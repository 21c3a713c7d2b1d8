"""Drop-in parity: bin/rsem-run-em and bin/rsem-run-gibbs against the reference executables
(oracle/_ref, built by oracle/Makefile) on the same generated inputs; where they are not built, against what they
wrote on those inputs (tests/golden/reference, see rsem_files.reference_run).

Tolerances (north_star: theta / TPM within 1e-6 relative after the same iteration count; Gibbs: same
seed -> same draws):
  .theta (raw and polished)   1e-6 relative for theta >= 1e-7, 1e-12 absolute below
  .model tables (%.10g)       1e-6 relative / 1e-9 absolute
  .ofg conprb / ncpv          1e-6 relative
  result rows (%.2f)          0.011 absolute, or 1e-6 relative for large values
  .countvectors               byte-identical
"""
import filecmp
import os

import numpy as np
import pytest

import rsem_files as rf

pytestmark = pytest.mark.gpu

CASES = {
    # name: (read_type, generator options)
    "se_noq": (0, dict(M=200, N1=3000, N0=150, read_len=50, maxL=200)),
    "se_q_rspd_polyA": (1, dict(M=150, N1=2500, N0=120, read_len=60, var_len=8, est_rspd=1, polyA=125, probF=0.7, spurious=0.05)),
    "pe_noq": (2, dict(M=150, N1=2000, N0=100, read_len=40, var_len=4, maxL=400, spurious=0.05)),
    "pe_q_rspd": (3, dict(M=200, N1=2500, N0=100, read_len=50, est_rspd=1, probF=0.3, spurious=0.1)),
    "se_q_revonly": (1, dict(M=100, N1=1500, N0=50, read_len=45, est_rspd=1, probF=0.0)),
    "se_noq_fraglen": (0, dict(M=100, N1=1500, N0=80, read_len=50, var_len=10, maxL=300, frag_mean=180, frag_sd=30)),
    "pe_q_polyA": (3, dict(M=120, N1=1500, N0=60, read_len=50, polyA=125, omit=5)),
}


def _num_rows_close(a_rows, b_rows):
    assert len(a_rows) == len(b_rows)
    for ra, rb in zip(a_rows, b_rows):
        assert len(ra) == len(rb)
        try:
            xa, xb = np.array(ra, float), np.array(rb, float)
        except ValueError:
            assert ra == rb
            continue
        assert np.all(np.abs(xa - xb) <= 0.011 + 1e-6 * np.abs(xb)), (ra[:5], rb[:5])


@pytest.fixture(scope="module")
def workdir(tmp_path_factory, built):
    return tmp_path_factory.mktemp("dropin")


@pytest.fixture
def live_ref():
    if not rf.have_ref():
        pytest.skip("oracle/_ref binaries not available (the .ofg and BAM files this test needs are not stored)")


@pytest.mark.parametrize("rounds", [13, 3])
@pytest.mark.parametrize("name", list(CASES))
def test_em_matches_reference(workdir, name, rounds):
    rt, opts = CASES[name]
    base = rf.gen_dataset(str(workdir / f"{name}_base"), read_type=rt, seed=7, **opts)
    ref = rf.clone(base, str(workdir / f"{name}_{rounds}_ref"))
    ours = rf.clone(base, str(workdir / f"{name}_{rounds}_ours"))
    pr = rf.reference_run(f"em_{name}_{rounds}", ref, lambda: rf.run_em(ref, rt, "ref", rounds=rounds, threads=2))
    po = rf.run_em(ours, rt, "ours", rounds=rounds)
    # same number of rounds and the same progress lines
    lr = [l for l in pr.stdout.splitlines() if l.startswith("ROUND = ")]
    lo = [l for l in po.stdout.splitlines() if l.startswith("ROUND = ")]
    assert len(lr) == len(lo) == rounds
    raw_r, pol_r = rf.read_theta(f"{ref}/s.stat/s.theta")
    raw_o, pol_o = rf.read_theta(f"{ours}/s.stat/s.theta")
    assert rf.close_rel(raw_o, raw_r, 1e-6), rf.max_rel(raw_o, raw_r)
    assert rf.close_rel(pol_o, pol_r, 1e-6), rf.max_rel(pol_o, pol_r)
    mr, mo = rf.read_tokens(f"{ref}/s.stat/s.model"), rf.read_tokens(f"{ours}/s.stat/s.model")
    assert mr.shape == mo.shape
    assert np.all(np.abs(mo - mr) <= 1e-9 + 1e-6 * np.abs(mr)), np.max(np.abs(mo - mr))
    if os.path.exists(f"{ref}/s.temp/s.ofg"):   # written by a live reference run only (rsem_files.UNSTORED)
        Mr, N0r, rp_r, sid_r, c_r = rf.read_ofg(f"{ref}/s.temp/s.ofg")
        Mo, N0o, rp_o, sid_o, c_o = rf.read_ofg(f"{ours}/s.temp/s.ofg")
        assert (Mr, N0r) == (Mo, N0o) and np.array_equal(rp_r, rp_o) and np.array_equal(sid_r, sid_o)
        assert np.all(np.abs(c_o - c_r) <= 1e-6 * np.abs(c_r))
    _num_rows_close(rf.read_res(f"{ours}/s.temp/s.iso_res"), rf.read_res(f"{ref}/s.temp/s.iso_res"))
    _num_rows_close(rf.read_res(f"{ours}/s.temp/s.gene_res"), rf.read_res(f"{ref}/s.temp/s.gene_res"))


@pytest.mark.parametrize("threads,nsamples,gap", [(1, 7, 1), (3, 10, 2)])
def test_gibbs_same_seed_same_draws(workdir, live_ref, threads, nsamples, gap):
    rt, opts = CASES["se_q_rspd_polyA"]
    base = rf.gen_dataset(str(workdir / f"gibbs_base_{threads}"), read_type=rt, seed=3, **dict(opts, omit=4))
    rf.run_em(base, rt, "ref", rounds=12, threads=1)   # reference EM produces .ofg / .model / result rows
    ref = rf.clone(base, str(workdir / f"gibbs_ref_{threads}"))
    ours = rf.clone(base, str(workdir / f"gibbs_ours_{threads}"))
    rf.run_gibbs(ref, "ref", 15, nsamples, gap, threads, 12345)
    rf.run_gibbs(ours, "ours", 15, nsamples, gap, threads, 12345)
    for t in range(threads):
        assert filecmp.cmp(f"{ref}/s.temp/s.countvectors{t}", f"{ours}/s.temp/s.countvectors{t}", shallow=False)
    _num_rows_close(rf.read_res(f"{ours}/s.temp/s.iso_res"), rf.read_res(f"{ref}/s.temp/s.iso_res"))
    _num_rows_close(rf.read_res(f"{ours}/s.temp/s.gene_res"), rf.read_res(f"{ref}/s.temp/s.gene_res"))


def test_gibbs_prior_and_pseudocount(workdir, live_ref):
    rt, opts = CASES["se_noq"]
    base = rf.gen_dataset(str(workdir / "gibbs_prior_base"), read_type=rt, seed=5, **opts)
    rf.run_em(base, rt, "ref", rounds=12, threads=1)
    M = opts["M"]
    with open(f"{base}/prior.txt", "w") as f:
        rng = np.random.default_rng(0)
        for i in range(M):
            f.write(f"{rng.uniform(0.1, 3.0):.4f} comment\n")
    for tag, extra in (("pc", ["--pseudo-count", "0.1"]), ("prior", ["--prior", "prior.txt"])):
        ref = rf.clone(base, str(workdir / f"gibbs_{tag}_ref"))
        ours = rf.clone(base, str(workdir / f"gibbs_{tag}_ours"))
        rf.run_gibbs(ref, "ref", 10, 6, 1, 2, 99, extra=extra)
        rf.run_gibbs(ours, "ours", 10, 6, 1, 2, 99, extra=extra)
        for t in range(2):
            assert filecmp.cmp(f"{ref}/s.temp/s.countvectors{t}", f"{ours}/s.temp/s.countvectors{t}", shallow=False)
        _num_rows_close(rf.read_res(f"{ours}/s.temp/s.iso_res"), rf.read_res(f"{ref}/s.temp/s.iso_res"))


def test_no_alignable_reads(workdir):
    """N1 == 0 special case (EM.cpp:615-638): empty .theta / .model, zero result rows; no GPU work"""
    base = rf.gen_dataset(str(workdir / "n1zero_base"), read_type=0, M=30, N1=0, N0=50)
    ref, ours = rf.clone(base, str(workdir / "n1zero_ref")), rf.clone(base, str(workdir / "n1zero_ours"))
    env_rounds = 3
    rf.run_em(ours, 0, "ours", rounds=env_rounds, gibbs_out=False)
    exe = os.path.join(rf.REF_DIR, "rsem-run-em-rounds")
    import subprocess
    rf.reference_run("n1zero", ref, lambda: subprocess.run([exe, "ref/r", "0", "s", "s.temp/s", "s.stat/s"], cwd=ref, check=True,
                                                           stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True))
    assert os.path.getsize(f"{ours}/s.stat/s.theta") == 0 and os.path.getsize(f"{ours}/s.stat/s.model") == 0
    assert filecmp.cmp(f"{ref}/s.temp/s.iso_res", f"{ours}/s.temp/s.iso_res", shallow=False)
    assert filecmp.cmp(f"{ref}/s.temp/s.gene_res", f"{ours}/s.temp/s.gene_res", shallow=False)


@pytest.mark.parametrize("rt,sampling", [(3, False), (0, False), (1, True)])
def test_posterior_bam(workdir, live_ref, rt, sampling):
    """-b (EM.cpp:504-536, BamWriter.h): every alignment line of the input comes back with MAPQ and ZW:f from the posteriors;
    --sampling draws one alignment per read with the seeded MT19937 (sampling.h:50-65)"""
    from bam_reader import read_bam
    base = rf.gen_dataset(str(workdir / f"bam_base_{rt}"), read_type=rt, M=80, N1=1500, N0=70, read_len=50, sam=1, seed=13 + rt)
    ref, ours = rf.clone(base, str(workdir / f"bam_ref_{rt}")), rf.clone(base, str(workdir / f"bam_ours_{rt}"))
    extra = ["-b", "aln.sam", "0"] + (["--sampling", "--seed", "4242"] if sampling else [])
    rf.run_em(ref, rt, "ref", rounds=13, threads=2, gibbs_out=False, extra=extra)
    po = rf.run_em(ours, rt, "ours", rounds=13, threads=3, gibbs_out=False, extra=extra)
    assert "Bam output file is generated!" in po.stdout
    tr, rr, a = read_bam(f"{ref}/s.transcript.bam")
    to, ro, b = read_bam(f"{ours}/s.transcript.bam")
    assert (tr, rr) == (to, ro) and len(a) == len(b)
    for x, y in zip(b, a):
        zx, zy = x["tags"].pop("ZW", None), y["tags"].pop("ZW", None)
        assert (zx is None) == (zy is None) == bool(y["flag"] & 4)
        if zy is not None:
            assert abs(zx[1] - zy[1]) <= 1e-6 + 1e-6 * abs(zy[1])
            if sampling:
                assert zx[1] in (0.0, 1.0)
            assert abs(x["mapq"] - y["mapq"]) <= (0 if zx[1] == zy[1] else 1)
            x["mapq"] = y["mapq"]
        assert x == y


def test_bam_of_a_sample_without_alignable_reads(workdir):
    """N1 == 0 with -b: the input file is copied as it is (EM.cpp:627-633)"""
    base = rf.gen_dataset(str(workdir / "bam_n1zero"), read_type=0, M=30, N1=0, N0=50, sam=1)
    rf.run_em(base, 0, "ours", rounds=3, gibbs_out=False, extra=["-b", "aln.sam", "0"])
    assert filecmp.cmp(f"{base}/aln.sam", f"{base}/s.transcript.bam", shallow=False)


def test_em_two_gpus_matches_reference(workdir, live_ref):
    """RSEM_B200_DEVICES=0,1: reads sharded over two GPUs (same rule as the reference's threads), counts and model
    statistics summed with ncclAllReduce inside the library.  Needs a machine with >= 2 GPUs."""
    import rsem_b200
    if rsem_b200.load_library().device_count() < 2:
        pytest.skip("needs two GPUs")
    rt, opts = CASES["pe_q_rspd"]
    base = rf.gen_dataset(str(workdir / "mgpu_base"), read_type=rt, seed=9, **opts)
    ref, ours = rf.clone(base, str(workdir / "mgpu_ref")), rf.clone(base, str(workdir / "mgpu_ours"))
    rf.run_em(ref, rt, "ref", rounds=14, threads=2)
    os.environ["RSEM_B200_DEVICES"] = "0,1"
    try:
        po = rf.run_em(ours, rt, "ours", rounds=14)
    finally:
        del os.environ["RSEM_B200_DEVICES"]
    assert "GPU 1 : N = " in po.stdout
    raw_r, pol_r = rf.read_theta(f"{ref}/s.stat/s.theta")
    raw_o, pol_o = rf.read_theta(f"{ours}/s.stat/s.theta")
    assert rf.close_rel(raw_o, raw_r, 1e-6) and rf.close_rel(pol_o, pol_r, 1e-6)
    mr, mo = rf.read_tokens(f"{ref}/s.stat/s.model"), rf.read_tokens(f"{ours}/s.stat/s.model")
    assert np.all(np.abs(mo - mr) <= 1e-9 + 1e-6 * np.abs(mr))
    _, _, rp_r, sid_r, c_r = rf.read_ofg(f"{ref}/s.temp/s.ofg")
    _, _, rp_o, sid_o, c_o = rf.read_ofg(f"{ours}/s.temp/s.ofg")
    assert np.array_equal(rp_r, rp_o) and np.array_equal(sid_r, sid_o) and np.all(np.abs(c_o - c_r) <= 1e-6 * np.abs(c_r))
    _num_rows_close(rf.read_res(f"{ours}/s.temp/s.iso_res"), rf.read_res(f"{ref}/s.temp/s.iso_res"))
