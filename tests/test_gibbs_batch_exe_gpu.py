"""bin/rsem-run-gibbs-batch against bin/rsem-run-gibbs run once per manifest line (every file byte for byte), against the
stored reference runs of the golden data sets, and against the reference binary where oracle/_ref is built.

The generated samples share one reference (gen_dataset --sample-seed); rsem-run-em-batch --gibbs-out writes their .ofg.
They cover both sides of the batch's size rule (a sample below 1248 reads and one without alignable reads take the
single-sample path), giant components (--spurious 0.01), -p not dividing NSAMPLES, -p above NSAMPLES, --pseudo-count
and --prior."""
import filecmp
import os
import re
import shutil
import subprocess

import pytest

import rsem_files as rf
from test_gibbs_multi_gpu import GOLDEN, _golden

pytestmark = pytest.mark.gpu

EXE = os.path.join(rf.BIN_DIR, "rsem-run-gibbs-batch")
M = 400

# (gen_dataset options, manifest arguments after imdName statName)
SPECS = [
    (dict(N1=6000, N0=50), "6 20 1 -p 3 --seed 11"),
    (dict(N1=3000, N0=20, spurious=0.01), "0 8 3 -p 2 --seed 12 --pseudo-count 0.1"),
    (dict(N1=600, N0=10), "4 6 1 -p 2 --seed 13 --pseudo-count 0.1"),
    (dict(N1=2500, N0=30, expressed_frac=0.3), "5 4 2 -p 6 --seed 14 --prior prior.txt"),
    (dict(N1=0, N0=40), "2 4 1 --seed 15"),
    (dict(N1=4000, N0=5, spurious=0.01), "3 10 1 -p 4 --seed 16 --pseudo-count 0.1 --prior prior.txt"),
]


@pytest.fixture(scope="module")
def samples(built, tmp_path_factory):
    """the generated samples after rsem-run-em-batch --gibbs-out"""
    root = tmp_path_factory.mktemp("gbexe")
    for k, (gen, _) in enumerate(SPECS):
        rf.gen_dataset(str(root / f"d{k}"), read_type=0, M=M, seed=7, sample_seed=200 + k, **gen)
    with open(root / "em_manifest", "w") as f:
        f.write("".join(f"d{k}/s d{k}/s.temp/s d{k}/s.stat/s --gibbs-out\n" for k in range(len(SPECS))))
    subprocess.run([os.path.join(rf.BIN_DIR, "rsem-run-em-batch"), "d0/ref/r", "0", "em_manifest", "-q"], cwd=root, check=True,
                   stdout=subprocess.DEVNULL)
    for k, (gen, _) in enumerate(SPECS):   # a sample without alignable reads: its .ofg is the header, its model any sample's
        if gen["N1"] == 0:
            with open(root / f"d{k}" / "s.temp" / "s.ofg", "w") as f:
                f.write(f"{M} {gen['N0']}\n")
            shutil.copy(root / "d0" / "s.stat" / "s.model", root / f"d{k}" / "s.stat" / "s.model")
    with open(root / "prior.txt", "w") as f:
        f.write("".join(f"{0.05 + (i % 5) * 0.3:.2f} prior\n" for i in range(M)))
    return str(root)


def _files(d, threads):
    return [f"s.temp/s.countvectors{t}" for t in range(threads)] + ["s.temp/s.iso_res", "s.temp/s.gene_res"]


def _threads(args):
    a = args.split()
    p = int(a[a.index("-p") + 1]) if "-p" in a else 1
    return max(1, min(p, int(a[1])))


def test_generated_samples_match_single_runs(samples, tmp_path):
    batch, single = str(tmp_path / "batch"), str(tmp_path / "single")
    shutil.copytree(samples, batch)
    shutil.copytree(samples, single)
    with open(os.path.join(batch, "manifest"), "w") as f:
        f.write("".join(f"d{k}/s.temp/s d{k}/s.stat/s {args}\n" for k, (_, args) in enumerate(SPECS)))
    env = dict(os.environ, RSEM_B200_TIMING="1")
    p = subprocess.run([EXE, "d0/ref/r", "manifest"], cwd=batch, env=env, capture_output=True, text=True)
    assert p.returncode == 0, p.stderr[-3000:]
    m = re.search(r"(\d+) samples in the batch, (\d+) on the single-sample path", p.stderr)
    assert m and (int(m.group(1)), int(m.group(2))) == (4, 2), p.stderr
    heads = re.findall(r"^== sample (\S+) \(manifest line (\d+)\)$", p.stdout, flags=re.M)
    assert heads == [(f"d{k}/s.temp/s", str(k + 1)) for k in range(len(SPECS))]
    blocks = re.split(r"^== sample .*$\n", p.stdout, flags=re.M)[1:]
    for k, (_, args) in enumerate(SPECS):
        q = subprocess.run([os.path.join(rf.BIN_DIR, "rsem-run-gibbs"), "d0/ref/r", f"d{k}/s.temp/s",
                            f"d{k}/s.stat/s", *args.split()], cwd=single, capture_output=True, text=True)
        assert q.returncode == 0, q.stderr[-2000:]
        assert blocks[k] == q.stdout, k
        for f in _files(f"d{k}", _threads(args)):
            assert filecmp.cmp(os.path.join(batch, f"d{k}", f), os.path.join(single, f"d{k}", f), shallow=False), (k, f)
        assert not os.path.exists(os.path.join(batch, f"d{k}", f"s.temp/s.countvectors{_threads(args)}"))


@pytest.mark.parametrize("name", ["pe_q_rspd", "se_noq"])
def test_golden_clones(tmp_path, built, name):
    """a manifest of three clones of a golden data set with the stored run's arguments reproduces the stored files"""
    base = _golden(tmp_path, name)
    root = tmp_path / "clones"
    os.makedirs(root)
    shutil.copytree(os.path.join(base, "ref"), root / "ref")
    for k in range(3):
        shutil.copytree(os.path.join(base, "s.temp"), root / f"c{k}" / "s.temp")
        shutil.copytree(os.path.join(base, "s.stat"), root / f"c{k}" / "s.stat")
    g = GOLDEN
    with open(root / "manifest", "w") as f:
        f.write("".join(f"c{k}/s.temp/s c{k}/s.stat/s {g['burnin']} {g['nsamples']} {g['gap']} -p {g['threads']} "
                        f"--seed {g['seed']}\n" for k in range(3)))
    p = subprocess.run([EXE, "ref/r", "manifest", "-q"], cwd=root, capture_output=True, text=True)
    assert p.returncode == 0, p.stderr[-2000:]
    stored = tmp_path / (name + ".stored")
    for k in range(3):
        for t in range(g["threads"]):
            assert filecmp.cmp(root / f"c{k}" / "s.temp" / f"s.countvectors{t}", stored / f"countvectors{t}", shallow=False)
        assert filecmp.cmp(root / f"c{k}" / "s.temp" / "s.iso_res", stored / "iso_res_gibbs", shallow=False)
        assert filecmp.cmp(root / f"c{k}" / "s.temp" / "s.gene_res", stored / "gene_res_gibbs", shallow=False)


@pytest.mark.skipif(not rf.have_ref(), reason="oracle/_ref not built")
def test_reference_binary(samples, tmp_path):
    """a batched sample above 1248 reads against the reference's rsem-run-gibbs"""
    ours, ref = str(tmp_path / "ours"), str(tmp_path / "ref")
    for d in (ours, ref):
        shutil.copytree(os.path.join(samples, "d0"), d)
    with open(os.path.join(ours, "manifest"), "w") as f:
        f.write("s.temp/s s.stat/s 4 6 1 -p 2 --seed 99\n")
    p = subprocess.run([EXE, "ref/r", "manifest", "-q"], cwd=ours, capture_output=True, text=True)
    assert p.returncode == 0, p.stderr[-2000:]
    rf.run_gibbs(ref, "ref", 4, 6, 1, 2, 99)
    for f in _files(ref, 2):
        assert filecmp.cmp(os.path.join(ours, f), os.path.join(ref, f), shallow=False), f
