"""bin/rsem-simulate-reads-batch: for every manifest line the read files, the .sim.*.results tables and the line's
stdout block must be byte-identical to a separate bin/rsem-simulate-reads run of that line, and where the line is one
of the stored cases of test_simulate_gpu.py, also to the reference simulator's (its stored digests, or
oracle/_ref/rsem-simulate-reads).

One lane runs consecutive samples of different shapes on one context, which keeps its buffers from run to run: every
manifest mixes theta0 0 and 0.2, two seeds, N = 0, models edited on the same reference (an all-zero reachable
QProfile block, zeroed RSPD bins, a single-end model with a mate-length distribution) and, at the default window, a
1 M-read line between lines of a few thousand reads (the buffers grow and are then reused smaller).  Lanes 0,0 .. 0,0,0,0
(and 0,1 with two GPUs) must write what one lane writes.  The C ABI is checked through capi.py: a reference kept on the
context by sim_upload_refs gives the runs what a reference passed in the params gives."""
import hashlib
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import rsem_files as rf
import test_simulate_gpu as ts

pytestmark = pytest.mark.gpu

BATCH = os.path.join(rf.ROOT, "bin", "rsem-simulate-reads-batch")


def _digests(d):
    return {f: hashlib.sha256(open(os.path.join(d, f), "rb").read()).hexdigest() for f in sorted(os.listdir(d))}


def _zero_qprofile(lines):
    """test_simulate_gpu.test_zero_profile_rows's edit: the QProfile block of the most common quality set to 0"""
    k = next(i for i, l in enumerate(lines) if l.strip() == "100" and len(lines[i + 1].split()) == 100)
    init = [float(x) for x in lines[k + 1].split()]
    q = max(range(100), key=lambda i: init[i])
    k0 = next(i for i, l in enumerate(lines) if l.strip() == "100 5")
    for r in range(5):
        lines[k0 + 1 + q * 6 + r] = " ".join(["0"] * 5)
    return lines


def _foreign_model(tmp_path, src):
    """the model of golden set src without its mw block (which is tied to src's reference): a model of another read
    type for the reference of the manifest"""
    g = ts._golden(tmp_path, src)
    lines = open(g / "out" / "model20").read().split("\n")
    M = int(open(g / "ref" / "r.ti").readline().split()[0])
    k = max(i for i, x in enumerate(lines) if x.strip() == str(M))
    return lambda _: lines[:k] + [""]


class Line:
    """one manifest line: the inputs of case directory d, and where its batch outputs and its single run go"""

    def __init__(self, d, theta0, n, seed, key=None, quiet=False):
        self.d, self.theta0, self.n, self.seed, self.key, self.quiet = d, theta0, n, seed, key, quiet

    def fields(self, out):
        f = [str(self.d / "model"), str(self.d / "res.tsv"), str(self.theta0), str(self.n), os.path.join(out, "s")]
        if self.seed is not None:
            f += ["--seed", str(self.seed)]
        return f + (["-q"] if self.quiet else [])


def _single(ref, line, out, env):
    """-> stdout of bin/rsem-simulate-reads for the line, its files in out; a stored case is also checked against the
    reference simulator (test_simulate_gpu._compare)"""
    shutil.rmtree(out, ignore_errors=True)
    if line.key:
        stdout = ts._compare(line.d, line.key, line.theta0, line.n, line.seed, env=env)
        shutil.copytree(str(line.d) + ".gpu", out)
        return stdout
    os.makedirs(out)
    p = subprocess.run([ts.BIN, ref, *line.fields(out)], capture_output=True, text=True, env={**os.environ, **env})
    assert p.returncode == 0, p.stderr
    return p.stdout


def _batch(tmp_path, ref, lines, env, tag, lanes=None, extra=()):
    """runs the batch on the lines (outputs in tmp_path/<tag>/<i>); -> the blocks of stdout, in manifest order"""
    root = tmp_path / tag
    shutil.rmtree(root, ignore_errors=True)
    os.makedirs(root)
    outs = []
    with open(root / "manifest", "w") as f:
        for i, l in enumerate(lines):
            outs.append(str(root / str(i)))
            os.makedirs(outs[-1])
            f.write(" ".join(l.fields(outs[-1])) + "\n")
    e = {**os.environ, **env}
    if lanes:
        e["RSEM_B200_DEVICES"] = lanes
    p = subprocess.run([BATCH, ref, str(root / "manifest"), *extra], capture_output=True, text=True, env=e)
    assert p.returncode == 0, p.stderr
    if "-q" in extra:
        return outs, p.stdout
    blocks = re.split(r"^== sample .*\n", p.stdout, flags=re.M)
    assert blocks[0] == "" and len(blocks) == len(lines) + 1, p.stdout[:2000]
    heads = re.findall(r"^== sample (.*) \((.*) line (\d+)\)$", p.stdout, flags=re.M)
    assert [int(h[2]) for h in heads] == list(range(1, len(lines) + 1))
    return outs, blocks[1:]


def _check_against_single(tmp_path, ref, lines, env, tag):
    outs, blocks = _batch(tmp_path, ref, lines, env, tag)
    for i, l in enumerate(lines):
        single = str(tmp_path / tag / f"single{i}")
        stdout = _single(ref, l, single, env)
        assert _digests(outs[i]) == _digests(single), f"line {i + 1}"
        assert blocks[i] == stdout, f"line {i + 1}"
        shutil.rmtree(single)
        shutil.rmtree(outs[i])   # the 1 M-read files are large
    return blocks


def _manifest(tmp_path, name, window):
    """the lines of one golden reference; returns (reference prefix, lines)"""
    c = lambda key, edit=None: ts._case(tmp_path, key, name, edit)
    d0, d2 = c(f"sim_{name}_0.0"), c(f"sim_{name}_0.2")
    lines = [Line(d0, 0.0, 3000, 11, f"sim_{name}_0.0"), Line(d2, 0.2, 0, 5)]
    if window is None:
        d1m = c("sim_1m") if name == "se_noq" else d2
        lines += [Line(d1m, 0.05, 1000000, 3, "sim_1m" if name == "se_noq" else None)]
    lines += [Line(d2, 0.2, 3000, 11, f"sim_{name}_0.2"), Line(d2, 0.2, 2500, 12)]
    if name == "pe_q_rspd":
        lines += [Line(c("sim_zero_rows", _zero_qprofile), 0.2, 4000, 17, "sim_zero_rows"),
                  Line(c("sim_rspd_fail", ts._zero_rspd_bins), 0.1, 5000, 9, "sim_rspd_fail")]
    elif name in ("se_q_polyA", "se_q_rspd"):
        lines += [Line(c(f"zero_rows_{name}", _zero_qprofile), 0.1, 4000, 23)]
        if name == "se_q_rspd":
            lines += [Line(c(f"rspd_fail_{name}", ts._zero_rspd_bins), 0.1, 5000, 29)]
    elif name == "se_noq":
        lines += [Line(c("sim_se_mld", ts._se_with_mld), 0.1, 5000, 21, "sim_se_mld")]
    if name in ("se_noq", "pe_noq"):   # single-end and paired-end samples on one context, in both orders
        other = c("other_type", _foreign_model(tmp_path, "pe_noq" if name == "se_noq" else "se_noq"))
        lines[1:1] = [Line(other, 0.1, 3000, 41)]
        lines += [Line(other, 0.2, 8000, 42)]
    if window is not None:
        lines += [Line(d2, 0.1, 20000, 5, f"sim_win_{name}" if name in ("pe_q_rspd", "se_noq") else None)]
        if lines[-1].key:
            lines[-1].d = c(lines[-1].key)
    lines += [Line(d0, 0.0, 1500, 31), Line(d2, 0.2, 0, 6)]
    return str(d0 / "ref" / "r"), lines


@pytest.mark.parametrize("window", [None, "3000"], ids=["default_window", "small_window"])
@pytest.mark.parametrize("name", ts.SETS)
def test_manifest_matches_single_runs(tmp_path, built, name, window):
    env = {"RSEM_B200_SIM_WINDOW": window} if window else {}
    ref, lines = _manifest(tmp_path, name, window)
    blocks = _check_against_single(tmp_path, ref, lines, env, "batch")
    if window is None:
        assert "GEN 1000000" in blocks[3 if name in ("se_noq", "pe_noq") else 2]


def test_allele_specific_reference(tmp_path, built):
    d = ts._case(tmp_path, "sim_allele", "se_q_rspd", extra_col=True)
    grp = [int(x) for x in open(d / "ref" / "r.grp").read().split()]
    M = grp[-1] - 1
    ta = [1]   # as test_simulate_gpu.test_allele_specific_reference builds them
    while ta[-1] <= M:
        a = ta[-1]
        ta.append(a + 2 if a + 1 <= M and not any(a < g <= a + 1 for g in grp) else a + 1)
    gt = [ta.index(g) for g in grp]
    open(d / "ref" / "r.ta", "w").write("\n".join(map(str, ta)) + "\n")
    open(d / "ref" / "r.gt", "w").write("\n".join(map(str, gt)) + "\n")
    lines = [Line(d, 0.2, 3000, 11, "sim_allele"), Line(d, 0.1, 0, 4), Line(d, 0.1, 5000, 12)]
    outs, blocks = _batch(tmp_path, str(d / "ref" / "r"), lines, {}, "allele")
    for i, l in enumerate(lines):
        assert os.path.exists(os.path.join(outs[i], "s.sim.alleles.results"))
    _check_against_single(tmp_path, str(d / "ref" / "r"), lines, {}, "allele")


def _many(tmp_path):
    """48 small samples of one reference, distinct seeds, two models"""
    plain = ts._case(tmp_path, "many_plain", "pe_q_rspd")
    fail = ts._case(tmp_path, "many_fail", "pe_q_rspd", ts._zero_rspd_bins)
    lines = [Line(fail if k % 3 == 2 else plain, (0.0, 0.1, 0.2)[k % 3], 300 + 97 * k, 1000 + k) for k in range(48)]
    return str(plain / "ref" / "r"), lines


def _device_count():
    import rsem_b200
    return rsem_b200.load_library().device_count()


def test_lanes_write_what_one_lane_writes(tmp_path, built):
    ref, lines = _many(tmp_path)
    outs, one = _batch(tmp_path, ref, lines, {}, "one")
    want = [_digests(o) for o in outs]
    lists = ["0,0", "0,0,0", "0,0,0,0"] + (["0,1"] if _device_count() >= 2 else [])
    for lanes in lists:
        outs, blocks = _batch(tmp_path, ref, lines, {}, "lanes" + lanes.replace(",", ""), lanes=lanes)
        assert [_digests(o) for o in outs] == want, lanes
        assert blocks == one, lanes
    for i in (0, 17, 47):   # and a few of them against single runs
        assert _single(ref, lines[i], str(tmp_path / f"single{i}"), {}) == one[i]
        assert _digests(str(tmp_path / f"single{i}")) == want[i]


def _reads(out):
    f = [x for x in os.listdir(out) if x.endswith((".fa", ".fq"))]
    return sum(1 for _ in open(os.path.join(out, f[0]))) // (4 if f[0].endswith(".fq") else 2)


def test_quiet_lines_and_lines_without_seed(tmp_path, built):
    d = ts._case(tmp_path, "quiet_case", "se_q_polyA")
    ref = str(d / "ref" / "r")
    lines = [Line(d, 0.1, 1200000, 8, quiet=True), Line(d, 0.1, 2000, None), Line(d, 0.2, 3000, None, quiet=True),
             Line(d, 0.1, 2000, 9)]
    outs, blocks = _batch(tmp_path, ref, lines, {}, "quiet")
    assert blocks[0] == _single(ref, lines[0], str(tmp_path / "single0"), {})
    assert "GEN" not in blocks[0] and blocks[2].startswith("Total number of resimulation is ")
    for i in (1, 2):
        assert _reads(outs[i]) == lines[i].n
        assert os.path.exists(os.path.join(outs[i], "s.sim.genes.results"))
        assert re.fullmatch(("Refs.loadRefs finished!\n" if i == 1 else "") + r"Total number of resimulation is \d+\n", blocks[i])
    outs_q, stdout = _batch(tmp_path, ref, lines, {}, "batch_quiet", extra=("-q",))
    assert "==" not in stdout and "GEN" not in stdout
    assert stdout.count("Total number of resimulation is") == 4
    assert _digests(outs_q[3]) == _digests(outs[3])


# ---- the C ABI: a reference kept on the context --------------------------------------------------------------------
def _abi_params(rng, M, model_type, seed, n, keep):
    """tables of a synthetic model (type 0 or 2, no qualities, no estRSPD); keep holds the arrays alive"""
    from rsem_b200 import capi
    import ctypes as C

    def dp(a):
        a = np.ascontiguousarray(a, np.float64)
        keep.append(a)
        return a.ctypes.data_as(C.POINTER(C.c_double))

    def lendist(lb, ub):
        pdf = np.concatenate([[0.0], rng.random(ub - lb)])
        pdf /= pdf.sum()
        return capi.LenDist(lb, ub, ub - lb, dp(pdf), dp(np.cumsum(pdf)))

    theta = np.concatenate([[0.05], rng.random(M)])
    theta[1:] *= 0.95 / theta[1:].sum()
    p = capi.SimParams()
    p.model_type, p.M, p.seed, p.exact_body, p.N, p.window_words = model_type, M, seed, 0, n, 0
    p.theta_cdf = dp(np.cumsum(theta))
    p.ori_prob0 = 0.5
    p.gld = lendist(50, 300)
    p.has_mld = 1 if model_type == 2 else 0
    if p.has_mld:
        p.mld = lendist(20, 60)
    pro_rows = 60 if model_type == 2 else 300
    p.pro_rows = pro_rows
    p.profile_cdf = dp(np.cumsum(rng.random((pro_rows * 5, 5)) + 0.1, axis=1))
    p.noise_cdf = dp(np.cumsum(rng.random(5) + 0.1))
    return p


def test_capi_uploaded_reference(built):
    import ctypes as C
    import rsem_b200
    from rsem_b200 import capi
    rng = np.random.default_rng(3)
    M = 40
    tot = rng.integers(300, 900, M + 1).astype(np.int32)
    tot[0] = 0
    full = tot.copy()
    seq_off = np.zeros(M + 2, np.uint64)
    seq_off[2:] = np.cumsum(tot[1:])
    seq_off[1] = 0
    seq = rng.integers(0, 5, int(seq_off[-1]), dtype=np.uint8)
    keep = []
    runs = [_abi_params(rng, M, 0, 7, 30000, keep), _abi_params(rng, M, 2, 8, 4000, keep)]

    def run(ctx, p):
        ctx.sim_begin(p)
        text = [b"", b""]
        while True:
            n, t = ctx.sim_next()
            if n == 0:
                break
            text = [text[0] + t[0], text[1] + t[1]]
        counts, resim, _ = ctx.sim_end(M)
        return text, counts.tolist(), resim

    want = []
    with capi.Context(0) as ctx:
        for p in runs:
            p.seq_off = seq_off.ctypes.data_as(C.POINTER(C.c_uint64))
            p.seq = seq.ctypes.data_as(C.POINTER(C.c_uint8))
            p.tot_len = tot.ctypes.data_as(C.POINTER(C.c_int32))
            p.full_len = full.ctypes.data_as(C.POINTER(C.c_int32))
            want.append(run(ctx, p))
    assert want[0][0][0] and want[1][0][1]
    for order in ([0, 1], [1, 0]):
        with capi.Context(0) as ctx:
            ctx.sim_upload_refs(seq_off, seq, tot, full)
            for k in order + order:
                p = runs[k]
                p.seq_off = p.seq = p.tot_len = p.full_len = None
                assert run(ctx, p) == want[k]
    with capi.Context(0) as ctx:   # no uploaded reference: refused
        with pytest.raises(rsem_b200.capi.RsemB200Error):
            ctx.sim_begin(runs[0])
