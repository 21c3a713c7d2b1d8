"""Readers for RSEM's intermediate / output files, and helpers that run the reference binaries
(oracle/_ref) and the drop-in executables (bin/) on a generated dataset.  Test infrastructure."""
import hashlib
import io
import json
import os
import shutil
import subprocess
import tarfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
BIN_DIR = os.path.join(ROOT, "bin")
GEN = os.path.join(ROOT, "tools", "gen_dataset")
REF_RUNS = os.path.join(ROOT, "tests", "golden", "reference")
# not stored: read indices are rebuilt from the reads; .ofg and BAM files of even the small cases are hundreds of KB
UNSTORED = (".ridx", ".ofg", ".bam")


def have_ref():
    return all(os.path.exists(os.path.join(REF_DIR, b)) for b in ("rsem-run-em-rounds", "rsem-run-gibbs", "rsem-build-read-index"))


def _tree_digests(d):
    out = {}
    for dp, _, fs in os.walk(d):
        for f in fs:
            p = os.path.join(dp, f)
            with open(p, "rb") as fh:
                out[os.path.relpath(p, d)] = hashlib.sha256(fh.read()).hexdigest()
    return out


def _add_bytes(tar, name, data):
    ti = tarfile.TarInfo(name)
    ti.size = len(data)
    tar.addfile(ti, io.BytesIO(data))


def reference_run(key, d, run, out=None, digests_only=False):
    """What a reference binary prints and writes when run on the data set in directory d (into d, or into out).

    With oracle/_ref present, run() executes it (and RSEM_B200_RECORD_REFERENCE=1 stores the result as
    tests/golden/reference/<key>.tar.xz: stdout, stderr, the files the run created or changed apart from UNSTORED,
    and a digest of the input files).  Without it, those outputs are restored from the stored copy, after checking
    that d holds the same inputs the reference was run on.  digests_only: for outputs that are compared byte for byte,
    only the SHA-256 of each file is stored; the result's .digests maps each file the run wrote to its digest."""
    out = out or d
    inputs = hashlib.sha256(repr(sorted(_tree_digests(d).items())).encode()).hexdigest()
    before = _tree_digests(out)
    path = os.path.join(REF_RUNS, key + ".tar.xz")
    if have_ref():
        p = run()
        p.digests = {rel: h for rel, h in _tree_digests(out).items() if before.get(rel) != h and not rel.endswith(UNSTORED)}
        if os.environ.get("RSEM_B200_RECORD_REFERENCE") == "1":
            os.makedirs(REF_RUNS, exist_ok=True)
            with tarfile.open(path, "w:xz") as tar:
                for name, text in (("inputs.sha256", inputs), ("returncode", str(p.returncode)), ("stdout", p.stdout or ""),
                                   ("stderr", p.stderr or "")):
                    _add_bytes(tar, name, text.encode())
                if digests_only:
                    _add_bytes(tar, "digests.json", json.dumps(p.digests, sort_keys=True).encode())
                else:
                    for rel in sorted(p.digests):
                        tar.add(os.path.join(out, rel), arcname="files/" + rel)
        return p
    if not os.path.exists(path):
        import pytest
        pytest.skip(f"needs oracle/_ref or tests/golden/reference/{key}.tar.xz")
    with tarfile.open(path) as tar:
        text = {n: tar.extractfile(n).read().decode() for n in ("inputs.sha256", "returncode", "stdout", "stderr")}
        assert text["inputs.sha256"] == inputs, f"{key}: the generated inputs differ from those the reference was run on"
        names = tar.getnames()
        digests = json.loads(tar.extractfile("digests.json").read()) if "digests.json" in names else None
        for m in tar.getmembers():
            if m.name.startswith("files/"):
                m.name = m.name[len("files/"):]
                tar.extract(m, out, filter="data")
    if digests is None:
        digests = {rel: h for rel, h in _tree_digests(out).items() if before.get(rel) != h}
    return types.SimpleNamespace(returncode=int(text["returncode"]), stdout=text["stdout"], stderr=text["stderr"], digests=digests)


def gen_dataset(out, **kw):
    args = [GEN, "--out", out]
    for k, v in kw.items():
        args += ["--" + k.replace("_", "-"), str(v)]
    subprocess.check_call(args, stderr=subprocess.DEVNULL)
    return out


def read_files(d, read_type, tag="alignable"):
    ext = "fq" if read_type & 1 else "fa"
    if read_type >= 2:
        return [f"{d}/s.temp/s_{tag}_1.{ext}", f"{d}/s.temp/s_{tag}_2.{ext}"]
    return [f"{d}/s.temp/s_{tag}.{ext}"]


def clone(src, dst):
    if os.path.exists(dst):
        shutil.rmtree(dst)
    shutil.copytree(src, dst)
    return dst


def run_em(d, read_type, which, rounds=None, min_rounds=None, threads=1, gibbs_out=True, extra=(), check=True):
    """which = 'ref' (oracle/_ref/rsem-run-em-rounds) or 'ours' (bin/rsem-run-em).  Returns stdout."""
    env = dict(os.environ)
    if rounds is not None:
        env["RSEM_MAX_ROUND"] = str(rounds)
        env["RSEM_MIN_ROUND"] = str(min_rounds if min_rounds is not None else min(20, rounds))
    if which in ("ref", "ref_unpatched"):
        # "ref_unpatched": oracle/_ref/rsem-run-em, the reference compiled without the MAX/MIN_ROUND environment hook
        exe = os.path.join(REF_DIR, "rsem-run-em-rounds" if which == "ref" else "rsem-run-em")
        subprocess.check_call([os.path.join(REF_DIR, "rsem-build-read-index"), "32", str(read_type & 1), "1", *read_files(d, read_type)])
    else:
        exe = os.path.join(BIN_DIR, "rsem-run-em")
    cmd = [exe, "ref/r", str(read_type), "s", "s.temp/s", "s.stat/s", "-p", str(threads)]
    if gibbs_out:
        cmd.append("--gibbs-out")
    cmd += list(extra)
    p = subprocess.run(cmd, cwd=d, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    if check and p.returncode != 0:
        raise RuntimeError(f"{exe} failed ({p.returncode}):\n{p.stdout[-2000:]}\n{p.stderr[-2000:]}")
    return p


def run_gibbs(d, which, burnin, nsamples, gap, threads, seed, extra=(), check=True):
    exe = os.path.join(REF_DIR if which == "ref" else BIN_DIR, "rsem-run-gibbs")
    cmd = [exe, "ref/r", "s.temp/s", "s.stat/s", str(burnin), str(nsamples), str(gap), "-p", str(threads), "--seed", str(seed), "-q", *extra]
    p = subprocess.run(cmd, cwd=d, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    if check and p.returncode != 0:
        raise RuntimeError(f"{exe} failed ({p.returncode}):\n{p.stdout[-2000:]}\n{p.stderr[-2000:]}")
    return p


def read_theta(path):
    with open(path) as f:
        n = int(f.readline())
        raw = np.array(f.readline().split(), dtype=np.float64)
        pol = np.array(f.readline().split(), dtype=np.float64)
    assert len(raw) == n and len(pol) == n
    return raw, pol


def read_tokens(path):
    with open(path) as f:
        return np.array(f.read().split(), dtype=np.float64)


def read_res(path):
    """row-major result file -> list of rows (lists of strings)"""
    with open(path) as f:
        return [line.rstrip("\n").split("\t") for line in f]


def read_ofg(path):
    with open(path) as f:
        M, N0 = f.readline().split()
        row_ptr, sid, conprb = [0], [], []
        for line in f:
            t = line.split()
            sid += [int(x) for x in t[0::2]]
            conprb += [float(x) for x in t[1::2]]
            row_ptr.append(len(sid))
    return int(M), int(N0), np.array(row_ptr, np.uint64), np.array(sid, np.int32), np.array(conprb, np.float64)


def read_dat(path, paired):
    with open(path) as f:
        hdr = f.readline().split()
        N = int(hdr[0])
        row_ptr, sid, pos, ins = [0], [], [], []
        for _ in range(N):
            t = [int(x) for x in f.readline().split()]
            k, rest = t[0], t[1:]
            step = 3 if paired else 2
            sid += rest[0::step]
            pos += rest[1::step]
            if paired:
                ins += rest[2::step]
            row_ptr.append(len(sid))
    return (np.array(row_ptr, np.uint64), np.array(sid, np.int32), np.array(pos, np.int32),
            np.array(ins, np.int32) if paired else None)


def close_rel(a, b, rtol, floor=1e-7, atol=1e-12):
    """north_star tolerance: relative error on entries >= floor of the reference, absolute below"""
    a, b = np.asarray(a), np.asarray(b)
    big = np.abs(b) >= floor
    ok_big = np.all(np.abs(a[big] - b[big]) <= rtol * np.abs(b[big]))
    ok_small = np.all(np.abs(a[~big] - b[~big]) <= atol + rtol * np.abs(b[~big]))
    return bool(ok_big and ok_small)


def max_rel(a, b, floor=1e-7):
    a, b = np.asarray(a), np.asarray(b)
    big = np.abs(b) >= floor
    return float(np.max(np.abs(a[big] - b[big]) / np.abs(b[big]))) if big.any() else 0.0


# ---------------------------------------------------------------------------------------------------
# parsers producing the arrays the C ABI / the oracle take
_CODE = np.full(256, 255, np.uint8)
for _ch, _v in (("A", 0), ("C", 1), ("G", 2), ("T", 3), ("N", 4)):
    _CODE[ord(_ch)] = _v
    _CODE[ord(_ch.lower())] = _v


def read_seq(path):
    """ref.seq -> dict(seq_off, seq, full_len, tot_len, mask_off, mask_words, has_polyA); index 0 unused"""
    seq_off, full_len, tot_len, mask_off = [0], [0], [0], [0]
    seqs, masks = [], []
    pos = mpos = 0
    with open(path) as f:
        while True:
            line = f.readline()
            if not line.strip():
                break
            fl, tl = (int(x) for x in line.split())
            f.readline()  # name
            s = f.readline().rstrip("\n")
            w = [int(x) for x in f.readline().split()]
            seq_off.append(pos); full_len.append(fl); tot_len.append(tl); mask_off.append(mpos)
            seqs.append(_CODE[np.frombuffer(s.encode(), np.uint8)][:tl])
            masks += w
            pos += tl
            mpos += len(w)
    seq_off.append(pos)
    return dict(M=len(full_len) - 1, seq_off=np.array(seq_off[:-1] + [pos], np.uint64)[: len(full_len)],
                seq=np.concatenate(seqs) if seqs else np.zeros(0, np.uint8), full_len=np.array(full_len, np.int32),
                tot_len=np.array(tot_len, np.int32), mask_off=np.array(mask_off, np.uint64),
                mask_words=np.array(masks, np.uint32), has_polyA=bool(np.any(np.array(full_len) < np.array(tot_len))))


def _single_lq(s, has_polyA, seed_len):
    """SingleReadQ.h:63-95"""
    n = len(s)
    if n < seed_len:
        return True
    if not has_polyA:
        return False
    t1 = int(0.9 * n - 1.5 * np.sqrt(n) + 0.5)
    t2 = (25 - 1) // 2 + 1
    numA, numT = s.count("A"), s.count("T")
    numAO, numTO = s[:25].count("A"), s[max(n - 25, 0):].count("T")
    if numA >= t1:
        return numAO >= t2
    if numT >= t1:
        return numTO >= t2
    return False


def read_reads(d, read_type, tag, has_polyA, seed_len):
    """-> dict(n, off[2], base[2], qual[2], lowq) for the read set `tag` (un / alignable / max)"""
    hasq, paired = bool(read_type & 1), read_type >= 2
    files = read_files(d, read_type, tag)
    per_mate = []
    for fn in files:
        seqs, quals = [], []
        if os.path.exists(fn):
            with open(fn) as f:
                lines = f.read().split("\n")
            step = 4 if hasq else 2
            for i in range(0, len(lines) - 1, step):
                seqs.append(lines[i + 1])
                if hasq:
                    quals.append(lines[i + 3])
        per_mate.append((seqs, quals))
    n = len(per_mate[0][0])
    out = dict(n=n, off=[], base=[], qual=[], n_mates=2 if paired else 1, has_qual=hasq)
    for seqs, quals in per_mate:
        lens = np.array([len(s) for s in seqs], np.uint64)
        off = np.zeros(n + 1, np.uint64)
        off[1:] = np.cumsum(lens)
        out["off"].append(off)
        out["base"].append(_CODE[np.frombuffer("".join(seqs).encode(), np.uint8)] if n else np.zeros(0, np.uint8))
        out["qual"].append((np.frombuffer("".join(quals).encode(), np.uint8) - 33).astype(np.uint8) if hasq and n else None)
    lq = np.zeros(n, np.uint8)
    for i in range(n):
        if not paired:
            lq[i] = _single_lq(per_mate[0][0][i], has_polyA, seed_len)
        else:
            a, b = per_mate[0][0][i], per_mate[1][0][i]
            if len(a) < seed_len or len(b) < seed_len:
                lq[i] = 1
            else:
                lq[i] = _single_lq(a, has_polyA, seed_len) and _single_lq(b, has_polyA, seed_len)
    out["lowq"] = lq
    return out


def read_mparams(path):
    t = open(path).read().split()
    return dict(minL=int(t[0]), maxL=int(t[1]), probF=float(t[2]), estRSPD=int(t[3]) != 0, B=int(t[4]),
                mate_minL=int(t[5]), mate_maxL=int(t[6]), mean=float(t[7]), sd=float(t[8]), seedLen=int(t[9]))


def read_model(path, M):
    """.model -> dict of tables (model_file_description.txt)"""
    t = open(path).read().split()
    it = iter(t)
    nxt = lambda: next(it)
    m = dict(model_type=int(nxt()), M=M)
    m["ori0"] = float(nxt())

    def lendist():
        lb, ub, span = int(nxt()), int(nxt()), int(nxt())
        pdf = np.zeros(span + 1)
        pdf[1:] = [float(nxt()) for _ in range(span)]
        return dict(lb=lb, ub=ub, span=span, pdf=pdf, cdf=np.cumsum(pdf))
    m["gld"] = lendist()
    if m["model_type"] >= 2:
        m["mld"] = lendist()
    else:
        m["mld"] = lendist() if int(nxt()) > 0 else None
    m["est_rspd"] = int(nxt()) != 0
    if m["est_rspd"]:
        B = int(nxt())
        pdf = np.zeros(B + 2)
        pdf[1:B + 1] = [float(nxt()) for _ in range(B)]
    else:
        B = 20
        pdf = np.zeros(B + 2)
        pdf[1:B + 1] = 1.0 / B
    cdf = np.zeros(B + 2)
    cdf[1:B + 1] = np.cumsum(pdf[1:B + 1])
    m["B"], m["rspd_pdf"], m["rspd_cdf"] = B, pdf, cdf
    if m["model_type"] & 1:
        n = int(nxt())
        m["qd_init"] = np.array([float(nxt()) for _ in range(n)])
        m["qd_tran"] = np.array([float(nxt()) for _ in range(n * n)])
    rows, nc = int(nxt()), int(nxt())
    m["pro_len"] = 0 if m["model_type"] & 1 else rows
    m["profile"] = np.array([float(nxt()) for _ in range(rows * 25)])
    if m["model_type"] & 1:
        r2, c2 = int(nxt()), int(nxt())
        m["noise"] = np.array([float(nxt()) for _ in range(r2 * c2)])
    else:
        c2 = int(nxt())
        m["noise"] = np.array([float(nxt()) for _ in range(c2)])
    assert int(nxt()) == M
    m["mw"] = np.array([float(nxt()) for _ in range(M + 1)])
    return m
