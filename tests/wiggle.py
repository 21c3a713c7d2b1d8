"""Inputs and comparisons for the rsem-bam2wig / rsem-bam2readdepth tests: BAM files written record by record (raw
optional-field bytes included), sorted BAMs, and runs of the reference tools next to ours.  Test infrastructure."""
import hashlib
import os
import struct
import subprocess

import rsem_files as rf
import tbam2gbam as tg

TOOLS = {"wig": "rsem-bam2wig", "depth": "rsem-bam2readdepth"}
OUT = {"wig": "out.wig", "depth": "out.depth"}
SELFTEST = tg.SELFTEST
M, I, D, N, S, H, P, EQ, X = range(9)   # CIGAR operation codes


def ref_exe(tool):
    return os.path.join(rf.REF_DIR, TOOLS[tool])


def our_exe(tool):
    return os.path.join(rf.BIN_DIR, TOOLS[tool])


def args(tool, infile, nfw=False):
    if tool == "wig":
        return [infile, OUT[tool], "trk"] + (["--no-fractional-weight"] if nfw else [])
    return [infile, OUT[tool]]


# ---- BAM records -------------------------------------------------------------------------------------------------------
def zwf(x):
    return b"ZWf" + struct.pack("<f", x)


def zwf_bits(bits):
    return b"ZWf" + struct.pack("<I", bits)


def zwd(x):
    return b"ZWd" + struct.pack("<d", x)


def record(qname, flag, tid, pos, cigar, aux=b"", l_seq=None, mapq=255):
    """one BAM record with its block_size: cigar = [(length, op)], SEQ of l_seq N bases (default: the query length)"""
    if l_seq is None:
        l_seq = sum(n for n, op in cigar if op in (M, I, S, EQ, X))
    cig = b"".join(struct.pack("<I", n << 4 | op) for n, op in cigar)
    name = qname.encode() + b"\0"
    core = struct.pack("<iiBBHHHiiii", tid, pos, len(name), mapq, 4680, len(cigar), flag, l_seq, -1, -1, 0)
    body = core + name + cig + b"\xff" * ((l_seq + 1) // 2) + b"\xff" * l_seq + aux
    return struct.pack("<i", len(body)) + body


def write_bam(path, refs, records, text=None):
    if text is None:
        text = "@HD\tVN:1.4\tSO:coordinate\n" + "".join(f"@SQ\tSN:{n}\tLN:{l}\n" for n, l in refs)
    d = b"BAM\1" + struct.pack("<i", len(text)) + text.encode() + struct.pack("<i", len(refs))
    for name, length in refs:
        d += struct.pack("<i", len(name) + 1) + name.encode() + b"\0" + struct.pack("<I", length)
    with open(path, "wb") as f:
        f.write(tg.bgzf(d + b"".join(records)))


def sort_bam(src, dst, threads=4):
    subprocess.check_call([SELFTEST, "--bam-sort", src, dst, str(threads)], stdout=subprocess.DEVNULL)


# ---- runs ----------------------------------------------------------------------------------------------------------------
def rundir(d, name):
    w = d.rstrip("/") + "_" + name
    os.makedirs(w, exist_ok=True)
    if not os.path.lexists(os.path.join(w, "in.bam")) and os.path.exists(os.path.join(d, "in.bam")):
        os.symlink(os.path.join(d, "in.bam"), os.path.join(w, "in.bam"))
    return w


def run_ours(d, tool, name, nfw=False, env=None, infile="in.bam"):
    w = rundir(d, name)
    e = dict(os.environ)
    e.update(env or {})
    p = subprocess.run([our_exe(tool), *args(tool, infile, nfw)], cwd=w, stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                       text=True, env=e)
    path = os.path.join(w, OUT[tool])
    p.output = open(path, "rb").read() if os.path.exists(path) else None
    return p


def run_pair(key, d, tool, nfw=False, infile="in.bam", env=None):
    """the reference and ours on d/in.bam, each in its own directory -> (reference result with .digests, ours with
    .output).  Without oracle/_ref the reference's stdout, status and digests come from
    tests/golden/reference/wiggle_<key>."""
    tag = tool + ("_nfw" if nfw else "")
    wr = rundir(d, "ref_" + tag)

    def run():
        return subprocess.run([ref_exe(tool), *args(tool, infile, nfw)], cwd=wr, stdout=subprocess.PIPE,
                              stderr=subprocess.PIPE, text=True)
    ref = rf.reference_run("wiggle_" + key, d, run, out=wr, digests_only=True)
    ours = run_ours(d, tool, "ours_" + tag, nfw, env, infile)
    return ref, ours


def sha(b):
    return hashlib.sha256(b).hexdigest()


def check_same(key, d, tool, nfw=False, env=None):
    ref, ours = run_pair(key, d, tool, nfw, env=env)
    assert ours.returncode == ref.returncode, ours.stderr
    assert ours.stdout == ref.stdout
    assert ours.output is not None and sha(ours.output) == ref.digests.get(OUT[tool], sha(b"")), \
        (ours.output or b"")[:2000].decode(errors="replace")
    return ref, ours
