"""Inputs and comparisons for the rsem-tbam2gbam tests: genome-mode data sets, BAM files written from SAM text or
directly, the decoded canonical text of a genome BAM, and runs of the reference tool next to ours.  Test infrastructure."""
import hashlib
import json
import os
import re
import struct
import subprocess
import zlib

import bam_reader
import rsem_files as rf

REF_EXE = os.path.join(rf.REF_DIR, "rsem-tbam2gbam")
OUR_EXE = os.path.join(rf.BIN_DIR, "rsem-tbam2gbam")
SELFTEST = os.path.join(rf.BIN_DIR, "rsem-b200-host-selftest")


def bgzf(data):
    """BGZF blocks of <= 0xff00 bytes and the EOF marker (SAM specification 4.1)"""
    out = []
    for a in range(0, len(data), 0xff00):
        chunk = data[a:a + 0xff00]
        co = zlib.compressobj(6, zlib.DEFLATED, -15)
        c = co.compress(chunk) + co.flush()
        out.append(b"\x1f\x8b\x08\x04\0\0\0\0\0\xff\x06\0BC\x02\0" + struct.pack("<H", len(c) + 25) + c
                   + struct.pack("<II", zlib.crc32(chunk) & 0xffffffff, len(chunk)))
    out.append(bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000"))
    return b"".join(out)


def header_only_bam(path, text, refs):
    d = b"BAM\1" + struct.pack("<i", len(text)) + text.encode() + struct.pack("<i", len(refs))
    for name, length in refs:
        d += struct.pack("<i", len(name) + 1) + name.encode() + b"\0" + struct.pack("<i", length)
    with open(path, "wb") as f:
        f.write(bgzf(d))


def sam_to_bam(sam, bam, weight_step=0.0):
    """SAM -> BAM with our reader / writer; weight_step > 0 gives every mapped record MAPQ and a ZW:f as rsem-run-em -b"""
    args = [SELFTEST, "--bam-copy", sam, bam, "1"] + ([repr(weight_step)] if weight_step else [])
    subprocess.check_call(args, stdout=subprocess.DEVNULL)


def read_ti(path):
    """Transcript::read (Transcript.h:119-148) restated: [(id, name, gene_id, gene_name, seqname, strand, length, exons)]"""
    lines = open(path).read().split("\n")
    M, typ = (int(x) for x in lines[0].split())
    out, i = [], 1
    for _ in range(M):
        tid, _, tname = lines[i].partition("\t")
        gid, _, gname = lines[i + 1].partition("\t")
        seqname = lines[i + 2]
        strand, length = lines[i + 3].split()
        nums = [int(x) for x in lines[i + 4].split()]
        exons = list(zip(nums[1::2], nums[2::2]))
        assert len(exons) == nums[0]
        out.append((tid, tname, gid, gname, seqname, strand, int(length), exons))
        i += 6
    return typ, out


def canonical(path):
    """the decoded genome BAM as text: header (argv[0] of our @PG CL: replaced), references, then one JSON line per
    record with every field and the tags in order, floats by their exact value"""
    text, refs, recs = bam_reader.read_bam(path)
    text = re.sub(r"(?m)^(@PG\tID:rsem-tbam2gbam\tCL:)\S+", r"\1<argv0>", text)
    lines = [json.dumps(text), json.dumps(refs)]
    for r in recs:
        tags = [[k, t, v.hex() if isinstance(v, float) else v] for k, (t, v) in r["tags"].items()]
        rr = {k: r[k] for k in ("qname", "flag", "tid", "pos", "mapq", "bin", "cigar", "mtid", "mpos", "tlen", "seq", "qual")}
        lines.append(json.dumps([rr, tags]))
    return "\n".join(lines) + "\n"


def _rundir(d, name):
    w = d.rstrip("/") + "_" + name
    os.makedirs(w, exist_ok=True)
    for f in ("ref", "in.bam"):
        if not os.path.lexists(os.path.join(w, f)):
            os.symlink(os.path.join(d, f), os.path.join(w, f))
    return w


def run_pair(key, d, ours_args=(), env=None, ref_args=()):
    """the reference and ours on d/ref/r + d/in.bam, both as `<exe> ref/r in.bam g.bam`, each in its own directory.
    -> (reference result, our CompletedProcess, sha256 of the reference's canonical text, our canonical text or None).
    Without oracle/_ref the reference's stdout, status and digests come from tests/golden/reference/tbam2gbam_<key>."""
    wr = _rundir(d, "ref")

    def run():
        p = subprocess.run([REF_EXE, "ref/r", "in.bam", "g.bam", *ref_args], cwd=wr, stdout=subprocess.PIPE,
                           stderr=subprocess.PIPE, text=True)
        if p.returncode == 0:
            with open(os.path.join(wr, "g.txt"), "w") as f:
                f.write(canonical(os.path.join(wr, "g.bam")))
        return p
    ref = rf.reference_run("tbam2gbam_" + key, d, run, out=wr, digests_only=True)
    wo = _rundir(d, "ours")
    e = dict(os.environ)
    e.update(env or {})
    ours = subprocess.run([OUR_EXE, "ref/r", "in.bam", "g.bam", *ours_args], cwd=wo, stdout=subprocess.PIPE,
                          stderr=subprocess.PIPE, text=True, env=e)
    text = canonical(os.path.join(wo, "g.bam")) if ours.returncode == 0 else None
    return ref, ours, ref.digests.get("g.txt"), text


def sha(text):
    return hashlib.sha256(text.encode()).hexdigest()
