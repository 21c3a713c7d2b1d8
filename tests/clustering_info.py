"""Helpers for the rsem-for-ebseq-calculate-clustering-info tests and benchmark: the input cases, a seeded generator of
family-structured transcriptomes, a Python restatement of the reference's FASTA reading (loadRef,
EBSeq/calcClusteringInfo.cpp:61-90), the binding of oracle/libkmer_oracle.so (the sort-based C restatement of the
counts), and the reference run.  Test infrastructure."""
import ctypes as C
import os
import subprocess

import numpy as np

import rsem_files as rf

TOOL = "rsem-for-ebseq-calculate-clustering-info"
BIN = os.path.join(rf.BIN_DIR, TOOL)
REF_BIN = os.path.join(rf.REF_DIR, TOOL)
ORACLE = os.path.join(rf.ROOT, "oracle", "libkmer_oracle.so")
FA, OUT = "t.fa", "t.out"

_CODE = np.full(256, 4, np.uint8)
for _i, _ch in enumerate(b"ACGT"):
    _CODE[_ch] = _CODE[_ch + 32] = _i


# ---- inputs ------------------------------------------------------------------------------------------------------
def family_transcriptome(total_bases, seed, iupac=False):
    """-> (names, sequences as bytes) of about total_bases bases: gene families whose isoforms are subsets of one set of
    exons (so they share bodies), some N runs inside gene bodies (shared by the isoforms), soft-masked lowercase
    stretches, a few exact copies under other names and, with iupac, IUPAC codes in place of some bases"""
    rng = np.random.default_rng(seed)
    acgt = np.frombuffer(b"ACGT", np.uint8)
    names, seqs, total, fam = [], [], 0, 0
    while total < total_bases:
        n_ex = int(rng.integers(1, 9))
        lens = rng.integers(40, 700, n_ex)
        body = acgt[rng.integers(0, 4, int(lens.sum()))]
        if rng.random() < 0.08:   # an N run inside the gene body
            a = int(rng.integers(0, len(body)))
            body[a:a + int(rng.integers(5, 80))] = ord("N")
        if iupac and rng.random() < 0.3:
            at = rng.integers(0, len(body), 3)
            body[at] = np.frombuffer(b"RYK", np.uint8)
        bounds = np.concatenate([[0], np.cumsum(lens)])
        for i in range(int(rng.integers(1, 5))):
            keep = rng.random(n_ex) < 0.7
            keep[int(rng.integers(0, n_ex))] = True
            s = np.concatenate([body[bounds[e]:bounds[e + 1]] for e in range(n_ex) if keep[e]])
            if rng.random() < 0.15:   # soft-masked stretch
                a = int(rng.integers(0, len(s)))
                seg = s[a:a + int(rng.integers(10, 200))]
                s[a:a + len(seg)] = np.where(seg == ord("N"), seg, seg + 32)
            name = f"FAM{fam}.{i}" + (f" gene=G{fam} len={len(s)}" if rng.random() < 0.3 else "")
            names.append(name.encode())
            seqs.append(s.tobytes())
            total += len(s)
            if rng.random() < 0.01:
                names.append(f"COPY_OF_FAM{fam}.{i}".encode())
                seqs.append(seqs[-1])
                total += len(s)
        fam += 1
    return names, seqs


def to_fasta(names, seqs, width=60, eol=b"\n"):
    out = []
    for n, s in zip(names, seqs):
        out.append(b">" + n + eol)
        out.extend(s[i:i + width] + eol for i in range(0, len(s), width))
    return b"".join(out)


def _random(rng, n, alphabet=b"ACGT"):
    return np.frombuffer(alphabet, np.uint8)[rng.integers(0, len(alphabet), n)].tobytes()


def _crlf_iupac():
    rng = np.random.default_rng(5)
    core = _random(rng, 300)
    names, seqs = [], []
    for i in range(12):
        s = bytearray(_random(rng, int(rng.integers(20, 120))) + core[: int(rng.integers(30, 300))] + _random(rng, 40))
        for j in rng.integers(0, len(s), 4):
            s[j] = b"RYKMSWBDHVrykn-.*"[int(rng.integers(0, 17))]
        s = bytes(s).lower() if i % 3 == 0 else bytes(s)
        names.append(f"tr{i} some description".encode())
        seqs.append(s)
    return to_fasta(names, seqs, width=50, eol=b"\r\n")


def _dups():
    rng = np.random.default_rng(6)
    a, b, c = _random(rng, 200), _random(rng, 150), _random(rng, 90)
    names = [b"a", b"a_copy", b"b", b"a", b"c", b"b_lower", b"d"]
    seqs = [a, a, b, a, c, b.lower(), c[:40] + _random(rng, 60)]
    return to_fasta(names, seqs, width=70)


def _self_repeats():
    rng = np.random.default_rng(7)
    names, seqs = [], []
    for i in range(8):   # tandem repeats within each transcript only; the units differ between transcripts
        unit = _random(rng, int(rng.integers(3, 30)))
        seqs.append(unit * int(rng.integers(5, 20)) + _random(rng, 20))
        names.append(f"rep{i}".encode())
    seqs.append(seqs[0][:50])   # one that does share with rep0
    names.append(b"rep0_part")
    return to_fasta(names, seqs)


def _n_runs():
    rng = np.random.default_rng(8)
    names, seqs = [], []
    for i in range(6):
        seqs.append(_random(rng, 60) + b"N" * int(rng.integers(5, 40)) + _random(rng, 60) + b"n" * (i % 3) * 7)
        names.append(f"nrun{i}".encode())
    seqs.append(b"N" * 30)
    names.append(b"all_n")
    return to_fasta(names, seqs)


def _length_k(k):
    rng = np.random.default_rng(9)
    x = _random(rng, k + 30)
    names = [b"exact_k", b"k_minus_1", b"k_plus_1", b"exact_k_copy", b"long", b"k_minus_1_inside"]
    seqs = [x[:k], x[1:k], x[:k + 1], x[:k], x, x[5:k + 4]]
    return to_fasta(names, seqs, width=7)


QUIRK5 = b">a\nACGTRACGT\n>empty\n>b\nacgtyacgt\n>c\nAAAA\n>d\r\nACGTN\r\nACGT\n"
SMALL_FAMILY = lambda: to_fasta(*family_transcriptome(120_000, 21, iupac=True))
FAMILY_K = (1, 5, 25, 31, 32, 33, 64, 65, 150)

# key -> (k argument, FASTA bytes): every case the GPU tests run through the executable (and the C restatement checks)
DEVICE_CASES = {
    "ebseq_quirk5": ("5", lambda: QUIRK5),
    "ebseq_crlf_iupac": ("7", _crlf_iupac),
    "ebseq_dups": ("11", _dups),
    "ebseq_self_repeats": ("9", _self_repeats),
    "ebseq_n_runs": ("12", _n_runs),
    "ebseq_length_k": ("20", lambda: _length_k(20)),
    **{f"ebseq_k{k}": (str(k), SMALL_FAMILY) for k in FAMILY_K},
    "ebseq_family_k25": ("25", lambda: to_fasta(*family_transcriptome(3_000_000, 33))),
    "ebseq_family_k100": ("100", lambda: to_fasta(*family_transcriptome(3_000_000, 33))),
}
# cases without device work: no transcripts, no k-mer positions, or k <= 0 (atoi)
HOST_CASES = {
    "ebseq_no_header": ("5", lambda: b"ACGT\n>a\nACGTACGT\n>b\nACGTACGT\n"),
    "ebseq_all_short": ("50", lambda: QUIRK5),
    "ebseq_k0": ("0", lambda: QUIRK5),
    "ebseq_k_minus3": ("-3", lambda: QUIRK5),
    "ebseq_k_text": ("abc", lambda: QUIRK5),
    "ebseq_k0_one": ("0", lambda: b">only one\nACGTTT\n"),
}


def atoi(s):
    """C atoi for the arguments used here: leading sign and digits, 0 when there are none"""
    s = s.lstrip()
    i = 1 if s[:1] in ("-", "+") else 0
    while i < len(s) and s[i].isdigit():
        i += 1
    return int(s[:i]) if i and s[:i] not in ("-", "+") else 0


# ---- restatements ------------------------------------------------------------------------------------------------
def load_ref(data):
    """loadRef's reading of a FASTA (getline semantics) -> (names, offsets, base codes, warnings)"""
    lines = data.split(b"\n")
    if lines and lines[-1] == b"":   # nothing after a final '\n' is a line
        lines.pop()
    names, seqs, warnings = [], [], []
    it = iter(lines)
    line = next(it, None)
    while line is not None and line[:1] == b">":
        tag, raw = line[1:], []
        line = next(it, None)
        while line is not None and line[:1] != b">":
            raw.append(line)
            line = next(it, None)
        seq = b"".join(raw)
        if not seq:
            warnings.append(tag.split(b"\0")[0])
            continue
        names.append(tag)
        seqs.append(seq)
    off = np.zeros(len(seqs) + 1, np.uint64)
    off[1:] = np.cumsum([len(s) for s in seqs]) if seqs else []
    bases = _CODE[np.frombuffer(b"".join(seqs), np.uint8)] if seqs else np.zeros(0, np.uint8)
    return names, off, bases, warnings


def oracle_counts(k, off, bases):
    dll = C.CDLL(ORACLE)
    off, bases = np.ascontiguousarray(off, np.uint64), np.ascontiguousarray(bases, np.uint8)
    n = len(off) - 1
    counts = np.zeros(max(n, 1), np.uint64)
    assert dll.ko_shared_counts(C.c_int32(k), C.c_uint64(n), off.ctypes.data_as(C.POINTER(C.c_uint64)),
                                bases.ctypes.data_as(C.POINTER(C.c_uint8)), counts.ctypes.data_as(C.POINTER(C.c_uint64))) == 0
    return counts[:n]


def eff_lengths(k, off):
    return np.maximum(np.diff(off.astype(np.int64)) - k + 1, 0)


def output_text(names, counts, effl):
    """the output file (setprecision(6) is %.6g), :132-141"""
    return b"".join(n + b"\t" + (b"-1" if e == 0 else b"%.6g" % (int(c) / int(e))) + b"\n"
                    for n, c, e in zip(names, counts, effl))


def stdout_text(k, warnings):
    return "".join(f"Warning: Fasta entry {w.decode()} has an empty sequence! It is omitted!\n" for w in warnings) + \
        f"The reference is loaded.\nAll possbile {k} mers are generated.\nAll {k} mers are sorted.\n" \
        "Clustering information is calculated.\n"


# ---- runs --------------------------------------------------------------------------------------------------------
def write_case(d, data):
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, FA), "wb") as f:
        f.write(data)
    return d


def run(exe, d, k, env=None):
    return subprocess.run([exe, k, FA, OUT], cwd=d, capture_output=True, text=True, env=env)


def reference(key, d, k):
    """the reference tool's stdout and output digest on the case in d (oracle/_ref, or the stored run)"""
    import pytest
    if rf.have_ref() and not os.path.exists(REF_BIN):
        pytest.skip(f"oracle/_ref has no {TOOL}: rebuild the oracle (oracle/ebseq.mk)")
    return rf.reference_run(key, d, lambda: run(REF_BIN, d, k), digests_only=True)
