#!/usr/bin/env python
"""Whole-executable timing of rsem-for-ebseq-calculate-clustering-info (H100) on a seeded synthetic transcriptome:
gene families whose isoforms share exon bodies, N runs, soft-masked lowercase stretches and a few exact copies
(tests/clustering_info.py).  With --reference the reference tool (oracle/_ref, built by oracle/ebseq.mk) runs on the
same file, and both stdout and the output file must be byte-identical before any number is printed.

Reported, as one JSON line:
  ours_wall_s, ours_load_s     wall time of the executable, and its FASTA load (RSEM_B200_TIMING=1)
  ours_device_s                device time per K9 phase (CUDA events): pack, insert, count
  passes, positions, table_slots, positions_per_s (positions over the executable's wall time)
  fasta_sha256, output_sha256 the generated input and our output file, so runs on other machines can be compared
  ref_wall_s, speedup_wall     with --reference
  gpu                          name, power limit and SM clock of the card (nvidia-smi), read in the same run"""
import argparse
import filecmp
import hashlib
import json
import os
import re
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import clustering_info as ci  # noqa: E402


def _size(s):
    mult = {"K": 10 ** 3, "M": 10 ** 6, "G": 10 ** 9}
    return int(float(s[:-1]) * mult[s[-1].upper()]) if s[-1].upper() in mult else int(s)


def _timed(exe, d, k, env=None):
    t0 = time.perf_counter()
    p = ci.run(exe, d, str(k), env=env)
    return p, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", default="33M", help="bases of the transcriptome, e.g. 33M or 400M")
    ap.add_argument("--k", type=int, default=25)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--reference", action="store_true", help="also run the reference tool and compare the outputs")
    a = ap.parse_args()
    if a.reference and not os.path.exists(ci.REF_BIN):
        sys.exit(f"{ci.REF_BIN} is not built (oracle/ebseq.mk needs the reference sources)")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    out = {"size": a.size, "k": a.k, "seed": a.seed, "gpu": gpu}
    with tempfile.TemporaryDirectory(prefix="rsem_ebseq_") as tmp:
        t0 = time.perf_counter()
        names, seqs = ci.family_transcriptome(_size(a.size), a.seed)
        data = ci.to_fasta(names, seqs)
        out.update(transcripts=len(names), bases=sum(len(s) for s in seqs), generate_s=round(time.perf_counter() - t0, 2))
        del seqs
        ours = ci.write_case(os.path.join(tmp, "ours"), data)
        out["fasta_sha256"] = hashlib.sha256(data).hexdigest()
        del data
        p, wall = _timed(ci.BIN, ours, a.k, env={**os.environ, "RSEM_B200_TIMING": "1"})
        assert p.returncode == 0, p.stderr[-2000:]
        m = re.search(r"FASTA load ([\d.]+) s, total [\d.]+ s; device: pack ([\d.]+) s, insert ([\d.]+) s, count ([\d.]+) s, "
                      r"(\d+) passes, (\d+) positions, (\d+) table slots", p.stderr)
        out.update(ours_wall_s=round(wall, 3), ours_load_s=float(m.group(1)),
                   ours_device_s={"pack": float(m.group(2)), "insert": float(m.group(3)), "count": float(m.group(4))},
                   passes=int(m.group(5)), positions=int(m.group(6)), table_slots=int(m.group(7)),
                   positions_per_s=round(int(m.group(6)) / wall))
        with open(os.path.join(ours, ci.OUT), "rb") as f:
            out["output_sha256"] = hashlib.sha256(f.read()).hexdigest()
        if a.reference:
            ref = os.path.join(tmp, "ref")
            os.makedirs(ref)
            os.link(os.path.join(ours, ci.FA), os.path.join(ref, ci.FA))
            r, rwall = _timed(ci.REF_BIN, ref, a.k)
            assert r.returncode == 0, r.stderr[-2000:]
            assert r.stdout == p.stdout, "stdout differs"
            assert filecmp.cmp(os.path.join(ref, ci.OUT), os.path.join(ours, ci.OUT), shallow=False), "output differs"
            out.update(identical_output=True, ref_wall_s=round(rwall, 2), speedup_wall=round(rwall / wall, 1))
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
