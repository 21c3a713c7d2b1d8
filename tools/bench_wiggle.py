"""Benchmark of bin/rsem-bam2wig and bin/rsem-bam2readdepth against the reference's tools (oracle/_ref).

Generates a paired-end data set in genome mode with the arguments tools/bench_tbam2gbam.py uses, gets its transcript BAM
from bin/rsem-run-em -b and its genome BAM from bin/rsem-tbam2gbam, sorts both with rsem-b200-host-selftest --bam-sort,
then times, in the same call, the reference and ours: rsem-bam2wig on the sorted genome BAM and rsem-bam2readdepth on
the sorted transcript BAM.  Checks that the outputs' SHA-256 and stdout are equal and prints one JSON line: wall times,
our phases from RSEM_B200_TIMING=1, and the card's name and power limit read in the same call.

  python tools/bench_wiggle.py [--N1 10000000] [--M 20000] [--work DIR]
"""
import argparse
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
import rsem_files as rf  # noqa: E402
import tbam2gbam as tg  # noqa: E402
import wiggle as wg  # noqa: E402


def sha_file(path):
    h = hashlib.sha256()
    with open(path, "rb") as f:
        for block in iter(lambda: f.read(1 << 24), b""):
            h.update(block)
    return h.hexdigest()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N1", type=int, default=10_000_000, help="paired-end reads")
    ap.add_argument("--M", type=int, default=20000)
    ap.add_argument("--avg-family", type=float, default=5.0, help="mean isoforms per gene (alignments per read)")
    ap.add_argument("--work", default=None, help="directory for the data (default: a temporary one)")
    a = ap.parse_args()
    work = a.work or tempfile.mkdtemp(prefix="bench_wiggle_")
    os.makedirs(work, exist_ok=True)
    d = os.path.join(work, "d")
    threads = str(os.cpu_count() or 8)
    t0 = time.time()
    rf.gen_dataset(d, read_type=3, M=a.M, N1=a.N1, N0=a.N1 // 50, genome=1, sam=1, polyA=0, seed=21,
                   avg_family=a.avg_family)
    rf.run_em(d, 3, "ours", threads=os.cpu_count() or 8, gibbs_out=False, extra=("-b", "aln.sam", "0"))
    os.remove(os.path.join(d, "aln.sam"))
    subprocess.check_call([tg.OUR_EXE, "ref/r", "s.transcript.bam", "g.bam"], cwd=d, stdout=subprocess.DEVNULL)
    wg.sort_bam(os.path.join(d, "s.transcript.bam"), os.path.join(d, "t.sorted.bam"), int(threads))
    wg.sort_bam(os.path.join(d, "g.bam"), os.path.join(d, "g.sorted.bam"), int(threads))
    for f in ("s.transcript.bam", "g.bam"):
        os.remove(os.path.join(d, f))
    t_prep = time.time() - t0
    print(f"inputs ready in {t_prep:.1f} s", file=sys.stderr, flush=True)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                         text=True).stdout.strip()

    def run(exe, args, env=None):
        e = dict(os.environ)
        e.update(env or {})
        t = time.time()
        p = subprocess.run([exe, *args], cwd=d, env=e, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
        dt = time.time() - t
        print(f"{exe}: {dt:.1f} s", file=sys.stderr, flush=True)
        if p.returncode != 0:
            raise RuntimeError(f"{exe} failed ({p.returncode}): {p.stderr[-2000:]}")
        return dt, p

    out = {"gpu": gpu, "N1_pairs": a.N1, "M": a.M, "cpus": os.cpu_count(), "prep_s": round(t_prep, 1),
           "genome_bam_bytes": os.path.getsize(os.path.join(d, "g.sorted.bam")),
           "transcript_bam_bytes": os.path.getsize(os.path.join(d, "t.sorted.bam"))}
    ok = True
    for tool, bam, args in (("wig", "g.sorted.bam", ["g.sorted.bam", "{}.wig", "bench"]),
                            ("depth", "t.sorted.bam", ["t.sorted.bam", "{}.depth"])):
        t_ours, po = run(wg.our_exe(tool), [x.format("ours") for x in args], {"RSEM_B200_TIMING": "1"})
        t_ref, pr = run(wg.ref_exe(tool), [x.format("ref") for x in args])
        ext = args[1][2:]
        equal = sha_file(os.path.join(d, "ours" + ext)) == sha_file(os.path.join(d, "ref" + ext))
        m = re.search(r"timing: .*", po.stderr)
        phases = {k.strip(): float(v) for k, v in re.findall(r"([a-z+ ]+?) ([0-9.]+) s", m.group(0))} if m else {}
        out[wg.TOOLS[tool]] = {"input": bam, "ref_wall_s": round(t_ref, 3), "ours_wall_s": round(t_ours, 3),
                               "speedup": round(t_ref / t_ours, 2), "ours_phases_s": phases,
                               "ours_timing_line": m.group(0) if m else None,
                               "output_bytes": os.path.getsize(os.path.join(d, "ours" + ext)),
                               "outputs_equal": equal, "stdout_equal": po.stdout == pr.stdout}
        ok = ok and equal and po.stdout == pr.stdout
    print(json.dumps(out))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
