"""Benchmark of bin/rsem-tbam2gbam against the reference's rsem-tbam2gbam (oracle/_ref) on one genome-mode data set.

Generates a paired-end data set in genome mode (tools/gen_dataset --genome 1 --sam 1), gets its transcript BAM from
bin/rsem-run-em -b (MAPQ and ZW from our EM, as the driver produces it), then times the reference and ours on it in the
same call, checks that the decoded outputs are equal and prints one JSON line: wall times, our phases from
RSEM_B200_TIMING=1, and the card's name and power limit read in the same call.

  python tools/bench_tbam2gbam.py [--N1 10000000] [--M 20000] [--threads 0] [--work DIR]
"""
import argparse
import gzip
import json
import os
import re
import struct
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import rsem_files as rf  # noqa: E402
import tbam2gbam as tg  # noqa: E402


def same_records(a, b):
    """-> the two BAM files hold the same header, apart from argv[0] in our @PG CL:, and the same record bytes.  Streams
    both decompressed files, so that outputs of many GB compare in bounded memory and time."""
    fa, fb = gzip.open(a, "rb"), gzip.open(b, "rb")

    def header(f):
        h = f.read(8)
        text = f.read(struct.unpack_from("<i", h, 4)[0]).rstrip(b"\0").decode()
        n_ref = struct.unpack("<i", f.read(4))[0]
        refs = []
        for _ in range(n_ref):
            name = f.read(struct.unpack("<i", f.read(4))[0])
            refs.append((name, f.read(4)))
        return re.sub(r"(?m)^(@PG\tID:rsem-tbam2gbam\tCL:)\S+", r"\1<argv0>", text), refs
    if header(fa) != header(fb):
        return False
    while True:   # after the header the streams are the records: compare them in large chunks
        x, y = fa.read(1 << 24), fb.read(1 << 24)
        if x != y:
            return False
        if not x:
            return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N1", type=int, default=10_000_000, help="paired-end reads")
    ap.add_argument("--M", type=int, default=20000)
    ap.add_argument("--avg-family", type=float, default=5.0, help="mean isoforms per gene (alignments per read)")
    ap.add_argument("--threads", type=int, default=0, help="-p for ours (0: the default, no -p, as the driver runs it)")
    ap.add_argument("--work", default=None, help="directory for the data (default: a temporary one)")
    a = ap.parse_args()
    work = a.work or tempfile.mkdtemp(prefix="bench_tbam2gbam_")
    os.makedirs(work, exist_ok=True)
    d = os.path.join(work, "d")
    t0 = time.time()
    rf.gen_dataset(d, read_type=3, M=a.M, N1=a.N1, N0=a.N1 // 50, genome=1, sam=1, polyA=0, seed=21,
                    avg_family=a.avg_family)
    t_gen = time.time() - t0
    print(f"generated in {t_gen:.1f} s", file=sys.stderr, flush=True)
    t0 = time.time()
    p = rf.run_em(d, 3, "ours", threads=os.cpu_count() or 8, gibbs_out=False, extra=("-b", "aln.sam", "0"))
    t_em = time.time() - t0
    print(f"rsem-run-em -b in {t_em:.1f} s", file=sys.stderr, flush=True)
    os.replace(os.path.join(d, "s.transcript.bam"), os.path.join(d, "in.bam"))
    os.remove(os.path.join(d, "aln.sam"))
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                         text=True).stdout.strip()

    def run(exe, name, args=(), env=None):
        w = tg._rundir(d, name)
        e = dict(os.environ)
        e.update(env or {})
        t = time.time()
        p = subprocess.run([exe, "ref/r", "in.bam", "g.bam", *args], cwd=w, env=e, stdout=subprocess.PIPE,
                           stderr=subprocess.PIPE, text=True)
        dt = time.time() - t
        print(f"{exe}: {dt:.1f} s", file=sys.stderr, flush=True)
        if p.returncode != 0:
            raise RuntimeError(f"{exe} failed ({p.returncode}): {p.stderr[-2000:]}")
        return w, dt, p
    wo, t_ours, po = run(tg.OUR_EXE, "ours", ("-p", str(a.threads)) if a.threads else (), {"RSEM_B200_TIMING": "1"})
    print(po.stderr.strip(), file=sys.stderr, flush=True)
    wr, t_ref, pr = run(tg.REF_EXE, "ref")
    same_stdout = pr.stdout == po.stdout
    equal = same_records(os.path.join(wr, "g.bam"), os.path.join(wo, "g.bam"))
    m = re.search(r"rsem-tbam2gbam timing: .*", po.stderr)
    phases = {}
    if m:
        for k, v in re.findall(r"([a-z+ ]+?) ([0-9.]+) s", m.group(0)):
            phases[k.strip()] = float(v)
    print(json.dumps({
        "gpu": gpu, "N1_pairs": a.N1, "M": a.M, "out_bam_bytes": os.path.getsize(os.path.join(wo, "g.bam")),
        "in_bam_bytes": os.path.getsize(os.path.join(d, "in.bam")),
        "ref_wall_s": round(t_ref, 3), "ours_wall_s": round(t_ours, 3), "speedup": round(t_ref / t_ours, 2),
        "ours_phases_s": phases, "ours_timing_line": m.group(0) if m else None,
        "outputs_equal": equal, "stdout_equal": same_stdout,
        "gen_s": round(t_gen, 1), "rsem_run_em_b_s": round(t_em, 1), "cpus": os.cpu_count(),
    }))
    return 0 if equal and same_stdout else 1


if __name__ == "__main__":
    sys.exit(main())
