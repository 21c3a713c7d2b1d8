"""rsem-run-gibbs-batch against bin/rsem-run-gibbs run once per sample (and, with --reference, oracle/_ref/rsem-run-gibbs
on a time-bounded subset), with the driver's Gibbs arguments for --calc-pme / --calc-ci (200 1000 1 -p 8
--pseudo-count 0.1, rsem-calculate-expression).

Three workloads, against one reference of --transcripts transcripts (50 000 by default):
  single-cell        --samples samples of --reads reads, few families expressed (--expressed-frac 0.05), no spurious hits:
                     many small components, every sample in the batch (K13);
  single-cell-giant  the same with --spurious 0.01: most reads join one giant component (one walker per chain);
  bulk               --bulk-samples samples of --bulk-reads reads, above the batch's size rule (2^19 reads): every sample
                     on the single-sample path of rsem-run-gibbs.
The .ofg / .model inputs come from rsem-run-em-batch --gibbs-out (not timed).  Every output file of the batch run is
compared with bin/rsem-run-gibbs's before any time is printed.  Prints one JSON line per workload: wall time per sample of
both programs (and of the reference), K13 device time (CUDA events), the share of chain cycles spent in the per-kept-draw
O(M) work (ChainSync::prof[3]), the phase split of the batch run, the bytes of count-vector text written, and the card's
name and power limit read in the same run.  The work directory is deleted at the end.

  python tools/bench_gibbs_batch.py [--samples 16] [--reads 75000] [--bulk-samples 1] [--bulk-reads 600000]
                                    [--transcripts 50000] [--reference] [--reference-seconds 600] [--workdir DIR]
"""
import argparse
import filecmp
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import rsem_files as rf  # noqa: E402

GIBBS_ARGS = "200 1000 1 -p 8 --pseudo-count 0.1"
THREADS = 8


def log(msg):
    print(f"[bench_gibbs_batch {time.strftime('%H:%M:%S')}] {msg}", file=sys.stderr, flush=True)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, text=True, check=True).stdout.splitlines()[0]
    name, power = [x.strip() for x in out.split(",")]
    return name, power


def make(root, n, reads, M, spurious, frac):
    """n samples sharing one reference, after rsem-run-em-batch --gibbs-out"""
    os.makedirs(root)
    for k in range(n):
        rf.gen_dataset(os.path.join(root, f"d{k}"), read_type=0, M=M, N1=reads, N0=reads // 20, seed=5, sample_seed=300 + k,
                       spurious=spurious, expressed_frac=frac)
    with open(os.path.join(root, "em_manifest"), "w") as f:
        f.write("".join(f"d{k}/s d{k}/s.temp/s d{k}/s.stat/s --gibbs-out\n" for k in range(n)))
    subprocess.run([os.path.join(rf.BIN_DIR, "rsem-run-em-batch"), "d0/ref/r", "0", "em_manifest", "-q", "-p", "8"], cwd=root,
                   check=True, stdout=subprocess.DEVNULL)


def files(k):
    return [f"d{k}/s.temp/s.countvectors{t}" for t in range(THREADS)] + [f"d{k}/s.temp/s.iso_res", f"d{k}/s.temp/s.gene_res"]


def workload(work, name, n, reads, M, spurious, frac, reference, ref_seconds):
    root = os.path.join(work, name)
    log(f"{name}: generating {n} samples of {reads} reads")
    make(root, n, reads, M, spurious, frac)
    single = root + ".single"
    shutil.copytree(root, single)
    with open(os.path.join(root, "manifest"), "w") as f:
        f.write("".join(f"d{k}/s.temp/s d{k}/s.stat/s {GIBBS_ARGS} --seed {17 + k}\n" for k in range(n)))
    log(f"{name}: rsem-run-gibbs-batch")
    t0 = time.time()
    p = subprocess.run([os.path.join(rf.BIN_DIR, "rsem-run-gibbs-batch"), "d0/ref/r", "manifest", "-q"], cwd=root,
                       env=dict(os.environ, RSEM_B200_TIMING="1"), capture_output=True, text=True)
    t_batch = time.time() - t0
    if p.returncode != 0:
        raise RuntimeError(p.stderr[-3000:])
    log(f"{name}: bin/rsem-run-gibbs once per sample")
    t0 = time.time()
    for k in range(n):
        subprocess.run([os.path.join(rf.BIN_DIR, "rsem-run-gibbs"), "d0/ref/r", f"d{k}/s.temp/s", f"d{k}/s.stat/s",
                        *GIBBS_ARGS.split(), "--seed", str(17 + k), "-q"], cwd=single, check=True, capture_output=True)
    t_single = time.time() - t0
    for k in range(n):
        for f in files(k):
            if not filecmp.cmp(os.path.join(root, f), os.path.join(single, f), shallow=False):
                raise RuntimeError(f"{name}: {f} differs between rsem-run-gibbs-batch and rsem-run-gibbs")
    err = p.stderr
    m1 = re.search(r"(\d+) samples in the batch, (\d+) on the single-sample path; K13 ([\d.]+) ms, (\d+) jobs, (\d+) teams of "
                   r"(\d+) worker CTAs, per-kept-draw work ([\d.]+) of chain cycles", err)
    m2 = re.search(r"load\+components ([\d.]+) s, device ([\d.]+) s, copies back ([\d.]+) s, writers ([\d.]+) s \(thread seconds\), "
                   r"count-vector text (\d+) bytes", err)
    res = dict(workload=name, samples=n, reads=reads, transcripts=M, spurious=spurious, expressed_frac=frac,
               gibbs_args=GIBBS_ARGS, batch_s_per_sample=t_batch / n, single_s_per_sample=t_single / n,
               speedup=t_single / t_batch, batched=int(m1.group(1)), single_path=int(m1.group(2)),
               k13_ms=float(m1.group(3)), jobs=int(m1.group(4)), teams=int(m1.group(5)), worker_ctas=int(m1.group(6)),
               per_kept_draw_share=float(m1.group(7)), phase_s=dict(load_components=float(m2.group(1)),
                                                                     device=float(m2.group(2)), copies_back=float(m2.group(3)),
                                                                     writers_thread_s=float(m2.group(4))),
               countvector_bytes=int(m2.group(5)), reference_s_per_sample="not measured")
    if reference and rf.have_ref():
        ref = root + ".ref"
        shutil.copytree(single, ref)
        done, t0 = 0, time.time()
        for k in range(n):
            if time.time() - t0 > ref_seconds:
                break
            log(f"{name}: reference rsem-run-gibbs on sample {k}")
            subprocess.run([os.path.join(rf.REF_DIR, "rsem-run-gibbs"), "d0/ref/r", f"d{k}/s.temp/s", f"d{k}/s.stat/s",
                            *GIBBS_ARGS.split(), "--seed", str(17 + k), "-q"], cwd=ref, check=True, capture_output=True)
            done += 1
        res.update(reference_s_per_sample=(time.time() - t0) / done, reference_samples=done)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=16)
    ap.add_argument("--reads", type=int, default=75000)
    ap.add_argument("--bulk-samples", type=int, default=1)
    ap.add_argument("--bulk-reads", type=int, default=600000)
    ap.add_argument("--transcripts", type=int, default=50000)
    ap.add_argument("--reference", action="store_true")
    ap.add_argument("--reference-seconds", type=float, default=600.0)
    ap.add_argument("--workdir", default=None)
    ap.add_argument("--only", default=None, help="comma-separated workload names")
    a = ap.parse_args()
    work = tempfile.mkdtemp(prefix="bench_gibbs_batch_", dir=a.workdir)
    try:
        name, power = card()
        specs = [("single-cell", a.samples, a.reads, 0.0, 0.05), ("single-cell-giant", a.samples, a.reads, 0.01, 0.05),
                 ("bulk", a.bulk_samples, a.bulk_reads, 0.0, 1.0)]
        for wl, n, reads, spurious, frac in specs:
            if a.only and wl not in a.only.split(","):
                continue
            res = workload(work, wl, n, reads, a.transcripts, spurious, frac, a.reference, a.reference_seconds)
            res.update(gpu=name, power_limit=power)
            print(json.dumps(res), flush=True)
    finally:
        shutil.rmtree(work, ignore_errors=True)


if __name__ == "__main__":
    main()
