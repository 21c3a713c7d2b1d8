"""rsem-run-em-batch against bin/rsem-run-em run once per sample (and, with --reference, oracle/_ref/rsem-run-em).

Two workloads, one on each side of the rule that sends a sample to the batch (K12) or to the single-sample path:
  single-cell  many samples (default 264: two per H100 SM) of 5e4-5e5 reads against one reference of 50 000
               transcripts, few families expressed (--expressed-frac 0.05): every sample goes to the batch;
  bulk         a few samples with more than 2^20 alignments: every sample finishes on the single-sample path.
Every run is free-running (no RSEM_MAX_ROUND).  --reference times the reference on the single-cell workload only.  The outputs of the runs are compared before any time is printed.
Prints one JSON line per workload: wall time per sample of each program, K12 device time per sample-round (CUDA
events), K12's achieved bytes/s on 12 H + 16 N + 16 (m + 1) per sample-round against 3.35 TB/s, the phase split of
the batch run, and the card's name and power limit read in the same run.

  python tools/bench_em_batch.py [--samples 264] [--reads-min 50000] [--reads-max 500000] [--bulk-samples 3]
                                 [--bulk-reads 2000000] [--reference] [--workdir DIR]
"""
import argparse
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import rsem_files as rf  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def log(msg):
    print(f"[bench_em_batch {time.strftime('%H:%M:%S')}] {msg}", file=sys.stderr, flush=True)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, text=True, check=True).stdout.splitlines()[0]
    name, power = [x.strip() for x in out.split(",")]
    return name, power


def generate(root, n, reads_min, reads_max, M, frac, seed):
    rng = np.random.default_rng(seed)
    dirs = []
    for k in range(n):
        d = os.path.join(root, f"s{k}")
        N1 = int(rng.integers(reads_min, reads_max + 1))
        rf.gen_dataset(d, read_type=0, M=M, N1=N1, N0=N1 // 20, avg_family=2, seed=11, sample_seed=1000 + k,
                       expressed_frac=frac)
        if dirs:   # the reference is byte-identical in every sample (--sample-seed): keep one copy
            shutil.rmtree(os.path.join(d, "ref"))
            os.symlink(os.path.join(dirs[0], "ref"), os.path.join(d, "ref"))
        dirs.append(d)
        if (k + 1) % 32 == 0:
            log(f"generated {k + 1} of {n} samples")
    return dirs


def frozen_bytes_per_round(d):
    """12 H + 16 N + 16 (m + 1) of one frozen round in the sample's compact transcript space"""
    row_ptr, sid = rf.read_dat(os.path.join(d, "s.temp", "s.dat"), False)[:2]
    return 12 * len(sid) + 16 * (len(row_ptr) - 1) + 16 * (len(np.unique(np.abs(sid))) + 1)


def run_batch(root, dirs):
    with open(os.path.join(root, "manifest"), "w") as f:
        for d in dirs:
            b = os.path.basename(d)
            f.write(f"{b}/s {b}/s.temp/s {b}/s.stat/s\n")
    env = dict(os.environ, RSEM_B200_TIMING="1")
    t0 = time.perf_counter()
    p = subprocess.run([os.path.join(rf.BIN_DIR, "rsem-run-em-batch"), f"{os.path.basename(dirs[0])}/ref/r", "0",
                        "manifest", "-p", str(os.cpu_count())], cwd=root, env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.PIPE, text=True)
    wall = time.perf_counter() - t0
    if p.returncode != 0:
        raise RuntimeError(p.stderr[-3000:])
    k12 = re.search(r"K12 ([0-9.]+) ms over (\d+) sample-rounds", p.stderr)
    ph = re.search(r"load ([0-9.]+) s, model rounds ([0-9.]+) s, frozen rounds ([0-9.]+) s, final pass ([0-9.]+) s, "
                   r"writers ([0-9.]+) s", p.stderr)
    blocks = re.split(r"^== sample ", p.stdout, flags=re.M)[1:]
    frozen_rounds = [sum(1 for l in b.splitlines() if l.startswith("ROUND = ") and int(l.split()[2].rstrip(",")) > 10)
                     for b in blocks]
    return wall, float(k12.group(1)), int(k12.group(2)), [float(x) for x in ph.groups()], frozen_rounds


def run_each(dirs, exe_args, tag):
    """one process per sample on a copy of its directory; returns the summed wall time and the copies"""
    total, copies = 0.0, []
    for d in dirs:
        c = d + "_" + tag
        shutil.copytree(d, c, symlinks=True)
        if tag == "ref":   # the reference's rsem-run-em reads the read index rsem-calculate-expression builds first
            subprocess.check_call([os.path.join(rf.REF_DIR, "rsem-build-read-index"), "32", "0", "1",
                                   *rf.read_files(c, 0)], stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
        t0 = time.perf_counter()
        subprocess.run([*exe_args, "ref/r", "0", "s", "s.temp/s", "s.stat/s", "-p", str(os.cpu_count())], cwd=c,
                       check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
        total += time.perf_counter() - t0
        copies.append(c)
    return total, copies


def check_same(dirs, copies, what):
    for d, c in zip(dirs, copies):
        for x, y in zip(rf.read_theta(os.path.join(d, "s.stat", "s.theta")), rf.read_theta(os.path.join(c, "s.stat", "s.theta"))):
            if not rf.close_rel(x, y, 1e-6):
                raise AssertionError(f"{d}: theta differs from {what} by {rf.max_rel(x, y)}")


def workload(name, root, dirs, reference):
    bytes_per_round = [frozen_bytes_per_round(d) for d in dirs]
    wall_b, k12_ms, k12_rounds, phases, frozen = run_batch(root, dirs)
    log(f"{name}: rsem-run-em-batch {wall_b:.2f} s, K12 {k12_ms:.1f} ms over {k12_rounds} sample-rounds, "
        f"{sum(b * r for b, r in zip(bytes_per_round, frozen)) / max(k12_ms * 1e-3, 1e-12) / 1e9:.1f} GB/s, phases {phases}")
    wall_s, singles = run_each(dirs, [os.path.join(rf.BIN_DIR, "rsem-run-em")], "single")
    log(f"{name}: rsem-run-em per sample {wall_s:.2f} s")
    check_same(dirs, singles, "bin/rsem-run-em")
    out = dict(workload=name, samples=len(dirs), batch_s_per_sample=wall_b / len(dirs),
               rsem_run_em_s_per_sample=wall_s / len(dirs))
    if reference:
        wall_r, refs = run_each(dirs, [os.path.join(rf.REF_DIR, "rsem-run-em")], "ref")
        check_same(dirs, refs, "the reference")
        out["reference_s_per_sample"] = wall_r / len(dirs)
        out["reference_threads"] = os.cpu_count()
    if k12_rounds:
        k12_bytes = sum(b * r for b, r in zip(bytes_per_round, frozen))
        out.update(k12_us_per_sample_round=1e3 * k12_ms / k12_rounds, k12_sample_rounds=k12_rounds,
                   k12_bytes_per_s=k12_bytes / (k12_ms * 1e-3), k12_share_of_hbm=k12_bytes / (k12_ms * 1e-3) / HBM_BYTES_PER_S)
    out["batch_phases_s"] = dict(zip(("load", "model_rounds", "frozen_rounds", "final_pass", "writers"), phases))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=264)
    ap.add_argument("--reads-min", type=int, default=50000)
    ap.add_argument("--reads-max", type=int, default=500000)
    ap.add_argument("--M", type=int, default=50000)
    ap.add_argument("--expressed-frac", type=float, default=0.05)
    ap.add_argument("--bulk-samples", type=int, default=3)
    ap.add_argument("--bulk-reads", type=int, default=2000000)
    ap.add_argument("--reference", action="store_true")
    ap.add_argument("--workdir", default=None)
    a = ap.parse_args()
    name, power = card()
    work = a.workdir or tempfile.mkdtemp(prefix="bench_em_batch_")
    try:
        for wl, n, lo, hi, frac in (("single-cell", a.samples, a.reads_min, a.reads_max, a.expressed_frac),
                                    ("bulk", a.bulk_samples, a.bulk_reads, a.bulk_reads, 1.0)):
            if n <= 0:
                continue
            root = os.path.join(work, wl)
            os.makedirs(root, exist_ok=True)
            dirs = generate(root, n, lo, hi, a.M, frac, seed=len(wl))
            res = workload(wl, root, dirs, a.reference and wl == "single-cell")
            res.update(M=a.M, reads=[lo, hi], expressed_frac=frac, gpu=name, power_limit=power)
            print(json.dumps(res), flush=True)
    finally:
        if not a.workdir:
            shutil.rmtree(work, ignore_errors=True)


if __name__ == "__main__":
    main()
