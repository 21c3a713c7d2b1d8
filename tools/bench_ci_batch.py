"""rsem-calculate-credibility-intervals-batch against bin/rsem-calculate-credibility-intervals run once per sample, with
the driver's --calc-ci --single-cell-prior arguments (0.95 1000 50 1024 -p 8 --pseudo-count 0.1, rsem-calculate-expression).

A single-cell cohort of --samples samples of --reads reads against one reference of --transcripts transcripts (few
families expressed, as tools/bench_gibbs_batch.py's single-cell workload): .ofg / .model from rsem-run-em-batch
--gibbs-out and count vectors from rsem-run-gibbs-batch with the driver's Gibbs arguments (200 1000 1 -p 8
--pseudo-count 0.1), none of it timed.  Then, --repeats times and alternating, each in its own copy of the cohort:
  single   bin/rsem-calculate-credibility-intervals once per sample;
  batch    the batch on one lane;
  lanes    the batch on --lanes lanes of device 0 (RSEM_B200_DEVICES=0,0,...; default host cores / 8, at least 2).
Every result file of every run is compared with the single runs' before any time is printed.  Prints one JSON line:
wall seconds per sample of each way (best and all repeats), the host sampling time (RSEM_B200_TIMING: the single runs'
sampling seconds times their sampler threads, the batch's sampler thread-seconds) and the Phase II device time of the
last repeat, the host core count, and the card's name and power limit read in the same run.  The work directory is
deleted at the end.

  python tools/bench_ci_batch.py [--samples 16] [--reads 75000] [--transcripts 50000] [--lanes K] [--repeats 1]
                                 [--workdir DIR]
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
CI_ARGS = "0.95 1000 50 1024 -p 8 --pseudo-count 0.1"
SINGLE = os.path.join(rf.BIN_DIR, "rsem-calculate-credibility-intervals")
BATCH = os.path.join(rf.BIN_DIR, "rsem-calculate-credibility-intervals-batch")


def log(msg):
    print(f"[bench_ci_batch {time.strftime('%H:%M:%S')}] {msg}", file=sys.stderr, flush=True)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, text=True, check=True).stdout.splitlines()[0]
    name, power = [x.strip() for x in out.split(",")]
    return name, power


def make(root, n, reads, M):
    """n samples sharing one reference, after rsem-run-em-batch --gibbs-out and rsem-run-gibbs-batch"""
    os.makedirs(root)
    for k in range(n):
        rf.gen_dataset(os.path.join(root, f"d{k}"), read_type=0, M=M, N1=reads, N0=reads // 20, seed=5, sample_seed=300 + k,
                       spurious=0.0, expressed_frac=0.05)
    with open(os.path.join(root, "em_manifest"), "w") as f:
        f.write("".join(f"d{k}/s d{k}/s.temp/s d{k}/s.stat/s --gibbs-out\n" for k in range(n)))
    subprocess.run([os.path.join(rf.BIN_DIR, "rsem-run-em-batch"), "d0/ref/r", "0", "em_manifest", "-q", "-p", "8"], cwd=root,
                   check=True, stdout=subprocess.DEVNULL)
    with open(os.path.join(root, "gibbs_manifest"), "w") as f:
        f.write("".join(f"d{k}/s.temp/s d{k}/s.stat/s {GIBBS_ARGS} --seed {17 + k}\n" for k in range(n)))
    subprocess.run([os.path.join(rf.BIN_DIR, "rsem-run-gibbs-batch"), "d0/ref/r", "gibbs_manifest", "-q"], cwd=root,
                   check=True, stdout=subprocess.DEVNULL)
    with open(os.path.join(root, "manifest"), "w") as f:
        f.write("".join(f"d{k}/s.temp/s d{k}/s.stat/s {CI_ARGS} --seed {29 + k}\n" for k in range(n)))


def run_single(root, n):
    env = dict(os.environ, RSEM_B200_TIMING="1")
    sampling = device = 0.0
    t0 = time.time()
    for k in range(n):
        p = subprocess.run([SINGLE, "d0/ref/r", f"d{k}/s.temp/s", f"d{k}/s.stat/s", *CI_ARGS.split(), "--seed", str(29 + k),
                            "-q"], cwd=root, env=env, capture_output=True, text=True)
        if p.returncode != 0:
            raise RuntimeError(p.stderr[-3000:])
        m = re.search(r"sampling \(host, (\d+) threads\) ([\d.]+) s, intervals [\d.]+ s; device: transpose ([\d.]+) s, "
                      r"sums ([\d.]+) s, sort ([\d.]+) s, intervals ([\d.]+) s", p.stderr)
        sampling += int(m.group(1)) * float(m.group(2))
        device += sum(float(m.group(i)) for i in range(3, 7))
    return time.time() - t0, sampling, device


def run_batch(root, lanes):
    env = dict(os.environ, RSEM_B200_TIMING="1")
    env.pop("RSEM_B200_DEVICES", None)
    env.pop("RSEM_B200_DEVICE", None)
    if lanes > 1:
        env["RSEM_B200_DEVICES"] = ",".join(["0"] * lanes)
    t0 = time.time()
    p = subprocess.run([BATCH, "d0/ref/r", "manifest", "-q"], cwd=root, env=env, capture_output=True, text=True)
    wall = time.time() - t0
    if p.returncode != 0:
        raise RuntimeError(p.stderr[-3000:])
    sampling = device = 0.0
    for m in re.finditer(r"sampling ([\d.]+) thread-s .*device: transpose ([\d.]+) s, sums ([\d.]+) s, sort ([\d.]+) s, "
                         r"intervals ([\d.]+) s", p.stderr):
        sampling += float(m.group(1))
        device += sum(float(m.group(i)) for i in range(2, 6))
    return wall, sampling, device


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=16)
    ap.add_argument("--reads", type=int, default=75000)
    ap.add_argument("--transcripts", type=int, default=50000)
    ap.add_argument("--lanes", type=int, default=0, help="lanes on device 0 (0: host cores / 8, at least 2)")
    ap.add_argument("--repeats", type=int, default=1)
    ap.add_argument("--workdir", default=None)
    a = ap.parse_args()
    cores = os.cpu_count()
    lanes = a.lanes or max(2, cores // 8)
    n = a.samples
    work = tempfile.mkdtemp(prefix="bench_ci_batch_", dir=a.workdir)
    try:
        name, power = card()
        base = os.path.join(work, "cohort")
        log(f"generating {n} samples of {a.reads} reads, EM and Gibbs (not timed)")
        make(base, n, a.reads, a.transcripts)
        times = {"single": [], "batch": [], "lanes": []}
        last = {}
        for r in range(a.repeats):
            for way in times:
                d = os.path.join(work, f"{way}{r}")
                shutil.copytree(base, d)
                log(f"repeat {r}: {way}")
                res = run_single(d, n) if way == "single" else run_batch(d, 1 if way == "batch" else lanes)
                times[way].append(res[0])
                last[way] = res
            for way in ("batch", "lanes"):
                for k in range(n):
                    for f in ("s.iso_res", "s.gene_res"):
                        rel = os.path.join(f"d{k}", "s.temp", f)
                        if not filecmp.cmp(os.path.join(work, f"single{r}", rel), os.path.join(work, f"{way}{r}", rel),
                                           shallow=False):
                            raise RuntimeError(f"{rel} differs between the single runs and the {way} run")
            for way in times:
                shutil.rmtree(os.path.join(work, f"{way}{r}"))
        res = dict(workload="single-cell", samples=n, reads=a.reads, transcripts=a.transcripts, ci_args=CI_ARGS,
                   gibbs_args=GIBBS_ARGS, lanes=lanes, host_cores=cores, repeats=a.repeats,
                   s_per_sample={w: min(t) / n for w, t in times.items()},
                   all_s_per_sample={w: [x / n for x in t] for w, t in times.items()},
                   host_sampling_thread_s={w: last[w][1] for w in last},
                   phase2_device_s={w: last[w][2] for w in last}, gpu=name, power_limit=power)
        print(json.dumps(res), flush=True)
    finally:
        shutil.rmtree(work, ignore_errors=True)


if __name__ == "__main__":
    main()
