"""rsem-simulate-reads-batch against bin/rsem-simulate-reads run once per sample, on two workloads on either side of the
trade-off between fixed cost and device time:
  replicates  --replicates samples of --replicate-reads paired-end reads with qualities (the pe_q_rspd golden model):
              the device draws most of the time;
  cells       --cells samples of --cell-reads single-end reads (the se_noq golden model): the fixed cost of a run
              (process, context, reference, tables) dominates.
Each sample has its own seed and theta0 against one reference.  Every workload is timed --repeats times in three ways,
alternating: bin/rsem-simulate-reads once per sample, the batch with one lane, and the batch with
RSEM_B200_DEVICES=0,0,0,0 (four lanes on one card).  Every output file of every run is compared (SHA-256) with the
first run's before any time is printed.  Prints one JSON line per workload: wall seconds per sample of each way (best
and all repeats), the per-lane device phase times and host load / write times of the last batch runs
(RSEM_B200_TIMING=1), and the card's name and power limit read in the same run.  The work directory is deleted at the end.

  python tools/bench_simulate_batch.py [--replicates 8] [--replicate-reads 20000000] [--cells 256] [--cell-reads 100000]
                                       [--repeats 2] [--workloads replicates,cells] [--workdir DIR]
"""
import argparse
import hashlib
import json
import os
import random
import shutil
import subprocess
import sys
import tarfile
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SINGLE = os.path.join(ROOT, "bin", "rsem-simulate-reads")
BATCH = os.path.join(ROOT, "bin", "rsem-simulate-reads-batch")


def log(msg):
    print(f"[bench_simulate_batch {time.strftime('%H:%M:%S')}] {msg}", file=sys.stderr, flush=True)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, text=True, check=True).stdout.splitlines()[0]
    name, power = [x.strip() for x in out.split(",")]
    return name, power


def inputs(work, name):
    """the golden data set's reference and model, and a results file with random TPMs"""
    d = os.path.join(work, name)
    with tarfile.open(os.path.join(ROOT, "tests", "golden", name + ".tar.gz")) as t:
        t.extractall(work, filter="data")
    M = int(open(os.path.join(d, "ref", "r.ti")).readline().split()[0])
    rng = random.Random(7)
    rows = ["transcript_id\tgene_id\tlength\teffective_length\texpected_count\tTPM\tFPKM\tIsoPct"]
    rows += [f"T{i}\tG\t1\t1\t1\t{rng.uniform(0, 100):.2f}\t0\t0" for i in range(1, M + 1)]
    open(os.path.join(d, "res.tsv"), "w").write("\n".join(rows) + "\n")
    return os.path.join(d, "ref", "r"), os.path.join(d, "out", "model20"), os.path.join(d, "res.tsv")


def digests(out):
    h = {}
    for f in sorted(os.listdir(out)):
        s = hashlib.sha256()
        with open(os.path.join(out, f), "rb") as fi:
            for b in iter(lambda: fi.read(1 << 24), b""):
                s.update(b)
        h[f] = s.hexdigest()
    return h


def workload(work, tag, name, n, reads, repeats):
    ref, model, res = inputs(work, name)
    root = os.path.join(work, tag)
    lines = [[model, res, str((0.05, 0.1, 0.2)[k % 3]), str(reads), os.path.join(root, f"s{k}", "s"), "--seed", str(100 + k)]
             for k in range(n)]
    manifest = os.path.join(work, tag + ".manifest")
    open(manifest, "w").write("".join(" ".join(l) + "\n" for l in lines))
    ways = {"single": None, "batch_1_lane": {}, "batch_4_lanes": {"RSEM_B200_DEVICES": "0,0,0,0"}}
    walls = {w: [] for w in ways}
    lanes = {}
    want = None
    for rep in range(repeats):
        for way, env in ways.items():
            shutil.rmtree(root, ignore_errors=True)
            for k in range(n):
                os.makedirs(os.path.join(root, f"s{k}"))
            e = {**os.environ, "RSEM_B200_TIMING": "1", **(env or {})}
            t0 = time.perf_counter()
            if env is None:
                for l in lines:
                    subprocess.run([SINGLE, ref, *l, "-q"], check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL, env=e)
            else:
                p = subprocess.run([BATCH, ref, manifest, "-q"], check=True, stdout=subprocess.DEVNULL, stderr=subprocess.PIPE,
                                   text=True, env=e)
            walls[way].append((time.perf_counter() - t0) / n)
            if env is not None:
                lanes[way] = [x for x in p.stderr.splitlines() if "timing: lane" in x]
            got = [digests(os.path.join(root, f"s{k}")) for k in range(n)]
            if want is None:
                want = got
            assert got == want, f"{tag}: {way} wrote different files"
            log(f"{tag} repeat {rep} {way}: {walls[way][-1]:.4f} s per sample")
    shutil.rmtree(root, ignore_errors=True)
    return {w: {"best_s_per_sample": min(v), "s_per_sample": v} for w, v in walls.items()}, lanes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replicates", type=int, default=8)
    ap.add_argument("--replicate-reads", type=int, default=20000000)
    ap.add_argument("--cells", type=int, default=256)
    ap.add_argument("--cell-reads", type=int, default=100000)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--workloads", default="replicates,cells")
    ap.add_argument("--workdir", default=None)
    a = ap.parse_args()
    name, power = card()
    work = tempfile.mkdtemp(prefix="bench_sim_batch_", dir=a.workdir)
    try:
        for tag in a.workloads.split(","):
            n, reads, data = {"replicates": (a.replicates, a.replicate_reads, "pe_q_rspd"),
                              "cells": (a.cells, a.cell_reads, "se_noq")}[tag]
            walls, lanes = workload(work, tag, data, n, reads, a.repeats)
            print(json.dumps({"workload": tag, "samples": n, "reads_per_sample": reads, "model": data, "wall": walls,
                              "lanes": lanes, "gpu": name, "power_limit": power}), flush=True)
    finally:
        shutil.rmtree(work, ignore_errors=True)


if __name__ == "__main__":
    main()
