#!/usr/bin/env python
"""Whole-executable timing of rsem-calculate-credibility-intervals (H100) against the reference tool on one generated
dataset.  The count vectors come from bin/rsem-run-gibbs (driver defaults: NCV = 1000 count vectors, NSPC = 50 samples
each).  Both tools run with -p THREADS on the same copies of imd; the appended iso_res / gene_res rows must be
byte-identical before any number is printed.

Reported, as one JSON line:
  ref_phase1_s / ref_phase2_s   the reference's sampling and interval phases, split at its stdout line
                                "Sampling is finished!" (stdout line-buffered with stdbuf, each line timestamped)
  ours_*                        host sampling, K8 wall time, device time per K8 phase (CUDA events, RSEM_B200_TIMING=1)
  gpu                           name, power limit and SM clock of the card (nvidia-smi)"""
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

TOOL = "rsem-calculate-credibility-intervals"


def _timed_lines(cmd, cwd, env=None):
    """-> (returncode, [(seconds since start, line)], stderr, wall seconds)"""
    t0 = time.perf_counter()
    p = subprocess.Popen(cmd, cwd=cwd, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    lines = [(time.perf_counter() - t0, l.rstrip("\n")) for l in p.stdout]
    err = p.stderr.read()
    p.wait()
    return p.returncode, lines, err, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--M", type=int, default=50_000)
    ap.add_argument("--N1", type=int, default=200_000)
    ap.add_argument("--ncv", type=int, default=1000)
    ap.add_argument("--nspc", type=int, default=50)
    ap.add_argument("--burnin", type=int, default=200)
    ap.add_argument("--threads", type=int, default=8)
    ap.add_argument("--seed", type=int, default=42)
    a = ap.parse_args()
    ref_bin = os.path.join(rf.REF_DIR, TOOL)
    if not os.path.exists(ref_bin):
        sys.exit(f"{ref_bin} is not built (oracle/ci.mk needs the reference sources)")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    out = {"transcripts": a.M, "reads": a.N1, "ncv": a.ncv, "nspc": a.nspc, "samples": a.ncv * a.nspc,
           "threads": a.threads, "gpu": gpu}
    with tempfile.TemporaryDirectory(prefix="rsem_ci_") as tmp:
        base = rf.gen_dataset(os.path.join(tmp, "base"), read_type=1, M=a.M, N1=a.N1, N0=a.N1 // 20, read_len=100, seed=11)
        rf.run_em(base, 1, "ours", rounds=20)
        rf.run_gibbs(base, "ours", a.burnin, a.ncv, 1, a.threads, a.seed)
        args = ["ref/r", "s.temp/s", "s.stat/s", "0.95", str(a.ncv), str(a.nspc), "1024", "-p", str(a.threads),
                "--seed", str(a.seed)]
        dirs = {w: rf.clone(base, os.path.join(tmp, w)) for w in ("ref", "ours")}
        stdbuf = shutil.which("stdbuf")
        rc, lines, err, wall = _timed_lines(([stdbuf, "-oL"] if stdbuf else []) + [ref_bin, *args], dirs["ref"])
        assert rc == 0, err[-2000:]
        split = next(t for t, l in lines if l == "Sampling is finished!")
        out.update(ref_wall_s=round(wall, 2), ref_phase1_s=round(split, 2), ref_phase2_s=round(wall - split, 2),
                   ref_stdout_line_buffered=bool(stdbuf))
        rc, lines, err, wall = _timed_lines([os.path.join(rf.BIN_DIR, TOOL), *args], dirs["ours"],
                                            env={**os.environ, "RSEM_B200_TIMING": "1"})
        assert rc == 0, err[-2000:]
        for f in ("s.iso_res", "s.gene_res"):
            assert filecmp.cmp(f"{dirs['ref']}/s.temp/{f}", f"{dirs['ours']}/s.temp/{f}", shallow=False), f"{f} differs"
        out["identical_rows"] = True
        m = re.search(r"sampling \(host, \d+ threads\) ([\d.]+) s, intervals ([\d.]+) s; device: transpose ([\d.]+) s, "
                      r"sums ([\d.]+) s, sort ([\d.]+) s, intervals ([\d.]+) s, (\d+) blocks, sample matrix (.*)", err)
        out.update(ours_wall_s=round(wall, 2), ours_sampling_s=float(m.group(1)), ours_phase2_s=float(m.group(2)),
                   ours_device_s={"transpose": float(m.group(3)), "sums": float(m.group(4)), "sort": float(m.group(5)),
                                  "intervals": float(m.group(6))},
                   ours_blocks=int(m.group(7)), ours_sample_matrix=m.group(8))
        out["speedup_wall"] = round(out["ref_wall_s"] / out["ours_wall_s"], 2)
        out["speedup_phase2"] = round(out["ref_phase2_s"] / out["ours_phase2_s"], 2)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
