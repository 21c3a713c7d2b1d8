#!/usr/bin/env python
"""Where the class-layout E-step (K2) spends its time: builds a bench.py workload matrix the way bench.py does, runs a
few frozen-conprb rounds with profiling on and prints, per persistent CTA of the last launch, its busy time, the time
its consumer warps spent blocked on staged data (mean over the warps), the rest of the busy time (compute, i.e. not
blocked on data) and the time a separate copy-issuing warp spent blocked on a free stage; and, over all CTAs, the
share of the consumer warps' busy time (SM cycles) spent in each phase of a batch: front (descriptor, ids and theta
gather until theta is usable), rows (the row walk), flush (fold +
reductions) and hand-over (releasing a stage -> the next stage's data seen); "other" is the rest (loop control, timer
reads, the time before the first and after the last tile).

  python tools/k2_anatomy.py [--workload C3] [--scale 1.0] [--per-cta]

Prints one JSON line (summary over the CTAs; with --per-cta also the per-CTA arrays, in microseconds).
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (matrix generator shared with the benchmark)

BIG = bench.BIG


def _summary(x):
    return {"min": round(float(x.min()), 1), "median": round(float(np.median(x)), 1), "max": round(float(x.max()), 1),
            "mean": round(float(x.mean()), 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="C3", choices=sorted(bench.WORKLOADS))
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--per-cta", action="store_true")
    args = ap.parse_args()

    import torch

    import rsem_b200

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    N, M, deg, zipf = bench.WORKLOADS[args.workload]
    if args.scale != 1.0:
        N = max(1000, int(N * args.scale))
    row_ptr, sid, conprb, ncpv, H = bench.gen_matrix_torch(torch, dev, N, M, deg, 1234, zipf)
    torch.cuda.synchronize()
    ctx = rsem_b200.Context(0)
    ctx.adopt_device_matrix(N, H, M, row_ptr.data_ptr(), sid.data_ptr(), conprb.data_ptr(), ncpv.data_ptr())
    n0 = N / 20
    theta0 = np.empty(M + 1)
    theta0[0] = max(n0 / (N + n0), 1e-8)
    theta0[1:] = (1 - theta0[0]) / M
    ctx.set_theta(theta0)
    ctx.em_rounds(12, 3, BIG, BIG, n0)  # builds the class layout, warms up
    ctx.set_profiling(True)
    ctx.estep_timing(reset=True)
    ctx.em_rounds(15, args.rounds, BIG, BIG, n0)
    ctx.sync()
    k2_ms, k2_n = ctx.estep_timing(reset=True)
    ctx.set_profiling(False)
    busy = ctx.estep_cta_times().astype(np.float64) / 1e3
    w = ctx.estep_wait_times().astype(np.float64)
    info = ctx.class_layout_info()
    ctx.close()
    if not info["built"] or w.size == 0:
        print(json.dumps({"error": "no profiled class-layout launch"}))
        return 1
    warps = w[:, 2]
    data_wait = w[:, 0] / warps / 1e3  # mean over the CTA's consumer warps
    compute = busy - data_wait
    warp_cycles = float((warps * w[:, 7]).sum())  # busy cycles of all consumer warps
    shares = {k: round(float(w[:, 3 + i].sum()) / warp_cycles, 4) for i, k in enumerate(("front", "rows", "flush", "hand_over"))}
    shares["other"] = round(1.0 - sum(shares.values()), 4)
    out = {"workload": args.workload, "reads": N, "hits": H, "gpu": torch.cuda.get_device_name(0),
           "k2_ms_per_launch_with_profiling": round(k2_ms / k2_n, 4), "ctas": int(busy.size),
           "consumer_warps_per_cta": int(warps[0]), "bytes_per_round": info["bytes_per_round"],
           "busy_us": _summary(busy), "data_wait_us_per_warp": _summary(data_wait), "compute_us_per_warp": _summary(compute),
           "producer_wait_us": _summary(w[:, 1] / 1e3),
           "data_wait_share_of_busy": round(float(data_wait.sum() / busy.sum()), 4),
           "producer_wait_share_of_busy": round(float((w[:, 1] / 1e3).sum() / busy.sum()), 4),
           "phase_share_of_warp_cycles": shares,
           "sm_cycles_per_ns": round(float(w[:, 7].sum() / (busy.sum() * 1e3)), 3),
           "note": "last profiled launch; data wait = time a consumer warp blocked on its staged data (mean over the CTA's "
                   "warps), compute = busy - data wait; profiling adds %globaltimer reads around every wait"}
    if args.per_cta:
        out["per_cta"] = {"busy_us": busy.round(1).tolist(), "data_wait_us": data_wait.round(1).tolist(),
                          "compute_us": compute.round(1).tolist(), "producer_wait_us": (w[:, 1] / 1e3).round(1).tolist()}
    print(json.dumps(out), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
