#!/usr/bin/env python
"""Whole-executable timing of rsem-run-gibbs (H100) against the reference on one generated dataset; checks that the
count vectors are byte-identical.  Tooling for profiles/.

--devices 0,1,...: instead, rsem-run-gibbs on device 0 alone and with RSEM_B200_DEVICES set to the list, alternating, in
one call (the EM inputs come from bin/rsem-run-em, so no reference binary is needed); checks that both write the same
count vectors and reports the wall times with the name and power limit of every card, read in the same call."""
import argparse
import filecmp
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import rsem_files as rf  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--read-type", type=int, default=1)
    ap.add_argument("--N1", type=int, default=1_000_000)
    ap.add_argument("--M", type=int, default=50_000)
    ap.add_argument("--avg-family", type=float, default=10)
    ap.add_argument("--read-len", type=int, default=100)
    ap.add_argument("--burnin", type=int, default=50)
    ap.add_argument("--nsamples", type=int, default=64)
    ap.add_argument("--gap", type=int, default=1)
    ap.add_argument("--chains", type=int, default=8)
    ap.add_argument("--devices", default=None, help="compare one device with this RSEM_B200_DEVICES list")
    ap.add_argument("--repeats", type=int, default=3, help="--devices: timed runs of each, alternating")
    a = ap.parse_args()
    if a.devices:
        return compare_devices(a)
    cores = os.cpu_count() or 1
    with tempfile.TemporaryDirectory(prefix="rsem_gibbs_") as tmp:
        base = rf.gen_dataset(os.path.join(tmp, "base"), read_type=a.read_type, M=a.M, N1=a.N1, N0=a.N1 // 20,
                              avg_family=a.avg_family, read_len=a.read_len, seed=11)
        rf.run_em(base, a.read_type, "ref", rounds=12, threads=cores)
        n_entries = sum(len(l.split()) // 2 for l in open(f"{base}/s.temp/s.ofg")) - 1
        out = {"reads": a.N1, "transcripts": a.M, "ofg_entries": n_entries, "chains": a.chains,
               "sweeps_per_chain": a.burnin + 1 + (a.nsamples // a.chains - 1) * a.gap, "host_cores": cores}
        for which in ("ref", "ours"):
            d = rf.clone(base, os.path.join(tmp, which))
            t0 = time.perf_counter()
            os.environ["RSEM_B200_TIMING"] = "1"
            p = rf.run_gibbs(d, which, a.burnin, a.nsamples, a.gap, a.chains, 777)
            out[which + "_wall_s"] = round(time.perf_counter() - t0, 3)
            if which == "ours":
                out["ours_phases"] = [l for l in p.stderr.splitlines() if "timing" in l or "cycles" in l]
        out["identical_countvectors"] = all(filecmp.cmp(f"{tmp}/ref/s.temp/s.countvectors{t}", f"{tmp}/ours/s.temp/s.countvectors{t}",
                                                         shallow=False) for t in range(a.chains))
        out["speedup_wall"] = round(out["ref_wall_s"] / out["ours_wall_s"], 2)
        print(json.dumps(out))


def compare_devices(a):
    cards = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit", "--format=csv,noheader"], check=True,
                           capture_output=True, text=True).stdout.strip().splitlines()
    with tempfile.TemporaryDirectory(prefix="rsem_gibbs_") as tmp:
        base = rf.gen_dataset(os.path.join(tmp, "base"), read_type=a.read_type, M=a.M, N1=a.N1, N0=a.N1 // 20,
                              avg_family=a.avg_family, read_len=a.read_len, seed=11)
        for k in ("RSEM_B200_DEVICES", "RSEM_B200_DEVICE"):
            os.environ.pop(k, None)
        rf.run_em(base, a.read_type, "ours", rounds=12)
        out = {"reads": a.N1, "transcripts": a.M, "chains": a.chains, "devices": a.devices, "cards": cards,
               "sweeps_per_chain": a.burnin + 1 + (a.nsamples // a.chains - 1) * a.gap}
        walls = {"one": [], "list": []}
        os.environ["RSEM_B200_TIMING"] = "1"
        for r in range(a.repeats + 1):   # run 0 of each is a warm-up (page cache, driver start)
            for key in ("one", "list"):
                if key == "list":
                    os.environ["RSEM_B200_DEVICES"] = a.devices
                d = rf.clone(base, os.path.join(tmp, key))
                t0 = time.perf_counter()
                p = rf.run_gibbs(d, "ours", a.burnin, a.nsamples, a.gap, a.chains, 777)
                wall = time.perf_counter() - t0
                os.environ.pop("RSEM_B200_DEVICES", None)
                if r > 0:
                    walls[key].append(round(wall, 3))
                out[key + "_phases"] = [l for l in p.stderr.splitlines() if l.startswith("rsem-run-gibbs timing")]
        out["one_wall_s"], out["list_wall_s"] = walls["one"], walls["list"]
        out["identical_countvectors"] = all(filecmp.cmp(f"{tmp}/one/s.temp/s.countvectors{t}", f"{tmp}/list/s.temp/s.countvectors{t}",
                                                         shallow=False) for t in range(a.chains))
        out["identical_results"] = all(filecmp.cmp(f"{tmp}/one/s.temp/{f}", f"{tmp}/list/s.temp/{f}", shallow=False)
                                       for f in ("s.iso_res", "s.gene_res"))
        if walls["one"]:
            out["speedup_median_wall"] = round(sorted(walls["one"])[len(walls["one"]) // 2] /
                                               sorted(walls["list"])[len(walls["list"]) // 2], 3)
        print(json.dumps(out))


if __name__ == "__main__":
    main()
