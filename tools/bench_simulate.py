"""Wall time of bin/rsem-simulate-reads against the reference simulator (oracle/_ref/rsem-simulate-reads) on the
paired-end model with qualities of the pe_q_rspd golden data set (2 x 50 bases, estRSPD), same seed.

  python tools/bench_simulate.py --reads 2000000 [--reads 20000000] [--no-ref] [--out DIR]
  python tools/bench_simulate.py --reads 20000000 --devices 0,1 [--repeat 3]

Prints one JSON line per run: wall seconds, reads/s, the simulator's device / file-write split
(RSEM_B200_TIMING) and whether the outputs are byte-identical to the reference's.  With --devices, one device
(RSEM_B200_DEVICES unset) and the list (RSEM_B200_DEVICES=LIST) are run alternately --repeat times each, after a first
pair of runs whose files must be identical; no reference run."""
import argparse
import filecmp
import json
import os
import random
import subprocess
import sys
import tarfile
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, action="append")
    ap.add_argument("--no-ref", action="store_true")
    ap.add_argument("--out", default=None)
    ap.add_argument("--devices", default=None, help="comma-separated device list to compare with one device")
    ap.add_argument("--repeat", type=int, default=3)
    a = ap.parse_args()
    work = tempfile.mkdtemp(prefix="bench_sim_", dir=a.out)
    with tarfile.open(os.path.join(ROOT, "tests", "golden", "pe_q_rspd.tar.gz")) as t:
        t.extractall(work, filter="data")
    d = os.path.join(work, "pe_q_rspd")
    M = int(open(os.path.join(d, "ref", "r.ti")).readline().split()[0])
    rng = random.Random(1)
    with open(os.path.join(d, "res.tsv"), "w") as f:
        f.write("transcript_id\tgene_id\tlength\teffective_length\texpected_count\tTPM\tFPKM\tIsoPct\n")
        for i in range(1, M + 1):
            f.write(f"T{i}\tG\t1\t1\t1\t{rng.uniform(0, 100):.2f}\t0\t0\n")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    if a.devices:
        for n in a.reads or [2000000]:
            print(json.dumps(compare_devices(d, work, n, a.devices, a.repeat, gpu)), flush=True)
        return
    for n in a.reads or [2000000]:
        res = {"reads": n, "gpu": gpu}
        runs = [("gpu", os.path.join(ROOT, "bin", "rsem-simulate-reads"))]
        if not a.no_ref:
            runs.append(("ref", os.path.join(ROOT, "oracle", "_ref", "rsem-simulate-reads")))
        for tag, exe in runs:
            prefix = os.path.join(work, f"{tag}_{n}")
            t0 = time.perf_counter()
            p = subprocess.run([exe, os.path.join(d, "ref", "r"), os.path.join(d, "out", "model20"),
                                os.path.join(d, "res.tsv"), "0.1", str(n), prefix, "--seed", "7", "-q"],
                               capture_output=True, text=True, env={**os.environ, "RSEM_B200_TIMING": "1"})
            wall = time.perf_counter() - t0
            if p.returncode != 0:
                sys.exit(f"{tag} failed: {p.stderr}")
            res[f"{tag}_s"] = round(wall, 3)
            res[f"{tag}_reads_per_s"] = round(n / wall)
            if tag == "gpu":
                res["gpu_timing"] = [l for l in p.stderr.splitlines() if "timing" in l]
        if not a.no_ref:
            res["identical"] = all(filecmp.cmp(os.path.join(work, f"gpu_{n}{s}"), os.path.join(work, f"ref_{n}{s}"), shallow=False)
                                   for s in ("_1.fq", "_2.fq", ".sim.isoforms.results", ".sim.genes.results"))
        for f in os.listdir(work):
            if f.startswith(("gpu_", "ref_")):
                os.remove(os.path.join(work, f))
        print(json.dumps(res), flush=True)


def _run(d, prefix, n, devices):
    env = {**os.environ, "RSEM_B200_TIMING": "1"}
    env.pop("RSEM_B200_DEVICES", None)
    if devices:
        env["RSEM_B200_DEVICES"] = devices
    t0 = time.perf_counter()
    p = subprocess.run([os.path.join(ROOT, "bin", "rsem-simulate-reads"), os.path.join(d, "ref", "r"),
                        os.path.join(d, "out", "model20"), os.path.join(d, "res.tsv"), "0.1", str(n), prefix, "--seed",
                        "7", "-q"], capture_output=True, text=True, env=env)
    wall = time.perf_counter() - t0
    if p.returncode != 0:
        sys.exit(f"RSEM_B200_DEVICES={devices} failed: {p.stderr}")
    return wall, [l for l in p.stderr.splitlines() if "timing" in l]


def compare_devices(d, work, n, devices, repeat, gpu):
    """one device against the list: identical files first, then alternating timed runs"""
    sfx = ("_1.fq", "_2.fq", ".sim.isoforms.results", ".sim.genes.results")
    one, many = os.path.join(work, f"one_{n}"), os.path.join(work, f"many_{n}")
    _run(d, one, n, None)
    _run(d, many, n, devices)
    res = {"reads": n, "gpu": gpu, "devices": devices,
           "identical": all(filecmp.cmp(one + s, many + s, shallow=False) for s in sfx), "one_s": [], "list_s": []}
    for _ in range(repeat):
        for key, dev, prefix in (("one_s", None, one), ("list_s", devices, many)):
            wall, timing = _run(d, prefix, n, dev)
            res[key].append(round(wall, 3))
            res[key.replace("_s", "_timing")] = timing
    for f in os.listdir(work):
        if f.startswith(("one_", "many_")):
            os.remove(os.path.join(work, f))
    return res


if __name__ == "__main__":
    main()
