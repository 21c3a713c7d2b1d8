"""Wall time of bin/rsem-simulate-reads against the reference simulator (oracle/_ref/rsem-simulate-reads) on the
paired-end model with qualities of the pe_q_rspd golden data set (2 x 50 bases, estRSPD), same seed.

  python tools/bench_simulate.py --reads 2000000 [--reads 20000000] [--no-ref] [--out DIR]

Prints one JSON line per run: wall seconds, reads/s, the simulator's device / file-write split
(RSEM_B200_TIMING) and whether the outputs are byte-identical to the reference's."""
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


if __name__ == "__main__":
    main()
