#!/usr/bin/env python
"""Generate tests/golden/*.tar.gz: small inputs + the outputs of the REFERENCE binaries on them.

The reference ships no golden vectors for the EM / Gibbs path (SURVEY.md section 4), so parity is pinned against
outputs of the reference itself: oracle/_ref/* are compiled by oracle/Makefile from the sources where they lie in
/root/reference.  This script only runs in the build container (it needs oracle/_ref); the fixtures it writes are
committed and are all the tests need.

    python tools/make_golden.py            # regenerates every case (deterministic: fixed generator seeds)
"""
import os
import shutil
import subprocess
import sys
import tarfile
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import rsem_files as rf  # noqa: E402

CASES = {
    # name: (read_type, generator options)   -- no poly(A), no --fragment-length-mean unless noted
    "se_noq": (0, dict(M=60, N1=400, N0=30, read_len=40, maxL=120, seed=21)),
    "se_q_rspd": (1, dict(M=60, N1=400, N0=30, read_len=45, var_len=5, est_rspd=1, probF=0.6, seed=22)),
    "pe_noq": (2, dict(M=50, N1=350, N0=25, read_len=36, var_len=3, maxL=320, spurious=0.05, seed=23)),
    "pe_q_rspd": (3, dict(M=60, N1=400, N0=30, read_len=40, est_rspd=1, probF=0.4, spurious=0.1, seed=24)),
    "se_q_polyA": (1, dict(M=40, N1=300, N0=20, read_len=50, polyA=125, omit=3, seed=25)),
}
GIBBS = dict(burnin=10, nsamples=6, gap=2, threads=2, seed=4242)


def main():
    if not rf.have_ref():
        sys.exit("oracle/_ref is missing: run `make -C oracle ref` in the build container")
    out_dir = os.path.join(ROOT, "tests", "golden")
    os.makedirs(out_dir, exist_ok=True)
    for name, (rt, opts) in CASES.items():
        with tempfile.TemporaryDirectory() as tmp:
            base = rf.gen_dataset(os.path.join(tmp, "base"), read_type=rt, **opts)
            pack = os.path.join(tmp, name)
            shutil.copytree(base, pack)
            os.makedirs(os.path.join(pack, "out"))
            for rounds in (1, 20, 25):
                run = rf.clone(base, os.path.join(tmp, f"run{rounds}"))
                rf.run_em(run, rt, "ref", rounds=rounds, min_rounds=rounds, threads=1)
                shutil.copy(f"{run}/s.stat/s.theta", f"{pack}/out/theta{rounds}")
                if rounds != 25:
                    shutil.copy(f"{run}/s.stat/s.model", f"{pack}/out/model{rounds}")
                if rounds == 20:
                    shutil.copy(f"{run}/s.temp/s.ofg", f"{pack}/out/ofg20")
                    shutil.copy(f"{run}/s.temp/s.iso_res", f"{pack}/out/iso_res20")
                    shutil.copy(f"{run}/s.temp/s.gene_res", f"{pack}/out/gene_res20")
                    rf.run_gibbs(run, "ref", GIBBS["burnin"], GIBBS["nsamples"], GIBBS["gap"], GIBBS["threads"], GIBBS["seed"])
                    for t in range(GIBBS["threads"]):
                        shutil.copy(f"{run}/s.temp/s.countvectors{t}", f"{pack}/out/countvectors{t}")
                    shutil.copy(f"{run}/s.temp/s.iso_res", f"{pack}/out/iso_res_gibbs")
                    shutil.copy(f"{run}/s.temp/s.gene_res", f"{pack}/out/gene_res_gibbs")
            with open(f"{pack}/out/README", "w") as f:
                f.write(f"case {name}: read_type {rt}, generator options {opts}\n"
                        f"reference: oracle/_ref/rsem-run-em-rounds -p 1 with RSEM_MAX_ROUND = RSEM_MIN_ROUND = 1 / 20 / 25,\n"
                        f"oracle/_ref/rsem-run-gibbs {GIBBS} on the 20-round outputs\n")
            tar_path = os.path.join(out_dir, name + ".tar.gz")
            with tarfile.open(tar_path, "w:gz") as tar:
                tar.add(pack, arcname=name, filter=lambda ti: None if ti.name.endswith(".ridx") else ti)
            print(f"{tar_path}: {os.path.getsize(tar_path) / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
