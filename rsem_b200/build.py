"""In-tree build of every native artefact (called by __graft_entry__.build()).

  rsem_b200/librsem_b200.so   CUDA kernels + C ABI, sm_90a only
  bin/rsem-run-em, bin/rsem-run-gibbs, bin/rsem-parse-alignments, bin/rsem-simulate-reads,
  bin/rsem-calculate-credibility-intervals, bin/rsem-for-ebseq-calculate-clustering-info, bin/rsem-tbam2gbam,
  bin/rsem-bam2wig, bin/rsem-bam2readdepth, bin/rsem-run-em-batch, bin/rsem-run-gibbs-batch
                              C++ drop-in executables (link the .so)
  tools/gen_dataset           synthetic intermediate-file generator (tooling)
  oracle/librsem_oracle.so    CPU restatement (test infrastructure)
  oracle/libkmer_oracle.so    CPU restatement of the k-mer counts (test infrastructure)
  oracle/_ref/*               reference binaries, only when /root/reference is present
"""
from __future__ import annotations

import glob
import os
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "rsem_b200", "csrc")
HOST = os.path.join(ROOT, "rsem_b200", "host")
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
              "-diag-suppress", "177"]


def _newer(target: str, sources) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources)


def _run(cmd, **kw):
    print("+", " ".join(cmd), file=sys.stderr, flush=True)
    subprocess.check_call(cmd, **kw)


def build_lib(force: bool = False) -> str:
    out = os.path.join(ROOT, "rsem_b200", "librsem_b200.so")
    srcs = sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cpp")))
    deps = srcs + glob.glob(os.path.join(CSRC, "*.cuh")) + [os.path.join(ROOT, "include", "rsem_b200.h")]
    if force or _newer(out, deps):
        _run([NVCC, *NVCC_FLAGS, "-shared", "-o", out, *srcs, "-ldl"])
    return out


def build_host(force: bool = False):
    os.makedirs(os.path.join(ROOT, "bin"), exist_ok=True)
    common = sorted(glob.glob(os.path.join(HOST, "*.cpp")))
    mains = [s for s in common if os.path.basename(s).startswith("main_")]
    shared = [s for s in common if s not in mains]
    # the simulator's tables and the credibility-interval sampler are built in files compiled with the reference's flags
    # for simulation.cpp and calcCI.cpp (-O3 -ffast-math, reference Makefile:39,72-73), so that they carry the same bits;
    # the link step adds no -ffast-math (no crtfastmath.o, which would set flush-to-zero for the whole process)
    ffm = sorted(glob.glob(os.path.join(HOST, "ffm", "*.cpp")))
    deps = common + ffm + glob.glob(os.path.join(HOST, "*.hpp")) + [os.path.join(ROOT, "include", "rsem_b200.h")]
    ffm_objs = []
    for src in ffm:
        obj = os.path.join(ROOT, "build", "host", os.path.basename(src)[:-4] + ".o")
        os.makedirs(os.path.dirname(obj), exist_ok=True)
        if force or _newer(obj, deps):
            _run(["g++", "-O3", "-ffast-math", "-std=c++17", "-Wall", "-I", os.path.join(ROOT, "include"), "-c", "-o", obj, src])
        ffm_objs.append(obj)
    for m in mains:
        name = {"main_em.cpp": "rsem-run-em", "main_gibbs.cpp": "rsem-run-gibbs", "main_simulate.cpp": "rsem-simulate-reads",
                "main_selftest.cpp": "rsem-b200-host-selftest", "main_parse.cpp": "rsem-parse-alignments",
                "main_ci.cpp": "rsem-calculate-credibility-intervals",
                "main_clustering_info.cpp": "rsem-for-ebseq-calculate-clustering-info",
                "main_tbam2gbam.cpp": "rsem-tbam2gbam", "main_bam2wig.cpp": "rsem-bam2wig",
                "main_bam2readdepth.cpp": "rsem-bam2readdepth", "main_em_batch.cpp": "rsem-run-em-batch",
                "main_gibbs_batch.cpp": "rsem-run-gibbs-batch"}[os.path.basename(m)]
        out = os.path.join(ROOT, "bin", name)
        ffm_use = {"rsem-simulate-reads": "sim_tables.o", "rsem-calculate-credibility-intervals": "ci_sample.o"}
        extra = [o for o in ffm_objs if os.path.basename(o) == ffm_use.get(name)]
        if force or _newer(out, deps + [os.path.join(ROOT, "rsem_b200", "librsem_b200.so")]):
            _run(["g++", "-O2", "-std=c++17", "-Wall", "-pthread", "-I", os.path.join(ROOT, "include"), "-o", out, m, *shared, *extra,
                  "-L", os.path.join(ROOT, "rsem_b200"), "-lrsem_b200", "-Wl,-rpath,$ORIGIN/../rsem_b200",
                  "-static-libstdc++", "-static-libgcc", "-lz"])


def build_tools(force: bool = False):
    src = os.path.join(ROOT, "tools", "gen_dataset.cpp")
    out = os.path.join(ROOT, "tools", "gen_dataset")
    if force or _newer(out, [src]):
        _run(["g++", "-O2", "-std=c++17", "-o", out, src])
    # micro-benchmarks: red / ldg throughput per lane mapping; HBM read rate per copy geometry
    for name in ("red_bench", "hbm_read"):
        src = os.path.join(ROOT, "tools", "micro", name + ".cu")
        out = os.path.join(ROOT, "tools", "micro", name)
        if os.path.exists(src) and (force or _newer(out, [src])):
            _run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-o", out, src])


def build_oracle():
    # building the checker is not using it; `make ref` is a no-op when /root/reference is absent
    _run(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "all"])
    _run(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "-f", "simulate.mk"])
    _run(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "-f", "ci.mk"])
    _run(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "-f", "ebseq.mk"])
    _run(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "-f", "tbam2gbam.mk"])
    _run(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "-f", "wiggle.mk"])


def build_all(force: bool = False):
    build_lib(force)
    if glob.glob(os.path.join(HOST, "main_*.cpp")):
        build_host(force)
    build_tools(force)
    build_oracle()


if __name__ == "__main__":
    build_all(force="--force" in sys.argv)
