"""rsem_b200 - H100 (sm_90a) implementation of RSEM's EM / Gibbs estimation hot path.

The product is `librsem_b200.so` (hand-written CUDA behind the C ABI of include/rsem_b200.h) and the
drop-in executables `bin/rsem-run-em` / `bin/rsem-run-gibbs` (C++ hosts in rsem_b200/host/).  This
Python package is a thin ctypes mirror of the C ABI used by the tests and by bench.py; it contains
no arithmetic of its own and no CPU fallback.
"""
from .capi import Batch, Context, GibbsBatch, Lib, RsemB200Error, load_library  # noqa: F401
