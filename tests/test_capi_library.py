"""CPU checks of the boundary: the C-ABI library loads, exports every symbol include/rsem_b200.h declares, and
refuses to compute without a GPU (no fallback).  No compute calls here."""
import ctypes
import os
import re
import subprocess

import pytest

import rsem_files as rf

HEADER = os.path.join(rf.ROOT, "include", "rsem_b200.h")


def declared_symbols():
    text = open(HEADER).read()
    return sorted(set(re.findall(r"^(?:int|const char\*)\s+(rsem_b200_\w+)\s*\(", text, flags=re.M)))


def test_library_exports_every_declared_symbol(built):
    import rsem_b200
    from rsem_b200 import capi
    names = declared_symbols()
    assert len(names) >= 25
    dll = ctypes.CDLL(capi.LIB_PATH)
    for n in names:
        assert hasattr(dll, n), f"{n} declared in include/rsem_b200.h but not exported"
    assert sorted(capi.SYMBOLS) == names, "rsem_b200/capi.py mirror out of sync with the header"
    assert rsem_b200.load_library().version() == 100


def test_no_cpu_fallback(built, tmp_path):
    """without a CUDA device every path fails loudly: the library returns an error, the executables exit(-1)"""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    import rsem_b200
    with pytest.raises(rsem_b200.RsemB200Error):
        rsem_b200.Context(0)
    d = rf.gen_dataset(str(tmp_path / "d"), read_type=0, M=20, N1=50, N0=5)
    p = rf.run_em(d, 0, "ours", rounds=2, check=False)
    assert p.returncode == 255 and "CUDA" in p.stderr


def test_product_does_not_link_the_oracle(built):
    """the oracle is test infrastructure: neither the library nor the executables may depend on it"""
    for f in ("rsem_b200/librsem_b200.so", "bin/rsem-run-em", "bin/rsem-run-gibbs"):
        out = subprocess.run(["ldd", os.path.join(rf.ROOT, f)], stdout=subprocess.PIPE, text=True).stdout
        assert "oracle" not in out
    for dirpath, _, files in os.walk(os.path.join(rf.ROOT, "rsem_b200")):
        for fn in files:
            if fn == "build.py":  # builds the checker (make -C oracle) but never loads or calls it
                continue
            if fn.endswith((".py", ".cpp", ".hpp", ".cu", ".cuh")):
                text = open(os.path.join(dirpath, fn)).read()
                assert "rsem_oracle" not in text and "oracle_binding" not in text, f"{fn} references the oracle"


def test_usage_messages_match_reference_convention():
    for exe, n in (("rsem-run-em", 6), ("rsem-run-gibbs", 7)):
        p = subprocess.run([os.path.join(rf.BIN_DIR, exe)], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
        assert p.returncode == 255 and p.stdout.startswith("Usage")
