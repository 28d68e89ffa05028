"""CPU-side checks of the drop-in boundary: the shared library loads, exports exactly the
symbols include/diskann_b200.h declares, and fails loudly (no CPU fallback) without a GPU."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "diskann_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(dab_[a-z0-9_]+)\s*\(", text)))


def test_header_binding_and_library_agree():
    import diskann_b200
    declared = declared_symbols()
    assert sorted(diskann_b200.SYMBOLS) == declared
    L = diskann_b200.lib()  # raises if the .so is missing or lacks a symbol
    for name in declared:
        assert hasattr(L, name), name
    out = subprocess.run(["nm", "-D", "--defined-only", diskann_b200.LIB_PATH], capture_output=True, text=True).stdout
    exported = sorted(set(re.findall(r" T (dab_[a-z0-9_]+)", out)))
    assert exported == declared


def test_library_is_sm90a_and_self_contained():
    import diskann_b200
    out = subprocess.run(["cuobjdump", "-lelf", diskann_b200.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out and "sm_100" not in out and "sm_80" not in out
    ldd = subprocess.run(["ldd", diskann_b200.LIB_PATH], capture_output=True, text=True).stdout
    assert "torch" not in ldd and "oracle" not in ldd  # plain C ABI, no torch types, never links the oracle


def test_product_never_imports_the_oracle():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "diskann_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".hpp", ".cpp")):
                text = open(os.path.join(dirpath, f)).read()
                assert "oracle" not in text.lower(), os.path.join(dirpath, f)


def test_fails_loudly_without_a_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    import diskann_b200 as dab
    with pytest.raises(dab.DabError) as e:
        dab.GpuIndex(dab.DType.f32, dab.Metric.L2, 8, 10)
    assert e.value.code == 6 and "no CPU fallback" in str(e.value)
    with pytest.raises(dab.DabError) as e:
        dab.pair_distances(np.zeros((1, 4), np.float32), np.zeros((1, 4), np.float32), dab.Metric.L2)
    assert e.value.code == 6


def test_argument_validation_happens_before_any_device_work():
    import diskann_b200 as dab
    L = dab.lib()
    h = C.c_void_p()
    assert L.dab_create(C.byref(h), 9, 2, 8, 10, 1, 4, 0) == 1      # unknown dtype
    assert b"dtype" in L.dab_last_error()
    assert L.dab_create(C.byref(h), 0, 7, 8, 10, 1, 4, 0) == 1      # unknown metric
    assert L.dab_create(C.byref(h), 0, 2, 0, 10, 1, 4, 0) == 1      # dim 0
    assert L.dab_create(C.byref(h), 0, 2, 8, 0, 0, 4, 0) == 1       # empty index
    assert L.dab_create(None, 0, 2, 8, 10, 1, 4, 0) == 1
    assert L.dab_search_batch(None, None, 0, 1, 1, 1, None, None, None, None, None) == 1
    assert L.dab_pair_distances(0, 0, 9, 4, None, None, 0, None, 0) == 1
    L.dab_destroy(None)  # no-op
    assert dab.Metric.Cosine == 0 and dab.Metric.InnerProduct == 1 and dab.Metric.L2 == 2 and dab.Metric.CosineNormalized == 3


def test_rust_sys_crate_is_generated_from_the_header():
    """ffi/diskann-b200-sys/src/lib.rs declares exactly the header's entry points (tools/gen_ffi.py --check)."""
    import subprocess
    import sys
    assert subprocess.run([sys.executable, os.path.join(ROOT, "tools", "gen_ffi.py"), "--check"]).returncode == 0
    text = open(os.path.join(ROOT, "ffi", "diskann-b200-sys", "src", "lib.rs")).read()
    import diskann_b200._lib as L
    for name in L.SYMBOLS:
        assert f"pub fn {name}(" in text, name
