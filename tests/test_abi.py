"""CPU-side checks of the drop-in boundary: libx265cu.so builds for sm_90a, loads without a GPU and
exports every symbol include/x265_b200.h declares; compute entry points refuse to run without CUDA
(no CPU fallback)."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    txt = open(os.path.join(ROOT, "include", "x265_b200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(x265cu_\w+)\s*\(", txt)))


def test_header_symbols_exported():
    from x265_b200 import build
    lib = C.CDLL(build.build())
    syms = declared_symbols()
    assert len(syms) >= 30
    missing = [s for s in syms if not hasattr(lib, s)]
    assert not missing, missing


def test_no_cpu_fallback():
    import x265_b200
    lib = x265_b200.load(need_gpu=False)
    if lib.L.x265cu_device_count() > 0:
        pytest.skip("GPU present")
    with pytest.raises(x265_b200.CudaUnavailable):
        x265_b200.Lib(need_gpu=True)
    assert lib.L.x265cu_get_primitive(8, b"pu.sad", 2, 0, 0) is None
    assert lib.L.x265cu_create(0) is None


def test_job_layouts_match_header():
    from x265_b200 import lib as L
    assert L.CMP_JOB.itemsize == 32 and L.BLK_JOB.itemsize == 56
    assert L.INTERP_JOB.itemsize == 32 and L.ME_JOB.itemsize == 40 and L.INTRA_JOB.itemsize == 8
    assert L.PRED_JOB.itemsize == 20            # x265cu_pred_job


def test_mvcost_table_matches_oracle():
    import numpy as np
    import x265_b200
    from common import load_oracle, ptr
    lib = x265_b200.load(need_gpu=False)
    O = load_oracle(8)
    for lam in (4.0, 11.3137, 57.0175, 724.0773):
        a = lib.mvcost_table(lam, 4096)
        b = np.zeros(2 * 4096 + 1, np.uint16)
        O.orc_mvcost_table(C.c_double(lam), 4096, ptr(b))
        assert np.array_equal(a, b)
