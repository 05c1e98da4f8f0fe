"""CPU check of the per-size work lists of the frame analyser's residual and intra launches (geometry.h tuBy / cuBy): per
CTU row, the TU lists by luma TU size (8, 16, 32) and the CU lists by CU size (8, 16, 32, 64) partition the row's slice of
the TU and CU tables, each list holds only its size, keeps the table order, and its row offsets slice it by CTU row as
rowTu / rowCu slice the tables."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from frame_helpers import stride_for

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def geo(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("geolists") / "libgeolists.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-o", so, os.path.join(HERE, "geometry_lists_capi.cpp")])
    lib = C.CDLL(so)
    lib.geo_get.argtypes = [C.c_int, C.c_void_p]
    return lib


def fetch(geo, what, n=None):
    if n is None:
        n = geo.geo_get(what, None)
    out = np.zeros(max(n, 1), np.int32)
    assert geo.geo_get(what, out.ctypes.data) == n
    return out[:n]


@pytest.mark.parametrize("size", [(200, 136), (200, 200), (352, 288), (1920, 1080), (3840, 2160), (7680, 4320)])
@pytest.mark.parametrize("rect,amp", [(1, 0), (1, 1)])
def test_size_lists_partition_each_row(geo, size, rect, amp):
    W, H = size
    counts = np.zeros(3, np.int64)
    geo.geo_build(W, H, stride_for(W), 2, rect, amp, counts.ctypes.data_as(C.c_void_p))
    ntu, ncu, rows = (int(x) for x in counts)
    tu_size = np.minimum(fetch(geo, 0, ntu), 32)                # luma TU size of every TU
    cu_size = fetch(geo, 1, ncu)
    for table, sizes, base, nk, row_of in ((2, tu_size, 10, 3, fetch(geo, 2)), (3, cu_size, 30, 4, fetch(geo, 3))):
        lists = [fetch(geo, base + k) for k in range(nk)]
        offs = [fetch(geo, base + 10 + k) for k in range(nk)]
        assert sum(len(l) for l in lists) == len(sizes)
        for k in range(nk):
            assert len(offs[k]) == rows + 1 and offs[k][0] == 0 and offs[k][-1] == len(lists[k])
            assert (np.diff(offs[k]) >= 0).all()
            assert (sizes[lists[k]] == 8 << k).all()
        for r in range(rows):
            parts = [lists[k][offs[k][r]:offs[k][r + 1]] for k in range(nk)]
            for p in parts:
                assert (np.diff(p) > 0).all()                    # table order
            got = np.sort(np.concatenate(parts))
            assert np.array_equal(got, np.arange(row_of[r], row_of[r + 1])), (table, r)
