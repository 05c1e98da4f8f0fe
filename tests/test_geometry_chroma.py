"""CPU check of the host-side geometry of the analyser's 4:2:0 chroma residual stage (x265_b200/csrc/geometry.h, compiled here
with g++ through tests/geometry_chroma_capi.cpp): the chroma TU list and its level offsets, the chroma pixels the chroma MC can read
against the chroma plane allocation (what x265cu_analyser_enable_chroma_residual and every bit-3 run check), and the host's
chroma QP map against the oracle's (which tests/test_chroma_residual_oracle_vs_ref.py pins to the real Quant::setChromaQP)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from chroma_helpers import load_oracle_chroma
from frame_helpers import MARGIN_X, MARGIN_Y, stride_for, qp_max

HERE = os.path.dirname(os.path.abspath(__file__))
SIZES = [(200, 136), (352, 288), (1920, 1080), (3840, 2160), (256, 128), (200, 200)]


@pytest.fixture(scope="module")
def geo(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("geoc") / "libgeoc.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-o", so, os.path.join(HERE, "geometry_chroma_capi.cpp")])
    return C.CDLL(so)


def build(geo, W, H, rect=1, amp=0):
    counts = np.zeros(5, np.int64)
    geo.geo_build(W, H, stride_for(W), 1, rect, amp, counts.ctypes.data_as(C.c_void_p))
    nj, ncu, ntu, rows, ncoef = [int(x) for x in counts]

    def get(fn, what, dtype, n):
        out = np.zeros(n, dtype)
        assert fn(*what, out.ctypes.data_as(C.c_void_p)) == 0
        return out
    cus = get(geo.geo_get, (1,), np.int64, ncu * 4).reshape(-1, 4)
    tus = get(geo.geo_get, (2,), np.int32, ntu * 3).reshape(-1, 3)
    rowTu = get(geo.geo_get, (6,), np.int32, rows + 1)
    ctu = get(geo.geo_chroma_tus, (), np.int64, ntu * 4).reshape(-1, 4)
    return dict(ncoef=ncoef, rows=rows, cus=cus, tus=tus, rowTu=rowTu, ctu=ctu)


def reach(geo, W, H, tu0, tu1, my=MARGIN_Y // 2, mx=MARGIN_X // 2):
    r = (C.c_int * 4)()
    ok = geo.geo_chroma_reach(W, H, int(tu0), int(tu1), stride_for(W) // 2, mx, my, r)
    return bool(ok), tuple(r)


@pytest.mark.parametrize("size", SIZES)
def test_chroma_tus(geo, size):
    """Chroma TUs: half the luma TU at half its coordinates, inside the chroma picture, and their levels tile [0, ncoef / 4)
    exactly, CU by CU in the luma TU order."""
    W, H = size
    g = build(geo, W, H)
    cus, tus, ctu = g["cus"], g["tus"], g["ctu"]
    cu = cus[tus[:, 0]]
    T = np.minimum(cu[:, 2], 32)
    assert np.array_equal(ctu[:, 0], (cu[:, 0] + tus[:, 1]) // 2) and np.array_equal(ctu[:, 1], (cu[:, 1] + tus[:, 2]) // 2)
    assert np.array_equal(ctu[:, 2], T // 2) and set(ctu[:, 2].tolist()) <= {4, 8, 16}
    assert (ctu[:, 0] >= 0).all() and (ctu[:, 1] >= 0).all()
    assert (ctu[:, 0] + ctu[:, 2] <= W // 2).all() and (ctu[:, 1] + ctu[:, 2] <= H // 2).all()
    assert g["ncoef"] % 4 == 0
    ends = ctu[:, 3] + ctu[:, 2] ** 2
    assert ctu[0, 3] == 0 and np.array_equal(ctu[1:, 3], ends[:-1]) and ends[-1] == g["ncoef"] // 4
    first = np.r_[True, tus[1:, 0] != tus[:-1, 0]]
    assert np.array_equal(ctu[first, 3], cus[tus[first, 0], 3] // 4)


@pytest.mark.parametrize("size", SIZES)
def test_chroma_reach(geo, size):
    """What the chroma MC can read: columns -39 .. W/2 + S/2 + 6 and rows -37 .. H/2 + S/2 + 4 for the largest CU size S
    present.  The chroma allocation (margins 48 x 40) holds it for the whole frame and for every CTU row; a margin 4 rows
    smaller does not."""
    W, H = size
    g = build(geo, W, H)
    ok, r = reach(geo, W, H, 0, len(g["tus"]))
    smax = int(g["cus"][:, 2].max())
    assert ok and r == (-39, -37, W // 2 + smax // 2 + 6, H // 2 + smax // 2 + 4), r
    assert not reach(geo, W, H, 0, len(g["tus"]), my=MARGIN_Y // 2 - 4)[0]
    for row in range(g["rows"]):
        ok, rr = reach(geo, W, H, g["rowTu"][row], g["rowTu"][row + 1])
        assert ok and rr[1] >= r[1] and rr[3] <= r[3]


@pytest.mark.parametrize("depth", [8, 10])
def test_chroma_qp_host(geo, depth):
    """The QPs x265cu_analyser_enable_chroma_residual computes on the host equal the oracle driver's."""
    O = load_oracle_chroma(depth)
    for qp in range(qp_max(depth) + 1):
        for off in range(-12, 13):
            assert geo.geo_chroma_qp(qp, off, depth) == O.orc_chroma_qp(qp, off), (qp, off)
