"""Adaptive quantisation: the plain-C restatement of calcAdaptiveQuantFrame (oracle/oracle_aq.c) against the REAL function
on a real Frame (oracle/ref_shim_aq.cpp), every output compared (doubles by bit pattern, arrays including the words the
reference leaves alone); and the library's host finish, x265cu_aq_finish from libx265cu.so (no device), against the
restatement on the restatement's energies and totals.  Where oracle/_ref is absent the reference's stored results
(tests/golden/aq_ref.json) stand in for it.  CPU only."""
import ctypes as C

import numpy as np
import pytest

import aq_helpers as A
import x265_b200

MATRIX = A.param_matrix()


@pytest.fixture(scope="module")
def cu():
    return x265_b200.load(need_gpu=False)


@pytest.mark.parametrize("case", A.PICTURES, ids=[c[0] for c in A.PICTURES])
def test_aq_oracle_matches_reference(request, case):
    name, W, H, depth, c420, content = case
    R = A.AqRefResults(request, depth)
    pic = A.make_picture(case)
    for prm in MATRIX:
        R.same(A.key(prm), lambda: A.reference(pic, W, H, depth, prm), A.oracle(pic, W, H, depth, prm))


def _lib_finish(cu, pic, W, H, depth, prm):
    """x265cu_aq_finish on the oracle's energies and totals, its arrays prefilled as the oracle's: (rc, outputs)."""
    from x265_b200.lib import AqOut, AqParams
    e, t = A.oracle_energy(pic, W, H, depth, prm[2])
    _, count, n8 = A.geometry(W, H, prm[2])
    qo = A.quant_offsets(count)
    mode, s, qg, wp, var, use_qo = prm
    p = AqParams(aqMode=mode, qgSize=qg, weightp=wp, variance=var, aqStrength=s, quantOffsets=qo.ctypes.data if use_qo else None)
    qp, iq, bv = A.prefilled(count)
    iq8 = np.zeros(n8, np.int32)
    wps, wpd, fv = np.zeros(3, np.uint64), np.zeros(3, np.uint64), np.zeros(1)
    out = AqOut(qp.ctypes.data, iq.ctypes.data, iq8.ctypes.data if qg == 8 else None, wps.ctypes.data, wpd.ctypes.data,
                bv.ctypes.data, fv.ctypes.data)
    rc = cu.L.x265cu_aq_finish(depth, W, H, C.byref(p), e.ctypes.data, t.ctypes.data, C.byref(out))
    return rc, A.outputs(prm, qp, iq, iq8, wps, wpd, bv, fv[0])


@pytest.mark.parametrize("case", A.PICTURES, ids=[c[0] for c in A.PICTURES])
def test_aq_finish_matches_oracle(cu, case):
    """The library's finish equals the restatement bit for bit; it refuses only the fades-grid case it documents."""
    name, W, H, depth, c420, content = case
    pic = A.make_picture(case)
    refused = 0
    for prm in MATRIX:
        rc, got = _lib_finish(cu, pic, W, H, depth, prm)
        if A.finish_refused(W, H, prm):
            assert rc == -1 and "fades pass" in cu.last_error(), prm
            refused += 1
            continue
        assert rc == 0, (prm, cu.last_error())
        want = A.oracle(pic, W, H, depth, prm)
        assert A.same_outputs(want, got), (prm, {k: (want[k], got[k]) for k in want})
    assert refused == 0 or (W % 16 == 8 or H % 16 == 8)


def test_aq_quirks_are_reached():
    """The 328x184 pictures of the matrix reach the qgSize 8 quirks: blockCount above the blocks the loops visit (the
    averages divide by it) and the 8x8 reduction's stride differing from the loop's row."""
    W, H = 328, 184
    nb, count, _ = A.geometry(W, H, 8)
    assert nb < count and (W + 7) // 8 != 2 * ((W // 2 + 7) >> 3)
    pic = A.make_picture(("", W, H, 10, True, "fullrange"))
    o = A.oracle(pic, W, H, 10, (2, 1.0, 8, 0, 1, 0))
    assert o["invQscaleFactor8x8"].min() > 0 and o["frameVariance"] > 0


def test_aq_weightp_correction_wraps(cu):
    """wp_ssd -= (sum * sum + n / 2) / n in uint64: on a white 3840x2160 10-bit picture sum * sum wraps, and the finish
    wraps exactly as the restatement does."""
    from x265_b200.lib import AqOut, AqParams
    W, H = 3840, 2160
    n = W * H
    s = n * 1023
    t = np.array([s, n * 1023 * 1023, 0, 0, 0, 0], np.uint64)
    e = np.zeros(A.geometry(W, H, 32)[0], np.uint32)
    p = AqParams(aqMode=0, qgSize=32, weightp=1, aqStrength=1.0)
    wps, wpd = np.zeros(3, np.uint64), np.zeros(3, np.uint64)
    out = AqOut(None, None, None, wps.ctypes.data, wpd.ctypes.data, None, None)
    assert cu.L.x265cu_aq_finish(10, W, H, C.byref(p), e.ctypes.data, t.ctypes.data, C.byref(out)) == 0
    want = (n * 1023 * 1023 - ((s * s) % 2 ** 64 + n // 2) % 2 ** 64 // n) % 2 ** 64
    assert int(wps[0]) == s and int(wpd[0]) == want and (s * s) >= 2 ** 64


@pytest.mark.parametrize("what,kw", [("aq-mode 4", dict(aqMode=4)), ("hevc-aq", dict(hevcAq=1)), ("HDR10 opt", dict(hdr10Opt=1)),
                                     ("aq-motion", dict(aqMotion=1)), ("qgSize", dict(qgSize=12)), ("depth", dict(depth=12)),
                                     ("odd", dict(width=63)), ("8x8", dict(only8x8=True))])
def test_aq_finish_refusals(cu, what, kw):
    from x265_b200.lib import AqOut, AqParams
    depth, W = kw.pop("depth", 8), kw.pop("width", 64)
    only8 = kw.pop("only8x8", False)
    p = AqParams(aqMode=2, qgSize=8 if only8 else 32, aqStrength=1.0)
    for k, v in kw.items():
        setattr(p, k, v)
    e, t = np.zeros(64, np.uint32), np.zeros(6, np.uint64)
    iq8 = np.zeros(16, np.int32)
    out = AqOut(None, None, iq8.ctypes.data if only8 else None, None, None, None, None)
    assert cu.L.x265cu_aq_finish(depth, W, 64, C.byref(p), e.ctypes.data, t.ctypes.data, C.byref(out)) == -1
    assert "x265cu_aq_finish" in cu.last_error()
