"""GPU parity of the frame analyser's per-CU stages: the luma residual chain (k_cu_residual, one launch per luma TU size over
its own work list) and the intra mode search (k_intra_cu, a warp per 8x8 CU or per 16x16 quadrant, angular modes in the
vertical-family frame against the transposed source).  Every result of the stages -- cu_sse, cu_numsig, cu_ref, the levels,
the four recon planes and intra_cost -- is compared bit for bit with the oracle's frame driver:
  * 8 and 10 bit, smooth and noise content, flat black and flat maximum pictures (numSig 0, the DC-only shortcut and the
    reconstruction clip), at QP 0 and the top QP, on a 200x136 picture whose last CTU row is 8 pixels high;
  * a CTU-row range analysed alone;
  * a 1920x1152 picture, on which every per-size launch runs more than one grid-stride pass on a 132-SM H100, against the
    driver's first CTU rows of the full-frame geometry."""
import numpy as np
import pytest

from common import load_oracle
from frame_helpers import (Workload, cpu_analyse, lambda_for, qp_max, run_analyser, assert_frame_equal, tu_classes,
                           recon_overshoot, pad_plane, MARGIN_X, MARGIN_Y)
from me_helpers import mvcost_table

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cu():
    import x265_b200
    return x265_b200.load()


def workload(W, H, depth, qp, content):
    """content "smooth" / "noise", or "black" / "white": every plane (source and references) one constant value."""
    flat = content in ("black", "white")
    wl = Workload(W, H, depth=depth, numRefs=2, method=3, subme=3, merange=57, rect=1, qp=qp,
                  content=None if flat else content)
    if flat:
        v = 0 if content == "black" else (1 << depth) - 1
        for plane in [wl.fenc] + wl.refs:
            plane[...] = v
    return wl


def oracle(wl, max_ctu_rows=0):
    O = load_oracle(wl.depth)
    return cpu_analyse(O, "orc_analyse_frame", wl, mvcost_table(O, lambda_for(wl.params["qp"], wl.depth)), threads=8,
                       max_ctu_rows=max_ctu_rows)


CASES = [(content, depth, qp) for content in ("smooth", "noise", "black", "white") for depth in (8, 10)
         for qp in (0, qp_max(depth))]


@pytest.mark.parametrize("content,depth,qp", CASES, ids=["%s-%d-qp%d" % c for c in CASES])
def test_cu_stages_frame(cu, content, depth, qp):
    W, H = 200, 136
    assert (H - 1) % 64 + 1 == 8
    wl = workload(W, H, depth, qp, content)
    want = oracle(wl)
    n = tu_classes(want)
    if content in ("black", "white"):
        assert n["zero"] == sum(n.values()), n            # a constant picture predicts itself: numSig 0 everywhere
    elif content == "noise" and qp == 0:
        assert n["full"] > 0, n
    elif content == "smooth" and qp == qp_max(depth):
        assert n["zero"] > 0, n
    an = run_analyser(cu, wl, lam=lambda_for(qp, depth))
    assert_frame_equal(an, want, wl)
    an.close()


def test_cu_stages_dc_only_and_clip(cu):
    """The DC-only inverse transform and the reconstruction clip: the source is a white picture with a black rectangle,
    the references black, so that most TUs carry a large constant residual."""
    W, H = 200, 136
    wl = workload(W, H, 8, 0, "black")
    img = np.full((H, W), 255, np.uint8)
    img[40:90, 37:141] = 0
    wl.fenc[...] = pad_plane(img, 8)[0]                 # margins extended as the device extends them
    want = oracle(wl)
    n = tu_classes(want)
    assert n["dc"] > 0 and n["full"] > 0, n
    assert recon_overshoot(load_oracle(8), want, wl) > 0
    an = run_analyser(cu, wl, lam=lambda_for(0, 8))
    assert_frame_equal(an, want, wl)
    an.close()


def _row_slices(an, want, wl, c0, c1):
    """The stage outputs of the CUs [c0, c1) and of their picture rows, against the driver's frame `want`."""
    for k in ("cu_sse", "cu_numsig", "cu_ref", "intra_cost"):
        assert np.array_equal(np.asarray(getattr(an, k))[c0:c1], want[k][c0:c1]), k
    off = want["cu_coef_off"]
    k0 = int(off[c0]); k1 = int(off[c1 - 1]) + int(want["cus"][c1 - 1][2]) ** 2
    assert np.array_equal(an.fetch("coef")[k0:k1], want["coef"][k0:k1])
    y0 = int(want["cus"][c0][1]) // 64 * 64; y1 = min((int(want["cus"][c1 - 1][1]) // 64 + 1) * 64, wl.H)
    W = wl.W
    for d in range(4):
        got = an.fetch("recon%d" % d).reshape(wl.fenc.shape)[MARGIN_Y + y0:MARGIN_Y + y1, MARGIN_X:MARGIN_X + W]
        assert np.array_equal(got, want["recon"][d][MARGIN_Y + y0:MARGIN_Y + y1, MARGIN_X:MARGIN_X + W]), "recon depth %d" % d


@pytest.mark.parametrize("depth", [8, 10])
def test_cu_stages_row_range(cu, depth):
    """CTU rows [1, 3) of a 4-row picture analysed alone: the launches read only their rows' slices of the per-size lists."""
    import x265_b200
    W, H, qp = 200, 200, 30
    wl = workload(W, H, depth, qp, "noise")
    want = oracle(wl)
    p = wl.params
    an = x265_b200.Analyser(cu, W, H, depth=depth, numRefs=p["numRefs"], method=p["method"], subme=p["subme"],
                            merange=p["merange"], rect=p["rect"], qp=qp, lam=lambda_for(qp, depth))
    for r, ref in enumerate(wl.refs):
        an.set_ref(r, ref[MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W])
    for k in ("cu_sse", "cu_numsig", "cu_ref", "intra_cost"):
        getattr(an, k)[...] = 0
    an.analyse_rows(np.ascontiguousarray(wl.fenc[MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W]), wl.field, 1, 3)
    _, _, c0, nc = an.row_range(1, 3)
    _row_slices(an, want, wl, c0, c0 + nc)
    # the rows outside the range were not written
    _, _, c3, _ = an.row_range(3, 4)
    assert not np.asarray(an.intra_cost)[c3:].any()
    an.close()


@pytest.mark.timeout(600)
def test_cu_stages_multi_pass(cu):
    """1920x1152 (540 CTUs): more list entries than each per-size launch has CTA slots, so every launch strides over its
    list; the first two CTU rows against the driver over the full-frame geometry."""
    W, H, depth, qp = 1920, 1152, 8, 30
    wl = workload(W, H, depth, qp, "smooth")
    want = oracle(wl, max_ctu_rows=2)
    an = run_analyser(cu, wl, lam=lambda_for(qp, depth))
    assert an.ncu == want["ncu"]
    counts = np.bincount(np.asarray(want["cus"][:, 2]).astype(np.int64) // 8, minlength=9)
    sms = 132                                            # H100 SXM
    # intra lists of 32 (a CTA each), 16 and 8 (four per CTA), 16 CTAs per SM; the TU lists are longer or take fewer CTAs
    assert counts[4] > 16 * sms and counts[2] // 4 > 16 * sms and counts[1] // 4 > 16 * sms
    _row_slices(an, want, wl, 0, want["ncu_run"])
    an.close()
