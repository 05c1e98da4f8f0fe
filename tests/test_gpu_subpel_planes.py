"""GPU checks of the frame analyser's quarter-pel phase planes (MePlanes, me.cuh; analyser.cuh): every reference carries 15
interpolated copies, built on every run, and the sub-pel refinement reads its candidates from them as full-pel blocks.
The planes are compared pixel for pixel with the oracle's luma_hpp / luma_vpp / luma_hvpp over the rectangle the build
promises, a row-range run is compared with a full-frame run, and a frame whose vectors run far off every picture edge is
compared with the oracle's frame driver."""
import numpy as np
import pytest

from common import load_oracle, ptr, IP
from frame_helpers import Workload, cpu_analyse, lambda_for, run_analyser, assert_frame_equal, MARGIN_X, MARGIN_Y
from me_helpers import mvcost_table

pytestmark = pytest.mark.gpu

# the rectangle the build writes, picture-relative: columns [-PLANE_X, W + PLANE_X), rows [-PLANE_Y, H + PLANE_Y)
# (AN_PLANE_X / AN_PLANE_Y, analyser.cuh)
PLANE_X, PLANE_Y = 80, 76
# what the sub-pel refinement can read, inclusive: columns [-76, W + 74], rows [-71, H + 70] (analyser.cuh)
READ_X0, READ_X1, READ_Y0, READ_Y1 = -76, 74, -71, 70


@pytest.fixture(scope="module")
def cu():
    import x265_b200
    return x265_b200.load()


def oracle_planes(O, wl, ref):
    """The 16 phase planes of reference `ref` of the workload by the oracle, over the build rectangle; the rest 0."""
    src = wl.refs[ref]
    stride = wl.stride
    w, h = wl.W + 2 * PLANE_X, wl.H + 2 * PLANE_Y
    off = (MARGIN_Y - PLANE_Y) * stride + (MARGIN_X - PLANE_X)
    out = np.zeros((16,) + src.shape, src.dtype)
    out[0] = src
    for yf in range(4):
        for xf in range(4):
            if not (xf | yf):
                continue
            d = out[yf * 4 + xf]
            if not yf:
                O.orc_interp_hpp(ptr(src, off), IP(stride), ptr(d, off), IP(stride), xf, 8, w, h)
            elif not xf:
                O.orc_interp_vpp(ptr(src, off), IP(stride), ptr(d, off), IP(stride), yf, 8, w, h)
            else:       # the oracle's hvpp takes blocks of up to 64x64
                for y in range(0, h, 64):
                    for x in range(0, w, 64):
                        o = off + y * stride + x
                        O.orc_interp_hvpp(ptr(src, o), IP(stride), ptr(d, o), IP(stride), xf, yf, 8, min(64, w - x), min(64, h - y))
    return out


def assert_planes_equal(an, O, wl):
    for r in range(len(wl.refs)):
        want = oracle_planes(O, wl, r)
        for ph in range(16):
            got = an.fetch(("plane", r, ph))
            bad = np.argwhere(got != want[ph])
            assert len(bad) == 0, ("ref", r, "phase", ph, len(bad), (bad[:4] - (MARGIN_Y, MARGIN_X)).tolist())


PLANE_CASES = [(8, "smooth"), (8, "noise"), (10, "smooth"), (10, "full10")]


@pytest.mark.parametrize("depth,content", PLANE_CASES, ids=["%d-%s" % c for c in PLANE_CASES])
def test_phase_planes(cu, depth, content):
    """Every pixel of every phase plane equals the oracle's interpolation inside the build rectangle and is 0 outside it."""
    assert -PLANE_X <= READ_X0 and READ_X1 < PLANE_X and -PLANE_Y <= READ_Y0 and READ_Y1 < PLANE_Y
    wl = Workload(200, 136, depth=depth, numRefs=2, content=content)
    O = load_oracle(depth)
    an = run_analyser(cu, wl)
    assert_planes_equal(an, O, wl)
    an.close()


def test_row_range_builds_planes(cu):
    """A row-range run on a fresh analyser builds the whole rectangle (a PU of any CTU row can reach every row of it), and
    its ME results equal those of a full-frame run."""
    wl = Workload(256, 320, depth=8, numRefs=2, field="mixed")
    O = load_oracle(8)
    full = run_analyser(cu, wl)
    want = full.me_packed.copy()
    full.close()
    import x265_b200
    p = wl.params
    an = x265_b200.Analyser(cu, wl.W, wl.H, depth=8, numRefs=p["numRefs"], method=p["method"], subme=p["subme"],
                            merange=p["merange"], rect=p["rect"], qp=p["qp"], lam=lambda_for(p["qp"], 8), amp=p["amp"])
    for r, ref in enumerate(wl.refs):
        an.set_ref(r, ref[MARGIN_Y:MARGIN_Y + wl.H, MARGIN_X:MARGIN_X + wl.W])
    r0, r1 = 2, 4
    an.analyse_rows(np.ascontiguousarray(wl.fenc[MARGIN_Y:MARGIN_Y + wl.H, MARGIN_X:MARGIN_X + wl.W]), wl.field, r0, r1)
    assert_planes_equal(an, O, wl)
    j0, nj, _, _ = an.row_range(r0, r1)
    assert nj > 0 and np.array_equal(an.me_packed[j0:j0 + nj], want[j0:j0 + nj])
    an.close()


def final_blocks(wl, res):
    """(left, top, right, bottom) picture-relative full-pel columns / rows of every job's final block on its phase plane."""
    jobs, me = res["jobs"], res["me_out"].reshape(-1, 4)
    y, x = np.divmod(jobs["offset"].astype(np.int64), wl.stride)
    bx, by = me[:, 1].astype(np.int64) >> 2, me[:, 2].astype(np.int64) >> 2
    return x + bx, y + by, x + bx + jobs["pw"] - 1, y + by + jobs["ph"] - 1


FAR_CASES = {"star_chroma": dict(chroma=True), "hex_10bit": dict(method=1, subme=7, depth=10)}


@pytest.mark.timeout(300)
@pytest.mark.parametrize("name", sorted(FAR_CASES))
def test_far_off_every_edge(cu, name):
    """Predictors far off the picture (the search windows collapse against the clip on every side): final blocks lie more
    than 16 pixels past every picture edge and within 8 pixels of the left, top and bottom sides of the readable
    rectangle, none outside it, and every output equals the oracle's frame driver."""
    kw = dict(depth=8, numRefs=2, method=3, subme=3, merange=92, field="far")
    kw.update(FAR_CASES[name])
    wl = Workload(512, 320, **kw)
    O = load_oracle(wl.depth)
    want = cpu_analyse(O, "orc_analyse_frame", wl, mvcost_table(O, lambda_for(30, wl.depth)), threads=8)
    l, t, r, b = final_blocks(wl, want)
    assert l.min() <= READ_X0 + 8 and r.max() >= wl.W + 16, (l.min(), r.max())
    assert t.min() <= READ_Y0 + 8 and b.max() >= wl.H + READ_Y1 - 8, (t.min(), b.max())
    assert l.min() >= READ_X0 and r.max() <= wl.W + READ_X1 and t.min() >= READ_Y0 and b.max() <= wl.H + READ_Y1
    an = run_analyser(cu, wl)
    assert_frame_equal(an, want, wl)
    an.close()
