"""GPU parity of the per-CU sub-pel refinement (k_me_subpel_group: one warp runs the sub-pel rounds of the 2Nx2N / 2NxN /
Nx2N PUs of a CU 64 or CU 32 and evaluates each distinct candidate position once, over the 16x16 blocks the asking PUs
cover).  Every ME result (cost, mv) of the analyser is compared with the oracle's frame driver on a picture with whole
CTUs and a cut last CTU row and column: 8 and 10 bit, subme 2 / 3 / 4 / 7, with and without the chroma-SATD term, with and
without AMP (whose parts stay on the per-PU launch, as a job list), on smooth content (the PUs of a CU mostly share their
positions), noise (they mostly do not), flat areas (zero costs and pre-check winners), and with a predictor field that gives
the PUs of one CU different starts.  A run over CTU-row ranges must equal the full frame."""
import numpy as np
import pytest

from common import load_oracle
from frame_helpers import Workload, cpu_analyse, lambda_for, run_analyser, MARGIN_X, MARGIN_Y
from me_helpers import mvcost_table

pytestmark = pytest.mark.gpu

W, H = 264, 200                                       # 4 x 3 whole CTUs; the last CTU column is 8 wide (no CU), the last row 8 high

CASES = {
    "smooth8_s3_chroma": dict(depth=8, subme=3, chroma=True),
    "noise8_s3_chroma": dict(depth=8, subme=3, chroma=True, noise=True),
    "smooth8_s2": dict(depth=8, subme=2, chroma=True),                       # subme 2: no chroma term
    "smooth8_s3_norect": dict(depth=8, subme=3, chroma=True, rect=0),        # one PU per CU
    "noise8_s7_amp": dict(depth=8, subme=7, amp=1, noise=True),
    "smooth8_s3_amp_chroma": dict(depth=8, subme=3, chroma=True, amp=1),
    "smooth10_s4_amp_chroma": dict(depth=10, subme=4, chroma=True, amp=1),
    "noise10_s7_amp_chroma": dict(depth=10, subme=7, chroma=True, amp=1, noise=True),
    "noise10_s4": dict(depth=10, subme=4, noise=True),
    "smooth10_s3_chroma": dict(depth=10, subme=3, chroma=True),
    "mixed8_s3_chroma": dict(depth=8, subme=3, chroma=True, field="mixed"),  # the PUs of a CU start from different vectors
    "mixed10_s7_amp_chroma": dict(depth=10, subme=7, chroma=True, amp=1, field="mixed", noise=True),
    "true8_s4_chroma": dict(depth=8, subme=4, chroma=True, field="true"),    # every PU converges on the same vector
    "flat8_s3_static": dict(depth=8, subme=3, chroma=True, content="flat", motion=(0, 0), field="zero"),
    "flat10_s7_amp_chroma": dict(depth=10, subme=7, chroma=True, amp=1, content="flat"),
}


@pytest.fixture(scope="module")
def cu():
    import x265_b200
    return x265_b200.load()


def _workload(depth, subme, chroma=False, amp=0, rect=1, **kw):
    return Workload(W, H, depth=depth, numRefs=2, method=3, subme=subme, merange=57, rect=rect, qp=30, chroma=chroma, amp=amp, **kw)


def _want(wl):
    O = load_oracle(wl.depth)
    return cpu_analyse(O, "orc_analyse_frame", wl, mvcost_table(O, lambda_for(30, wl.depth)), threads=8, stages=1)


def _assert_me_equal(me, want, jobs):
    bad = np.nonzero((me[:, :3] != want[:, :3]).any(axis=1))[0]
    assert len(bad) == 0, (len(bad), len(me), jobs[bad[:4]].tolist(), me[bad[:4]].tolist(), want[bad[:4]].tolist())


@pytest.mark.timeout(300)
@pytest.mark.parametrize("name", sorted(CASES))
def test_subpel_groups(cu, name):
    wl = _workload(**CASES[name])
    want = _want(wl)
    an = run_analyser(cu, wl)
    assert an.njobs == want["njobs"]
    jobs = an.fetch("jobs")
    sides = {(int(w), int(h)) for w, h in zip(jobs["pw"], jobs["ph"])}
    assert {(64, 64), (32, 32)} <= sides and ((64, 32) in sides) == bool(wl.params["rect"])      # the PUs this kernel refines
    me = an.fetch("me_out").reshape(-1, 4)
    _assert_me_equal(me, want["me_out"], want["jobs"])
    an.close()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("depth,amp", [(8, 0), (10, 1)])
def test_subpel_groups_row_ranges(cu, depth, amp):
    """CTU-row ranges analysed in any order give the ME results of the full frame."""
    import x265_b200
    wl = _workload(depth, 4, chroma=True, amp=amp, noise=True)
    full = run_analyser(cu, wl)
    want = full.fetch("me_out").reshape(-1, 4).copy()
    nrows = full.ctu_rows
    full.close()
    assert nrows == 4
    p = wl.params
    an = x265_b200.Analyser(cu, W, H, depth=depth, numRefs=p["numRefs"], method=p["method"], subme=p["subme"],
                            merange=p["merange"], rect=p["rect"], qp=p["qp"], lam=lambda_for(p["qp"], depth), amp=p["amp"])
    for r, ref in enumerate(wl.refs):
        an.set_ref(r, ref[MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W])
    an.enable_chroma()
    mx, my = MARGIN_X // 2, MARGIN_Y // 2

    def inner(c):
        return np.ascontiguousarray(c[my:my + H // 2, mx:mx + W // 2])
    for r in range(len(wl.refs)):
        an.set_ref_chroma(r, inner(wl.refC[r][0]), inner(wl.refC[r][1]))
    an.load_chroma(inner(wl.fencC[0]), inner(wl.fencC[1]))
    fenc = np.ascontiguousarray(wl.fenc[MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W])
    seen = 0
    for r0, r1 in ((2, 3), (0, 2), (3, 4)):
        an.analyse_rows(fenc, wl.field, r0, r1)
        j0, nj, _, _ = an.row_range(r0, r1)
        me = an.fetch("me_out").reshape(-1, 4)
        _assert_me_equal(me[j0:j0 + nj], want[j0:j0 + nj], an.fetch("jobs")[j0:j0 + nj])
        seen += nj
    assert seen == an.njobs
    an.close()
