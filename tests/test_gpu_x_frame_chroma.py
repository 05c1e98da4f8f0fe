"""GPU parity of the frame analyser with the chroma-SATD term of subpelCompare switched on (x265cu_analyser_enable_chroma:
the ME stage runs the chroma instantiations of k_me on resident 4:2:0 planes) against the oracle's frame driver, which
tests/test_frame_oracle_vs_ref.py::test_frame_driver_chroma pins to the real MotionEstimate (Yuv setSourcePU, bChroma).
The kernels are the ones tests/test_gpu_me.py::test_me_batch_chroma covers; the analyser glue (plane residency, border
extension, argument passing) first ran green on the round-1 driver box (GPUTEST_r01.json).  Kept in a file that sorts last so that a fault here cannot disturb the verified tests."""
import numpy as np
import pytest

from common import load_oracle
from frame_helpers import Workload, cpu_analyse, lambda_for, MARGIN_X, MARGIN_Y
from me_helpers import mvcost_table

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cu():
    import x265_b200
    return x265_b200.load()


@pytest.mark.timeout(180)
@pytest.mark.parametrize("depth", [8, 10])
@pytest.mark.parametrize("noise", [False, True])
def test_frame_analysis_chroma(cu, depth, noise):
    import x265_b200
    O = load_oracle(depth)
    qp = 30
    W, H = 200, 136
    wl = Workload(W, H, depth=depth, numRefs=2, method=3, subme=3, merange=57, rect=1, qp=qp, noise=noise, chroma=True)
    tab = mvcost_table(O, lambda_for(qp, depth))
    want = cpu_analyse(O, "orc_analyse_frame", wl, tab, threads=8)
    p = wl.params
    an = x265_b200.Analyser(cu, W, H, depth=depth, numRefs=p["numRefs"], method=p["method"], subme=p["subme"],
                            merange=p["merange"], rect=p["rect"], qp=qp, lam=lambda_for(qp, depth))
    an.enable_chroma()
    mx, my = MARGIN_X // 2, MARGIN_Y // 2

    def inner(c):
        return np.ascontiguousarray(c[my:my + H // 2, mx:mx + W // 2])
    for r, ref in enumerate(wl.refs):
        an.set_ref(r, ref[MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W])
        an.set_ref_chroma(r, inner(wl.refC[r][0]), inner(wl.refC[r][1]))
    fenc = np.ascontiguousarray(wl.fenc[MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W])
    an.load_chroma(inner(wl.fencC[0]), inner(wl.fencC[1]))
    an.analyse(fenc, wl.field)
    assert an.njobs == want["njobs"]
    me = an.fetch("me_out").reshape(-1, 4)
    bad = np.nonzero((me[:, :3] != want["me_out"][:, :3]).any(axis=1))[0]
    assert len(bad) == 0, (len(bad), want["jobs"][bad[:3]].tolist(), me[bad[:3]].tolist(), want["me_out"][bad[:3]].tolist())
    assert np.array_equal(an.cu_ref, want["cu_ref"])
    assert np.array_equal(an.fetch("coef"), want["coef"])
    assert np.array_equal(an.cu_numsig, want["cu_numsig"]) and np.array_equal(an.cu_sse, want["cu_sse"])
    assert np.array_equal(an.intra_cost, want["intra_cost"])
    an.close()


@pytest.mark.timeout(180)
@pytest.mark.parametrize("depth", [8, 10])
def test_frame_analysis_amp(cu, depth):
    """rect + AMP PU set (presets slower / veryslow): the host geometry (CPU-checked against the oracle by tests/test_geometry.py)
    feeding the same kernels; every AMP PU size is covered at job level by tests/test_gpu_me.py."""
    import x265_b200
    O = load_oracle(depth)
    qp = 30
    W, H = 200, 136
    wl = Workload(W, H, depth=depth, numRefs=2, method=3, subme=4, merange=57, rect=1, qp=qp, noise=False, amp=1)
    tab = mvcost_table(O, lambda_for(qp, depth))
    want = cpu_analyse(O, "orc_analyse_frame", wl, tab, threads=8)
    p = wl.params
    an = x265_b200.Analyser(cu, W, H, depth=depth, numRefs=p["numRefs"], method=p["method"], subme=p["subme"],
                            merange=p["merange"], rect=p["rect"], qp=qp, lam=lambda_for(qp, depth), amp=1)
    for r, ref in enumerate(wl.refs):
        an.set_ref(r, ref[MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W])
    fenc = np.ascontiguousarray(wl.fenc[MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W])
    an.analyse(fenc, wl.field)
    assert an.njobs == want["njobs"] and an.ncu == want["ncu"]
    assert np.array_equal(an.fetch("jobs"), want["jobs"]), "job lists differ"
    me = an.fetch("me_out").reshape(-1, 4)
    bad = np.nonzero((me[:, :3] != want["me_out"][:, :3]).any(axis=1))[0]
    assert len(bad) == 0, (len(bad), want["jobs"][bad[:3]].tolist(), me[bad[:3]].tolist(), want["me_out"][bad[:3]].tolist())
    assert np.array_equal(an.cu_ref, want["cu_ref"]) and np.array_equal(an.fetch("coef"), want["coef"])
    assert np.array_equal(an.cu_sse, want["cu_sse"]) and np.array_equal(an.intra_cost, want["intra_cost"])
    an.close()
