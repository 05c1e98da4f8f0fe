"""GPU parity of the per-cell pre-checks (k_me_precheck_cell: one table of 4x4 SADs and chroma Hadamard sums per 16x16 cell,
every job folded from it) on frames whose cells are mostly away from the picture edge, so that the table path rather than the
per-PU fallback decides almost every job.  Every ME result is compared with the oracle's frame driver."""
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


def _run(cu, depth, noise, amp, subme):
    import x265_b200
    O = load_oracle(depth)
    qp = 30
    W, H = 512, 320
    wl = Workload(W, H, depth=depth, numRefs=2, method=3, subme=subme, merange=57, rect=1, qp=qp, noise=noise, chroma=True, amp=amp)
    tab = mvcost_table(O, lambda_for(qp, depth))
    want = cpu_analyse(O, "orc_analyse_frame", wl, tab, threads=8, stages=1)
    p = wl.params
    an = x265_b200.Analyser(cu, W, H, depth=depth, numRefs=p["numRefs"], method=p["method"], subme=p["subme"],
                            merange=p["merange"], rect=p["rect"], qp=qp, lam=lambda_for(qp, depth), amp=amp)
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
    an.close()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("depth", [8, 10])
@pytest.mark.parametrize("noise", [False, True])
def test_precheck_cells_chroma(cu, depth, noise):
    _run(cu, depth, noise, amp=0, subme=3)


@pytest.mark.timeout(300)
def test_precheck_cells_chroma_amp(cu):
    _run(cu, 10, False, amp=1, subme=4)
