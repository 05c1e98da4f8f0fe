"""GPU parity of the frame analyser across the quantiser's QP range.  The residual chain of k_cu_residual has its own
restatement of the quantiser (resid_quant's scale chains indexed by qp % 6 and shifts from qp / 6, the int16 clip of the
levels, the DC-only shortcut and the clip of the reconstruction), and the mv cost lambda of each QP decides the searches: at QP 0 SAD ties do, at the top QP
the MVP does.  Every case of test_frame_oracle_vs_ref.py::test_frame_driver_qp, which pins the oracle's frame driver to
the reference on the same workloads, is compared bit for bit with that driver, with the same host-checked
preconditions; at 512x320, where most search windows are away from the picture edge, the cut and the flat areas run
with the shared-memory-window search on and off (X265CU_ME_WINDOW)."""
import pytest

from common import load_oracle
from frame_helpers import (Workload, cpu_analyse, lambda_for, qp_max, run_analyser, assert_frame_equal, assert_qp_case_reaches,
                           QP_CASES)
from me_helpers import mvcost_table

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cu():
    import x265_b200
    return x265_b200.load()


def _frame(content, depth, qp, chroma, W, H):
    """The workload and the oracle's frame, after asserting that the case reaches what it is for."""
    wl = Workload(W, H, depth=depth, numRefs=2, method=3, subme=3, merange=57, rect=1, qp=qp, content=content, chroma=chroma)
    O = load_oracle(depth)
    want = cpu_analyse(O, "orc_analyse_frame", wl, mvcost_table(O, lambda_for(qp, depth)), threads=8)
    assert_qp_case_reaches(O, content, wl, want)
    return wl, want


@pytest.mark.parametrize("content,depth,qp,chroma", QP_CASES, ids=["%s-%d-qp%d" % c[:3] for c in QP_CASES])
def test_qp_frame(cu, content, depth, qp, chroma):
    wl, want = _frame(content, depth, qp, chroma, 200, 136)
    an = run_analyser(cu, wl, lam=lambda_for(qp, depth))
    assert_frame_equal(an, want, wl)
    an.close()


WINDOW_CASES = [(content, depth, qp, window) for content in ("cut", "flat") for depth in (8, 10) for qp in (0, qp_max(depth))
                for window in ("1", "0")]
_want = {}


def unclamped(jobs):
    """Fraction of the jobs whose search window is not cut by the picture edge."""
    span = jobs["mvmax"].astype(int) - jobs["mvmin"]
    return float((span == 2 * jobs["merange"][:, None].astype(int)).all(axis=1).mean())


@pytest.mark.timeout(300)
@pytest.mark.parametrize("content,depth,qp,window", WINDOW_CASES, ids=["%s-%d-qp%d-window%s" % c for c in WINDOW_CASES])
def test_qp_frame_window(cu, content, depth, qp, window, monkeypatch):
    """512x320: the per-cell pre-check and star tables and the window raster decide most jobs, here under the costs of the
    QP extremes, with every SAD tied (cut) or many tied (flat)."""
    key = (content, depth, qp)
    if key not in _want:
        _want.clear()
        _want[key] = _frame(content, depth, qp, content == "flat", 512, 320)
    wl, want = _want[key]
    assert unclamped(want["jobs"]) > 0.5
    monkeypatch.setenv("X265CU_ME_WINDOW", window)
    an = run_analyser(cu, wl, lam=lambda_for(qp, depth))
    assert_frame_equal(an, want, wl)
    an.close()
