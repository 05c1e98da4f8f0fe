"""GPU parity of the frame analyser's motion search over the search space the default workload never reaches: other search
methods, sub-pel levels and ranges, far / true / zero / mixed predictor fields, flat areas that make SADs tie, and 10-bit
content that uses every bit.  Every case names the state it is there to reach and asserts, on the host, that its inputs
reach it.  Every ME result, and the residual and intra outputs, are compared with the oracle's frame driver
(tests/test_frame_oracle_vs_ref.py pins that driver to the reference on the same options).  The STAR cases run with the
shared-memory-window search on and off (X265CU_ME_WINDOW).  Most frames are 512x320, so that most 16x16 cells are away
from the picture edge."""
import numpy as np
import pytest

from common import load_oracle
from frame_helpers import Workload, cpu_analyse, lambda_for, run_analyser, assert_frame_equal, MARGIN_X, MARGIN_Y
from me_helpers import mvcost_table

pytestmark = pytest.mark.gpu

MEW_MAP_ROWS = 23            # raster rows a cell's SAD maps hold (me_window.cuh)
CELL_WINDOW_BYTES = 208 * 160  # window budget of an 8-bit 16x16 cell group (me_window.cuh: mew_smem_bytes)


def outside_x(jobs):
    return int(((jobs["mvmin"][:, 0] > 0) | (jobs["mvmax"][:, 0] < 0)).sum())


def flat_4x4(wl):
    """Fraction of the source's 4x4 blocks that are constant."""
    img = wl.fenc[MARGIN_Y:MARGIN_Y + wl.H, MARGIN_X:MARGIN_X + wl.W].astype(np.int64)
    b = img[:wl.H // 4 * 4, :wl.W // 4 * 4].reshape(wl.H // 4, 4, wl.W // 4, 4)
    return float((b.max(axis=(1, 3)) == b.min(axis=(1, 3))).mean())


def cand_ties(jobs):
    """(jobs whose candidate 0 equals the MVP, jobs whose two candidates are equal) -- both skipped by the pre-checks."""
    c0, c1 = jobs["mvc"][:, 0:2], jobs["mvc"][:, 2:4]
    return int((c0 == jobs["qmvp"]).all(axis=1).sum()), int((c0 == c1).all(axis=1).sum())


def raster_rows(jobs):
    """Most raster rows of a job's search range (step 5)."""
    return int(((jobs["mvmax"][:, 1].astype(int) - jobs["mvmin"][:, 1]) // 5 + 1).max())


def window_bytes(jobs):
    """Largest 8-bit search window of one 16x16 PU: its range plus the block."""
    span = jobs["mvmax"].astype(int) - jobs["mvmin"] + 16
    return int((span[:, 0] * span[:, 1]).max())


def _method(m):
    return lambda wl, jobs: (jobs["method"] == m).all()


# name: (state reached, Workload options, host precondition on (workload, oracle job list))
CASES = {
    "dia_subme0": ("ultrafast's DIA with subme 0: every group through the global-memory kernel",
                   dict(method=0, subme=0), _method(0)),
    "hex_subme2": ("x265's default preset, HEX with subme 2, never run through the analyser before",
                   dict(method=1, subme=2), _method(1)),
    "full_r8": ("FULL search with merange 8", dict(method=5, subme=3, merange=8), _method(5)),
    "star_c3_true": ("the c3 path (STAR, subme 3, chroma) with the true motion as predictor: early star exits",
                     dict(chroma=True, field="true"),
                     lambda wl, jobs: (np.abs(jobs["qmvp"] - np.outer(jobs["ref"] + 1, (12, -8))) <= 2).all()),
    "placebo": ("preset placebo: STAR subme 5, AMP, merange 92, 5 references, chroma; windows over the shared-memory budget",
                dict(numRefs=5, subme=5, amp=1, merange=92, chroma=True),
                lambda wl, jobs: window_bytes(jobs) > CELL_WINDOW_BYTES and raster_rows(jobs) > MEW_MAP_ROWS),
    "star_r16": ("merange 16: the star's only far level is distance 16", dict(merange=16),
                 lambda wl, jobs: (jobs["mvmax"][:, 0].astype(int) - jobs["mvmin"][:, 0]).max() == 32),
    "star_r64": ("merange 64: star level 6, no cell star table, more raster rows than the SAD maps hold",
                 dict(merange=64, subme=4), lambda wl, jobs: raster_rows(jobs) > MEW_MAP_ROWS),
    "star_r127": ("merange 127, the largest the job record holds: every window over budget",
                  dict(merange=127), lambda wl, jobs: window_bytes(jobs) > CELL_WINDOW_BYTES and jobs["merange"].max() == 127),
    "far_static": ("far predictors on a static clip: MV 0 wins and the star starts outside its x range",
                   dict(field="far", motion=(0, 0), chroma=True), lambda wl, jobs: outside_x(jobs) > 0.9 * len(jobs)),
    "far_static_hex10": ("the same start outside the range for HEX, 10 bit", dict(field="far", motion=(0, 0), method=1, subme=2, depth=10),
                         lambda wl, jobs: outside_x(jobs) > 0.9 * len(jobs)),
    "far_moving_r92": ("far predictors on moving content, merange 92: windows clamped at the picture edge",
                       dict(field="far", merange=92, subme=5),
                       lambda wl, jobs: (jobs["mvmin"][:, 0] == jobs["mvmax"][:, 0]).any() and outside_x(jobs) > 0.9 * len(jobs)),
    "zero": ("an all-zero field: no MV 0 check and no candidates", dict(field="zero", chroma=True),
             lambda wl, jobs: not jobs["qmvp"].any() and not jobs["mvc"].any()),
    "mixed": ("mixed per-block vectors: candidate 0 equal to the MVP, candidates equal to each other",
              dict(field="mixed", chroma=True), lambda wl, jobs: min(cand_ties(jobs)) > 0.05 * len(jobs)),
    "flat": ("letterbox bars and constant rectangles: tied SADs in the arg-mins, tables and rasters",
             dict(content="flat", chroma=True), lambda wl, jobs: flat_4x4(wl) > 0.3),
    "flat_static_zero": ("flat areas that do not move, searched from MV 0: SAD 0 ties everywhere there",
                         dict(content="flat", motion=(0, 0), field="zero", subme=4), lambda wl, jobs: flat_4x4(wl) > 0.3),
    "full10": ("10-bit content using all 10 bits, 0 to 1023: u16 SAD prefix sums near their limit, packed 10-bit sub-pel",
               dict(content="full10", chroma=True, depth=10, subme=4),
               lambda wl, jobs: wl.fenc.min() == 0 and wl.fenc.max() == 1023 and (wl.fenc & 3).any()),
    "odd_size": ("200x136, not a multiple of 16: partial CTUs and cells at the right and bottom edges",
                 dict(field="mixed", depth=10, W=200, H=136), lambda wl, jobs: wl.W % 16 and wl.H % 16),
}
STAR = [k for k in CASES if CASES[k][1].get("method", 3) == 3]
PARAMS = [(k, w) for k in CASES for w in (("1", "0") if k in STAR else ("1",))]


@pytest.fixture(scope="module")
def cu():
    import x265_b200
    return x265_b200.load()


_want = {}


def _case(name):
    """The case's workload and the oracle's frame (computed once for both window settings)."""
    if name not in _want:
        opts = dict(CASES[name][1])
        W, H = opts.pop("W", 512), opts.pop("H", 320)
        kw = dict(depth=8, numRefs=2, method=3, subme=3, merange=57, rect=1, qp=30)
        kw.update(opts)
        wl = Workload(W, H, **kw)
        O = load_oracle(wl.depth)
        tab = mvcost_table(O, lambda_for(30, wl.depth))
        _want.clear()
        _want[name] = wl, cpu_analyse(O, "orc_analyse_frame", wl, tab, threads=8)
    return _want[name]


@pytest.mark.timeout(300)
@pytest.mark.parametrize("name,window", PARAMS, ids=["%s-window%s" % p for p in PARAMS])
def test_search_space(cu, name, window, monkeypatch):
    wl, want = _case(name)
    assert CASES[name][2](wl, want["jobs"]), "the inputs do not reach: " + CASES[name][0]
    monkeypatch.setenv("X265CU_ME_WINDOW", window)
    an = run_analyser(cu, wl)
    assert_frame_equal(an, want, wl)
    an.close()


# parameters the device cannot run as the reference does, or that the quantiser does not have: the analyser refuses them
REFUSED = [dict(method=2), dict(method=4), dict(method=6), dict(method=-1), dict(merange=128), dict(merange=-1),
           dict(subme=8), dict(subme=-1), dict(W=0), dict(W=204), dict(H=132), dict(H=-8),
           dict(qp=-1), dict(qp=52), dict(depth=10, qp=-1), dict(depth=10, qp=64), dict(qp=-6),
           dict(lam=-0.5), dict(lam=float("inf")), dict(lam=float("nan"))]


@pytest.mark.parametrize("bad", REFUSED, ids=[",".join("%s=%s" % kv for kv in b.items()) for b in REFUSED])
def test_analyser_refuses(cu, bad):
    import x265_b200
    kw = dict(W=64, H=64, method=3, subme=3, merange=57, depth=8, qp=30, lam=None)
    kw.update(bad)
    with pytest.raises(RuntimeError, match="x265cu_analyser_create: (search method|merange|subme|width and height|qp|lambda)"):
        x265_b200.Analyser(cu, kw.pop("W"), kw.pop("H"), numRefs=1, rect=1, **kw)
    # the limits themselves are accepted
    for ok in (dict(method=5, merange=0, subme=0), dict(method=0, merange=127, subme=7), dict(qp=0, lam=0.0), dict(qp=51),
               dict(depth=10, qp=0), dict(depth=10, qp=63, lam=1e6)):
        kw = dict(depth=8, qp=30)
        kw.update(ok)
        x265_b200.Analyser(cu, 64, 64, numRefs=1, rect=1, **kw).close()
