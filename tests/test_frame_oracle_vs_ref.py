"""Pins the oracle's frame-level CTU-analysis driver against the same driver running on the REAL
reference code (MotionEstimate class + C primitive table, oracle/_ref; its stored results where oracle/_ref is not
built, tests/ref_results.py).  CPU only."""
import numpy as np
import pytest

from common import load_oracle
from frame_helpers import Workload, cpu_analyse, lambda_for, assert_qp_case_reaches, MVRANGE, QP_CASES
from me_helpers import mvcost_table
from ref_results import RefResults

COMPARED = ("njobs", "ncu", "jobs", "me_out", "cu_jobs", "cus", "cu_ref", "coef", "cu_sse", "cu_numsig", "recon", "intra_cost")


def compare(G, a, wl, tab):
    """The oracle's frame `a` against the reference driver on the same workload."""
    G.same("frame", lambda: {k: v for k, v in cpu_analyse(G.R, "x265ref_analyse_frame", wl, tab, threads=4).items() if k in COMPARED},
           {k: v for k, v in a.items() if k in COMPARED})


@pytest.mark.parametrize("depth", [8, 10])
@pytest.mark.parametrize("noise", [False, True])
def test_frame_driver(depth, noise, request):
    G = RefResults(request, depth)
    O = load_oracle(depth)
    qp = 30
    wl = Workload(200, 136, depth=depth, numRefs=2, method=3, subme=3, merange=57, rect=1, qp=qp, noise=noise)
    G.same("lambda", lambda: G.R.x265ref_lambda(qp), lambda_for(qp, depth))
    tab = mvcost_table(O, lambda_for(qp, depth))
    a = cpu_analyse(O, "orc_analyse_frame", wl, tab, threads=4)
    assert a["njobs"] > 2000 and a["cu_numsig"].sum() > 0
    compare(G, a, wl, tab)


@pytest.mark.parametrize("depth", [8, 10])
@pytest.mark.parametrize("noise", [False, True])
def test_frame_driver_chroma(depth, noise, request):
    """The same frame with 4:2:0 chroma planes: every ME job runs as the encoder's setSourcePU(Yuv, ..., bChroma = true) call,
    i.e. with the chroma-SATD term of subpelCompare for the PUs that have one (motion.cpp:204-212, 1601-1661)."""
    G = RefResults(request, depth)
    O = load_oracle(depth)
    qp = 30
    wl = Workload(200, 136, depth=depth, numRefs=2, method=3, subme=3, merange=57, rect=1, qp=qp, noise=noise, chroma=True)
    tab = mvcost_table(O, lambda_for(qp, depth))
    a = cpu_analyse(O, "orc_analyse_frame", wl, tab, threads=4)
    compare(G, a, wl, tab)
    # the term is really on: results differ from the luma-only run of the same frame
    wl.chroma = False
    c = cpu_analyse(O, "orc_analyse_frame", wl, tab, threads=4)
    assert np.array_equal(a["jobs"], c["jobs"])
    assert (a["me_out"][:, 0] != c["me_out"][:, 0]).mean() > 0.3


def outside_x(jobs):
    """Jobs whose search range excludes 0 in x: where MV 0 wins their pre-checks, the search starts outside the range."""
    return int(((jobs["mvmin"][:, 0] > 0) | (jobs["mvmax"][:, 0] < 0)).sum())


# (name, depth, Workload options): the predictor fields, motions, contents and search methods beyond the default workload
SEARCH_SPACE = [
    ("far_static_star_chroma", 8, dict(field="far", motion=(0, 0), chroma=True)),
    ("far_static_star_chroma", 10, dict(field="far", motion=(0, 0), chroma=True)),
    ("far_static_hex", 8, dict(field="far", motion=(0, 0), method=1, subme=2)),
    ("far_static_dia", 10, dict(field="far", motion=(0, 0), method=0, subme=0)),
    ("far_moving_star92", 8, dict(field="far", merange=92, subme=5)),
    ("flat_chroma", 8, dict(content="flat", chroma=True)),
    ("flat_static_zero", 8, dict(content="flat", motion=(0, 0), field="zero")),
    ("true", 8, dict(field="true")),
    ("zero", 10, dict(field="zero", chroma=True)),
    ("mixed_chroma", 8, dict(field="mixed", chroma=True)),
    ("full10_chroma", 10, dict(content="full10", chroma=True)),
    ("full10_mixed_amp", 10, dict(content="full10", field="mixed", subme=4, amp=1)),
]


@pytest.mark.parametrize("name,depth,opts", SEARCH_SPACE, ids=["%s-%d" % (c[0], c[1]) for c in SEARCH_SPACE])
def test_frame_driver_search_space(name, depth, opts, request):
    """The frame driver on the workload options of frame_helpers: far predictors (with a static clip MV 0 wins and the
    search starts outside its x range), the true motion, an all-zero field, mixed per-block vectors, flat areas that make
    SADs tie, and 10-bit content using every bit."""
    G = RefResults(request, depth)
    O = load_oracle(depth)
    qp = 30
    kw = dict(numRefs=2, method=3, subme=3, merange=57, rect=1, qp=qp)
    kw.update(opts)
    wl = Workload(200, 136, depth=depth, **kw)
    tab = mvcost_table(O, lambda_for(qp, depth))
    a = cpu_analyse(O, "orc_analyse_frame", wl, tab, threads=4)
    if opts.get("field") == "far":
        assert outside_x(a["jobs"]) > 0.9 * a["njobs"]
    if opts.get("content") == "full10":
        assert wl.fenc.min() == 0 and wl.fenc.max() == 1023 and (wl.fenc & 3).any()
    compare(G, a, wl, tab)


@pytest.mark.parametrize("content,depth,qp,chroma", QP_CASES, ids=["%s-%d-qp%d" % c[:3] for c in QP_CASES])
def test_frame_driver_qp(content, depth, qp, chroma, request):
    """The frame driver across the quantiser's QP range (frame_helpers.QPS: every qp % 6 and every qp / 6 from 0 to the
    top), with the mv cost of each QP.  A cut from black ("cut") at every QP: constant white TUs take the DC-only
    shortcut, 10-bit levels reach the int16 clip at QP 0 and 3, ringing reaches the reconstruction clip, and every SAD
    ties, so that the mv cost alone decides the searches.  Noise and flat areas with chroma at the lowest and highest QP:
    full TUs, all-zero TUs and TUs with one nonzero AC level."""
    G = RefResults(request, depth)
    O = load_oracle(depth)
    wl = Workload(200, 136, depth=depth, numRefs=2, method=3, subme=3, merange=57, rect=1, qp=qp, content=content, chroma=chroma)
    tab = mvcost_table(O, lambda_for(qp, depth))
    a = cpu_analyse(O, "orc_analyse_frame", wl, tab, threads=4)
    assert_qp_case_reaches(O, content, wl, a)
    compare(G, a, wl, tab)


@pytest.mark.parametrize("depth", [8, 10])
def test_frame_driver_amp(depth, request):
    """rect + AMP partitions (presets slower / veryslow, BASELINE configs[3..4]): 2NxnU / 2NxnD / nLx2N / nRx2N of CUs >= 16."""
    G = RefResults(request, depth)
    O = load_oracle(depth)
    qp = 30
    wl = Workload(200, 136, depth=depth, numRefs=2, method=3, subme=4, merange=57, rect=1, qp=qp, amp=1)
    tab = mvcost_table(O, lambda_for(qp, depth))
    a = cpu_analyse(O, "orc_analyse_frame", wl, tab, threads=4)
    sizes = {(int(j["pw"]), int(j["ph"])) for j in a["jobs"]}
    assert {(64, 16), (64, 48), (16, 64), (48, 64), (32, 8), (32, 24), (8, 32), (24, 32), (16, 4), (16, 12), (4, 16), (12, 16)} <= sizes
    compare(G, a, wl, tab)
