"""Pins the oracle's frame-level CTU-analysis driver against the same driver running on the REAL
reference code (MotionEstimate class + C primitive table, oracle/_ref; its stored results where oracle/_ref is not
built, tests/ref_results.py).  CPU only."""
import numpy as np
import pytest

from common import load_oracle
from frame_helpers import Workload, cpu_analyse, lambda_for, MVRANGE
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
