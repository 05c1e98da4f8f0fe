"""Pins the oracle's 4:2:0 chroma residual stage (oracle/frame_chroma.h: stage bit 3) against the same driver on
the REAL reference code (the chroma pu filter entries in predInterChromaPixel's order, the C primitive table; oracle/_ref, or
its stored results, tests/golden/chroma_residual_ref.json), and the oracle's chroma QP mapping against the real
Quant::setChromaQP.  CPU only."""

import numpy as np
import pytest

from chroma_helpers import cpu_analyse_chroma, chroma_inner, load_oracle_chroma, ChromaRefResults, OFFSETS
from frame_helpers import Workload, lambda_for, qp_max, QP_CASES
from me_helpers import mvcost_table


def chroma_levels(res):
    """(plane, T/2 x T/2 levels) of every chroma TU of a result, in the layout of coef_c."""
    for pl in range(2):
        for (x, y, S), off in zip(res["cus"].tolist(), res["cu_coef_off"].tolist()):
            T = min(S, 32)
            Tc = T // 2
            for t in range((S // T) ** 2):
                o = off // 4 + t * Tc * Tc
                yield pl, res["coef_c"][pl][o:o + Tc * Tc].reshape(Tc, Tc)


def summary(res, wl):
    """What the chroma stage outputs (recon planes: their picture area), plus the reference choice it used."""
    return dict(qpc=list(res["qpc"]), cu_ref=res["cu_ref"], coef_c=res["coef_c"], cu_sse_c=res["cu_sse_c"], cu_numsig_c=res["cu_numsig_c"],
                recon_c=[chroma_inner(wl, res["recon_c"][d][k]) for d in range(4) for k in range(2)])


def run(G, O, wl, offsets=(0, 0)):
    qp = wl.params["qp"]
    tab = mvcost_table(O, lambda_for(qp, wl.depth))
    a = cpu_analyse_chroma(O, "orc_analyse_frame_chroma", wl, tab, offsets=offsets)
    G.same("chroma", lambda: summary(cpu_analyse_chroma(G.R, "x265ref_analyse_frame_chroma", wl, tab, offsets=offsets), wl), summary(a, wl))
    return a


@pytest.mark.parametrize("depth", [8, 10])
@pytest.mark.parametrize("noise", [False, True])
def test_chroma_residual_driver(depth, noise, request):
    G = ChromaRefResults(request, depth)
    O = load_oracle_chroma(depth)
    wl = Workload(200, 136, depth=depth, numRefs=2, method=3, subme=3, merange=57, rect=1, qp=30, noise=noise, chroma=True)
    a = run(G, O, wl)
    assert a["cu_numsig_c"].sum() > 0 and a["cu_sse_c"].sum() > 0
    # the stage changes no luma output: the same frame without bit 3
    b = cpu_analyse_chroma(O, "orc_analyse_frame_chroma", wl, mvcost_table(O, lambda_for(30, depth)), stages=7)
    for k in ("me_out", "coef", "cu_sse", "cu_numsig", "cu_ref", "intra_cost"):
        assert np.array_equal(a[k], b[k]), k


@pytest.mark.parametrize("depth", [8, 10])
@pytest.mark.parametrize("offsets", [(-12, 12), (12, -12)])
def test_chroma_residual_offsets(depth, offsets, request):
    """The PPS + slice chroma QP offsets at both ends of their range, one per plane."""
    G = ChromaRefResults(request, depth)
    O = load_oracle_chroma(depth)
    wl = Workload(200, 136, depth=depth, numRefs=2, method=3, subme=3, merange=57, rect=1, qp=30, noise=True, chroma=True)
    a = run(G, O, wl, offsets)
    assert a["qpc"][0] != a["qpc"][1]


@pytest.mark.parametrize("content,depth,qp,chroma", QP_CASES, ids=["%s-%d-qp%d" % c[:3] for c in QP_CASES])
def test_chroma_residual_qp(content, depth, qp, chroma, request):
    """The QP cases of the luma stage with chroma planes: every qp % 6 and qp / 6 through the chroma QP map; a cut from black
    ("cut") gives DC-only chroma TUs and reconstructions that reach the clip."""
    G = ChromaRefResults(request, depth)
    O = load_oracle_chroma(depth)
    wl = Workload(200, 136, depth=depth, numRefs=2, method=3, subme=3, merange=57, rect=1, qp=qp, content=content, chroma=True)
    a = run(G, O, wl)
    if content == "cut":
        dc = sum(1 for _, lv in chroma_levels(a) if np.count_nonzero(lv) == 1 and lv[0, 0])
        assert dc > 0


@pytest.mark.parametrize("field,depth,opts", [("far", 8, dict(motion=(0, 0))), ("far", 10, dict()), ("mixed", 8, dict()),
                                               ("mixed", 10, dict(amp=1, subme=4))])
def test_chroma_residual_fields(field, depth, opts, request):
    """Predictor fields whose vectors reach the search clamps ("far") or mix zero, full-pel and fractional vectors ("mixed"):
    the chroma MC reads the reference margins."""
    G = ChromaRefResults(request, depth)
    O = load_oracle_chroma(depth)
    kw = dict(numRefs=2, method=3, subme=3, merange=57, rect=1, qp=30, chroma=True, field=field)
    kw.update(opts)
    wl = Workload(200, 136, depth=depth, **kw)
    a = run(G, O, wl)
    if field == "far":
        # some chosen vectors move the block by more than a CTU
        mv = a["me_out"][a["cu_jobs"][np.arange(a["ncu"]), a["cu_ref"]]]
        assert (np.abs(mv[:, 1:3]) > 4 * 64).any()


@pytest.mark.parametrize("depth", [8, 10])
def test_chroma_qp_map(depth, request):
    """The oracle's restatement of Quant::setChromaQP against the real one (a subclass reaches the protected method), for
    every quantiser QP 0..51 + QP_BD_OFFSET and every offset -12..12."""
    G = ChromaRefResults(request, depth)
    O = load_oracle_chroma(depth)
    grid = [(qp, off) for qp in range(qp_max(depth) + 1) for off in range(-12, 13)]
    mine = [O.orc_chroma_qp(qp, off) for qp, off in grid]

    def ref():
        return [G.R.x265ref_chroma_qp(qp, off) for qp, off in grid]
    G.same("map", ref, mine)
    assert min(mine) == 0 and max(mine) == qp_max(depth) and set(OFFSETS) <= {off for _, off in grid}
