"""Pins the oracle's weighted P-slice references (oracle/frame_wref.h) against the REAL reference code (oracle/_ref, or its
stored results, tests/golden/wref_ref.json): the planes the search reads (MotionReference::init + applyWeight), and the whole
frame driver on them: every ME result and reference choice, and the luma and chroma levels, SSE, numSig and recon of every
CU, whose weighted prediction comes from the real predInterLumaShort / predInterChromaShort + addWeightUni.  CPU only."""

import numpy as np
import pytest

from chroma_helpers import chroma_inner
from frame_helpers import MARGIN_X, MARGIN_Y
from wref_helpers import (WrefRefResults, load_oracle_wref, fade_workload, search_planes, plane_area, cpu_analyse_wref, table,
                          entry, identity, MIXES)

# (denom, w0, offset) of the plane build: denominators 0 and 7, w0 0 / 1 << denom / 127 / 255, offsets -128 / 0 / 127
PLANE_CASES = [(0, 0, -128), (0, 1, 0), (0, 127, 127), (0, 255, -128), (7, 0, 127), (7, 128, 0), (7, 127, -128), (7, 255, 127),
               (3, 11, 40)]


@pytest.mark.parametrize("depth", [8, 10])
@pytest.mark.parametrize("H", [136, 200])
def test_wref_planes(depth, H, request):
    """Every plane of every case, margins included, on a height that is not a multiple of 64 (the last, partial CTU row of
    applyWeight): weighted luma, weighted chroma (chroma entries present), chroma copied (entry not present), and the whole
    reference unweighted when luma has no wtPresent."""
    G = WrefRefResults(request, depth)
    O = load_oracle_wref(depth)
    wl = fade_workload(200, H, depth, numRefs=1, noise=True)
    for denom, w0, off in PLANE_CASES:
        for chroma_present in (1, 0):
            tab = table([[entry(w0, denom, off), entry(w0, denom, -off if off != -128 else 127, chroma_present),
                          entry(255 - w0, denom, off, chroma_present)]])
            mine = search_planes(O, "orc_wref_planes", wl, tab)

            def ref():
                r = search_planes(G.R, "x265ref_wref_planes", wl, tab)
                return [plane_area(wl, r[0][0])] + [plane_area(wl, c, True) for c in r[1][0]] + [r[2]]
            got = [plane_area(wl, mine[0][0])] + [plane_area(wl, c, True) for c in mine[1][0]] + [mine[2]]
            G.same("planes %d %d %d %d" % (denom, w0, off, chroma_present), ref, got)
            # a weighted plane differs from the reference's pixels unless the weights are the identity
            assert mine[2] == [1]
            if (w0, off) != (1 << denom, 0):
                assert not np.array_equal(mine[0][0], wl.refs[0])
            same_cb = np.array_equal(plane_area(wl, mine[1][0][0], True), plane_area(wl, wl.refC[0][0], True))
            if not chroma_present or (w0, off) != (1 << denom, 0):
                assert same_cb == (not chroma_present)
    # luma not present: MotionReference::init gets no weights, whatever the chroma entries say
    tab = table([[entry(100, 6, 9, 0), entry(100, 6, 9), entry(100, 6, 9)]])
    mine = search_planes(O, "orc_wref_planes", wl, tab)
    G.same("unweighted", lambda: search_planes(G.R, "x265ref_wref_planes", wl, tab)[2], mine[2])
    assert mine[2] == [0] and np.array_equal(plane_area(wl, mine[0][0]), plane_area(wl, wl.refs[0]))


def test_wref_planes_subme2(request):
    """At subme 2 the search has no chroma-SATD term (numInterpPlanes = 1): chroma is not weighted even when present."""
    G = WrefRefResults(request, 8)
    O = load_oracle_wref(8)
    wl = fade_workload(200, 136, 8, numRefs=1, subme=2)
    tab = table([[entry(50, 5, 3), entry(50, 5, 3), entry(50, 5, 3)]])
    mine = search_planes(O, "orc_wref_planes", wl, tab)

    def ref():
        r = search_planes(G.R, "x265ref_wref_planes", wl, tab)
        return [plane_area(wl, r[0][0])] + [plane_area(wl, c, True) for c in r[1][0]]
    G.same("planes", ref, [plane_area(wl, mine[0][0])] + [plane_area(wl, c, True) for c in mine[1][0]])
    assert all(np.array_equal(plane_area(wl, mine[1][0][k], True), plane_area(wl, wl.refC[0][k], True)) for k in range(2))


def summary(res, wl):
    """Every output of the weighted driver: ME results, reference choice, luma levels / SSE / numSig / recon per CU, and the
    chroma ones (recon planes: their picture areas)."""
    inner = lambda p: p[MARGIN_Y:MARGIN_Y + wl.H, MARGIN_X:MARGIN_X + wl.W]
    return dict(me=res["me_out"][:, :3], cu_ref=res["cu_ref"], coef=res["coef"], sse=res["cu_sse"], ns=res["cu_numsig"],
                recon=[inner(res["recon"][d]) for d in range(4)], qpc=list(res["qpc"]), coef_c=res["coef_c"], sse_c=res["cu_sse_c"],
                ns_c=res["cu_numsig_c"], recon_c=[chroma_inner(wl, res["recon_c"][d][k]) for d in range(4) for k in range(2)])


DRIVER = [(d, noise, mix) for d in (8, 10) for noise in (False, True) for mix in ("one", "two", "three")]


@pytest.mark.parametrize("depth,noise,mix", DRIVER, ids=["%d-%s-%s" % (c[0], "noise" if c[1] else "smooth", c[2]) for c in DRIVER])
def test_wref_driver(depth, noise, mix, request):
    """Smooth and noisy textured fades with one to three references: weighted, luma-only weighted and unweighted ones."""
    G = WrefRefResults(request, depth)
    O = load_oracle_wref(depth)
    rows = MIXES[mix](depth)
    wl = fade_workload(200, 136, depth, numRefs=len(rows), noise=noise)
    tab = table(rows)
    a = cpu_analyse_wref(O, "orc", wl, tab)
    G.same("frame", lambda: summary(cpu_analyse_wref(G.R, "x265ref", wl, tab), wl), summary(a, wl))
    # weighting changes the search, not only the residual: against the same frame with every reference unweighted
    b = cpu_analyse_wref(O, "orc", wl, table([None] * len(rows)))
    weighted = np.array([r is not None and r[0][0] == 1 for r in rows])
    on = weighted[a["jobs"]["ref"]]
    moved = (a["me_out"][on, 1:3] != b["me_out"][on, 1:3]).any(axis=1).mean()
    assert moved > 0.1, moved
    # the weighted prediction reaches the chosen CUs of a weighted reference
    assert weighted[a["cu_ref"]].any()
    assert a["cu_numsig"].sum() > 0 and a["cu_numsig_c"].sum() > 0


@pytest.mark.parametrize("depth", [8, 10])
def test_wref_identity(depth, request):
    """An identity entry (w = 1 << denom, offset 0, wtPresent 1): the search reads the reference's own pixels, so its results
    are those of the unweighted frame, while the residual goes through the 14-bit path and weight_sp."""
    G = WrefRefResults(request, depth)
    O = load_oracle_wref(depth)
    wl = fade_workload(200, 136, depth, numRefs=2, noise=True)
    tab = table([[entry(64, 6, 0), identity(6), identity(6)], None])
    a = cpu_analyse_wref(O, "orc", wl, tab)
    G.same("frame", lambda: summary(cpu_analyse_wref(G.R, "x265ref", wl, tab), wl), summary(a, wl))
    b = cpu_analyse_wref(O, "orc", wl, table([None, None]))
    assert np.array_equal(a["me_out"], b["me_out"]) and np.array_equal(a["cu_ref"], b["cu_ref"])
