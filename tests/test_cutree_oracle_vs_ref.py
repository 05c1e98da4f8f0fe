"""cuTree's propagation chain: the plain-C restatement (oracle/oracle_cutree.c) against the REAL Lookahead::cuTree with
estimateCUPropagate and cuTreeFinish (oracle/ref_shim_cutree.cpp), every frame's whole propagateCost and qpCuTreeOffset
compared.  Where oracle/_ref is absent the reference's stored results (tests/golden/cutree_ref.json) stand in for it.

Also: the finish list is what the device chain hands the host.  Running cuTreeFinish on each listed frame's propagateCost
at the END of the chain gives the qpCuTreeOffset the reference computes at its call sites (VBV finishes inside the chain),
and every frame not listed keeps its qpCuTreeOffset.  CPU only."""
import numpy as np
import pytest

import cutree_helpers as T
import x265_b200

CASES = T.cases()
CLIP_PARAMS = [("clip_pyr0", T.params(bBPyramid=0)), ("clip_pyr1", T.params(bBPyramid=1)),
               ("clip_vbv", T.params(vbv=1, bBPyramid=1)), ("clip_wbipred", T.params(bEnableWeightedBiPred=1, bBPyramid=0))]


@pytest.fixture(scope="module")
def cu():
    return x265_b200.load(need_gpu=False)


def _pin(request, win):
    R = T.CutreeRefResults(request)
    prop, qp, fin = win.oracle()
    ref = {}

    def reference():
        if not ref:
            ref["prop"], ref["qp"] = win.reference()
        return ref
    R.same("propagateCost", lambda: reference()["prop"], prop)
    R.same("qpCuTreeOffset", lambda: reference()["qp"], qp)
    return prop, qp, fin


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_cutree_oracle_matches_reference(request, cu, case):
    name, w8, h8, types, prm, kw = case
    win = T.synth_window(cu, name, w8, h8, types, prm, **kw)
    prop, qp, fin = _pin(request, win)
    # the chain moved something (or, without an anchor to propagate into, left the pattern alone)
    assert fin or all(np.array_equal(p, T.pattern(f, win.ncu)) for f, p in enumerate(prop))


@pytest.mark.parametrize("name,prm", CLIP_PARAMS, ids=[c[0] for c in CLIP_PARAMS])
def test_cutree_oracle_matches_reference_clip(request, name, prm):
    """A real clip's estimates and AQ weights from the reference lookahead (x265ref_la_create_aq)."""
    win = T.clip_window(prm, T.CLIP_TYPES)
    prop, qp, fin = _pin(request, win)
    assert any(np.any(qp[f] != -1000.0 - f) for f, _ in fin)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_cutree_finish_list(cu, case):
    """cuTreeFinish on the listed frames' final propagateCost reproduces the chain's qpCuTreeOffset; no other frame's changes."""
    name, w8, h8, types, prm, kw = case
    win = T.synth_window(cu, name, w8, h8, types, prm, **kw)
    prop, qp, fin = win.oracle()
    done = set()
    for f, d in fin:
        if d < 0:
            continue
        assert np.array_equal(win.oracle_finish(f, d, prop[f]), qp[f], equal_nan=True), (f, d)   # log2 of a wrapped cost: NaN
        done.add(f)
    for f in range(win.n):
        if f not in done and not (fin and fin[0][1] < 0 and f == 0):
            assert np.all(qp[f] == -1000.0 - f), f


def test_cutree_overflow_case_reaches_the_wrap():
    """The overflow windows carry amounts past 2^21 (the device's serial replay, weight products that wrap) and
    intraCost * invQscale products past int32."""
    win = T.synth_window(x265_b200.load(need_gpu=False), "overflow_wrap", 9, 6, T.slice_types(9, 3),
                         T.params(bEnableWeightedBiPred=1), amount="overflow")
    prod = win.intra[1].astype(np.int64) * win.invq[1]
    assert (prod >= 2 ** 31).any() and ((prod < 2 ** 31) & (prod >= 2 ** 29)).any()


def test_cutree_estimates_cover_the_chain(cu):
    """Every window of the pin runs on exactly the estimates x265cu_cutree_estimates lists (the oracle refuses a missing one)."""
    for name, w8, h8, types, prm, kw in CASES:
        win = T.synth_window(cu, name, w8, h8, types, prm, **kw)
        win.oracle()
