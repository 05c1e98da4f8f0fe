"""weightAnalyse (encoder/weightPrediction.cpp:222-539): the plain-C restatement (oracle/oracle_weightp.c) equals the real
function on real Frames in every written entry of the weight table, its decision counters show every branch reached,
and the library's host decision (x265cu_weightp_decide), fed the restatement's costs, equals the restatement."""
import ctypes as C
import os

import numpy as np
import pytest

import weightp_helpers as WH
from common import ptr
from x265_b200.lib import WpFrame, WpParams, WpCand, WpEntry


_counters = {}


@pytest.mark.parametrize("case", WH.CASES, ids=[c[0] for c in WH.CASES])
def test_restatement_equals_reference(case):
    c = WH.Case(case)
    WH.oracle_counters(reset=True)
    got = c.written(WH.oracle_table(c))
    for k, v in WH.oracle_counters(reset=True).items():
        _counters[k] = _counters.get(k, 0) + v
    assert got == WH.expected(c)


def test_branch_reach():
    """every decision of the search is taken by some case of the matrix"""
    if len(_counters) == 0:
        for case in WH.CASES:
            c = WH.Case(case)
            WH.oracle_table(c)
            for k, v in WH.oracle_counters(reset=True).items():
                _counters[k] = _counters.get(k, 0) + v
    missing = [k for k in WH.COUNTERS if _counters.get(k, 0) == 0]
    assert not missing, missing


COST_CASES = [c for c in WH.CASES if c[8] not in ("none", "far") and c[2] <= 1920]


@pytest.mark.parametrize("case", COST_CASES, ids=[c[0] for c in COST_CASES])
def test_costs_equal_reference(case):
    """weightCost of every pin candidate, per list and plane, with and without motion compensation, equals the real
    mcLuma / mcChroma + weightCost (chroma planes included where the search itself never reaches them)"""
    from ref_results import digest
    c = WH.Case(case)
    got = {}
    for lst in range(c.nl):
        for plane in range(3 if c.csp else 1):
            for use in (0, 1) if c.mvs[lst] is not None else (0,):
                got["%d%d%d" % (lst, plane, use)] = WH.oracle_costs(c, lst, plane, use)
    if WH.load_ref_wp(c.depth) is None:
        want = WH.stored_costs(c.name)
        assert want is not None, "no stored reference costs for %s" % c.name
        assert {k: digest(v) for k, v in got.items()} == want
        return
    for k, v in got.items():
        r = WH.reference_costs(c, int(k[0]), int(k[1]), int(k[2]))
        assert np.array_equal(v, r), (k, np.nonzero(v != r)[0][:8])
    d = {k: digest(v) for k, v in got.items()}
    if os.environ.get("X265_WRITE_GOLDEN") == "1":
        WH.store("costs:" + c.name, d)
    else:
        assert WH.stored_costs(c.name) == d, "the reference's costs differ from the stored ones"


@pytest.mark.parametrize("case", WH.CASES[::3], ids=[c[0] for c in WH.CASES[::3]])
def test_host_decision_equals_restatement(case):
    import x265_b200
    lib = x265_b200.load(need_gpu=False)
    c = WH.Case(case)
    want = WH.oracle_table(c, fill=-7)
    got = np.full((2, 16, 3, 4), -7, np.int32)
    has = np.array([m is not None for m in c.mvs], np.int32)
    fn = WH.oracle_cost_fn(c)
    assert lib.L.x265cu_weightp_decide(c.depth, C.byref(c.params), C.byref(c.recs[1]), c.ref_records(), ptr(has), fn, None,
                                       ptr(got)) == 0
    assert np.array_equal(got, want)


def test_refusals():
    import x265_b200
    lib = x265_b200.load(need_gpu=False)
    fn = WH.WP_COST_FN(lambda *a: 0)
    f = WpFrame()
    refs = (C.POINTER(WpFrame) * 2)(C.pointer(f), C.pointer(f))
    has = np.zeros(2, np.int32)
    out = np.zeros((2, 16, 3, 4), np.int32)
    good = dict(sliceType=1, numRefIdx=(1, 0), bframes=3, width=328, height=184, csp=1)
    for depth, bad in [(12, {}), (8, dict(csp=2)), (8, dict(sliceType=2)), (8, dict(width=330)), (8, dict(height=0)),
                       (8, dict(numRefIdx=(0, 0))), (8, dict(numRefIdx=(17, 0))), (8, dict(sliceType=0, numRefIdx=(1, 0)))]:
        kw = dict(good, **bad)
        prm = WpParams(kw["sliceType"], (C.c_int32 * 2)(*kw["numRefIdx"]), kw["bframes"], kw["width"], kw["height"], kw["csp"])
        assert lib.L.x265cu_weightp_decide(depth, C.byref(prm), C.byref(f), refs, ptr(has), fn, None, ptr(out)) == -1
        assert "x265cu_weightp_decide" in lib.last_error()
    prm = WpParams(1, (C.c_int32 * 2)(1, 0), 3, 328, 184, 1)
    assert lib.L.x265cu_weightp_decide(8, C.byref(prm), C.byref(f), refs, ptr(has), WH.WP_COST_FN(), None, ptr(out)) == -1


def test_record_layouts():
    assert C.sizeof(WpFrame) == 112 and WpFrame.wp_sum.offset == 56 and WpFrame.poc.offset == 104
    assert C.sizeof(WpParams) == 28 and WpParams.csp.offset == 24
    assert C.sizeof(WpCand) == 16 and C.sizeof(WpEntry) == 16
