"""Pins the oracle's B slices (oracle/frame_bidir.h) against the REAL reference code (oracle/_ref, or its stored results,
tests/golden/bidir_ref.json): the BIDIR record of every CU (uni and bi costs, decision, references, zero flag, vectors), whose
bi-prediction comes from the real predInterLumaShort / predInterChromaShort + Yuv::addAvg, its costs from the real sa8d table
entries and its zero-try range test from the real MV::checkRange; and the luma and chroma levels, SSE, numSig, cu_ref and recon
of every CU, bi-predicted ones included.  Asserts on the oracle's decision counters that each content reaches the branch it is
there for.  CPU only."""

import pytest

from bidir_helpers import (BidirRefResults, load_oracle_bidir, bidir_workload, cpu_analyse_bidir, summary, CASES, case_id)


@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_bidir_driver(case, request):
    depth, (n0, n1), chroma, (W, H), qp, kind = case
    G = BidirRefResults(request, depth)
    O = load_oracle_bidir(depth)
    wl = bidir_workload(W, H, depth, n0, n1, kind, qp=qp)
    a = cpu_analyse_bidir(O, "orc", wl, n0, chroma)
    G.same("frame", lambda: summary(cpu_analyse_bidir(G.R, "x265ref", wl, n0, chroma), wl, chroma), summary(a, wl, chroma))
    n, bd = a["counts"], a["bidir"]
    assert n["bi"] + n["uni_l0"] + n["uni_l1"] == a["ncu"], n
    assert ((bd["interDir"] == 3) == (bd["biCost"] < bd["uniCost"])).all()
    assert (a["cu_ref"][bd["interDir"] == 3] == bd["ref"][bd["interDir"] == 3, 0]).all()
    assert (a["cu_ref"][bd["interDir"] == 2] >= n0).all() and (a["cu_ref"][bd["interDir"] == 1] < n0).all()
    if kind == "between":
        assert n["bi"] > 0.5 * a["ncu"], n
    elif kind == "cut":
        assert n["uni_l1"] > 0.5 * a["ncu"], n
    elif kind == "tie":
        assert n["tie_l0"] > 0 and n["uni_l1"] == 0, n
    else:
        assert n["zero_taken"] > 0 and n["zero_out_of_range"] > 0 and n["zero_skipped"] > 0, n
        assert n["zero_taken"] == int(bd["zero"].sum()) and (bd["mv"][bd["zero"] == 1] == 0).all()
    if qp == 22:
        assert a["cu_numsig"].sum() > 0
