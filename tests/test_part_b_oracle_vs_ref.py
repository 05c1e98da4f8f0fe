"""Pins the oracle's PART_B stage (oracle/frame_part_b.h, stage bit 6: the inter estimate of every partition of a B slice's CUs)
against the REAL reference code (oracle/_ref, or its stored results, tests/golden/part_b_ref.json): the PART_B record of every
CU byte for byte, the ME results it reads and the decision counters.  On the reference the bi try's cost comes from the real
setSourcePU / bufSATD / bufChromaSATD (pixelavg_pp from the real table where predInterSearch takes it), the final prediction
from a real Predict::motionCompensation of a B slice with every PU at its z-order offset, the zero try's range test from the
real MV::checkRange.  Asserts the stage's invariants, that each content reaches its branch, that the 2Nx2N entry is BIDIR's
uni estimate, and that a partition without a bi PU is the P slice's PART entry.  CPU only."""

import numpy as np
import pytest

from bidir_helpers import load_oracle_bidir, cpu_analyse_bidir
from part_helpers import load_oracle_part, cpu_analyse_part
from part_b_helpers import (PartBRefResults, load_oracle_part_b, load_ref_part_b, cpu_analyse_part_b, case_workload,
                            check_invariants, check_bidir_2nx2n, check_p_equivalence, summary, CASES, case_id)


@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_part_b_driver(case, request):
    depth, (n0, n1), geo, chroma_mode, size, qp, kind = case
    G = PartBRefResults(request, load_ref_part_b(depth))
    wl, n0, chroma = case_workload(case)
    # one thread: the drivers run every stage on the calling thread and start none
    a = cpu_analyse_part_b(load_oracle_part_b(depth), "orc", wl, n0, chroma, threads=1)
    G.same("frame", lambda: summary(cpu_analyse_part_b(G.R, "x265ref", wl, n0, chroma, threads=1)), summary(a))
    check_invariants(a, wl, n0)
    n = a["counts"]
    pb = a["part_b"]
    # the bi try's cost paths: chroma SATD needs chroma and subme > 2; a CU 16's AMP PUs have chroma blocks that are not
    # multiples of 4, so with AMP both paths occur
    if geo != (0, 0):
        assert n["bi_cu8"] > 0
        assert (n["chroma_satd"] > 0) == (chroma_mode == "s3")
        assert (n["avg_pp"] > 0) == (chroma_mode != "s3" or geo[1] == 1)
    else:
        assert n["bi_cu8"] == n["chroma_satd"] == n["avg_pp"] == 0
        assert (pb["cost"][:, 1:] == 0xffffffff).all()
    if kind == "average":
        assert n["bi"] > 0 if geo != (0, 0) else n["bi"] == 0
    if kind == "occlusion":
        both = (pb["interDir"] == 1).any(axis=2) & (pb["interDir"] == 2).any(axis=2)
        assert both.any(), "no partition whose PUs chose different lists"
    if kind == "cut":
        assert n["uni_l1"] > n["uni_l0"]
    if kind == "gpb":
        assert n["tie_l0"] > 0 and n["uni_l1"] == 0 and not (pb["interDir"] == 2).any()
    if kind == "static" and geo != (0, 0):
        assert min(n["zero_tried"], n["zero_taken"], n["zero_out_of_range"], n["zero_skipped"]) > 0, n
    # the 2Nx2N entry is BIDIR's uni estimate of the same inputs
    bd = cpu_analyse_bidir(load_oracle_bidir(depth), "orc", wl, n0, chroma, threads=1)
    assert np.array_equal(bd["me_out"][:, :3], a["me_out"][:, :3])
    check_bidir_2nx2n(a, bd["bidir"], a["me_out"])
    # a partition without a bi PU is the P slice's PART entry of the same inputs
    p = cpu_analyse_part(load_oracle_part(depth), "orc", wl, chroma, None, threads=1)
    assert np.array_equal(p["me_out"][:, :3], a["me_out"][:, :3])
    assert check_p_equivalence(a, p) > 0
