"""Pins the oracle's PART stage (oracle/frame_part.h) against the REAL reference code (oracle/_ref, or its stored results,
tests/golden/part_ref.json): the PART record of every CU byte for byte -- each partition's cost, sa8d, slots and vectors --
whose predictions come from a real Predict through PredictionUnits at the PUs' real z-order offsets (predInterLumaPixel /
predInterChromaPixel, or the Short paths + addWeightUni for a weighted slot) and whose costs come from the real sa8d table
entries; and the ME results the stage reads.  Asserts the stage's invariants on the oracle's result (part_helpers.check_invariants).
CPU only."""

import pytest

from part_helpers import (PartRefResults, load_oracle_part, cpu_analyse_part, case_workload, check_invariants, summary, CASES,
                          case_id)


@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_part_driver(case, request):
    depth, nr, geo, chroma, size, kind = case
    G = PartRefResults(request, depth)
    wl, tab = case_workload(case)
    # one thread: the drivers run every stage on the calling thread and start none
    a = cpu_analyse_part(load_oracle_part(depth), "orc", wl, chroma, tab, threads=1)
    G.same("frame", lambda: summary(cpu_analyse_part(G.R, "x265ref", wl, chroma, tab, threads=1)), summary(a))
    check_invariants(a, wl, kind)
    if geo == (0, 0):
        assert (a["part"]["cost"][:, 1:] == 0xffffffff).all()
