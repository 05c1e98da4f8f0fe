"""Pins the oracle's prediction costs (oracle/oracle_pred.c: orc_pred_cost, orc_pred_cost_batch) to the reference's Predict /
MotionEstimate classes (oracle/ref_shim.cpp: x265ref_pred_cost_batch) on the case families of tests/test_gpu_pred_paths.py
(pred_helpers.family): every PU shape swept through every luma / chroma phase pair on every kind of job, PUs at the picture
corners and edges with vectors at CUData::clipMv's limits, 0 / maxv content, and row pitches and PU positions of every
alignment.  Where oracle/_ref is not built the reference's stored results are compared instead (tests/ref_results.py).

The numpy restatement (tests/pred_numpy.py) is a third opinion on a sample of each family, and states the preconditions the
families promise: every read inside the picture's margins, and the clips the saturated content engages."""
import ctypes as C

import numpy as np
import pytest

import pred_helpers as ph
import pred_numpy as pn
from common import load_oracle, pixel_dtype
from ref_results import RefResults

DEPTHS = [8, 10]


def oracle_job_cost(O, pics, jb, chroma=True):
    """orc_pred_cost of one x265cu_pred_job record, its pointers computed here rather than by orc_pred_cost_batch"""
    es = np.dtype(pixel_dtype(pics.depth)).itemsize
    y, x = divmod(int(jb["offset"]), pics.stride)
    off, coff = pics.org + int(jb["offset"]), pics.corg + (y >> 1) * pics.cstride + (x >> 1)
    on = chroma and bool(jb["flags"] & 1)
    j = ph.OrcPredJob()
    j.fenc[0] = pics.fenc.ctypes.data + off * es
    if on:
        j.fenc[1], j.fenc[2] = pics.fc[0].ctypes.data + coff * es, pics.fc[1].ctypes.data + coff * es
    for l, dst in ((0, j.ref0), (1, j.ref1)):
        r = int(jb["ref%d" % l])
        if r >= 0:
            dst[0] = pics.refs[r].ctypes.data + off * es
            if on:
                dst[1], dst[2] = pics.rc[r][0].ctypes.data + coff * es, pics.rc[r][1].ctypes.data + coff * es
    j.stride, j.cstride, j.w, j.h = pics.stride, pics.cstride, int(jb["pw"]), int(jb["ph"])
    j.mv0[0], j.mv0[1] = (int(v) for v in jb["mv0"]); j.mv1[0], j.mv1[1] = (int(v) for v in jb["mv1"])
    j.cost, j.chroma, j.biAvgPP = int(jb["cost"]), int(on), int(jb["flags"] >> 1) & 1
    O.orc_pred_cost.argtypes = [C.POINTER(ph.OrcPredJob)]; O.orc_pred_cost.restype = C.c_int
    return int(O.orc_pred_cost(C.byref(j)))


@pytest.mark.parametrize("depth", DEPTHS)
@pytest.mark.parametrize("name", ph.FAMILIES)
def test_pred_family(depth, name, request):
    """The oracle's batch entry against the reference on the whole family, with and without chroma planes; against per-job
    orc_pred_cost and the numpy restatement on a sample; every job's reads inside the margins."""
    G = RefResults(request, depth)
    O = load_oracle(depth)
    pics, jobs, info = ph.family(name, depth)
    assert ph.reads_in_margins(pics, jobs).all()
    got = ph.oracle_batch(O, pics, jobs)
    luma = ph.oracle_batch(O, pics, jobs, chroma=False)
    for key, cost, chroma in (("costs", got, True), ("luma_costs", luma, False)):
        want = ph.ref_batch(G.R, pics, jobs, chroma) if G.R is not None else None
        if want is not None:
            bad = np.nonzero(want != cost)[0]
            assert bad.size == 0, (key, bad.size, [(int(i), jobs[i].tolist(), int(cost[i]), int(want[i])) for i in bad[:6]])
        G.same(key, lambda: want, cost)
    rng = np.random.default_rng(7 + depth)
    sample = rng.choice(len(jobs), min(len(jobs), 96), replace=False)
    for i in sample:
        assert oracle_job_cost(O, pics, jobs[i]) == got[i], (int(i), jobs[i].tolist())
        assert oracle_job_cost(O, pics, jobs[i], chroma=False) == luma[i], (int(i), jobs[i].tolist())
        c, reads, _ = pn.pred_cost(pics, jobs[i])
        assert c == got[i], ("numpy", int(i), jobs[i].tolist(), c, int(got[i]))
        assert pics.reads_inside(reads), (int(i), jobs[i].tolist(), reads)
        assert pn.pred_cost(pics, jobs[i], chroma_planes=False)[0] == luma[i], ("numpy luma", int(i), jobs[i].tolist())


@pytest.mark.parametrize("depth", DEPTHS)
def test_saturated_content_engages_the_clips(depth):
    """The saturated family reaches both ends of the pixel-path interpolation clip and of the addAvg clip (numpy restatement):
    at least 10 % of its one-list sub-pel jobs clip below 0 and above maxv, and so do 10 % of its addAvg jobs"""
    pics, jobs, _ = ph.family("saturated", depth)
    hits = {"interp": [0, 0, 0], "avg": [0, 0, 0]}
    for jb in jobs:
        _, _, st = pn.pred_cost(pics, jb)
        bi = jb["ref0"] >= 0 and jb["ref1"] >= 0
        if bi and not jb["flags"] & 2:
            k = "avg"
        elif not bi and ((jb["mv0"] if jb["ref0"] >= 0 else jb["mv1"]) & 3).any():
            k = "interp"
        else:
            continue
        hits[k][0] += 1
        hits[k][1] += st.get(k + "_lo", False)
        hits[k][2] += st.get(k + "_hi", False)
    for k, (n, lo, hi) in hits.items():
        assert n >= 50 and lo >= n // 10 and hi >= n // 10, (k, n, lo, hi)


def test_clip_family_reaches_the_box_limits():
    """The clip family's vectors reach every end of CUData::clipMv's box of their CU, and none leaves it"""
    pics, jobs, where = ph.family("clip", 8)
    ends = set()
    for jb, (s, cx, cy) in zip(jobs, where):
        xmin, xmax, ymin, ymax = ph.clip_box(pics.W, pics.H, cx, cy)
        for l in (0, 1):
            if jb["ref%d" % l] < 0:
                continue
            vx, vy = (int(v) for v in jb["mv%d" % l])
            assert xmin <= vx <= xmax and ymin <= vy <= ymax
            ends |= {("xmin", s) if vx == xmin else None, ("xmax", s) if vx == xmax else None,
                     ("ymin", s) if vy == ymin else None, ("ymax", s) if vy == ymax else None}
    ends.discard(None)
    assert ends == {(e, s) for e in ("xmin", "xmax", "ymin", "ymax") for s in (64, 32, 16, 8)}
