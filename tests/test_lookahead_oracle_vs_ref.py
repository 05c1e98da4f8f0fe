"""Pins the lookahead restatement (oracle/oracle_lookahead.c: lowresIntraEstimate + estimateFrameCost /
estimateCUCost) against the REAL classes compiled from /root/reference (Lowres::init,
LookaheadTLD::lowresIntraEstimate, CostEstimateGroup::singleCost) through oracle/_ref, or their stored results where
oracle/_ref is not built (tests/ref_results.py).  CPU only."""
import ctypes as C

import numpy as np
import pytest

from common import load_ref, load_oracle, ptr, P, I, IP, pixel_dtype
from frame_helpers import gen_luma, MARGIN_X, MARGIN_Y
from lookahead_helpers import OracleLookahead
from ref_results import RefResults

TRIPLES = [(0, 1, 1), (0, 2, 1), (0, 2, 2), (0, 3, 1), (0, 3, 2), (0, 3, 3), (1, 3, 2), (2, 3, 3)]


class RefLookahead:
    def __init__(self, R, frames, bframes=3, lslices=0, aq=0, chroma=None):
        self.R = R
        H, W = frames[0].shape
        self.keep = [np.ascontiguousarray(f) for f in frames]
        arr = (P * len(frames))(*[C.c_void_p(f.ctypes.data) for f in self.keep])
        R.x265ref_la_create.restype = P; R.x265ref_la_create.argtypes = [I, I, I, P, IP, I]
        R.x265ref_la_cost.restype = C.c_int64; R.x265ref_la_cost.argtypes = [P, I, I, I]
        R.x265ref_la_get.argtypes = [P, I, I, I, I, P]; R.x265ref_la_geometry.argtypes = [P, P]
        self.slices = None
        if aq:
            # adaptive quantisation on: real Frame objects, calcAdaptiveQuantFrame before lowresIntraEstimate
            cbs = [np.ascontiguousarray(c[0]) for c in chroma]; crs = [np.ascontiguousarray(c[1]) for c in chroma]
            self.keep += cbs + crs
            acb = (P * len(frames))(*[C.c_void_p(f.ctypes.data) for f in cbs]); acr = (P * len(frames))(*[C.c_void_p(f.ctypes.data) for f in crs])
            R.x265ref_la_create_aq.restype = P; R.x265ref_la_create_aq.argtypes = [I, I, I, P, P, P, IP, IP, I, I, I]
            self.h = R.x265ref_la_create_aq(W, H, len(frames), arr, acb, acr, W, W // 2, bframes, lslices, aq)
            if lslices:
                sl = np.zeros(2, np.int32); R.x265ref_la_slices.argtypes = [P, P]; R.x265ref_la_slices(self.h, ptr(sl))
                self.slices = (int(sl[0]), int(sl[1])) if sl[0] > 1 else None
        elif lslices:
            R.x265ref_la_create_slices.restype = P; R.x265ref_la_create_slices.argtypes = [I, I, I, P, IP, I, I]
            self.h = R.x265ref_la_create_slices(W, H, len(frames), arr, W, bframes, lslices)
            sl = np.zeros(2, np.int32); R.x265ref_la_slices.argtypes = [P, P]; R.x265ref_la_slices(self.h, ptr(sl))
            self.slices = (int(sl[0]), int(sl[1]))
        else:
            self.h = R.x265ref_la_create(W, H, len(frames), arr, W, bframes)
        g = np.zeros(7, np.int32); R.x265ref_la_geometry(self.h, ptr(g))
        self.w8, self.h8, self.stride, self.lw, self.lh = [int(x) for x in g[:5]]
        self.ncu = self.w8 * self.h8

    def cost(self, p0, p1, b):
        return int(self.R.x265ref_la_cost(self.h, p0, p1, b))

    def get(self, frame, what, d0=0, d1=0, dtype=np.int32, n=None):
        out = np.zeros(n if n is not None else self.ncu, dtype)
        assert self.R.x265ref_la_get(self.h, frame, what, d0, d1, ptr(out)) == 0
        return out


@pytest.mark.parametrize("depth", [8, 10])
@pytest.mark.parametrize("size,noise", [((416, 240), False), ((200, 136), True)])
def test_lookahead(depth, size, noise, request):
    G = RefResults(request, depth)
    O = load_oracle(depth)
    W, H = size
    frames = [gen_luma(W, H, i, s1=17.0, s2=11.0, bits=depth, noise=noise) for i in range(4)]
    ref = RefLookahead(G.R, frames) if G.R else None
    orc = OracleLookahead(O, frames, depth)
    G.same("geometry", lambda: (ref.w8, ref.h8, ref.stride), (orc.w8, orc.h8, orc.stride))
    # lowres planes incl. margins (Lowres::init)
    lw, lh = [int(x) for x in G.value("lowres_size", lambda: (ref.lw, ref.lh))]
    rows, vw = lh + 2 * MARGIN_Y, lw + 2 * MARGIN_X
    for k in range(4):
        G.same("plane%d" % k, lambda: ref.get(1, 7, k, 0, pixel_dtype(depth), rows * ref.stride).reshape(rows, ref.stride)[:, :vw],
               orc.fr[1]["planes"][k][:, :vw])
    for f in range(4):
        G.same("intraCost%d" % f, lambda: ref.get(f, 0), orc.fr[f]["intraCost"])
        G.same("intraMode%d" % f, lambda: ref.get(f, 1, dtype=np.uint8), orc.fr[f]["intraMode"])
        G.same("lowresCosts%d" % f, lambda: ref.get(f, 2, 0, 0, np.uint16), orc.fr[f]["lowresCosts"][(0, 0)])
        G.same("rowSatds%d" % f, lambda: ref.get(f, 3, 0, 0, np.int32, ref.h8), orc.fr[f]["rowSatds"][(0, 0)])
    for (p0, p1, b) in TRIPLES:
        t = "%d%d%d" % (p0, p1, b)
        c = orc.cost(p0, p1, b)
        G.same("cost" + t, lambda: ref.cost(p0, p1, b), c)
        d0, d1 = b - p0, p1 - b
        G.same("lowresCosts" + t, lambda: ref.get(b, 2, d0, d1, np.uint16), orc.fr[b]["lowresCosts"][(d0, d1)])
        G.same("rowSatds" + t, lambda: ref.get(b, 3, d0, d1, np.int32, ref.h8), orc.fr[b]["rowSatds"][(d0, d1)])
        G.same("mvs0" + t, lambda: ref.get(b, 4, 0, d0, np.int32, 2 * ref.ncu).reshape(-1, 2), orc.fr[b]["mvs"][(0, d0)])
        G.same("mvcosts0" + t, lambda: ref.get(b, 5, 0, d0), orc.fr[b]["mvcosts"][(0, d0)])
        if p1 > b:
            G.same("mvs1" + t, lambda: ref.get(b, 4, 1, d1, np.int32, 2 * ref.ncu).reshape(-1, 2), orc.fr[b]["mvs"][(1, d1)])
        G.same("costEst" + t, lambda: [int(x) for x in ref.get(b, 6, d0, d1, np.int64, 3)],
               list(orc.fr[b]["costEst"][(d0, d1)]) + [orc.fr[b]["intraMbs"].get(d0, 0)])


@pytest.mark.parametrize("depth,lslices", [(8, 4), (8, 8), (10, 4)])
def test_lookahead_cooperative_slices(depth, lslices, request):
    """estimateFrameCost as presets medium / slow run it (param.cpp:173 lookaheadSlices 8, :492 slow 4): the cooperative-slice
    path (slicetype.cpp:3075-3112, 3143-3173) of the REAL Lookahead (a pool without running workers: the caller processes
    every slice) against the oracle's slice loop -- frame costs, per-CU costs, row sums and motion fields."""
    G = RefResults(request, depth)
    O = load_oracle(depth)
    W, H = 1280, 720                                  # slices need a source height >= 720 (slicetype.cpp:1022-1026)
    frames = [gen_luma(W, H, i, bits=depth) for i in range(3)]
    ref = RefLookahead(G.R, frames, lslices=lslices) if G.R else None
    slices = tuple(int(x) for x in G.value("slices", lambda: ref.slices))
    assert slices[0] > 1, slices
    orc = OracleLookahead(O, frames, depth, slices=slices)
    for (p0, p1, b) in [(0, 1, 1), (0, 2, 1), (0, 2, 2)]:
        t = "%d%d%d" % (p0, p1, b)
        c = orc.cost(p0, p1, b)
        a = ref.cost(p0, p1, b) if ref else None
        d0, d1 = b - p0, p1 - b
        G.same("mvs0" + t, lambda: ref.get(b, 4, 0, d0, np.int32, 2 * ref.ncu).reshape(-1, 2), orc.fr[b]["mvs"][(0, d0)])
        G.same("lowresCosts" + t, lambda: ref.get(b, 2, d0, d1, np.uint16), orc.fr[b]["lowresCosts"][(d0, d1)])
        G.same("rowSatds" + t, lambda: ref.get(b, 3, d0, d1, np.int32, ref.h8), orc.fr[b]["rowSatds"][(d0, d1)])
        G.same("cost" + t, lambda: a, c)
    # and the slices change the result (otherwise the test would not see them): serial path on the same frames
    ser = OracleLookahead(O, frames, depth)
    assert any(ser.cost(*t) != orc.cost(*t) or not np.array_equal(ser.fr[t[2]]["mvs"][(0, t[2] - t[0])], orc.fr[t[2]]["mvs"][(0, t[2] - t[0])])
               for t in [(0, 1, 1), (0, 2, 2)])


def aq_inputs(request, depth, lslices, W=1280, H=720):
    """Frames of the AQ cases and the reference's (numCoopSlices, numRowsPerSlice) and per-frame Lowres::invQscaleFactor,
    which the code under test takes as inputs (there is no restatement of calcAdaptiveQuantFrame)."""
    from frame_helpers import gen_chroma
    G = RefResults(request, depth, name="aq_inputs[%d-%d]" % (depth, lslices))
    frames = [gen_luma(W, H, i, bits=depth) for i in range(3)]
    ref = None
    if G.R:
        chroma = [(gen_chroma(W, H, i, 1, bits=depth), gen_chroma(W, H, i, 2, bits=depth)) for i in range(3)]
        ref = RefLookahead(G.R, frames, lslices=lslices, aq=2, chroma=chroma)
    sl = G.value("slices", lambda: ref.slices or (0, 0))
    invq = list(G.value("invq", lambda: np.stack([ref.get(i, 8) for i in range(3)])).astype(np.int32))
    return frames, ref, (tuple(int(x) for x in sl) if sl[0] else None), invq


@pytest.mark.parametrize("depth,lslices", [(8, 0), (8, 8), (10, 0), (10, 4)])
def test_lookahead_with_adaptive_quant(depth, lslices, request):
    """The lookahead as preset medium runs it (aqMode AUTO_VARIANCE, param.cpp:268): Lowres::invQscaleFactor comes from the
    REAL calcAdaptiveQuantFrame (slicetype.cpp:444-694, real Frame objects with 4:2:0 chroma); with it as input the oracle's
    intra and frame-cost paths must reproduce costEstAq, the AQ-weighted row sums and the frame costs of the reference."""
    G = RefResults(request, depth)
    O = load_oracle(depth)
    frames, ref, slices, invq = aq_inputs(request, depth, lslices)
    assert any((q != 256).any() for q in invq), "AQ produced no offsets: the test would not see invQscale"
    orc = OracleLookahead(O, frames, depth, slices=slices, invq=invq)
    for f in range(3):
        G.same("intraCost%d" % f, lambda: ref.get(f, 0), orc.fr[f]["intraCost"])
        G.same("rowSatds%d" % f, lambda: ref.get(f, 3, 0, 0, np.int32, ref.h8), orc.fr[f]["rowSatds"][(0, 0)])
        G.same("costEst%d" % f, lambda: [int(x) for x in ref.get(f, 6, 0, 0, np.int64, 3)[:2]], list(orc.fr[f]["costEst"][(0, 0)]))
    for (p0, p1, b) in [(0, 1, 1), (0, 2, 1), (0, 2, 2)]:
        t = "%d%d%d" % (p0, p1, b)
        c = orc.cost(p0, p1, b)
        a = ref.cost(p0, p1, b) if ref else None
        d0, d1 = b - p0, p1 - b
        G.same("cost" + t, lambda: a, c)
        G.same("rowSatds" + t, lambda: ref.get(b, 3, d0, d1, np.int32, ref.h8), orc.fr[b]["rowSatds"][(d0, d1)])
        G.same("costEst" + t, lambda: [int(x) for x in ref.get(b, 6, d0, d1, np.int64, 3)[:2]], list(orc.fr[b]["costEst"][(d0, d1)]))


def _wp_stats(img):
    """Lowres::wp_sum[0] / wp_ssd[0] as calcAdaptiveQuantFrame leaves them (slicetype.cpp:49-57, 462-480, 665-676):
    sum of the luma samples and sum of squares minus the rounded mean-square term."""
    a = img.astype(np.int64)
    s, q, n = int(a.sum()), int((a * a).sum()), a.size
    return s, q - (s * s + n // 2) // n


@pytest.mark.parametrize("depth", [8, 10])
@pytest.mark.parametrize("case", ["same", "fade", "fade2", "bright", "offset", "noise_fade"])
def test_lookahead_weights_analyse(depth, case, request):
    """LookaheadTLD::weightsAnalyse + weightCostLuma (slicetype.cpp:807-961): the decision and the 4 re-weighted lowres
    planes of the oracle against the real class, on fades that take every exit of the analysis."""
    G = RefResults(request, depth)
    O = load_oracle(depth)
    W, H = 416, 240
    mx = (1 << depth) - 1
    base = gen_luma(W, H, 0, s1=17.0, s2=11.0, bits=depth, noise=case.startswith("noise")).astype(np.float64)
    nxt = gen_luma(W, H, 1, s1=17.0, s2=11.0, bits=depth, noise=case.startswith("noise")).astype(np.float64)
    sc = 1 << (depth - 8)
    # NB the analysis estimates the offset from full-resolution sums over the LOWRES area (slicetype.cpp:892-893), i.e. 4x the
    # true mean difference, so only (nearly) pure scalings end up weighted; "offset" exercises the rejected path
    cur = {"same": nxt, "fade": nxt * 0.78, "fade2": nxt * 0.55 + 1 * sc, "bright": nxt * 1.07, "offset": nxt + 21 * sc,
           "noise_fade": nxt * 0.6}[case]
    frames = [base.astype(pixel_dtype(depth)), np.clip(np.rint(cur), 0, mx).astype(pixel_dtype(depth))]
    ref = RefLookahead(G.R, frames) if G.R else None
    orc = OracleLookahead(O, frames, depth)
    lw, lh = [int(x) for x in G.value("lowres_size", lambda: (ref.lw, ref.lh))]
    rows = lh + 2 * MARGIN_Y
    planesize = rows * orc.stride
    # inputs: the lowres planes and intra costs of both frames, the reference's and the oracle's being the same
    bufs = [[np.ascontiguousarray(orc.fr[f]["planes"][k]).reshape(-1) for k in range(4)] for f in range(2)]
    G.same("planes", lambda: [[ref.get(f, 7, k, 0, pixel_dtype(depth), planesize) for k in range(4)] for f in range(2)], bufs)
    intra = orc.fr[1]["intraCost"]
    G.same("intra", lambda: ref.get(1, 0), intra)
    stats = np.array(list(_wp_stats(frames[1])) + list(_wp_stats(frames[0])), np.uint64)

    def ref_weights():
        out = np.zeros(2, np.int64)
        wref = np.zeros(4 * planesize, pixel_dtype(depth))
        G.R.x265ref_la_weights.argtypes = [P, I, I, P, P, P]
        got_r = G.R.x265ref_la_weights(ref.h, 1, 0, ptr(stats), ptr(out), ptr(wref))
        assert int(out[0]) == planesize and int(out[1]) == rows
        return [got_r, wref if got_r else 0]

    refarr = (P * 4)(*[C.c_void_p(b.ctypes.data) for b in bufs[0]])
    worc = np.zeros(4 * planesize, pixel_dtype(depth))
    wp = np.zeros(3, np.int32)
    O.orc_la_weights_analyse.argtypes = [P, P, P, IP, IP, I, I, IP, P, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, P]
    got_o = O.orc_la_weights_analyse(ptr(bufs[1][0]), refarr, ptr(worc), planesize, orc.stride, lw, lh,
                                     MARGIN_Y * orc.stride + MARGIN_X, ptr(intra),
                                     int(stats[0]), int(stats[1]), int(stats[2]), int(stats[3]), ptr(wp))
    G.same("weights", ref_weights, [got_o, worc if got_o else 0])
    assert (got_o == 0) == (case in ("same", "offset", "noise_fade")), (case, got_o)   # noise: inter never beats intra, no gain
    if got_o:
        assert 0 <= wp[0] <= 127 and 0 <= wp[1] <= 7 and -128 <= wp[2] <= 127
