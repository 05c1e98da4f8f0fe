"""Pins the lookahead restatement (oracle/oracle_lookahead.c: lowresIntraEstimate + estimateFrameCost /
estimateCUCost) against the REAL classes compiled from /root/reference (Lowres::init,
LookaheadTLD::lowresIntraEstimate, CostEstimateGroup::singleCost) through oracle/_ref, or their stored results where
oracle/_ref is not built (tests/ref_results.py).  CPU only."""
import ctypes as C

import numpy as np
import pytest

from common import load_ref, load_oracle, ptr, P, I, IP, pixel_dtype
from frame_helpers import gen_luma, MARGIN_X, MARGIN_Y
from lookahead_helpers import OracleLookahead, CONTENT_KINDS, content_frames, lowres_geometry, search_bounds
from ref_results import RefResults

TRIPLES = [(0, 1, 1), (0, 2, 1), (0, 2, 2), (0, 3, 1), (0, 3, 2), (0, 3, 3), (1, 3, 2), (2, 3, 3)]
# whole-frame geometries of tests/test_gpu_lookahead_shapes.py (lowres CU grids 120x68, 240x135, 130x65, 128x64, 68x120,
# 240x4, 4x135): 1080p and 2160p as presets medium to slower run them, the diagonal-length edges of the device wavefront,
# a portrait frame and the narrowest legal strips (64 px, the smallest picture at CTU 64, param.cpp:1597)
SHAPE_SIZES = [(1920, 1080), (3840, 2160), (2080, 1040), (2048, 1024), (1080, 1920), (3840, 64), (64, 2160)]


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
@pytest.mark.parametrize("size,noise", [((416, 240), False), ((200, 136), True)] + [(s, False) for s in SHAPE_SIZES])
def test_lookahead(depth, size, noise, request):
    G = RefResults(request, depth)
    O = load_oracle(depth)
    W, H = size
    frames = [gen_luma(W, H, i, s1=17.0, s2=11.0, bits=depth, noise=noise) for i in range(4)]
    ref = RefLookahead(G.R, frames) if G.R else None
    orc = OracleLookahead(O, frames, depth)
    _same_estimates(G, ref, orc, depth, TRIPLES)


def _same_estimates(G, ref, orc, depth, triples):
    """Lowres planes of frame 1, every frame's intra estimate, and per triple the frame cost, per-CU costs, row sums, motion
    fields (list 0 vectors and costs, list 1 vectors) and costEst / costEstAq / intraMbs of the oracle against the reference."""
    G.same("geometry", lambda: (ref.w8, ref.h8, ref.stride), (orc.w8, orc.h8, orc.stride))
    # lowres planes incl. margins (Lowres::init)
    lw, lh = [int(x) for x in G.value("lowres_size", lambda: (ref.lw, ref.lh))]
    rows, vw = lh + 2 * MARGIN_Y, lw + 2 * MARGIN_X
    for k in range(4):
        G.same("plane%d" % k, lambda: ref.get(1, 7, k, 0, pixel_dtype(depth), rows * ref.stride).reshape(rows, ref.stride)[:, :vw],
               orc.fr[1]["planes"][k][:, :vw])
    for f in range(len(orc.fr)):
        G.same("intraCost%d" % f, lambda: ref.get(f, 0), orc.fr[f]["intraCost"])
        G.same("intraMode%d" % f, lambda: ref.get(f, 1, dtype=np.uint8), orc.fr[f]["intraMode"])
        G.same("lowresCosts%d" % f, lambda: ref.get(f, 2, 0, 0, np.uint16), orc.fr[f]["lowresCosts"][(0, 0)])
        G.same("rowSatds%d" % f, lambda: ref.get(f, 3, 0, 0, np.int32, ref.h8), orc.fr[f]["rowSatds"][(0, 0)])
    for (p0, p1, b) in triples:
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
    _cooperative_slices(request, depth, lslices, 1280, 720)     # slices need a source height >= 720 (slicetype.cpp:1022-1026)


@pytest.mark.parametrize("depth,size,lslices", [(8, (1920, 1080), 8), (8, (3840, 2160), 4)], ids=["medium", "slow_2160"])
def test_lookahead_cooperative_slices_geometries(depth, size, lslices, request):
    """The cooperative-slice path at 1080p with preset medium's 8 slices (6 of 10 CU rows, the last of 18) and at 2160p with
    preset slow's 4 (33 / 33 / 33 / 36 rows): the geometries tests/test_gpu_lookahead_shapes.py runs on the device."""
    _cooperative_slices(request, depth, lslices, *size)


def _cooperative_slices(request, depth, lslices, W, H):
    G = RefResults(request, depth)
    O = load_oracle(depth)
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


# ---------------------------------------------------------------------------------------------------------------------
# the lookahead on content other than the moving clip (lookahead_helpers.content_frames): static and constant pictures,
# static flat areas, motion past the search range, a cut to noise, fades through black, the full 10-bit range
CONTENT_CASES = [(k, d) for k in CONTENT_KINDS for d in (8, 10) if k != "full10" or d == 10]
CONTENT_SIZES = [(416, 240), (200, 136)]               # 200x136: 100x68 lowres px, partial CUs on the right and at the bottom


def searched_fields(orc):
    """(frame, (list, distance), vectors, costs) of every motion field a triple searched (P triples also create the
    list-1 field of distance 0, which nothing searches)."""
    return [(b, k, f["mvs"][k], f["mvcosts"][k]) for b, f in enumerate(orc.fr) for k in f["mvs"] if k[1] > 0]


def assert_content_reaches(kind, depth, orc, triples):
    """What each kind is there for, asserted on the oracle's outputs, so that no case quietly stops reaching it."""
    fields = searched_fields(orc)
    if kind in ("static", "black", "white", "flat"):
        # the bidir zero-MV skip: the search result (which includes a vector cost) replaced by the bare SATD at (0, 0)
        assert any(((c == 0) & (m == 0).all(axis=1)).any() for _, _, m, c in fields), "no zero-MV skip"
    if kind in ("black", "white"):
        modes = np.concatenate([f["intraMode"] for f in orc.fr])
        assert (modes == modes[0]).all(), "a constant picture must leave a single intra mode (all 35 tie)"
    if kind == "fast":
        lx, hx, ly, hy = search_bounds(orc.w8, orc.h8)
        assert any(((m[:, 0] == lx) | (m[:, 0] == hx) | (m[:, 1] == ly) | (m[:, 1] == hy)).any() for _, _, m, _ in fields), \
            "no vector on its CU's search bound"
    if kind == "cut":
        n = len(orc.fr)
        across = [(p0, b) for (p0, p1, b) in triples if p1 == b and p0 < n // 2 <= b]
        assert across and all(orc.fr[b]["estIntraMbs"][(b - p0, 0)] > 0 for p0, b in across), "no intra CU across the cut"
        if depth == 10:
            assert any(((v & 0x3FFF) == 0x3FFF).any() for f in orc.fr for v in f["lowresCosts"].values()), \
                "10-bit noise must saturate a per-CU cost at LOWRES_COST_MASK"
    if kind == "fade":
        assert orc.fr[1]["estIntraMbs"][(1, 0)] > 0, "the P estimate from the black frame has no intra CU"


@pytest.mark.parametrize("size", CONTENT_SIZES, ids=["%dx%d" % s for s in CONTENT_SIZES])
@pytest.mark.parametrize("kind,depth", CONTENT_CASES)
def test_lookahead_content(kind, depth, size, request):
    """The comparisons of test_lookahead, plus every frame's lowres planes and the list-1 vector costs, on each kind of
    content_frames: the zero-MV skip and the bidir tie (static, constant, flat), the full-tie intra search (constant),
    vectors on the search bounds and far predictors (fast), intra CUs and saturated costs (cut, fade), the full 10-bit
    range (full10)."""
    G = RefResults(request, depth)
    O = load_oracle(depth)
    W, H = size
    frames = content_frames(kind, W, H, depth, 4)
    ref = RefLookahead(G.R, frames) if G.R else None
    orc = OracleLookahead(O, frames, depth)
    _same_estimates(G, ref, orc, depth, TRIPLES)
    _same_planes_and_list1_costs(G, ref, orc, depth, TRIPLES)
    assert_content_reaches(kind, depth, orc, TRIPLES)


def _same_planes_and_list1_costs(G, ref, orc, depth, triples):
    lw, lh = [int(x) for x in G.value("lowres_size", lambda: (ref.lw, ref.lh))]
    rows, vw = lh + 2 * MARGIN_Y, lw + 2 * MARGIN_X
    for f in range(len(orc.fr)):
        G.same("planes%d" % f, lambda: [ref.get(f, 7, k, 0, pixel_dtype(depth), rows * ref.stride).reshape(rows, ref.stride)[:, :vw]
                                        for k in range(4)], [orc.fr[f]["planes"][k][:, :vw] for k in range(4)])
    for (p0, p1, b) in triples:
        if p1 > b:
            G.same("mvcosts1%d%d%d" % (p0, p1, b), lambda: ref.get(b, 5, 1, p1 - b), orc.fr[b]["mvcosts"][(1, p1 - b)])


@pytest.mark.parametrize("lslices", [4, 8])
@pytest.mark.parametrize("kind", ["static", "fast"])
def test_lookahead_content_cooperative_slices(kind, lslices, request):
    """Cooperative slices at 1280x720 on static content (every slice's bottom row loses its predictors from below, which
    are all (0, 0) anyway) and on fast motion (each slice's bottom row then searches from the right neighbour alone)."""
    depth, W, H = 8, 1280, 720
    G = RefResults(request, depth)
    O = load_oracle(depth)
    frames = content_frames(kind, W, H, depth, 3)
    triples = [(0, 1, 1), (0, 2, 1), (0, 2, 2)]
    ref = RefLookahead(G.R, frames, lslices=lslices) if G.R else None
    slices = tuple(int(x) for x in G.value("slices", lambda: ref.slices))
    assert slices[0] > 1, slices
    orc = OracleLookahead(O, frames, depth, slices=slices)
    _same_estimates(G, ref, orc, depth, triples)
    assert_content_reaches(kind, depth, orc, triples)
    if kind == "fast":
        ser = OracleLookahead(O, frames, depth)
        for t in triples:
            ser.cost(*t)
        assert any(not np.array_equal(ser.fr[b]["mvs"][(0, b - p0)], orc.fr[b]["mvs"][(0, b - p0)]) for (p0, p1, b) in triples), \
            "the slices do not change the motion fields"


# (aqMode, strength, qgSize, weightp, variance, quantOffsets) of x265ref_la_create_aq: AUTO_VARIANCE, strength 1.0, qgSize 32
AQ_PARAMS = (2, 1.0, 32, 0, 0, 0)


def content_invq(kind, W, H, depth, frames):
    """Lowres::invQscaleFactor of every frame from the AQ restatement (aq_helpers.oracle), with chroma of the same kind."""
    import aq_helpers as A
    chroma = [(c1, c2) for c1, c2 in zip(content_frames(kind, W, H, depth, len(frames), 1), content_frames(kind, W, H, depth, len(frames), 2))]
    invq = [A.oracle((y, cb, cr), W, H, depth, AQ_PARAMS)["invQscaleFactor"].astype(np.int32) for y, (cb, cr) in zip(frames, chroma)]
    return chroma, invq


@pytest.mark.parametrize("depth", [8, 10])
@pytest.mark.parametrize("kind", ["flat", "static", "cut"])
def test_lookahead_content_with_adaptive_quant(kind, depth, request):
    """Adaptive quantisation on flat areas (zero-energy blocks), static and cut content: the AQ restatement's
    invQscaleFactor equals the real calcAdaptiveQuantFrame's, and with it every estimate equals the reference's."""
    G = RefResults(request, depth)
    O = load_oracle(depth)
    W, H = 416, 240
    frames = content_frames(kind, W, H, depth, 4)
    chroma, invq = content_invq(kind, W, H, depth, frames)
    assert any((q != 256).any() for q in invq), "AQ produced no offsets: the test would not see invQscale"
    ref = RefLookahead(G.R, frames, aq=2, chroma=chroma) if G.R else None
    for i in range(len(frames)):
        G.same("invq%d" % i, lambda: ref.get(i, 8), invq[i])
    orc = OracleLookahead(O, frames, depth, invq=invq)
    _same_estimates(G, ref, orc, depth, TRIPLES)
    assert_content_reaches(kind, depth, orc, TRIPLES)


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


# (reference, current) pictures of the weights analysis: fades that take every exit of the analysis
WEIGHTS_CASES = ["same", "fade", "fade2", "bright", "offset", "noise_fade", "from_black_dark", "from_black_bright", "to_black", "constant"]


def weights_frames(case, depth, W=416, H=240):
    """The two luma pictures of a WEIGHTS_CASES case.  NB the analysis estimates means from full-resolution sums over the
    LOWRES area (slicetype.cpp:892-893), i.e. 4x the true means, so only (nearly) pure scalings end up weighted; "offset"
    takes the rejected path.  The fades from black have a reference with wp_sum == wp_ssd == 0: the dark one (4x mean below
    127.5) keeps its offset, the bright one clamps it to 127 and divides by refMean == 0 (slicetype.cpp:921)."""
    mx = (1 << depth) - 1
    sc = 1 << (depth - 8)
    base = gen_luma(W, H, 0, s1=17.0, s2=11.0, bits=depth, noise=case.startswith("noise")).astype(np.float64)
    nxt = gen_luma(W, H, 1, s1=17.0, s2=11.0, bits=depth, noise=case.startswith("noise")).astype(np.float64)
    black = np.zeros_like(base)
    ref, cur = {"from_black_dark": (black, nxt * 0.15), "from_black_bright": (black, nxt * 0.6), "to_black": (base, black),
                "constant": (black + 60 * sc, black + 150 * sc)}.get(case, (base, None))
    if cur is None:
        cur = {"same": nxt, "fade": nxt * 0.78, "fade2": nxt * 0.55 + 1 * sc, "bright": nxt * 1.07, "offset": nxt + 21 * sc,
               "noise_fade": nxt * 0.6}[case]
    return [np.clip(np.rint(f), 0, mx).astype(pixel_dtype(depth)) for f in (ref, cur)]


def weights_offset_clamped(frames, depth):
    """Whether the analysis of `frames` clamps its first offset guess (slicetype.cpp:914-915), in the float arithmetic of
    the analysis: the curScale that follows divides by refMean."""
    f32 = np.float32
    lw, lh = [8 * g for g in lowres_geometry(*frames[0].shape[::-1])[:2]]
    (fs, fq), (rs, rq) = _wp_stats(frames[1]), _wp_stats(frames[0])
    fencMean = f32(f32(fs) / f32(lw * lh)) / f32(1 << (depth - 8))
    refMean = f32(f32(rs) / f32(lw * lh)) / f32(1 << (depth - 8))
    guess = np.sqrt(f32(fq) / f32(rq)) if fq and rq else f32(1.0)
    scale, denom = int(guess * f32(128) + f32(0.5)), 7
    while denom > 0 and scale > 127:
        denom, scale = denom - 1, scale >> 1
    off = int(fencMean - refMean * f32(min(scale, 127)) / f32(1 << denom) + f32(0.5))
    return not -128 <= off <= 127, float(refMean)


def weights_decision(case):
    """Lowres::weightedRef[].isWeighted of a case.  Not weighted: "same" and "offset" (no gain), noise (inter never beats
    intra), the fades from black (a constant reference never beats intra) and the constant pair (every CU is intra either
    way).  The fade to black ends weighted: scale 1/4, offset -128."""
    return int(case in ("fade", "fade2", "bright", "to_black"))


@pytest.mark.parametrize("depth", [8, 10])
@pytest.mark.parametrize("case", WEIGHTS_CASES)
def test_lookahead_weights_analyse(depth, case, request):
    """LookaheadTLD::weightsAnalyse + weightCostLuma (slicetype.cpp:807-961): the decision and the 4 re-weighted lowres
    planes of the oracle against the real class, on fades that take every exit of the analysis."""
    G = RefResults(request, depth)
    O = load_oracle(depth)
    frames = weights_frames(case, depth)
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
    assert got_o == weights_decision(case), (case, got_o)
    if case.startswith("from_black"):
        assert weights_offset_clamped(frames, depth) == (case == "from_black_bright", 0.0), case
    if got_o:
        assert 0 <= wp[0] <= 127 and 0 <= wp[1] <= 7 and -128 <= wp[2] <= 127
