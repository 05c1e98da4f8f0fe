"""Lookahead (BASELINE configs[1]) helpers: lowres plane construction as Lowres::init does it
(common/lowres.cpp:259-302), the oracle's job struct, and a small host-side cache that mirrors how
estimateFrameCost reuses motion vectors between (p0, p1, b) triples (slicetype.cpp:3121-3130)."""
import ctypes as C

import numpy as np

from common import P, I, IP, ptr, pixel_dtype
from frame_helpers import gen_luma, gen_chroma, pad_plane, MARGIN_X, MARGIN_Y, MVRANGE

LOOKAHEAD_LAMBDA = {8: 1.0, 10: 16.0}     # x265_lambda_tab[X265_LOOKAHEAD_QP = 12 + 6*(depth-8)] (constants.cpp:33-130)

# content_frames kinds, and what each one makes the lookahead do that the moving clip does not
CONTENT_KINDS = ("static", "black", "white", "flat", "fast", "cut", "fade", "full10")
FAST_MOTION = (44, -30)                   # px per frame: 22 / 15 lowres px, past the +-16 search range at every distance
CUT_SEED = 9001


def content_frames(kind, W, H, depth, n, plane=0):
    """n frames of lookahead content `kind`: luma (plane 0) or the 4:2:0 Cb / Cr plane (1 / 2) of the same pictures.
      static  one picture of the clip, repeated: every vector is (0, 0) and bidir ties list 0 (the zero-MV skip, the tie);
      black / white  constant 0 / maxv: every intra mode and every vector cost the same;
      flat    the clip with static letterbox bars and constant rectangles (frame_helpers._flat_areas);
      fast    the clip moving FAST_MOTION px per frame: vectors end on their CU's search bound, predictors lie far away;
      cut     the clip for the first n // 2 frames, then noise of another seed: the estimates across the cut go intra;
      fade    the clip scaled from black up and back down to black (frames 0 and n - 1 are black);
      full10  (10 bit) the clip over the whole 10-bit range, saturated at 0 and 1023."""
    assert kind in CONTENT_KINDS and (kind != "full10" or depth == 10), (kind, depth)
    if plane:
        gen = lambda i, **kw: gen_chroma(W, H, i, plane, bits=depth, **kw)
        shape = (H // 2, W // 2)
    else:
        gen = lambda i, **kw: gen_luma(W, H, i, bits=depth, **kw)
        shape = (H, W)
    if kind == "static":
        f = gen(0)
        return [f.copy() for _ in range(n)]
    if kind in ("black", "white"):
        return [np.full(shape, 0 if kind == "black" else (1 << depth) - 1, pixel_dtype(depth)) for _ in range(n)]
    if kind == "flat":
        return [gen(i, content="flat") for i in range(n)]
    if kind == "fast":
        return [gen(i, motion=FAST_MOTION) for i in range(n)]
    if kind == "cut":
        return [gen(i) if i < n // 2 else gen(i, seed=CUT_SEED, noise=True) for i in range(n)]
    if kind == "fade":
        half = (n - 1) / 2
        return [np.rint(gen(i).astype(np.float64) * min(min(i, n - 1 - i) / half, 1.0)).astype(pixel_dtype(depth)) for i in range(n)]
    return [gen(i, content="full10") for i in range(n)]


def search_bounds(w8, h8):
    """Per lowres CU, the qpel bounds (x min, x max, y min, y max) of its search: 8 px past the picture on every side
    (estimateCUCost, slicetype.cpp:3248-3251).  Vectors lie inside them, inclusive."""
    cx = np.arange(w8 * h8) % w8
    cy = np.arange(w8 * h8) // w8
    return 4 * (-cx * 8 - 8), 4 * ((w8 - cx - 1) * 8 + 8), 4 * (-cy * 8 - 8), 4 * ((h8 - cy - 1) * 8 + 8)


class OrcLaJob(C.Structure):
    _fields_ = [("fenc", P * 4), ("ref0", P * 4), ("ref1", P * 4), ("stride", IP), ("w8", I), ("h8", I), ("bidir", I),
                ("doSearch", I * 2), ("mvs", P * 2), ("mvcosts", P * 2), ("intraCost", P), ("invQscale", P), ("mvcost_tab", P),
                ("lowresCosts", P), ("rowSatds", P), ("out", C.c_int64 * 3), ("numSlices", I), ("rowsPerSlice", I)]


def lowres_geometry(W, H):
    w8 = ((W // 2) + 7) >> 3
    h8 = ((H // 2) + 7) >> 3
    stride = (W // 2 + 2 * MARGIN_X + 31) // 32 * 32
    return w8, h8, stride


def full_plane(img, depth):
    """Full-res luma in a PicYuv-like padded buffer (stride = CTU-aligned width + 2*96)."""
    H, W = img.shape
    stride = (W + 63) // 64 * 64 + 2 * MARGIN_X
    rows = (H + 63) // 64 * 64 + 2 * MARGIN_Y
    buf = np.zeros((rows, stride), pixel_dtype(depth))
    buf[MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W] = img
    buf[MARGIN_Y:MARGIN_Y + H, :MARGIN_X] = img[:, :1]
    buf[MARGIN_Y:MARGIN_Y + H, MARGIN_X + W:MARGIN_X + W + MARGIN_X] = img[:, -1:]
    buf[:MARGIN_Y, :] = buf[MARGIN_Y:MARGIN_Y + 1, :]
    buf[MARGIN_Y + H:MARGIN_Y + H + MARGIN_Y, :] = buf[MARGIN_Y + H - 1:MARGIN_Y + H, :]
    return buf, stride, MARGIN_Y * stride + MARGIN_X


def make_lowres(O, img, depth):
    """4 hpel planes with extended borders; returns (planes, stride, origin offset, w8, h8)."""
    H, W = img.shape
    w8, h8, ls = lowres_geometry(W, H)
    full, fs, forg = full_plane(img, depth)
    lw, lh = w8 * 8, h8 * 8
    planes = [np.zeros((lh + 2 * MARGIN_Y, ls), pixel_dtype(depth)) for _ in range(4)]
    lorg = MARGIN_Y * ls + MARGIN_X
    O.orc_frame_init_lowres(ptr(full, forg), *[ptr(p, lorg) for p in planes], IP(fs), IP(ls), lw, lh)
    for p in planes:
        O.orc_extend_pic_border(ptr(p, lorg), IP(ls), lw, lh, MARGIN_X, MARGIN_Y)
    return planes, ls, lorg, w8, h8


class OracleLookahead:
    def __init__(self, O, frames, depth, bframes=3, slices=None, invq=None):
        self.O, self.depth = O, depth
        self.slices = slices              # (numCoopSlices, numRowsPerSlice) or None: cooperative lookahead slices
        self.invq = invq                  # per frame Lowres::invQscaleFactor (int32 per lowres CU) or None: AQ off
        self.lam = LOOKAHEAD_LAMBDA[depth]
        self.tab = np.zeros(2 * MVRANGE + 1, np.uint16)
        O.orc_mvcost_table(C.c_double(self.lam), MVRANGE, ptr(self.tab))
        self.fr = []
        for fi, img in enumerate(frames):
            planes, ls, lorg, w8, h8 = make_lowres(O, img, depth)
            ncu = w8 * h8
            f = dict(planes=planes, intraCost=np.zeros(ncu, np.int32), intraMode=np.zeros(ncu, np.uint8),
                     lowresCosts={}, rowSatds={}, costEst={}, mvs={}, mvcosts={}, intraMbs={}, estIntraMbs={})
            lc = np.zeros(ncu, np.uint16); rs = np.zeros(h8, np.int32); ce = np.zeros(2, np.int64)
            O.orc_lowres_intra(ptr(planes[0], lorg), IP(ls), w8, h8, int(self.lam), ptr(invq[fi]) if invq is not None else None, ptr(f["intraCost"]), ptr(f["intraMode"]), ptr(lc), ptr(rs), ptr(ce))
            f["lowresCosts"][(0, 0)] = lc; f["rowSatds"][(0, 0)] = rs; f["costEst"][(0, 0)] = (int(ce[0]), int(ce[1]))
            self.fr.append(f)
        self.stride, self.org, self.w8, self.h8 = ls, lorg, w8, h8

    def cost(self, p0, p1, b):
        f = self.fr[b]
        d0, d1 = b - p0, p1 - b
        if (d0, d1) in f["costEst"]:
            return f["costEst"][(d0, d1)][0]
        ncu = self.w8 * self.h8
        j = OrcLaJob()
        es = np.dtype(pixel_dtype(self.depth)).itemsize
        for k in range(4):
            j.fenc[k] = f["planes"][k].ctypes.data + self.org * es
            j.ref0[k] = self.fr[p0]["planes"][k].ctypes.data + self.org * es
            j.ref1[k] = self.fr[p1]["planes"][k].ctypes.data + self.org * es
        j.stride, j.w8, j.h8, j.bidir = self.stride, self.w8, self.h8, int(b < p1)
        for lst, dist in ((0, d0), (1, d1)):
            new = (lst, dist) not in f["mvs"]
            if new:
                f["mvs"][(lst, dist)] = np.zeros((ncu, 2), np.int32); f["mvcosts"][(lst, dist)] = np.zeros(ncu, np.int32)
            j.doSearch[lst] = int(new and (lst == 0 or p1 > b))
            j.mvs[lst] = f["mvs"][(lst, dist)].ctypes.data; j.mvcosts[lst] = f["mvcosts"][(lst, dist)].ctypes.data
        if not (p1 > b):
            del_key = (1, d1)
            if del_key in f["mvs"] and j.doSearch[1] == 0 and not f["mvs"][del_key].any():
                pass
        if self.slices and self.slices[0] > 1 and (p1 > b or j.doSearch[0] or j.doSearch[1]):
            j.numSlices, j.rowsPerSlice = self.slices         # the cooperative path (slicetype.cpp:3143)
        j.intraCost = f["intraCost"].ctypes.data
        j.invQscale = self.invq[b].ctypes.data if self.invq is not None else None
        j.mvcost_tab = self.tab.ctypes.data + MVRANGE * 2
        lc = np.zeros(ncu, np.uint16); rs = np.zeros(self.h8, np.int32)
        j.lowresCosts = lc.ctypes.data; j.rowSatds = rs.ctypes.data
        self.O.orc_lookahead_frame_cost.argtypes = [C.POINTER(OrcLaJob)]
        self.O.orc_lookahead_frame_cost(C.byref(j))
        score = int(j.out[0])
        if b != p1:
            score = score * 100 // 130          # slicetype.cpp:3205-3206, bFrameBias = 0
        f["lowresCosts"][(d0, d1)] = lc; f["rowSatds"][(d0, d1)] = rs
        f["costEst"][(d0, d1)] = (score, int(j.out[1])); f["intraMbs"][d0] = f["intraMbs"].get(d0, 0) + int(j.out[2])
        f["estIntraMbs"][(d0, d1)] = int(j.out[2])      # this estimate's own count (intraMbs[d0] sums the estimates at d0)
        return score
