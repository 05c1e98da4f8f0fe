"""Weighted-prediction analysis (weightAnalyse, encoder/weightPrediction.cpp:222-539): pictures, the case matrix, the
plain-C restatement (oracle/oracle_weightp.c), the REAL function on real Frames (oracle/ref_shim_weightp.cpp) and its
stored results (tests/golden/weightp_ref.json) where oracle/_ref is not built."""
import ctypes as C
import json
import os

import numpy as np

from common import ROOT, P, I, ptr, pixel_dtype, load_oracle
from frame_helpers import gen_luma, gen_chroma
from lookahead_helpers import OracleLookahead
from aq_helpers import load_oracle_aq, AqParams
from x265_b200.lib import WpFrame, WpParams, WpCand, WpEntry, WP_COST_FN

GOLDEN = os.path.join(ROOT, "tests", "golden", "weightp_ref.json")
CMX, CMY = 48, 40                         # PicYuv 4:2:0 chroma margins

# content kinds: frames (ref0, fenc, ref1) at pocs (0, 1, 2)
KINDS = ("static", "fade_up", "fade_down", "to_black", "from_black", "offset", "constant", "motion_fade", "chroma_only",
         "luma_only", "fade_cb", "flat_ref_chroma")
# textured content moving by whole pixels: intraCost is high, so the compensated costs, not the intra cap, decide, and luma
# ends up weighted with the motion fields present (chroma is then analysed on compensated blocks).  The motion picks the
# chroma path of mcChroma: (3, -2) px -> lowres qpel (6, -4) -> hps + vsp; (4, -2) -> (8, -4) -> vpp.
NOISE_KINDS = ("noise_fade", "noise_fade_v", "noise_flat_chroma")
COUNTERS = ("early", "chroma_denom", "chroma_scale_skip", "offset_rescale", "rescale_refmean0", "delta_skip", "offset_break",
            "luma_denom", "reject_0998", "chroma_fixup", "list1", "path_copy", "path_hpp", "path_vpp", "path_hv",
            "mc_block", "copy_block", "orig_zero", "weighted")


def _scale(a, s, add, depth):
    return np.clip(np.rint(a.astype(np.float64) * s + add * (1 << (depth - 8))), 0, (1 << depth) - 1).astype(pixel_dtype(depth))


def _moving_noise(W, H, depth, motion, seed):
    """3 frames of one noise picture (smoothed over 2x2, so the lowres planes keep texture) displaced by `motion` px per
    frame, and the 4:2:0 chroma displaced by half of it"""
    dx, dy = motion
    rng = np.random.default_rng(seed)
    pad = 64
    big = rng.integers(0, 256, (H + 2 * pad + 1, W + 2 * pad + 1)).astype(np.float64)
    big = (big[:-1, :-1] + big[1:, :-1] + big[:-1, 1:] + big[1:, 1:]) / 4
    cbig = [rng.integers(16, 240, (H // 2 + pad + 1, W // 2 + pad + 1)).astype(np.float64) for _ in range(2)]
    cbig = [(c[:-1, :-1] + c[1:, :-1] + c[:-1, 1:] + c[1:, 1:]) / 4 for c in cbig]
    out = []
    for i in range(3):
        y = big[pad - dy * i:pad - dy * i + H, pad - dx * i:pad - dx * i + W] * (1 << (depth - 8))
        cs = [c[pad // 2 - dy // 2 * i:pad // 2 - dy // 2 * i + H // 2, pad // 2 - dx // 2 * i:pad // 2 - dx // 2 * i + W // 2]
              * (1 << (depth - 8)) for c in cbig]
        out.append((y, cs[0], cs[1]))
    return out


def pictures(kind, W, H, depth):
    """[(y, cb, cr)] of frames (ref0, fenc, ref1)"""
    if kind in NOISE_KINDS:
        frames = _moving_noise(W, H, depth, (4, -2) if kind == "noise_fade_v" else (3, -2), W + depth)
        ls, cbs, crs = (1.0, 0.75, 0.6), (1.0, 0.8, 0.7), (1.0, 0.7, 0.85)
        add = (0, 12, -6)
        return [(_scale(y, ls[i], add[i], depth), _scale(cb, cbs[i], 0, depth), _scale(cr, crs[i], 0, depth))
                for i, (y, cb, cr) in enumerate(frames)]
    motion = (12, -8) if kind == "motion_fade" else (3, -2)
    ys = [gen_luma(W, H, 0 if kind in ("static", "chroma_only") else i, bits=depth, motion=motion) for i in range(3)]
    cs = [[gen_chroma(W, H, 0 if kind in ("static", "luma_only") else i, pl, bits=depth, motion=motion) for pl in (1, 2)]
          for i in range(3)]
    ls, cbs, crs = (1.0, 1.0, 1.0), (1.0, 1.0, 1.0), (1.0, 1.0, 1.0)
    add = (0, 0, 0)
    if kind in ("fade_up", "motion_fade"):
        ls = cbs = crs = (0.55, 0.8, 1.0)
    elif kind == "fade_down":
        ls = cbs = crs = (1.0, 0.7, 0.5)
    elif kind == "to_black":
        ls = (1.0, 0.02, 1.0)
    elif kind == "from_black":
        ls = (0.0, 0.4, 0.0); add = (0, 150, 0)
    elif kind == "offset":
        add = (0, 24, -20)
    elif kind == "chroma_only":
        cbs = crs = (0.6, 1.0, 0.8)
    elif kind == "luma_only":
        ls = (0.6, 1.0, 0.75)
    elif kind == "fade_cb":
        ls = cbs = (0.6, 0.9, 1.0)
    elif kind == "flat_ref_chroma":
        ls = (0.6, 0.9, 0.7)
    out = []
    for i in range(3):
        y = _scale(ys[i], ls[i], add[i], depth)
        cb = _scale(cs[i][0], cbs[i], 0, depth)
        cr = _scale(cs[i][1], crs[i], 0, depth) if kind != "fade_cb" else cs[0][1].copy()
        if kind == "constant":
            v = (100, 140, 60)[i] << (depth - 8)
            y = np.full_like(y, v); cb = np.full_like(cb, v // 2 + 30); cr = np.full_like(cr, v)
        if kind == "flat_ref_chroma" and i != 1:
            cb = np.full_like(cb, 128 << (depth - 8)); cr = np.full_like(cr, 120 << (depth - 8))
        out.append((y, cb, cr))
    return out


# (name, kind, W, H, depth, csp, slice type, numRefIdx, motion fields)
def _case(kind, W, H, depth, csp, st, nref, mvs):
    return ("%s_%dx%d_%d_%s_%s%d_%s" % (kind, W, H, depth, "420" if csp else "400", st, nref, mvs), kind, W, H, depth, csp, st, nref, mvs)


CASES = [_case(k, 328, 184, 8, 1, "P", 1, "la") for k in KINDS]
CASES += [_case(k, 328, 184, 10, 1, "B", 3, "la") for k in KINDS]
CASES += [_case(k, 328, 184, 8, 1, "B", 1, "edge") for k in ("fade_up", "fade_cb", "flat_ref_chroma", "motion_fade")]
CASES += [_case(k, 328, 184, d, 1, st, n, m) for k in NOISE_KINDS for (d, st, n, m) in ((8, "P", 1, "la"), (10, "B", 3, "la"))]
CASES += [_case("noise_fade", 328, 184, 8, 1, "B", 1, "edge"), _case("noise_fade_v", 328, 184, 10, 1, "P", 1, "edge"),
          _case("noise_fade", 328, 184, 8, 0, "B", 1, "edge"), _case("noise_fade", 1920, 1080, 8, 1, "P", 1, "edge"),
          _case("fade_up", 328, 184, 8, 1, "B", 1, "rand"), _case("static", 328, 184, 8, 1, "P", 1, "rand")]
CASES += [_case("fade_up", 328, 184, 8, 0, "P", 3, "la"), _case("luma_only", 328, 184, 10, 0, "B", 1, "edge"),
          _case("fade_down", 328, 184, 10, 1, "P", 1, "edge"), _case("fade_up", 328, 184, 8, 1, "P", 1, "none"),
          _case("fade_up", 328, 184, 10, 1, "B", 3, "far"), _case("to_black", 328, 184, 8, 1, "B", 3, "none"),
          _case("fade_up", 1920, 1080, 8, 1, "P", 1, "la"), _case("motion_fade", 1920, 1080, 10, 1, "B", 3, "edge"),
          _case("fade_down", 3840, 2160, 8, 1, "P", 1, "edge")]
BFRAMES = 3


def _pad_chroma(pl):
    return np.pad(pl, ((CMY, CMY), (CMX, CMX + 8)), mode="edge")      # 8 extra columns: a stride wider than the row


def _wp_stats(depth, y, cb, cr, W, H):
    O = load_oracle_aq()
    prm = AqParams(aqMode=2, qgSize=32, weightp=1, aqStrength=1.0)
    w8, h8 = ((W // 2) + 7) >> 3, ((H // 2) + 7) >> 3
    qp = np.zeros(w8 * h8); iq = np.zeros(w8 * h8, np.int32); s = np.zeros(3, np.uint64); d = np.zeros(3, np.uint64)
    O.orc_aq(depth, ptr(y), W, ptr(cb) if cb is not None else None, ptr(cr) if cr is not None else None, W // 2, W, H,
             C.byref(prm), ptr(qp), ptr(iq), None, ptr(s), ptr(d), None, None)
    return s, d


class Case:
    """Every input of one analysis, on the host: planes, statistics, intraCost, motion fields, records."""

    def __init__(self, case):
        self.name, kind, W, H, depth, csp, st, nref, mvmode = case
        self.W, self.H, self.depth, self.csp, self.mvmode = W, H, depth, csp, mvmode
        self.nl = 1 if st == "P" else 2
        self.params = WpParams(1 if st == "P" else 0, (C.c_int32 * 2)(nref, nref if self.nl == 2 else 0), BFRAMES, W, H, csp)
        self.pics = pictures(kind, W, H, depth)
        la = OracleLookahead(load_oracle(depth), [p[0] for p in self.pics], depth, bframes=BFRAMES)
        self.la = la
        self.intraCost = la.fr[1]["intraCost"]
        self.poc = np.array([0, 1, 2] if mvmode != "far" else [0, BFRAMES + 3, 2 * BFRAMES + 6], np.int32)
        ncu = la.w8 * la.h8
        self.mvs = [None, None]
        if mvmode in ("la", "far", "edge"):
            la.cost(0, 1, 1) if self.nl == 1 else la.cost(0, 2, 1)
            self.mvs = [np.ascontiguousarray(la.fr[1]["mvs"][(l, 1)], np.int32) for l in range(self.nl)] + [None] * (2 - self.nl)
        if mvmode == "rand":
            # vectors unrelated to the content, half of them off a picture edge: the costs stay near the unweighted ones
            rng = np.random.default_rng(W * 5 + depth)
            lim = 4 * (la.w8 * 8 + 64)
            for l in range(self.nl):
                m = rng.integers(-64, 65, (ncu, 2)).astype(np.int32)
                far = rng.random(ncu) < 0.5
                m[far] = rng.integers(-lim, lim + 1, (int(far.sum()), 2))
                self.mvs[l] = m
        if mvmode == "edge":
            # the lookahead's field with one CU in 8 pointing off a picture edge, and every chroma fraction in the CUs
            # mcChroma compensates (pixel x < w8, y < h8)
            rng = np.random.default_rng(W * 7 + depth)
            lim = 4 * (la.w8 * 8 + 64)
            for l in range(self.nl):
                m = self.mvs[l]
                far = rng.random(ncu) < 0.125
                m[far] = rng.integers(-lim, lim + 1, (int(far.sum()), 2))
                for n, cu in enumerate(y * la.w8 + x // 8 for y in range(0, la.h8, 8) for x in range(0, la.w8, 8)):
                    m[cu] = ((n * 3) % 8 - 4, (n * 5) % 8 - 4)
        self.chroma = []
        self.stats = []
        for i, (y, cb, cr) in enumerate(self.pics):
            s, d = _wp_stats(depth, y, cb if csp else None, cr if csp else None, W, H)
            if kind == "static" and i == 1 and nref == 3:
                s, d = s * 3 // 2, d * 2          # statistics of a fade on identical pictures: origscore is 0
            if kind in ("fade_cb", "noise_flat_chroma") and i == 0 and (st == "B" or kind == "noise_flat_chroma"):
                d[1:] = 0                         # a flat reference chroma: guessScale past 127 at any denominator
            self.stats.append((s, d))
            self.chroma.append([_pad_chroma(cb), _pad_chroma(cr)] if csp else None)
        self.recs = [self.record(i) for i in range(3)]

    def record(self, i):
        la, es = self.la, np.dtype(pixel_dtype(self.depth)).itemsize
        r = WpFrame()
        for k in range(4):
            r.lowres[k] = la.fr[i]["planes"][k].ctypes.data + la.org * es
        r.lowresStride = la.stride
        if self.chroma[i] is not None:
            cs = self.chroma[i][0].shape[1]
            r.cb, r.cr = [c.ctypes.data + (CMY * cs + CMX) * es for c in self.chroma[i]]
            r.chromaStride = cs
        for k in range(3):
            r.wp_sum[k], r.wp_ssd[k] = int(self.stats[i][0][k]), int(self.stats[i][1][k])
        r.poc = int(self.poc[i])
        return r

    def ref_records(self):
        return (C.POINTER(WpFrame) * 2)(C.pointer(self.recs[0]), C.pointer(self.recs[2]) if self.nl == 2 else C.POINTER(WpFrame)())

    def mv_ptrs(self):
        return (C.c_void_p * 2)(*[m.ctypes.data if m is not None else None for m in self.mvs])

    def written(self, table):
        """the entries the reference writes: list < numPredDir, ref < numRefIdx[list]; luma only in 4:0:0 (the
        reference's chroma denominator there comes from uninitialised floats)"""
        t = np.asarray(table).reshape(2, 16, 3, 4)
        return [t[l, r, p].tolist() for l in range(self.nl) for r in range(self.params.numRefIdx[l])
                for p in range(3 if self.csp else 1)]


_libs = {}


def load_oracle_wp():
    if "orc" not in _libs:
        p = os.path.join(ROOT, "oracle", "liboracle_weightp.so")
        if not os.path.exists(p):
            import subprocess
            subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "-f", "Makefile.weightp", "oracle"])
        L = C.CDLL(p)
        L.orc_wp_costs.restype = None
        L.orc_wp_costs.argtypes = [I, C.POINTER(WpParams), C.POINTER(WpFrame), C.POINTER(WpFrame), P, P, I, C.POINTER(WpCand), I, P]
        L.orc_wp_analyse.restype = None
        L.orc_wp_analyse.argtypes = [I, C.POINTER(WpParams), C.POINTER(WpFrame), P, C.POINTER(C.POINTER(WpFrame)), C.POINTER(P), P]
        L.orc_wp_counters.restype = None
        L.orc_wp_counters.argtypes = [P, I]
        _libs["orc"] = L
    return _libs["orc"]


def load_ref_wp(depth):
    key = ("ref", depth)
    if key not in _libs:
        p = os.path.join(ROOT, "oracle", "_ref", "libx265ref_weightp%d.so" % depth)
        if not os.path.exists(p):
            return None
        L = C.CDLL(p)
        L.x265ref_weightp.restype = None
        L.x265ref_weightp.argtypes = [P, P, P, P, P, P, P, P, P]
        L.x265ref_weightp_costs.restype = None
        L.x265ref_weightp_costs.argtypes = [P, P, P, P, P, P, P, I, I, I, P, I, P]
        _libs[key] = L
    return _libs[key]


def oracle_table(c, fill=-7):
    O = load_oracle_wp()
    out = np.full((2, 16, 3, 4), fill, np.int32)
    O.orc_wp_analyse(c.depth, C.byref(c.params), C.byref(c.recs[1]), ptr(c.intraCost), c.ref_records(), c.mv_ptrs(), ptr(out))
    return out


def oracle_counters(reset=True):
    cnt = np.zeros(len(COUNTERS), np.int64)
    load_oracle_wp().orc_wp_counters(ptr(cnt), int(reset))
    return dict(zip(COUNTERS, cnt.tolist()))


def reference_table(c):
    """(table, intraCost) of the real weightAnalyse, or None without oracle/_ref"""
    R = load_ref_wp(c.depth)
    if R is None:
        return None
    out = np.zeros((2, 16, 3, 4), np.int32)
    intra = np.zeros(c.la.w8 * c.la.h8, np.int32)
    R.x265ref_weightp(*_shim_inputs(c), ptr(out), ptr(intra))
    return out, intra


def _shim_inputs(c):
    arr = lambda xs: (C.c_void_p * 3)(*[x.ctypes.data if x is not None else None for x in xs])
    order = (1, 0, 2)                     # the shim's frames: fenc, m_refFrameList[0][0], m_refFrameList[1][0]
    c._keep = [np.ascontiguousarray(np.array([np.concatenate(c.stats[i]) for i in order], np.uint64)),
               np.ascontiguousarray(c.poc[list(order)])]
    ys = [c.pics[i][0] for i in order]
    cbs = [c.pics[i][1] if c.csp else None for i in order]
    crs = [c.pics[i][2] if c.csp else None for i in order]
    return arr(ys), arr(cbs), arr(crs), C.byref(c.params), ptr(c._keep[1]), ptr(c._keep[0]), c.mv_ptrs()


# candidates of the cost pins: the unweighted reference, then w0 over 0..127 with every denominator and the offsets
# -128 / 0 / 127 (weight_pp's extremes)
PIN_CANDS = [(0, 0, 0, 0)] + [(1, w0, k % 8, (-128, 0, 127)[k % 3]) for k, w0 in enumerate(range(0, 128, 6))]


def oracle_costs(c, lst, plane, use_mvs, cands=PIN_CANDS):
    arr = (WpCand * len(cands))(*[WpCand(*x) for x in cands])
    out = np.zeros(len(cands), np.uint32)
    load_oracle_wp().orc_wp_costs(c.depth, C.byref(c.params), C.byref(c.recs[1]), C.byref(c.recs[2 * lst]), ptr(c.intraCost),
                                  c.mvs[lst].ctypes.data if use_mvs else None, plane, arr, len(cands), ptr(out))
    return out


def reference_costs(c, lst, plane, use_mvs, cands=PIN_CANDS):
    """the real mcLuma / mcChroma + weightCost on the case's frames, or None without oracle/_ref"""
    R = load_ref_wp(c.depth)
    if R is None:
        return None
    cd = np.ascontiguousarray(np.array(cands, np.int32))
    out = np.zeros(len(cands), np.uint32)
    R.x265ref_weightp_costs(*_shim_inputs(c), lst, plane, int(use_mvs), ptr(cd), len(cands), ptr(out))
    return out


_golden = {}


def stored(name):
    if not _golden:
        _golden.update(json.load(open(GOLDEN)) if os.path.exists(GOLDEN) else {})
    return _golden.get(name)


def store(name, written):
    stored(name)
    _golden[name] = written
    with open(GOLDEN, "w") as f:
        json.dump(_golden, f, indent=0, sort_keys=True)
        f.write("\n")


def stored_costs(name):
    return stored("costs:" + name)


def expected(c):
    """the reference's written entries: computed where oracle/_ref is built (and stored with X265_WRITE_GOLDEN=1), else
    read from tests/golden/weightp_ref.json"""
    r = reference_table(c)
    if r is None:
        want = stored(c.name)
        assert want is not None, "no stored reference result for %s in %s" % (c.name, GOLDEN)
        return want
    table, intra = r
    assert np.array_equal(intra, c.intraCost), "the oracle's intraCost differs from lowresIntraEstimate's"
    w = c.written(table)
    if os.environ.get("X265_WRITE_GOLDEN") == "1":
        store(c.name, w)
    elif stored(c.name) is not None:
        assert stored(c.name) == w, "the reference's result differs from %s" % GOLDEN
    return w


def oracle_cost_fn(c):
    """a cost provider for x265cu_weightp_decide backed by the restatement's weightCost"""
    O = load_oracle_wp()

    def fn(user, lst, plane, use_mvs, cands, n, costs):
        O.orc_wp_costs(c.depth, C.byref(c.params), C.byref(c.recs[1]), C.byref(c.recs[2 * lst]), ptr(c.intraCost),
                       c.mvs[lst].ctypes.data if use_mvs else None, plane, cands, n, C.cast(costs, P))
        return 0
    return WP_COST_FN(fn)
