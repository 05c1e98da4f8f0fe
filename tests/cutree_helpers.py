"""cuTree's propagation chain: windows of synthetic or real lookahead estimates, the plain-C restatement
(oracle/oracle_cutree.c), the REAL Lookahead::cuTree (oracle/ref_shim_cutree.cpp) and the stored results of the latter
(tests/golden/cutree_ref.json, tests/golden/cutree_clip.npz) where oracle/_ref is not built."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from common import ROOT, P, I, ptr
from ref_results import digest

DIST = 18
TYPE_I, TYPE_P, TYPE_B = 2, 3, 5
GOLDEN = os.path.join(ROOT, "tests", "golden", "cutree_ref.json")
CLIP = os.path.join(ROOT, "tests", "golden", "cutree_clip.npz")


class OrcFrame(C.Structure):
    _fields_ = [("intraCost", P), ("invQscale", P), ("propagateCost", P), ("lowresCosts", P * DIST * DIST),
                ("mvs", P * DIST * 2), ("sliceType", C.c_int32), ("reserved", C.c_int32),
                ("qpAqOffset", P), ("qpCuTreeOffset", P), ("weightedCostDelta", C.c_double * DIST)]


class OrcParams(C.Structure):
    _fields_ = [("bIntra", C.c_int32), ("lookaheadDepth", C.c_int32), ("bBPyramid", C.c_int32), ("bEnableWeightedBiPred", C.c_int32),
                ("vbv", C.c_int32), ("fpsNum", C.c_int32), ("fpsDenom", C.c_int32), ("qgSize", C.c_int32), ("qCompress", C.c_double)]


_libs = {}


def load_oracle_cutree():
    if "orc" not in _libs:
        p = os.path.join(ROOT, "oracle", "liboracle_cutree.so")
        if not os.path.exists(p):
            import subprocess
            subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "-f", "Makefile.cutree", "oracle"])
        L = C.CDLL(p)
        L.orc_cutree.restype = I
        L.orc_cutree.argtypes = [P, I, P, I, I, P, I]
        L.orc_cutree_finish.restype = None
        L.orc_cutree_finish.argtypes = [P, I, P, I, I, I, I]
        _libs["orc"] = L
    return _libs["orc"]


def load_ref_cutree(depth=8):
    key = ("ref", depth)
    if key not in _libs:
        p = os.path.join(ROOT, "oracle", "_ref", "libx265ref_cutree%d.so" % depth)
        if not os.path.exists(p):
            return None
        L = C.CDLL(p)
        L.x265ref_cutree.restype = None
        L.x265ref_cutree.argtypes = [P, I, P, I, I, P, P]
        L.x265ref_cutree_finish.restype = None
        L.x265ref_cutree_finish.argtypes = [P, I, P, I, I, I, I, P]
        _libs[key] = L
    return _libs[key]


def pattern(f, ncu):
    """What every frame's propagateCost holds before the chain (the shim's fill)."""
    return ((np.uint32(f + 1) * np.uint32(40503) + np.arange(ncu, dtype=np.uint32) * np.uint32(9973)) & 0xffff).astype(np.uint16)


def slice_types(n, bframes, intra0=True):
    """I (or P) at frame 0, then P every bframes + 1 frames, B between; the last frame is a P when the window ends mid-GOP
    only if it falls on the cadence (trailing B frames are what cuTree skips)."""
    return [TYPE_I if (i == 0 and intra0) else (TYPE_P if i % (bframes + 1) == 0 else TYPE_B) for i in range(n)]


def estimates(cu_lib, types, prm):
    """(p0, p1, b) the chain reads: x265cu_cutree_estimates (host code of the product library; needs no GPU)."""
    from x265_b200.lib import CutreeParams
    st = np.ascontiguousarray(types, np.int32)
    cap = 4 * (len(types) + 1) * DIST
    out = np.zeros(3 * cap, np.int32)
    p = CutreeParams(prm["bIntra"], prm["lookaheadDepth"], prm["bBPyramid"], prm["bEnableWeightedBiPred"], prm["vbv"],
                     prm["fpsNum"], prm["fpsDenom"])
    n = cu_lib.L.x265cu_cutree_estimates(st.ctypes.data, len(types) - 1, C.byref(p), out.ctypes.data, cap)
    assert n >= 0, cu_lib.last_error()
    return [tuple(int(v) for v in out[3 * k:3 * k + 3]) for k in range(n)]


def params(**kw):
    p = dict(bIntra=0, lookaheadDepth=40, bBPyramid=1, bEnableWeightedBiPred=0, vbv=0, fpsNum=25, fpsDenom=1, qgSize=32, qCompress=0.6)
    p.update(kw)
    return p


class Window:
    """One cuTree window as host arrays: per frame intraCost / invQscale / qpAqOffset, per estimate lowresCosts and
    the motion fields keyed (list, dist)."""

    def __init__(self, w8, h8, types, prm):
        self.w8, self.h8, self.ncu, self.types, self.prm = w8, h8, w8 * h8, list(types), prm
        self.n = len(types)
        self.nfull = 4 * self.ncu if prm["qgSize"] == 8 else self.ncu
        self.intra = [None] * self.n
        self.invq = [None] * self.n
        self.aq = [None] * self.n
        self.wcd = [np.zeros(DIST) for _ in range(self.n)]
        self.costs = {}                      # (b, d0, d1) -> uint16[ncu]
        self.mvs = {}                        # (b, list, dist) -> int32[ncu, 2]

    def _records(self, props, qps):
        recs = (OrcFrame * self.n)()
        keep = []
        for f in range(self.n):
            r = recs[f]
            arrs = [np.ascontiguousarray(self.intra[f], np.int32), np.ascontiguousarray(self.invq[f], np.int32),
                    np.ascontiguousarray(self.aq[f], np.float64)]
            keep += arrs
            r.intraCost, r.invQscale, r.qpAqOffset = arrs[0].ctypes.data, arrs[1].ctypes.data, arrs[2].ctypes.data
            r.propagateCost = props[f].ctypes.data if props is not None else None
            r.qpCuTreeOffset = qps[f].ctypes.data if qps is not None else None
            r.sliceType = self.types[f]
            for d in range(DIST):
                r.weightedCostDelta[d] = float(self.wcd[f][d])
        for (b, d0, d1), a in self.costs.items():
            a = np.ascontiguousarray(a, np.uint16); keep.append(a)
            recs[b].lowresCosts[d0][d1] = a.ctypes.data
        for (b, lst, dist), a in self.mvs.items():
            a = np.ascontiguousarray(a, np.int32); keep.append(a)
            recs[b].mvs[lst][dist] = a.ctypes.data
        return recs, keep

    def c_params(self):
        p = self.prm
        return OrcParams(p["bIntra"], p["lookaheadDepth"], p["bBPyramid"], p["bEnableWeightedBiPred"], p["vbv"], p["fpsNum"],
                         p["fpsDenom"], p["qgSize"], p["qCompress"])

    def oracle(self):
        """(propagateCost of every frame after the chain, as its pointer then points; qpCuTreeOffset; finish list)."""
        O = load_oracle_cutree()
        props = [pattern(f, self.ncu) for f in range(self.n)]
        qps = [np.full(self.nfull, -1000.0 - f) for f in range(self.n)]
        recs, keep = self._records(props, qps)
        prm = self.c_params()
        fin = np.zeros(2 * (self.n + 2), np.int32)
        nf = O.orc_cutree(C.cast(recs, P), self.n - 1, C.cast(C.pointer(prm), P), self.w8, self.h8, ptr(fin), self.n + 2)
        assert nf >= 0, "the window reaches estimateCUPropagate(0, 0, 0)"
        byaddr = {a.ctypes.data: a for a in props}
        out = [byaddr[recs[f].propagateCost].copy() for f in range(self.n)]
        return out, qps, [(int(fin[2 * k]), int(fin[2 * k + 1])) for k in range(nf)]

    def oracle_finish(self, f, d, prop):
        """The restated cuTreeFinish of frame f on `prop` (qpCuTreeOffset prefilled -1000 - f)."""
        O = load_oracle_cutree()
        props = [pattern(g, self.ncu) for g in range(self.n)]
        props[f] = np.ascontiguousarray(prop, np.uint16)
        qps = [np.full(self.nfull, -1000.0 - g) for g in range(self.n)]
        recs, keep = self._records(props, qps)
        prm = self.c_params()
        O.orc_cutree_finish(C.cast(recs, P), self.n - 1, C.cast(C.pointer(prm), P), self.w8, self.h8, f, d)
        return qps[f]

    def reference(self, depth=8):
        """The real Lookahead::cuTree: (propagateCost of every frame, qpCuTreeOffset of every frame)."""
        R = load_ref_cutree(depth)
        recs, keep = self._records(None, None)
        prm = self.c_params()
        prop = np.zeros(self.n * self.ncu, np.uint16)
        qp = np.zeros(self.n * self.nfull)
        R.x265ref_cutree(C.cast(recs, P), self.n - 1, C.cast(C.pointer(prm), P), self.w8, self.h8, ptr(prop), ptr(qp))
        return list(prop.reshape(self.n, self.ncu)), list(qp.reshape(self.n, self.nfull))

    def reference_finish(self, f, d, prop, depth=8):
        R = load_ref_cutree(depth)
        props = [None] * self.n
        props[f] = np.ascontiguousarray(prop, np.uint16)
        recs, keep = self._records(None, None)
        recs[f].propagateCost = props[f].ctypes.data
        prm = self.c_params()
        qp = np.zeros(self.nfull)
        R.x265ref_cutree_finish(C.cast(recs, P), self.n - 1, C.cast(C.pointer(prm), P), self.w8, self.h8, f, d, ptr(qp))
        return qp


def synth_window(cu_lib, name, w8, h8, types, prm, seed=1, depth=8, mv="random", amount="normal"):
    """Synthetic inputs for every estimate the chain reads.
    mv: random | edges (MVs off every picture edge) | zero_frac (whole-CU MVs) | one_cu (every MV aimed at one CU) | zero
    amount: normal | overflow (amounts past 2^21: the wrapped, order-dependent path) | int_min (intraCost 0 entries)"""
    rng = np.random.default_rng([seed, sum(map(ord, name))])
    win = Window(w8, h8, types, prm)
    ncu = w8 * h8
    imax = (1 << 14) if depth == 8 else (1 << 17)          # 10-bit lowres SATD costs run higher
    for f in range(win.n):
        win.intra[f] = rng.integers(1, imax, ncu).astype(np.int32)
        win.invq[f] = rng.integers(40, 1024, ncu).astype(np.int32)
        if amount == "overflow":
            big = rng.random(ncu) < 0.3                     # amounts past 2^21: the weight products wrap
            win.intra[f][big] = rng.integers(1 << 14, 1 << 15, big.sum())
            win.invq[f][big] = rng.integers(1 << 15, 0xffff, big.sum())
            wrap = rng.random(ncu) < 0.1                    # intraCost * invQscale itself past 2^31
            win.intra[f][wrap] = rng.integers(1 << 16, 1 << 20, wrap.sum())
            win.invq[f][wrap] = 0xffff
        if amount == "int_min":
            win.intra[f][rng.random(ncu) < 0.2] = 0
        win.aq[f] = rng.normal(0, 2, win.nfull)
        win.wcd[f] = rng.random(DIST) * 1.5 - 0.25
    cux, cuy = np.meshgrid(np.arange(w8), np.arange(h8))
    cux, cuy = cux.ravel(), cuy.ravel()
    for (p0, p1, b) in estimates(cu_lib, types, prm):
        d0, d1 = b - p0, p1 - b
        if (b, d0, d1) in win.costs:
            continue
        bidir = p1 > b
        lists = rng.integers(0, 4 if bidir else 2, ncu)
        cost = np.minimum(rng.integers(0, imax, ncu), (1 << 14) - 1)
        win.costs[(b, d0, d1)] = (cost | (lists << 14)).astype(np.uint16)
        for lst, dist in [(0, d0)] + ([(1, d1)] if bidir else []):
            if (b, lst, dist) in win.mvs:
                continue
            if mv == "random":
                m = rng.integers(-96, 97, (ncu, 2))
                m[rng.random(ncu) < 0.2] = 0
            elif mv == "edges":
                m = np.stack([(rng.integers(-2, 3, ncu) - cux * (rng.random(ncu) < 0.5)) * 32 + rng.integers(-31, 32, ncu),
                              (rng.integers(-2, 3, ncu) - cuy * (rng.random(ncu) < 0.5)) * 32 + rng.integers(-31, 32, ncu)], 1)
                far = rng.random(ncu) < 0.5
                m[far, 0] += (w8 - cux[far]) * 32 * np.sign(rng.random(far.sum()) - 0.5).astype(np.int64)
                m[far, 1] += (h8 - cuy[far]) * 32 * np.sign(rng.random(far.sum()) - 0.5).astype(np.int64)
            elif mv == "zero_frac":
                m = rng.integers(-3, 4, (ncu, 2)) * 32
            elif mv == "one_cu":
                tx, ty = w8 // 2, h8 // 2
                m = np.stack([(tx - cux) * 32, (ty - cuy) * 32], 1)
            else:
                m = np.zeros((ncu, 2), np.int64)
            win.mvs[(b, lst, dist)] = np.clip(m, -32768, 32767).astype(np.int32)
    return win


def clip_window(prm, types):
    """A real clip's lookahead window: the reference lookahead with AQ (x265ref_la_create_aq) estimates every triple the
    chain reads; stored in tests/golden/cutree_clip.npz (written with X265_WRITE_GOLDEN=1 while oracle/_ref is built)."""
    from common import load_ref
    R = load_ref(8)
    if R is not None and os.environ.get("X265_WRITE_GOLDEN") == "1":
        _write_clip(R, types)
    if not os.path.exists(CLIP):
        pytest.fail("no stored clip window in %s" % CLIP)
    z = np.load(CLIP)
    w8, h8 = int(z["geometry"][0]), int(z["geometry"][1])
    win = Window(w8, h8, types, prm)
    for f in range(win.n):
        win.intra[f] = z["intra%d" % f]
        win.invq[f] = z["invq%d" % f]
        win.aq[f] = np.zeros(win.nfull)
    for k in z.files:
        if k.startswith("costs_"):
            b, d0, d1 = map(int, k[6:].split("_"))
            win.costs[(b, d0, d1)] = z[k]
        if k.startswith("mvs_"):
            b, lst, dist = map(int, k[4:].split("_"))
            win.mvs[(b, lst, dist)] = z[k]
    return win


CLIP_TYPES = slice_types(13, 3)
CLIP_SIZE = (192, 112)


def _write_clip(R, types):
    from frame_helpers import gen_luma
    from test_lookahead_oracle_vs_ref import RefLookahead
    import x265_b200
    W, H = CLIP_SIZE
    frames = [gen_luma(W, H, i, s1=17.0, s2=11.0, bits=8, noise=False) for i in range(len(types))]
    chroma = [(np.ascontiguousarray(f[::2, ::2]), np.ascontiguousarray(f[1::2, 1::2])) for f in frames]
    ref = RefLookahead(R, frames, bframes=3, aq=1, chroma=chroma)
    cu = x265_b200.load(need_gpu=False)
    trip = set()
    for pyr in (0, 1):
        for vbv in (0, 1):
            trip |= set(estimates(cu, types, params(bBPyramid=pyr, vbv=vbv)))
    out = dict(geometry=np.array([ref.w8, ref.h8], np.int32))
    for f in range(len(types)):
        out["intra%d" % f] = ref.get(f, 0)
        out["invq%d" % f] = ref.get(f, 8)
    for (p0, p1, b) in sorted(trip):
        ref.cost(p0, p1, b)
        d0, d1 = b - p0, p1 - b
        out["costs_%d_%d_%d" % (b, d0, d1)] = ref.get(b, 2, d0, d1, np.uint16)
        out["mvs_%d_0_%d" % (b, d0)] = ref.get(b, 4, 0, d0, n=2 * ref.ncu).reshape(-1, 2)
        if p1 > b:
            out["mvs_%d_1_%d" % (b, d1)] = ref.get(b, 4, 1, d1, n=2 * ref.ncu).reshape(-1, 2)
    np.savez_compressed(CLIP, **out)


_golden = {}


class CutreeRefResults:
    """`same(key, ref_fn, value)`: `value` equals the real cuTree's result (computed while oracle/_ref is built, else the
    digest stored in tests/golden/cutree_ref.json).  X265_WRITE_GOLDEN=1 with oracle/_ref built stores the digests."""

    def __init__(self, request, depth=8):
        self.R = load_ref_cutree(depth)
        self.depth = depth
        self.test = "%s::%s" % (request.node.module.__name__, request.node.name)
        self.write = self.R is not None and os.environ.get("X265_WRITE_GOLDEN") == "1"
        if not _golden:
            _golden.update(json.load(open(GOLDEN)) if os.path.exists(GOLDEN) else {})
        if self.write:
            _golden[self.test] = {}
            request.addfinalizer(_save_golden)
        elif self.test not in _golden:
            pytest.fail("no stored reference results for %s in %s" % (self.test, GOLDEN))
        self.digests = _golden[self.test]

    def same(self, key, ref_fn, value):
        if self.R is None:
            assert digest(value) == self.digests[key], "%s differs from the reference's stored result" % key
            return
        r = ref_fn()
        for k, (a, b) in enumerate(zip(r if isinstance(r, list) else [r], value if isinstance(value, list) else [value])):
            assert np.array_equal(np.asarray(a), np.asarray(b), equal_nan=np.asarray(a).dtype.kind == "f"), "%s, item %d" % (key, k)
        assert digest(r) == digest(value), key
        if self.write:
            self.digests[key] = digest(r)
        else:
            assert digest(r) == self.digests[key], "the reference's %s differs from %s" % (key, GOLDEN)


def _save_golden():
    with open(GOLDEN, "w") as f:
        json.dump(_golden, f, indent=0, sort_keys=True)
        f.write("\n")


def cases():
    """(name, w8, h8, types, params, kwargs of synth_window): the CPU pin's and the GPU test's synthetic windows."""
    out = []
    for bf in (0, 1, 3, 4, 8):
        for pyr in (0, 1):
            if bf < 2 and pyr:
                continue
            out.append(("bf%d_pyr%d" % (bf, pyr), 11, 7, slice_types(2 * (bf + 1) + 1 + (bf > 0), bf), params(bBPyramid=pyr), {}))
    out += [
        ("wbipred", 11, 7, slice_types(9, 3), params(bEnableWeightedBiPred=1), {}),
        ("wbipred_pyr_bf4", 12, 6, slice_types(11, 4), params(bEnableWeightedBiPred=1, bBPyramid=1), {}),
        ("intra", 9, 6, slice_types(9, 3), params(bIntra=1), {}),
        ("intra_p0", 9, 6, slice_types(9, 3, intra0=False), params(bIntra=1), {}),
        ("depth0", 9, 6, slice_types(9, 3), params(lookaheadDepth=0), {}),
        ("depth0_intra", 9, 6, slice_types(5, 3), params(lookaheadDepth=0, bIntra=1), {}),
        ("depth40_trailing_b", 10, 6, slice_types(11, 3), params(), {}),
        ("numframes0", 8, 5, [TYPE_I], params(), {}),
        ("numframes0_intra", 8, 5, [TYPE_I], params(bIntra=1), {}),
        ("numframes0_depth0_intra", 8, 5, [TYPE_I], params(bIntra=1, lookaheadDepth=0), {}),
        ("all_b", 8, 5, [TYPE_I] + [TYPE_B] * 4, params(), {}),
        ("vbv", 11, 7, slice_types(13, 3), params(vbv=1), {}),
        ("vbv_pyr_bf8", 11, 7, slice_types(19, 8), params(vbv=1, bBPyramid=1), {}),
        ("qg8", 10, 6, slice_types(9, 3), params(qgSize=8), {}),
        ("qg8_vbv", 10, 6, slice_types(9, 3), params(qgSize=8, vbv=1), {}),
        ("fps_short", 9, 6, slice_types(9, 3), params(fpsNum=240, fpsDenom=1), {}),
        ("fps_long", 9, 6, slice_types(9, 3), params(fpsNum=1, fpsDenom=3), {}),
        ("mv_edges", 9, 7, slice_types(9, 3), params(), dict(mv="edges")),
        ("mv_zero_frac", 9, 7, slice_types(9, 3), params(), dict(mv="zero_frac")),
        ("mv_zero", 9, 7, slice_types(9, 3), params(), dict(mv="zero")),
        ("saturate_one_cu", 12, 8, slice_types(9, 3), params(), dict(mv="one_cu")),
        ("int_min", 9, 6, slice_types(9, 3), params(), dict(amount="int_min")),
        ("overflow_wrap", 9, 6, slice_types(9, 3), params(bEnableWeightedBiPred=1), dict(amount="overflow")),
        ("overflow_pyr", 9, 6, slice_types(11, 4), params(bBPyramid=1), dict(amount="overflow")),
        ("tenbit_costs", 10, 6, slice_types(9, 3), params(), dict(depth=10)),
        ("tenbit_one_cu", 10, 6, slice_types(9, 3), params(), dict(depth=10, mv="one_cu")),
        ("one_cu_wide", 1, 5, slice_types(9, 3), params(), {}),
        ("one_row", 9, 1, slice_types(9, 3), params(), dict(mv="edges")),
    ]
    return out
