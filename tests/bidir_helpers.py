"""Helpers of the frame analyser's B slices (x265cu_analyser_set_lists, stage bit 4): the CPU drivers with them
(oracle/frame_bidir.h, built by oracle/Makefile.bidir: liboracle_bidir{8,10}.so over the oracle, oracle/_ref/libx265ref_bidir{8,10}.so
over the reference), the ctypes view of their drv_bidir, B-frame workloads, a run of the CPU driver with a B slice, and the store
of the reference's results (tests/golden/bidir_ref.json) for where oracle/_ref is not built."""
import copy
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

from common import ROOT, P, I, pixel_dtype
from chroma_helpers import DrvChroma
from frame_helpers import DrvFrame, Workload, cpu_analyse, gen_luma, gen_chroma, pad_plane, pad_plane_c, MARGIN_X, MARGIN_Y
from ref_results import digest
from wref_helpers import mvcost_tab_for

_libs = {}
# decision counters of drv_bidir (frame_bidir.h)
COUNTERS = ("bi", "uni_l0", "uni_l1", "tie_l0", "zero_tried", "zero_taken", "zero_out_of_range", "zero_skipped")


def load_oracle_bidir(depth):
    """The oracle with B slices (built on first use where build() has not built it)."""
    if ("orc", depth) not in _libs:
        path = os.path.join(ROOT, "oracle", "liboracle_bidir%d.so" % depth)
        if not os.path.exists(path):
            subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "-f", "Makefile.bidir", "oracle"],
                                  stdout=subprocess.DEVNULL)
        _libs[("orc", depth)] = C.CDLL(path)
    return _libs[("orc", depth)]


def load_ref_bidir(depth):
    """The reference-from-source library with B slices, or None where oracle/_ref is not built."""
    if ("ref", depth) not in _libs:
        path = os.path.join(ROOT, "oracle", "_ref", "libx265ref_bidir%d.so" % depth)
        _libs[("ref", depth)] = C.CDLL(path) if os.path.exists(path) else None
    return _libs[("ref", depth)]


GOLDEN = os.path.join(ROOT, "tests", "golden", "bidir_ref.json")
_golden = {}


class BidirRefResults:
    """tests/ref_results.RefResults for the B slices, with its own store: `same(key, ref_fn, value)` asserts that `value`
    equals the reference's result (computed while oracle/_ref is built, else the stored digest).  X265_WRITE_GOLDEN=1 with
    oracle/_ref built stores the reference's digests instead of checking them."""

    def __init__(self, request, depth):
        self.R = load_ref_bidir(depth)
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
        assert digest(r) == digest(value), key
        if self.write:
            self.digests[key] = digest(r)
        else:
            assert digest(r) == self.digests[key], "the reference's %s differs from %s" % (key, GOLDEN)


def _save_golden():
    with open(GOLDEN, "w") as f:
        json.dump(_golden, f, indent=0, sort_keys=True)
        f.write("\n")


class DrvBidir(C.Structure):
    _fields_ = [("numRefL0", I), ("out", P), ("counts", I * len(COUNTERS))]


class BidirCu(C.Structure):
    """x265cu_bidir_cu (include/x265_b200.h)."""
    _fields_ = [("uniCost", C.c_uint32), ("biCost", C.c_uint32), ("interDir", C.c_int8), ("ref", C.c_int8 * 2), ("zero", C.c_uint8),
                ("mv", (C.c_int16 * 2) * 2)]


# ---- B-frame workloads ----
KINDS = ("between", "cut", "tie", "static")


def _field(W, H, vecs, jitter, seed):
    """[len(vecs)][fh][fw][2] qpel field: slot r's MVP = vecs[r] plus uniform jitter in [-jitter, jitter]."""
    rng = np.random.default_rng(seed)
    fw, fh = (W + 15) // 16, (H + 15) // 16
    f = np.zeros((len(vecs), fh, fw, 2), np.int16)
    for r, v in enumerate(vecs):
        for c in range(2):
            f[r, :, :, c] = v[c] + rng.integers(-jitter, jitter + 1, (fh, fw))
    return f


def bidir_workload(W, H, depth, n0, n1, kind, qp=22, seed=265, motion=(3, -2)):
    """A B frame (source: frame k of the synthetic clip, which moves by `motion` px per frame) with list 0 in slots [0, n0) and
    list 1 in [n0, n0 + n1), 4:2:0 planes throughout.  kind:
      "between": list-0 slot i = frame k - 1 - i, list-1 slot i = frame k + 1 + i, MVPs the true displacements +- 2 qpel: the
                 two lists' predictions average the per-frame noise away, so bi-prediction wins in most CUs;
      "cut":     list 0 is another clip (a cut after the list-0 references), list 1 as in "between": list-1 uni wins;
      "tie":     n0 == n1 and list-1 slot i is list-0 slot i (a picture in both lists, as in low-delay B): every L0 / L1 cost
                 ties, so list 0 wins;
      "static":  every slot is the source itself (a static noisy picture); the MVPs are zero in the left third of the picture
                 (both searched vectors zero: the zero try is skipped) and far elsewhere (nonzero searched vectors: the zero
                 pair is tried and taken where both MVPs lie in the zero try's range, refused by the range test where not)."""
    assert kind in KINDS, kind
    n = n0 + n1
    wl = Workload(W, H, depth=depth, numRefs=n, method=3, subme=3, merange=57, rect=1, qp=qp, seed=seed, chroma=True,
                  content="noise" if kind == "static" else None)
    k = 8
    gen = dict(bits=depth, seed=seed, motion=motion, noise=kind == "static")

    def frame(i, g=gen):
        return (pad_plane(gen_luma(W, H, i, **g), depth)[0],
                [pad_plane_c(gen_chroma(W, H, i, pl, **g), depth, wl.stride)[0] for pl in (1, 2)])
    if kind == "static":
        cur = frame(k)
        wl.fenc, wl.fencC = cur[0], cur[1]
        wl.refs = [cur[0].copy() for _ in range(n)]
        wl.refC = [[c.copy() for c in cur[1]] for _ in range(n)]
        fw = (W + 15) // 16
        far = _field(W, H, [(4 * 120, -4 * 90)] * n, 200, seed + 1)
        far[:, :, :fw // 3, :] = 0
        wl.field = far
        return wl
    wl.fenc, wl.fencC = frame(k)
    d = [i + 1 for i in range(n0)] + [-(i + 1) for i in range(n1)]
    pics = [frame(k - di) for di in d]
    if kind == "cut":
        other = dict(gen, seed=seed + 77, motion=(-5, 4))
        pics[:n0] = [frame(k - di, other) for di in d[:n0]]
    if kind == "tie":
        assert n0 == n1
        pics[n0:] = [(p[0].copy(), [c.copy() for c in p[1]]) for p in pics[:n0]]
        d[n0:] = d[:n0]
    wl.refs = [p[0] for p in pics]
    wl.refC = [p[1] for p in pics]
    wl.field = _field(W, H, [(4 * motion[0] * di, 4 * motion[1] * di) for di in d], 2, seed + 1)
    if kind == "tie":
        wl.field[n0:] = wl.field[:n0]
    return wl


def stages_for(chroma):
    """ME, luma residual, intra, BIDIR, and the chroma residual when chroma is on."""
    return 1 | 2 | 4 | 16 | (8 if chroma else 0)


class _BidirEntry:
    """Stands in for a driver entry point in frame_helpers.cpu_analyse: calls the B-slice one with `cr` and `b`."""

    def __init__(self, fn, cr, b):
        self.fn, self.cr, self.b = fn, cr, b
        fn.argtypes = [C.POINTER(DrvFrame), I, C.POINTER(DrvChroma), C.POINTER(DrvBidir)]
        fn.restype = I

    def __call__(self, frame, stages):
        assert self.fn(frame, stages, C.byref(self.cr), C.byref(self.b)) == 0


class _Lib:
    def __init__(self, name, entry):
        setattr(self, name, entry)


def cpu_analyse_bidir(lib, prefix, wl, n0, chroma, threads=4, max_ctu_rows=0):
    """The CPU driver with a B slice (prefix "orc": the oracle, "x265ref": the reference), list 0 = slots [0, n0), chroma
    planes in the ME, BIDIR and the chroma residual iff `chroma`.  Returns frame_helpers.cpu_analyse's result plus bidir
    (BIDIR_CU records), counts (COUNTERS) and, with chroma, chroma_helpers.cpu_analyse_chroma's chroma outputs."""
    from x265_b200.lib import BIDIR_CU
    fn_name = "%s_analyse_frame_bidir" % prefix
    W, H = wl.W, wl.H
    ctus = ((W + 63) // 64) * ((H + 63) // 64)
    maxcu = ctus * 85
    es = np.dtype(pixel_dtype(wl.depth)).itemsize
    out = dict(coef_c=[np.zeros(ctus * 4096, np.int16) for _ in range(2)],
               recon_c=[[np.zeros_like(wl.fencC[0]) for _ in range(2)] for _ in range(4)],
               cu_sse_c=np.zeros((maxcu, 2), np.uint64), cu_numsig_c=np.zeros((maxcu, 2), np.uint32),
               bidir=np.zeros(maxcu, BIDIR_CU))
    cr = DrvChroma()
    for k in range(2):
        cr.coef[k] = out["coef_c"][k].ctypes.data
        for d in range(4):
            cr.recon[d][k] = out["recon_c"][d][k].ctypes.data + wl.corg * es
    cr.cu_sse = out["cu_sse_c"].ctypes.data
    cr.cu_numsig = out["cu_numsig_c"].ctypes.data
    b = DrvBidir()
    b.numRefL0, b.out = n0, out["bidir"].ctypes.data
    sw = copy.copy(wl)
    sw.chroma = chroma
    res = cpu_analyse(_Lib(fn_name, _BidirEntry(getattr(lib, fn_name), cr, b)), fn_name, sw, mvcost_tab_for(wl), threads=threads,
                      stages=stages_for(chroma), max_ctu_rows=max_ctu_rows)
    nc = res["ncu"]
    res.update(bidir=out["bidir"][:nc], counts=dict(zip(COUNTERS, list(b.counts))))
    if chroma:
        n4 = res["ncoef"] // 4
        res.update(qpc=(cr.qpc[0], cr.qpc[1]), coef_c=[c[:n4] for c in out["coef_c"]], recon_c=out["recon_c"],
                   cu_sse_c=out["cu_sse_c"][:nc], cu_numsig_c=out["cu_numsig_c"][:nc])
    return res


def summary(res, wl, chroma):
    """Every output of the B-slice driver: the BIDIR records, ME results, reference choice, luma levels / SSE / numSig /
    recon per CU and, with chroma, the chroma ones (recon planes: their picture areas)."""
    from chroma_helpers import chroma_inner
    inner = lambda p: p[MARGIN_Y:MARGIN_Y + wl.H, MARGIN_X:MARGIN_X + wl.W]
    s = dict(bidir=np.frombuffer(res["bidir"].tobytes(), np.uint8), me=res["me_out"][:, :3], cu_ref=res["cu_ref"], coef=res["coef"], sse=res["cu_sse"],
             ns=res["cu_numsig"], recon=[inner(res["recon"][d]) for d in range(4)])
    if chroma:
        s.update(coef_c=res["coef_c"], sse_c=res["cu_sse_c"], ns_c=res["cu_numsig_c"],
                 recon_c=[chroma_inner(wl, res["recon_c"][d][k]) for d in range(4) for k in range(2)])
    return s


# (depth, (n0, n1), chroma, (W, H), qp, kind): "between" over every depth x lists x chroma, the sizes and QPs alternating;
# the other contents at both depths, both sizes and both QPs
SIZES = ((200, 136), (320, 256))
LISTS = ((1, 1), (2, 2), (1, 3))
CASES = ([(d, l, ch, SIZES[i % 2], (22, 37)[(i // 2) % 2], "between")
          for i, (d, l, ch) in enumerate((d, l, ch) for d in (8, 10) for l in LISTS for ch in (False, True))] +
         [(8, (1, 1), True, SIZES[0], 22, "cut"), (10, (1, 3), False, SIZES[1], 37, "cut"),
          (8, (2, 2), True, SIZES[0], 37, "tie"), (10, (1, 1), False, SIZES[0], 22, "tie"),
          (8, (1, 1), True, SIZES[0], 22, "static"), (10, (2, 2), True, SIZES[1], 37, "static"),
          (8, (1, 3), False, SIZES[1], 22, "static")])


def case_id(c):
    d, (n0, n1), ch, (W, H), qp, kind = c
    return "%s-%d-%d+%d-%s-%dx%d-qp%d" % (kind, d, n0, n1, "chroma" if ch else "luma", W, H, qp)
