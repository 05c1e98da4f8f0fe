"""Helpers of the frame analyser's weighted P-slice references (x265cu_analyser_set_ref_weights): the CPU drivers with them
(oracle/frame_wref.h, built by oracle/Makefile.wref: liboracle_wref{8,10}.so over the oracle, oracle/_ref/libx265ref_wref{8,10}.so
over the reference), the ctypes view of their drv_wref, fading workloads, weight tables, a run of the CPU driver with weights,
and the store of the reference's results (tests/golden/wref_ref.json) for where oracle/_ref is not built."""
import copy
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

from common import ROOT, P, I, pixel_dtype
from chroma_helpers import DrvChroma, cpu_analyse_chroma
from frame_helpers import DrvFrame, Workload, lambda_for, MARGIN_X, MARGIN_Y
from me_helpers import mvcost_table
from ref_results import digest

_libs = {}
PLANE_ARGS = [P, P, P, C.c_ssize_t, C.c_ssize_t, I, I, I, I, I, P, P, P, P]


def load_oracle_wref(depth):
    """The oracle with weighted references (built on first use where build() has not built it)."""
    if ("orc", depth) not in _libs:
        path = os.path.join(ROOT, "oracle", "liboracle_wref%d.so" % depth)
        if not os.path.exists(path):
            subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "-f", "Makefile.wref", "oracle"],
                                  stdout=subprocess.DEVNULL)
        L = C.CDLL(path)
        L.orc_wref_planes.argtypes = PLANE_ARGS
        _libs[("orc", depth)] = L
    return _libs[("orc", depth)]


def load_ref_wref(depth):
    """The reference-from-source library with weighted references, or None where oracle/_ref is not built."""
    if ("ref", depth) not in _libs:
        path = os.path.join(ROOT, "oracle", "_ref", "libx265ref_wref%d.so" % depth)
        L = None
        if os.path.exists(path):
            L = C.CDLL(path)
            L.x265ref_wref_planes.argtypes = PLANE_ARGS
        _libs[("ref", depth)] = L
    return _libs[("ref", depth)]


GOLDEN = os.path.join(ROOT, "tests", "golden", "wref_ref.json")
_golden = {}


class WrefRefResults:
    """tests/ref_results.RefResults for the weighted references, with its own store: `same(key, ref_fn, value)` asserts that
    `value` equals the reference's result (computed while oracle/_ref is built, else the stored digest).  X265_WRITE_GOLDEN=1
    with oracle/_ref built stores the reference's digests instead of checking them."""

    def __init__(self, request, depth):
        self.R = load_ref_wref(depth)
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


class DrvWref(C.Structure):
    _fields_ = [("wp", ((I * 4) * 3) * 16), ("refs", P * 16), ("refC", (P * 2) * 16)]


# ---- weight tables: [numRefs][3][4] int32 rows {wtPresent, inputWeight, log2WeightDenom, inputOffset} ----
def entry(w0, denom, offset, present=1):
    return [present, w0, denom, offset]


def identity(denom=6):
    """The entry of an unweighted plane in a weighted slice: w = 1 << denom, offset 0, wtPresent 0."""
    return entry(1 << denom, denom, 0, 0)


def table(rows):
    """rows: per reference None (unweighted) or three entries.  Returns the [numRefs][3][4] int32 table."""
    t = np.zeros((len(rows), 3, 4), np.int32)
    for r, row in enumerate(rows):
        if row is not None:
            t[r] = row
    return t


# the reference mixes of the tests: weighted (luma and chroma), luma-only weighted (chroma entries not present, one of them
# not the identity: the residual still applies it), unweighted with chroma entries present (the whole reference unweighted)
MIXES = {
    "one": lambda d: [[entry(46, 5, 14), entry(60, 6, 9), entry(70, 6, -11)]],
    "two": lambda d: [[entry(46, 5, 14), entry(60, 6, 9), entry(70, 6, -11)], None],
    "three": lambda d: [[entry(40, 5, 20), entry(33, 5, 2), entry(31, 5, -3)],
                        [entry(75, 6, 10), identity(6), entry(50, 6, 7, 0)],
                        [entry(64, 6, 0, 0), entry(70, 6, 5), entry(60, 6, -5)]],
}


def fade_workload(W, H, depth, numRefs, noise=False, subme=3, method=3, qp=30, seed=265, merange=57, gains=(0.62, 0.7, 0.78)):
    """A Workload whose references are the clip's frames darkened towards black (a fade in): reference r is the frame scaled by
    gains[r] plus a small lift, luma and chroma (chroma towards 128), so the source is brighter than every reference."""
    wl = Workload(W, H, depth=depth, numRefs=numRefs, method=method, subme=subme, merange=merange, rect=1, qp=qp, noise=noise,
                  seed=seed, chroma=True)
    maxv = (1 << depth) - 1
    s = 1 << (depth - 8)
    for r in range(numRefs):
        g = gains[r % len(gains)]
        wl.refs[r] = np.clip(np.rint(wl.refs[r] * g + 6 * s), 0, maxv).astype(pixel_dtype(depth))
        wl.refC[r] = [np.clip(np.rint((c.astype(np.float64) - 128 * s) * g + 128 * s + 3 * s), 0, maxv).astype(pixel_dtype(depth))
                      for c in wl.refC[r]]
    return wl


def search_planes(lib, fn, wl, tab):
    """Per reference the planes the search reads (lib's fn: orc_wref_planes / x265ref_wref_planes): ([luma], [[Cb, Cr]], weighted
    flags), in the workload's padded layouts."""
    p, es = wl.params, np.dtype(pixel_dtype(wl.depth)).itemsize
    ys, cs, flags = [], [], []
    for r in range(p["numRefs"]):
        oy = np.zeros_like(wl.refs[r])
        oc = [np.zeros_like(wl.refC[r][k]) for k in range(2)]
        row = np.ascontiguousarray(tab[r], np.int32)
        flags.append(getattr(lib, fn)(wl.refs[r].ctypes.data + wl.org * es, wl.refC[r][0].ctypes.data + wl.corg * es,
                                      wl.refC[r][1].ctypes.data + wl.corg * es, wl.stride, wl.cstride, wl.W, wl.H, p["method"],
                                      p["subme"], p["merange"], row.ctypes.data, oy.ctypes.data + wl.org * es,
                                      oc[0].ctypes.data + wl.corg * es, oc[1].ctypes.data + wl.corg * es))
        ys.append(oy)
        cs.append(oc)
    return ys, cs, flags


def plane_area(wl, plane, chroma=False):
    """The rows and columns of a padded plane that the margins and the picture cover (what applyWeight defines)."""
    if chroma:
        mx, my = MARGIN_X // 2, MARGIN_Y // 2
        return plane[:wl.H // 2 + 2 * my, :wl.W // 2 + 2 * mx]
    return plane[:wl.H + 2 * MARGIN_Y, :wl.W + 2 * MARGIN_X]


class _WrefFn:
    """A driver entry point with the weights as fourth argument, called as chroma_helpers calls the chroma one."""

    def __init__(self, fn, w):
        self.fn, self.w = fn, w
        fn.argtypes = [C.POINTER(DrvFrame), I, C.POINTER(DrvChroma), C.POINTER(DrvWref)]
        fn.restype = I

    def __call__(self, frame, stages, cr):
        return self.fn(frame, stages, cr, C.byref(self.w))


class _Lib:
    def __init__(self, name, entry):
        setattr(self, name, entry)


def cpu_analyse_wref(lib, prefix, wl, tab, offsets=(0, 0), threads=4, stages=15, max_ctu_rows=0, planes=None):
    """The CPU driver with weighted references (prefix "orc": the oracle, "x265ref": the reference): the search planes of
    every reference from the library's plane build (or `planes`, search_planes' result), the frame through
    <prefix>_analyse_frame_wref.  Returns cpu_analyse_chroma's result plus "planes"."""
    fn = "orc_analyse_frame_wref" if prefix == "orc" else "x265ref_analyse_frame_wref"
    if planes is None:
        planes = search_planes(lib, "orc_wref_planes" if prefix == "orc" else "x265ref_wref_planes", wl, tab)
    es = np.dtype(pixel_dtype(wl.depth)).itemsize
    w = DrvWref()
    for r in range(wl.params["numRefs"]):
        for k in range(3):
            for j in range(4):
                w.wp[r][k][j] = int(tab[r][k][j])
        w.refs[r] = wl.refs[r].ctypes.data + wl.org * es
        for k in range(2):
            w.refC[r][k] = wl.refC[r][k].ctypes.data + wl.corg * es
    sw = copy.copy(wl)
    sw.refs, sw.refC = planes[0], planes[1]
    res = cpu_analyse_chroma(_Lib(fn, _WrefFn(getattr(lib, fn), w)), fn, sw, mvcost_tab_for(wl), offsets=offsets,
                             threads=threads, stages=stages, max_ctu_rows=max_ctu_rows)
    res["planes"] = planes
    return res


def mvcost_tab_for(wl):
    """The mvcost table of the workload's QP (the one the analyser builds from lambda_for)."""
    from common import load_oracle
    return mvcost_table(load_oracle(wl.depth), lambda_for(wl.params["qp"], wl.depth))
