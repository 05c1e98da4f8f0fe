"""Helpers of the 4:2:0 chroma residual stage (analyser stage bit 3): the CPU drivers with that stage (oracle/frame_chroma.h,
built by oracle/Makefile.chroma: liboracle_chroma{8,10}.so over the oracle, oracle/_ref/libx265ref_chroma{8,10}.so over the
reference), the ctypes view of their drv_chroma_resid, a run of the CPU driver with the stage, and the store of the
reference's results (tests/golden/chroma_residual_ref.json) for where oracle/_ref is not built."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

from common import ROOT, P, I, pixel_dtype
from frame_helpers import DrvFrame, cpu_analyse
from ref_results import digest

OFFSETS = (-12, 0, 12)
_libs = {}


def load_oracle_chroma(depth):
    """The oracle with the chroma residual stage (built on first use where build() has not built it)."""
    if ("orc", depth) not in _libs:
        path = os.path.join(ROOT, "oracle", "liboracle_chroma%d.so" % depth)
        if not os.path.exists(path):
            subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "-f", "Makefile.chroma", "oracle"],
                                  stdout=subprocess.DEVNULL)
        L = C.CDLL(path)
        L.orc_chroma_qp.argtypes = [I, I]
        _libs[("orc", depth)] = L
    return _libs[("orc", depth)]


def load_ref_chroma(depth):
    """The reference-from-source library with the chroma residual stage, or None where oracle/_ref is not built."""
    if ("ref", depth) not in _libs:
        path = os.path.join(ROOT, "oracle", "_ref", "libx265ref_chroma%d.so" % depth)
        L = None
        if os.path.exists(path):
            L = C.CDLL(path)
            L.x265ref_chroma_qp.argtypes = [I, I]
        _libs[("ref", depth)] = L
    return _libs[("ref", depth)]


GOLDEN = os.path.join(ROOT, "tests", "golden", "chroma_residual_ref.json")
_golden = {}


class ChromaRefResults:
    """tests/ref_results.RefResults for the chroma stage, with its own store: `same(key, ref_fn, value)` asserts that `value`
    equals the reference's result (computed while oracle/_ref is built, else the stored digest).  X265_WRITE_GOLDEN=1 with
    oracle/_ref built stores the reference's digests instead of checking them."""

    def __init__(self, request, depth):
        self.R = load_ref_chroma(depth)
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
        assert digest(r) == digest(value), (key, r, value)
        if self.write:
            self.digests[key] = digest(r)
        else:
            assert digest(r) == self.digests[key], "the reference's %s differs from %s" % (key, GOLDEN)


def _save_golden():
    with open(GOLDEN, "w") as f:
        json.dump(_golden, f, indent=0, sort_keys=True)
        f.write("\n")


class DrvChroma(C.Structure):
    _fields_ = [("offset", I * 2), ("qpc", I * 2), ("coef", P * 2), ("recon", (P * 2) * 4), ("cu_sse", P), ("cu_numsig", P)]


class _ChromaEntry:
    """Stands in for a driver entry point in frame_helpers.cpu_analyse: calls the chroma one with `cr` as third argument."""

    def __init__(self, fn, cr):
        self.fn, self.cr, self.argtypes = fn, cr, None
        fn.argtypes = [C.POINTER(DrvFrame), I, C.POINTER(DrvChroma)]
        fn.restype = I

    def __call__(self, frame, stages):
        assert self.fn(frame, stages, C.byref(self.cr)) == 0


class _Lib:
    def __init__(self, name, entry):
        setattr(self, name, entry)


def cpu_analyse_chroma(lib, fn_name, wl, mvcost_tab, offsets=(0, 0), threads=4, stages=15, max_ctu_rows=0):
    """frame_helpers.cpu_analyse through the chroma entry point (oracle: orc_analyse_frame_chroma, reference:
    x265ref_analyse_frame_chroma).  Adds to the result: qpc (the two quantiser QPs), coef_c [2][ncoef / 4],
    recon_c [4][2] (margin-extended chroma planes, wl.fencC geometry), cu_sse_c / cu_numsig_c [ncu][2]."""
    assert wl.chroma
    W, H = wl.W, wl.H
    ctus = ((W + 63) // 64) * ((H + 63) // 64)
    maxcu = ctus * 85
    es = np.dtype(pixel_dtype(wl.depth)).itemsize
    out = dict(coef_c=[np.zeros(ctus * 4096, np.int16) for _ in range(2)],
               recon_c=[[np.zeros_like(wl.fencC[0]) for _ in range(2)] for _ in range(4)],
               cu_sse_c=np.zeros((maxcu, 2), np.uint64), cu_numsig_c=np.zeros((maxcu, 2), np.uint32))
    cr = DrvChroma()
    cr.offset[0], cr.offset[1] = offsets
    for k in range(2):
        cr.coef[k] = out["coef_c"][k].ctypes.data
        for d in range(4):
            cr.recon[d][k] = out["recon_c"][d][k].ctypes.data + wl.corg * es
    cr.cu_sse = out["cu_sse_c"].ctypes.data
    cr.cu_numsig = out["cu_numsig_c"].ctypes.data
    res = cpu_analyse(_Lib(fn_name, _ChromaEntry(getattr(lib, fn_name), cr)), fn_name, wl, mvcost_tab, threads=threads,
                      stages=stages, max_ctu_rows=max_ctu_rows)
    nc, n4 = res["ncu"], res["ncoef"] // 4
    res.update(qpc=(cr.qpc[0], cr.qpc[1]), coef_c=[c[:n4] for c in out["coef_c"]], recon_c=out["recon_c"],
               cu_sse_c=out["cu_sse_c"][:nc], cu_numsig_c=out["cu_numsig_c"][:nc])
    return res


def chroma_inner(wl, plane):
    """The picture area of a margin-extended chroma plane of the workload's geometry."""
    my, mx = wl.corg // wl.cstride, wl.corg % wl.cstride
    return plane[my:my + wl.H // 2, mx:mx + wl.W // 2]
