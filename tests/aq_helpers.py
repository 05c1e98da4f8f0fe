"""Adaptive quantisation (calcAdaptiveQuantFrame, encoder/slicetype.cpp:444-694): pictures, the parameter matrix, the
plain-C restatement (oracle/oracle_aq.c), the REAL function on a real Frame (oracle/ref_shim_aq.cpp) and the stored results
of the latter (tests/golden/aq_ref.json) where oracle/_ref is not built."""
import ctypes as C
import itertools
import json
import os

import numpy as np
import pytest

from common import ROOT, P, I, pixel_dtype
from ref_results import digest

GOLDEN = os.path.join(ROOT, "tests", "golden", "aq_ref.json")


class AqParams(C.Structure):
    """x265cu_aq_params / the oracle's and the shim's parameter record"""
    _fields_ = [("aqMode", C.c_int32), ("qgSize", C.c_int32), ("weightp", C.c_int32), ("variance", C.c_int32),
                ("hevcAq", C.c_int32), ("hdr10Opt", C.c_int32), ("aqMotion", C.c_int32), ("reserved", C.c_int32),
                ("aqStrength", C.c_double), ("quantOffsets", P)]


_libs = {}


def load_oracle_aq():
    if "orc" not in _libs:
        p = os.path.join(ROOT, "oracle", "liboracle_aq.so")
        if not os.path.exists(p):
            import subprocess
            subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "-f", "Makefile.aq", "oracle"])
        L = C.CDLL(p)
        L.orc_aq_energy.restype = None
        L.orc_aq_energy.argtypes = [I, P, I, P, P, I, I, I, I, P, P]
        L.orc_aq.restype = None
        L.orc_aq.argtypes = [I, P, I, P, P, I, I, I, P, P, P, P, P, P, P, P]
        _libs["orc"] = L
    return _libs["orc"]


def load_ref_aq(depth):
    key = ("ref", depth)
    if key not in _libs:
        p = os.path.join(ROOT, "oracle", "_ref", "libx265ref_aq%d.so" % depth)
        if not os.path.exists(p):
            return None
        L = C.CDLL(p)
        L.x265ref_aq.restype = None
        L.x265ref_aq.argtypes = [P, P, P, I, I, P, P, P, P, P, P, P, P]
        _libs[key] = L
    return _libs[key]


def geometry(W, H, qg):
    """(energy grid blocks, blockCount, w8 * h8)"""
    L = 8 if qg == 8 else 16
    w8, h8 = ((W // 2) + 7) >> 3, ((H // 2) + 7) >> 3
    return ((W + L - 1) // L) * ((H + L - 1) // L), (4 if qg == 8 else 1) * w8 * h8, w8 * h8


def picture(W, H, depth, content, seed=0):
    """(y, cb, cr) contiguous planes: smooth | noise | black | white | fullrange (noise over the whole 10-bit range with
    flat and saturated patches)."""
    rng = np.random.default_rng([seed, W, H, depth, sum(map(ord, content))])
    mx = (1 << depth) - 1
    dt = pixel_dtype(depth)

    def plane(w, h, k):
        if content == "black":
            return np.zeros((h, w), dt)
        if content == "white":
            return np.full((h, w), mx, dt)
        if content == "smooth":
            yy, xx = np.mgrid[0:h, 0:w]
            img = 128 + 60 * np.sin(xx / (17.0 + k)) + 40 * np.cos(yy / (11.0 + k)) + rng.integers(-3, 4, (h, w))
            return (np.clip(img, 0, 255).astype(np.int64) << (depth - 8)).astype(dt)
        img = rng.integers(0, mx + 1, (h, w))
        if content == "fullrange":
            img[: h // 3, : w // 2] = mx
            img[h // 2:, w // 3: w // 2] = 0
        return img.astype(dt)
    return plane(W, H, 0), plane(W // 2, H // 2, 1), plane(W // 2, H // 2, 2)


def quant_offsets(count, seed=3):
    return np.random.default_rng(seed).uniform(-4, 4, count).astype(np.float32)


def param_matrix():
    """(aqMode, strength, qgSize, weightp, variance, quantOffsets): every combination the reference can run (aqMode 0 with
    qgSize 8 is not one: Lowres allocates no invQscaleFactor without AQ and the qgSize 8 reduction reads it)."""
    out = []
    for mode, s, qg, wp, var, qo in itertools.product((0, 1, 2, 3), (0.0, 0.4, 1.0, 3.0), (8, 32), (0, 1), (0, 1), (0, 1)):
        if mode == 0 and qg == 8:
            continue
        out.append((mode, s, qg, wp, var, qo))
    return out


def key(prm):
    return "m%d_s%g_qg%d_wp%d_var%d_qo%d" % prm


def c_params(prm, qo_arr):
    mode, s, qg, wp, var, qo = prm
    return AqParams(aqMode=mode, qgSize=qg, weightp=wp, variance=var, aqStrength=s,
                    quantOffsets=qo_arr.ctypes.data if qo else None)


def prefilled(count):
    """What the shim leaves in the Lowres arrays before the call: qpAqOffset, invQscaleFactor, blockVariance."""
    i = np.arange(count)
    return -1000.0 - i, (7 + 3 * i).astype(np.int32), (0x5a5a0000 + i).astype(np.uint32)


def ptr(a):
    return a.ctypes.data if a is not None else None


def oracle(pic, W, H, depth, prm):
    """The restatement on the pixels: dict of every output (arrays prefilled as the shim prefills the reference's)."""
    O = load_oracle_aq()
    y, cb, cr = pic
    _, count, n8 = geometry(W, H, prm[2])
    qo = quant_offsets(count)
    p = c_params(prm, qo)
    qp, iq, bv = prefilled(count)
    iq8 = np.zeros(n8, np.int32)
    wps, wpd, fv = np.zeros(3, np.uint64), np.zeros(3, np.uint64), np.zeros(1)
    O.orc_aq(depth, ptr(y), W, ptr(cb), ptr(cr), W // 2, W, H, C.byref(p), ptr(qp), ptr(iq), ptr(iq8), ptr(wps), ptr(wpd),
             ptr(bv), ptr(fv))
    return outputs(prm, qp, iq, iq8, wps, wpd, bv, fv[0])


def outputs(prm, qp, iq, iq8, wps, wpd, bv, fv):
    """The outputs the reference has for these parameters (Lowres allocates the AQ arrays only with aqMode, blockVariance
    only with variance)."""
    mode, s, qg, wp, var, qo = prm
    r = dict(wp_sum=np.asarray(wps, np.uint64), wp_ssd=np.asarray(wpd, np.uint64))
    if mode:
        r.update(qpAqOffset=qp, invQscaleFactor=iq)
        if qg == 8:
            r["invQscaleFactor8x8"] = iq8
    if var:
        r.update(blockVariance=bv, frameVariance=float(fv))
    return r


def oracle_energy(pic, W, H, depth, qg):
    O = load_oracle_aq()
    y, cb, cr = pic
    nb, _, _ = geometry(W, H, qg)
    e, t = np.zeros(nb, np.uint32), np.zeros(6, np.uint64)
    O.orc_aq_energy(depth, ptr(y), W, ptr(cb), ptr(cr), W // 2, W, H, qg, ptr(e), ptr(t))
    return e, t


def reference(pic, W, H, depth, prm):
    R = load_ref_aq(depth)
    y, cb, cr = pic
    _, count, n8 = geometry(W, H, prm[2])
    qo = quant_offsets(count)
    p = c_params(prm, qo)
    qp, iq, bv = prefilled(count)
    qc = qp.copy()
    iq8 = np.zeros(n8, np.int32)
    wp, fv = np.zeros(6, np.uint64), np.zeros(1)
    R.x265ref_aq(ptr(y), ptr(cb), ptr(cr), W, H, C.byref(p), ptr(qp), ptr(qc), ptr(iq), ptr(iq8), ptr(bv), ptr(wp), ptr(fv))
    if prm[0]:
        assert np.array_equal(qp.view(np.uint64), qc.view(np.uint64)), "qpCuTreeOffset differs from qpAqOffset"
    return outputs(prm, qp, iq, iq8, wp[:3], wp[3:], bv, fv[0])


def same_outputs(a, b):
    """Every output equal, doubles by bit pattern."""
    if sorted(a) != sorted(b):
        return False
    for k in a:
        x, y = np.asarray(a[k]), np.asarray(b[k])
        if x.dtype.kind == "f":
            x, y = x.view(np.uint64), y.view(np.uint64)
        if x.shape != y.shape or not np.array_equal(x, y):
            return False
    return True


def finish_refused(W, H, prm):
    """x265cu_aq_finish refuses variance with weightp when weightp's rounding changes the fades pass's grid."""
    mode, s, qg, wp, var, qo = prm
    if not (wp and var):
        return False
    L = 8 if qg == 8 else 16
    wpad, hpad = ((W + 8) >> 4) << 4, ((H + 8) >> 4) << 4
    return (wpad + L - 1) // L != (W + L - 1) // L or (hpad + L - 1) // L != (H + L - 1) // L


# (name, W, H, depth, 4:2:0, content): the pictures of the CPU pin and of the device pass's GPU test
PICTURES = [("1080p_8_420_smooth", 1920, 1080, 8, True, "smooth"), ("1080p_10_400_noise", 1920, 1080, 10, False, "noise")]
PICTURES += [("328x184_%d_%s_%s" % (d, "420" if c else "400", t), 328, 184, d, c, t)
             for d in (8, 10) for c in (True, False) for t in ("smooth", "noise", "black", "white")]
PICTURES += [("328x184_10_420_fullrange", 328, 184, 10, True, "fullrange"),
             ("64x64_8_420_noise", 64, 64, 8, True, "noise"), ("64x64_10_420_fullrange", 64, 64, 10, True, "fullrange"),
             ("64x64_8_400_white", 64, 64, 8, False, "white"), ("64x64_10_400_black", 64, 64, 10, False, "black")]


def make_picture(case):
    name, W, H, depth, c420, content = case
    y, cb, cr = picture(W, H, depth, content)
    return (y, cb, cr) if c420 else (y, None, None)


_golden = {}


class AqRefResults:
    """`same(key, ref_fn, value)`: `value` equals the real calcAdaptiveQuantFrame's result (computed while oracle/_ref is
    built, else the digest stored in tests/golden/aq_ref.json).  X265_WRITE_GOLDEN=1 with oracle/_ref built stores them."""

    def __init__(self, request, depth):
        self.R = load_ref_aq(depth)
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
        assert same_outputs(r, value), (key, {k: (r[k], value.get(k)) for k in r})
        assert digest(r) == digest(value), key
        if self.write:
            self.digests[key] = digest(r)
        else:
            assert digest(r) == self.digests[key], "the reference's %s differs from %s" % (key, GOLDEN)


def _save_golden():
    with open(GOLDEN, "w") as f:
        json.dump(_golden, f, indent=0, sort_keys=True)
        f.write("\n")
