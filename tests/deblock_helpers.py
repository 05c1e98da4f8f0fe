"""Fixtures of the frame-level deblocking tests: random but legal per-4x4 decision maps (x265cu_deblock_unit records, raster
order) drawn per CTU as the encoder's final decisions could be, blocky or noisy picture content, and the oracle / reference
drivers over them.

A map holds a CU quadtree down to 8x8 (split where a CU crosses the right / bottom border, as CUData::calcCTUGeoms requires),
part sizes with AMP at CU >= 16 and NxN only for 8x8 intra CUs, a TU quadtree per CU with TUs of at most 32, intra / inter
mixes, per-TU luma cbf, per-CU QPs over the whole range (negative at 10 bit), reference picture ids and quarter-pel vectors
drawn from small pools so that equal vectors, |delta| = 3 and |delta| = 4 all occur, and rare transquant-bypass CUs.

The libraries are built by oracle/Makefile.deblock: liboracle_deblock{8,10}.so (the restatement) and, where the reference
sources are present, oracle/_ref/libx265ref_deblock{8,10}.so (the real Deblock).  The reference's results are stored in
tests/golden/deblock_ref.json for where oracle/_ref is not built."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

from common import ROOT, pixel_dtype, ptr
from ref_results import digest
from x265_b200.lib import DEBLOCK_UNIT, B_SLICE, P_SLICE, I_SLICE

GOLDEN = os.path.join(ROOT, "tests", "golden", "deblock_ref.json")
_libs = {}
_golden = {}


def load_oracle_deblock(depth):
    """The deblocking restatement (built on first use where build() has not built it)."""
    if ("orc", depth) not in _libs:
        path = os.path.join(ROOT, "oracle", "liboracle_deblock%d.so" % depth)
        if not os.path.exists(path):
            subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "-f", "Makefile.deblock", "oracle"],
                                  stdout=subprocess.DEVNULL)
        _libs[("orc", depth)] = C.CDLL(path)
    return _libs[("orc", depth)]


def load_ref_deblock(depth):
    """The real Deblock driver (x265ref_deblock_frame), or None where oracle/_ref is not built."""
    if ("ref", depth) not in _libs:
        path = os.path.join(ROOT, "oracle", "_ref", "libx265ref_deblock%d.so" % depth)
        _libs[("ref", depth)] = C.CDLL(path) if os.path.exists(path) else None
    return _libs[("ref", depth)]


class DeblockRefResults:
    """tests/ref_results.RefResults for the deblocking pin, with its own store: `same(key, ref_fn, value)` asserts that
    `value` equals the reference's result (computed while oracle/_ref is built, else the stored digest).
    X265_WRITE_GOLDEN=1 with oracle/_ref built stores the reference's digests instead of checking them."""

    def __init__(self, request, depth):
        self.R = load_ref_deblock(depth)
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


SIZE_2Nx2N, SIZE_2NxN, SIZE_Nx2N, SIZE_NxN, SIZE_2NxnU, SIZE_2NxnD, SIZE_nLx2N, SIZE_nRx2N = range(8)
MV_POOL = np.array([0, 3, 4, 7, 8, -4, -3, 1, 16, -16], np.int16)
# orc_deblock_frame's decision counters
COUNTERS = ["bs0", "bs1", "bs2", "beta_skip", "strong", "normal_both", "normal_one", "normal_neither", "chroma"]


def params_array(slice_type=B_SLICE, beta=0, tc=0, cb=0, cr=0, bypass=0):
    """x265cu_deblock_params as int32[6]"""
    return np.array([slice_type, beta, tc, cb, cr, bypass], np.int32)


def make_map(rng, width, height, ctu, depth, slice_type, mode="mixed", p_intra=0.25, p_bypass=0.0, split=None, num_refs=3):
    """(height / 4, width / 4) DEBLOCK_UNIT map.  mode (B slices): "mixed" (independent ids per list), "same" (bi units use the
    same picture in both lists), "swapped" (bi units use pictures 0 and 1 in either order)."""
    h4, w4 = height // 4, width // 4
    m = np.zeros((h4, w4), DEBLOCK_UNIT)
    split = split or {6: 0.7, 5: 0.55, 4: 0.45}
    qmin = -6 * (depth - 8)

    def draw_refs():
        if slice_type == P_SLICE:
            return (int(rng.integers(0, num_refs)), -1)
        d = int(rng.integers(0, 3))                   # 0: L0, 1: L1, 2: bi
        if d < 2:
            r = int(rng.integers(0, num_refs))
            return (r, -1) if d == 0 else (-1, r)
        if mode == "same":
            r = int(rng.integers(0, 2))
            return (r, r)
        if mode == "swapped":
            return (0, 1) if rng.random() < 0.5 else (1, 0)
        return (int(rng.integers(0, num_refs)), int(rng.integers(0, num_refs)))

    def draw_mv():
        return rng.choice(MV_POOL, 2)

    def fill_tu(x, y, log2t, d, min_d, max_d, cu):
        """TU quadtree leaf / split; x, y in units of 4"""
        if x * 4 >= width or y * 4 >= height:
            return
        if d < min_d or (d < max_d and log2t > 2 and rng.random() < 0.35):
            n = 1 << (log2t - 3)
            for qy in range(2):
                for qx in range(2):
                    fill_tu(x + qx * n, y + qy * n, log2t - 1, d + 1, min_d, max_d, cu)
            return
        n = max(1 << (log2t - 2), 1)
        sl = (slice(y, y + n), slice(x, x + n))
        m["tuDepth"][sl] = d
        if rng.random() < 0.5:
            m["flags"][sl] |= 2

    def fill_cu(x, y, log2):
        S = 1 << log2
        if x * 4 >= width or y * 4 >= height:
            return
        crosses = x * 4 + S > width or y * 4 + S > height
        if log2 > 3 and (crosses or rng.random() < split.get(log2, 0.0)):
            n = S // 8
            for qy in range(2):
                for qx in range(2):
                    fill_cu(x + qx * n, y + qy * n, log2 - 1)
            return
        n = S // 4
        sl = (slice(y, y + n), slice(x, x + n))
        intra = slice_type == I_SLICE or rng.random() < p_intra
        m["log2CuSize"][sl] = log2
        m["qp"][sl] = int(rng.integers(qmin, 52))
        m["flags"][sl] = (1 if intra else 0) | (4 if rng.random() < p_bypass else 0)
        if intra:
            ps = SIZE_NxN if log2 == 3 and rng.random() < 0.4 else SIZE_2Nx2N
            m["refPic"][sl] = -1
            m["mv"][sl] = 0
        else:
            choices = [SIZE_2Nx2N, SIZE_2NxN, SIZE_Nx2N] + ([SIZE_2NxnU, SIZE_2NxnD, SIZE_nLx2N, SIZE_nRx2N] if log2 >= 4 else [])
            ps = int(rng.choice(choices))
            # PU rectangles in units (x0, y0, w, h) relative to the CU
            q = n // 4
            pus = {SIZE_2Nx2N: [(0, 0, n, n)], SIZE_2NxN: [(0, 0, n, n // 2), (0, n // 2, n, n // 2)],
                   SIZE_Nx2N: [(0, 0, n // 2, n), (n // 2, 0, n // 2, n)],
                   SIZE_2NxnU: [(0, 0, n, q), (0, q, n, n - q)], SIZE_2NxnD: [(0, 0, n, n - q), (0, n - q, n, q)],
                   SIZE_nLx2N: [(0, 0, q, n), (q, 0, n - q, n)], SIZE_nRx2N: [(0, 0, n - q, n), (n - q, 0, q, n)]}[ps]
            for (px, py, pw, ph) in pus:
                psl = (slice(y + py, y + py + ph), slice(x + px, x + px + pw))
                r0, r1 = draw_refs()
                m["refPic"][psl] = (r0, r1)
                mv = np.zeros((2, 2), np.int16)
                for l, r in enumerate((r0, r1)):
                    if r >= 0:
                        mv[l] = draw_mv()
                    elif rng.random() < 0.5:
                        mv[l] = draw_mv()             # a stale vector in an unused list must not matter
                m["mv"][psl] = mv
        m["partSize"][sl] = ps
        min_d = 1 if log2 == 6 or ps == SIZE_NxN else 0
        max_d = min(log2 - 2, 3)
        fill_tu(x, y, log2, 0, min_d, max_d, None)

    ctu_log2 = ctu.bit_length() - 1
    for cy in range(0, height, ctu):
        for cx in range(0, width, ctu):
            fill_cu(cx // 4, cy // 4, ctu_log2)
    return np.ascontiguousarray(m)


def make_planes(rng, width, height, depth, content="blocky", chroma=True):
    """(luma, cb, cr) pictures (cb = cr = None without chroma).  "blocky": a smooth field plus per-8x8-block offsets of a few
    levels, so that the strong and the normal filters fire; "noise": uniform noise, mostly the d >= beta skip."""
    dt, mx = pixel_dtype(depth), (1 << depth) - 1

    def plane(w, h, blk):
        if content == "noise":
            return rng.integers(0, mx + 1, (h, w)).astype(dt)
        yy, xx = np.mgrid[0:h, 0:w]
        base = 128 + 50 * np.sin(xx / 41.0 + rng.random() * 6) + 35 * np.cos(yy / 29.0 + rng.random() * 6)
        offs = rng.integers(-5, 6, ((h + blk - 1) // blk, (w + blk - 1) // blk))
        offs = np.repeat(np.repeat(offs, blk, 0), blk, 1)[:h, :w]
        img = (base + offs) * (1 << (depth - 8)) + rng.integers(0, 1 << (depth - 8), (h, w))
        return np.clip(np.rint(img), 0, mx).astype(dt)

    luma = plane(width, height, 8)
    if not chroma:
        return luma, None, None
    return luma, plane(width // 2, height // 2, 4), plane(width // 2, height // 2, 4)


def oracle_deblock(depth, luma, cb, cr, units, prm, counters=None):
    """orc_deblock_frame on copies; returns (luma, cb, cr) and accumulates the decision counters into `counters` (int64[9])."""
    O = load_oracle_deblock(depth)
    y = luma.copy()
    u = cb.copy() if cb is not None else None
    v = cr.copy() if cr is not None else None
    cnt = np.zeros(len(COUNTERS), np.int64)
    rc = O.orc_deblock_frame(ptr(y), C.c_ssize_t(y.shape[1]), ptr(u) if u is not None else None, ptr(v) if v is not None else None,
                             C.c_ssize_t(u.shape[1] if u is not None else 0), y.shape[1], y.shape[0], ptr(units), ptr(prm), ptr(cnt))
    assert rc == 0
    if counters is not None:
        counters += cnt
    return y, u, v


def ref_deblock(depth, luma, cb, cr, units, prm, ctu):
    """x265ref_deblock_frame (the real Deblock over real CUData CTUs) on copies; None without oracle/_ref."""
    R = load_ref_deblock(depth)
    if R is None:
        return None
    y = luma.copy()
    u = cb.copy() if cb is not None else None
    v = cr.copy() if cr is not None else None
    rc = R.x265ref_deblock_frame(ptr(y), C.c_ssize_t(y.shape[1]), ptr(u) if u is not None else None, ptr(v) if v is not None else None,
                                 C.c_ssize_t(u.shape[1] if u is not None else 0), y.shape[1], y.shape[0], ctu, ptr(units), ptr(prm))
    assert rc == 0
    return y, u, v


# The cases of the oracle-vs-reference pin and of the device-vs-oracle test: (name, depth, width, height, ctu, slice, params
# kwargs, luma only, content, map kwargs)
def cases():
    out = []
    for depth in (8, 10):
        for st, sname in ((I_SLICE, "I"), (P_SLICE, "P"), (B_SLICE, "B")):
            out.append(("%s%d_200x136_ctu64" % (sname, depth), depth, 200, 136, 64, st, {}, False, "blocky", {}))
        out.append(("B%d_offs_lo" % depth, depth, 200, 136, 32, B_SLICE, dict(beta=-6, tc=-6, cb=-12, cr=12), False, "blocky", {}))
        out.append(("P%d_offs_hi" % depth, depth, 136, 104, 64, P_SLICE, dict(beta=6, tc=6, cb=12, cr=-12), False, "blocky", {}))
        out.append(("B%d_ctu32" % depth, depth, 200, 136, 32, B_SLICE, dict(beta=0, tc=2, cb=3, cr=-2), False, "blocky", {}))
        out.append(("B%d_64x64" % depth, depth, 64, 64, 64, B_SLICE, {}, False, "blocky", {}))
        out.append(("P%d_luma_only" % depth, depth, 200, 136, 64, P_SLICE, dict(beta=2, tc=-2), True, "blocky", {}))
        out.append(("B%d_noise" % depth, depth, 200, 136, 64, B_SLICE, {}, False, "noise", {}))
        out.append(("B%d_same_pic" % depth, depth, 200, 136, 64, B_SLICE, {}, False, "blocky", dict(mode="same", p_intra=0.05)))
        out.append(("B%d_swapped" % depth, depth, 200, 136, 32, B_SLICE, {}, False, "blocky", dict(mode="swapped", p_intra=0.05)))
        out.append(("B%d_tq_bypass" % depth, depth, 200, 136, 64, B_SLICE, dict(bypass=1), False, "blocky", dict(p_bypass=0.15)))
    return out


def case_inputs(case, seed=1234):
    """(luma, cb, cr, units, prm) of a case, deterministic."""
    name, depth, w, h, ctu, st, pk, luma_only, content, mk = case
    rng = np.random.default_rng([seed, sum(map(ord, name))])
    units = make_map(rng, w, h, ctu, depth, st, **mk)
    luma, cb, cr = make_planes(rng, w, h, depth, content, chroma=not luma_only)
    return luma, cb, cr, units, params_array(st, **pk)
