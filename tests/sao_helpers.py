"""Fixtures of the frame-level SAO tests: per-CTU parameter records (SAO_CTU, [3][numCtus], raster order) as the encoder's
final decisions could leave them, reconstructed and source pictures, and the oracle / reference drivers over them.

Pictures: a smooth field with noise, plus a flat area and areas at 0 and at the maximum (so that offsets clip); the source
is the reconstruction plus small noise, with one full-range area.  Records: every type on every plane, band positions with
the wrap at 28-31, offsets up to +-(OFFSET_THRESH - 1), Cr of the same type as Cb (as x265's decision leaves them) unless a
case asks otherwise, merged CTUs holding the copied parameters of their left / upper neighbour.

The libraries are built by oracle/Makefile.sao: liboracle_sao{8,10}.so (the restatement) and, where the reference sources
are present, oracle/_ref/libx265ref_sao{8,10}.so (the real SAO / Deblock / ParallelFilter).  The reference's results are
stored in tests/golden/sao_ref.json for where oracle/_ref is not built."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

import deblock_helpers as D
from common import ROOT, pixel_dtype, ptr
from ref_results import digest
from x265_b200.lib import SAO_CTU, B_SLICE

GOLDEN = os.path.join(ROOT, "tests", "golden", "sao_ref.json")
STATS_SHAPE = (2, 3, 5, 32)          # per CTU: [count, offsetOrg][plane][SaoType][class] = two SAO::PerPlane
MERGE_NONE, MERGE_LEFT, MERGE_UP = 0, 1, 2
# the decision counters of orc_sao_stats_frame / orc_sao_apply_frame
COUNTERS = ["stats_right", "stats_bottom", "stats_inner", "stats_top", "stats_left", "apply_off", "apply_eo0", "apply_eo1",
            "apply_eo2", "apply_eo3", "apply_bo", "band_wrap", "clip_lo", "clip_hi", "cr_cb_type", "cr_skipped", "bypass"]
_libs = {}
_golden = {}


def load_oracle_sao(depth):
    if ("orc", depth) not in _libs:
        path = os.path.join(ROOT, "oracle", "liboracle_sao%d.so" % depth)
        if not os.path.exists(path):
            subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "-f", "Makefile.sao", "oracle"],
                                  stdout=subprocess.DEVNULL)
        _libs[("orc", depth)] = C.CDLL(path)
    return _libs[("orc", depth)]


def load_ref_sao(depth):
    """The real SAO driver, or None where oracle/_ref is not built."""
    if ("ref", depth) not in _libs:
        path = os.path.join(ROOT, "oracle", "_ref", "libx265ref_sao%d.so" % depth)
        _libs[("ref", depth)] = C.CDLL(path) if os.path.exists(path) else None
    return _libs[("ref", depth)]


class SaoRefResults:
    """`same(key, ref_fn, value)` asserts that `value` equals the reference's result (computed while oracle/_ref is built,
    else the digest stored in tests/golden/sao_ref.json).  X265_WRITE_GOLDEN=1 with oracle/_ref built stores the digests."""

    def __init__(self, request, depth):
        self.R = load_ref_sao(depth)
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


def num_ctus(W, H, ctu):
    return ((W + ctu - 1) // ctu) * ((H + ctu - 1) // ctu)


def offset_thresh(depth):
    return 1 << min(depth - 5, 5)


def make_pictures(rng, W, H, depth, chroma=True, noise=3):
    """(rec, fenc): lists of 3 planes (None for absent chroma).  rec: a smooth field with noise, a flat area and areas at 0
    and at the maximum; fenc: rec plus noise of +-noise levels (scaled to the bit depth), with one full-range area."""
    dt, mx, sc = pixel_dtype(depth), (1 << depth) - 1, 1 << (depth - 8)

    def plane(w, h):
        yy, xx = np.mgrid[0:h, 0:w]
        base = 128 + 70 * np.sin(xx / 13.0 + rng.random() * 6) * np.cos(yy / 11.0 + rng.random() * 6)
        img = base * sc + rng.integers(-6 * sc, 6 * sc + 1, (h, w))
        r = np.clip(np.rint(img), 0, mx).astype(np.int64)
        fx, fy = int(rng.integers(0, max(w - w // 4, 1))), int(rng.integers(0, max(h - h // 4, 1)))
        r[fy:fy + h // 4, fx:fx + w // 4] = int(rng.integers(0, mx + 1))          # flat
        r[:h // 6, w - w // 5:] = 0                                               # clips low
        r[h - h // 6:, :w // 5] = mx                                              # clips high
        r[h // 3:h // 3 + h // 8, w // 3:w // 3 + w // 8] = rng.integers(0, mx + 1, (h // 8, w // 8))   # full range
        f = np.clip(r + rng.integers(-noise * sc, noise * sc + 1, (h, w)), 0, mx)
        f[h - h // 5:, w - w // 5:] = rng.integers(0, mx + 1, (h // 5, w // 5))  # a full-range source area
        return r.astype(dt), f.astype(dt)

    pl = [plane(W, H)] + ([plane(W // 2, H // 2), plane(W // 2, H // 2)] if chroma else [])
    rec = [p[0] for p in pl] + [None] * (3 - len(pl))
    fenc = [p[1] for p in pl] + [None] * (3 - len(pl))
    return rec, fenc


def make_params(rng, W, H, ctu, depth, p_off=0.15, p_merge=0.2, cr_mode="same", band_hi=0.4, types=None):
    """(params [3][n] SAO_CTU, merge [3][n] uint8).  cr_mode: "same" (Cr has Cb's type), "eo_mix" (Cr another edge type
    than Cb where both are EO), "cb_off" (Cb off, Cr on, in some CTUs)."""
    cols, rows = (W + ctu - 1) // ctu, (H + ctu - 1) // ctu
    n = cols * rows
    t = offset_thresh(depth) - 1
    prm = np.zeros((3, n), SAO_CTU)
    merge = np.zeros((3, n), np.uint8)
    for a in range(n):
        c, r = a % cols, a // cols
        if (c or r) and rng.random() < p_merge:
            m = MERGE_LEFT if c and (not r or rng.random() < 0.5) else MERGE_UP
            src = a - 1 if m == MERGE_LEFT else a - cols
            prm[:, a] = prm[:, src]
            merge[:, a] = m
            continue
        for p in range(3):
            if p == 2 and cr_mode == "same":
                ty = int(prm[1, a]["typeIdx"])
            elif p == 2 and cr_mode == "eo_mix" and 0 <= prm[1, a]["typeIdx"] < 4:
                ty = int(rng.integers(0, 4))
            elif p == 2 and cr_mode == "cb_off":
                ty = int(prm[1, a]["typeIdx"])
                if rng.random() < 0.5:
                    prm[1, a]["typeIdx"] = -1
                    ty = int(rng.integers(0, 5))
            else:
                ty = -1 if rng.random() < p_off else int(rng.choice(types) if types is not None else rng.integers(0, 5))
            rec = prm[p, a]
            rec["typeIdx"] = ty
            rec["bandPos"] = int(rng.integers(28, 32)) if rng.random() < band_hi else int(rng.integers(0, 32))
            if ty == 4:
                off = rng.integers(-t, t + 1, 4)
            else:                          # the signs x265's EO decision gives: classes 1, 2 >= 0, classes 3, 4 <= 0
                off = np.concatenate([rng.integers(0, t + 1, 2), rng.integers(-t, 1, 2)])
            ext = rng.random(4) < 0.3
            off[ext] = np.where(off[ext] >= 0, t, -t) if ty == 4 else np.array([t, t, -t, -t])[ext]
            rec["offset"] = off
    return prm, merge


def planes_args(planes):
    """(ptr y, ptr cb, ptr cr, stride, cstride) of a plane list"""
    y, u, v = planes
    return (ptr(y), ptr(u) if u is not None else None, ptr(v) if v is not None else None,
            C.c_ssize_t(y.shape[1]), C.c_ssize_t(u.shape[1] if u is not None else 0))


def _copies(planes):
    return [p.copy() if p is not None else None for p in planes]


def oracle_stats(depth, rec, fenc, ctu, counters=None):
    O = load_oracle_sao(depth)
    H, W = rec[0].shape
    out = np.full((num_ctus(W, H, ctu),) + STATS_SHAPE, 0x5A5A5A5A, np.int32)
    cnt = np.zeros(len(COUNTERS), np.int64)
    assert O.orc_sao_stats_frame(*planes_args(fenc), *planes_args(rec), W, H, ctu, ptr(out), ptr(cnt)) == 0
    if counters is not None:
        counters += cnt
    return out


def oracle_apply(depth, rec, ctu, params, sao_luma=1, sao_chroma=1, units=None, fenc=None, counters=None):
    O = load_oracle_sao(depth)
    H, W = rec[0].shape
    out = _copies(rec)
    f = fenc if fenc is not None else [None] * 3
    fa = planes_args(f) if f[0] is not None else (None, None, None, C.c_ssize_t(0), C.c_ssize_t(0))
    cnt = np.zeros(len(COUNTERS), np.int64)
    assert O.orc_sao_apply_frame(*planes_args(out), W, H, ctu, ptr(params), sao_luma, sao_chroma,
                                 ptr(units) if units is not None else None, *fa, ptr(cnt)) == 0
    if counters is not None:
        counters += cnt
    return out


def ref_stats(depth, rec, fenc, ctu):
    R = load_ref_sao(depth)
    H, W = rec[0].shape
    out = np.full((num_ctus(W, H, ctu),) + STATS_SHAPE, 0x5A5A5A5A, np.int32)
    assert R.x265ref_sao_stats_frame(*planes_args(rec), *planes_args(fenc), W, H, ctu, ptr(out)) == 0
    return out


def ref_apply(depth, rec, ctu, params, merge, sao_luma=1, sao_chroma=1, units=None, fenc=None):
    R = load_ref_sao(depth)
    H, W = rec[0].shape
    out = _copies(rec)
    f = fenc if fenc is not None else [None] * 3
    fa = planes_args(f) if f[0] is not None else (None, None, None, C.c_ssize_t(0), C.c_ssize_t(0))
    assert R.x265ref_sao_apply_frame(*planes_args(out), W, H, ctu, ptr(params), ptr(merge), sao_luma, sao_chroma,
                                     ptr(units) if units is not None else None, *fa) == 0
    return out


def ref_frame(depth, rec, fenc, ctu, units, dprm, params, merge, sao_luma=1, sao_chroma=1):
    """deblocking, statistics and apply interleaved in FrameFilter's order: (planes, stats)"""
    R = load_ref_sao(depth)
    H, W = rec[0].shape
    out = _copies(rec)
    st = np.full((num_ctus(W, H, ctu),) + STATS_SHAPE, 0x5A5A5A5A, np.int32)
    assert R.x265ref_sao_frame(*planes_args(out), *planes_args(fenc), W, H, ctu, ptr(units), ptr(dprm), ptr(params), ptr(merge),
                               sao_luma, sao_chroma, ptr(st)) == 0
    return out, st


# The cases of the oracle-vs-reference pin and of the device-vs-oracle test:
# (name, depth, width, height, ctu, chroma, params kwargs, (saoLuma, saoChroma), bypass)
# Right-edge CTU widths: 200 -> 8 / 4 (chroma) samples, 208 -> 16 / 8, 224 -> 32 / 16, so that both apply paths of the
# reference (ctuWidth % 16, sao.cpp:327 ...) run on the right edge in both planes.
def cases():
    out = []
    for d in (8, 10):
        out += [
            ("d%d_ctu64_200x136" % d, d, 200, 136, 64, True, {}, (1, 1), False),
            ("d%d_ctu64_224x136" % d, d, 224, 136, 64, True, {}, (1, 1), False),
            ("d%d_ctu32_208x104" % d, d, 208, 104, 32, True, {}, (1, 1), False),
            ("d%d_ctu16_200x72" % d, d, 200, 72, 16, True, {}, (1, 1), False),
            ("d%d_ctu64_luma_only" % d, d, 200, 136, 64, False, {}, (1, 0), False),
            ("d%d_one_ctu_wide" % d, d, 48, 136, 64, True, {}, (1, 1), False),
            ("d%d_two_ctus_wide" % d, d, 120, 136, 64, True, {}, (1, 1), False),
            ("d%d_one_row" % d, d, 224, 40, 64, True, {}, (1, 1), False),
            ("d%d_one_ctu" % d, d, 64, 64, 64, True, {}, (1, 1), False),
            ("d%d_bo_wrap" % d, d, 200, 136, 32, True, dict(types=[4], band_hi=0.9, p_off=0.0), (1, 1), False),
            ("d%d_merge" % d, d, 200, 136, 32, True, dict(p_merge=0.6), (1, 1), False),
            ("d%d_luma_off" % d, d, 200, 136, 64, True, {}, (0, 1), False),
            ("d%d_chroma_off" % d, d, 200, 136, 64, True, {}, (1, 0), False),
            ("d%d_cr_eo_mix" % d, d, 200, 136, 32, True, dict(cr_mode="eo_mix", types=[0, 1, 2, 3]), (1, 1), False),
            ("d%d_cr_cb_off" % d, d, 200, 136, 32, True, dict(cr_mode="cb_off"), (1, 1), False),
            ("d%d_bypass" % d, d, 200, 136, 64, True, {}, (1, 1), True),
            ("d%d_bypass_luma_only" % d, d, 208, 104, 32, False, {}, (1, 0), True),
        ]
    return out


def case_inputs(case, seed=4321):
    """(rec, fenc, params, merge, units) of a case, deterministic; units: the bypass map (None without bypass)."""
    name, depth, W, H, ctu, chroma, pk, flags, bypass = case
    rng = np.random.default_rng([seed, sum(map(ord, name))])
    rec, fenc = make_pictures(rng, W, H, depth, chroma)
    params, merge = make_params(rng, W, H, ctu, depth, **pk)
    units = D.make_map(rng, W, H, ctu, depth, B_SLICE, p_bypass=0.2) if bypass else None
    return rec, fenc, params, merge, units
