"""GPU: x265cu_deblock_rows / x265cu_sao_stats_rows / x265cu_sao_apply_rows against the whole-picture calls on the same inputs
(themselves checked against the restatements here), byte-exact: every CPU case over the bands of several partitions, out of
place and in place on per-band copies, with noise outside the rows a call reads and a sentinel outside the rows it writes,
inside guard bands with odd strides and an unaligned base; 3840x2160 and 7680x4320; the row-by-row lag order on one plane;
emulated row shards on the frame analyser; and the refusals."""
import ctypes as C

import numpy as np
import pytest

import deblock_helpers as D
import sao_helpers as S
from common import pixel_dtype
from test_filter_rows_cpu import DEBLOCK_CASES, SAO_CASES, bands, noise_outside
from test_gpu_deblock import GuardedPlane, assert_planes_equal, device_deblock, dparams
from test_gpu_sao import decide, device_apply, device_stats
from x265_b200 import shard
from x265_b200.lib import B_SLICE, SAO_STATS_PER_CTU, DeblockParams

pytestmark = pytest.mark.gpu
GARBAGE = 0x5A


@pytest.fixture(scope="module")
def cu():
    import x265_b200
    return x265_b200.load()


def sentinel_like(img):
    return np.full(img.shape, 0xA5 if img.dtype == np.uint8 else 0xA5A5, img.dtype)


class Planes:
    """(y, cb, cr) GuardedPlanes (None for absent chroma); `odd`: strides that are not multiples of 16 bytes and a base one
    pixel past an aligned address."""

    def __init__(self, cu, imgs, odd=False):
        W = imgs[0].shape[1]
        self.stride, self.cstride = (W + 7, W // 2 + 5) if odd else (W, W // 2)
        sh = 1 if odd else 0
        self.g = [GuardedPlane(cu, imgs[0], self.stride, shift=sh)] + \
                 [GuardedPlane(cu, p, self.cstride, shift=sh) if p is not None else None for p in imgs[1:]]

    @property
    def ptrs(self):
        return tuple(g.ptr if g is not None else None for g in self.g)

    @property
    def cs(self):
        return self.cstride if self.g[1] is not None else 0

    def expect(self, rows, want):
        """the allocations as uploaded, with rows [a, b) of each picture replaced by `want`'s"""
        out = []
        for g, (a, b), w in zip(self.g, rows, want):
            if g is None:
                continue
            e = g.expect_outside.copy()
            for y in range(a, b):
                e[g.org + y * g.stride:g.org + y * g.stride + g.w] = w[y]
            out.append(e)
        return out

    def check(self, rows, want, what):
        for k, (g, e) in enumerate(zip([g for g in self.g if g is not None], self.expect(rows, want))):
            got = g.download()
            assert np.array_equal(got, e), (what, "plane %d" % k, int(np.count_nonzero(got != e)))

    def free(self):
        for g in self.g:
            if g is not None:
                g.free()


# ---- deblocking ----

@pytest.mark.parametrize("case", DEBLOCK_CASES, ids=[c[0] for c in DEBLOCK_CASES])
def test_deblock_rows_match_frame(cu, case):
    """Every band of several partitions, out of place (dst starts as a sentinel) and in place on a per-band copy: the
    write range holds the frame call's values and nothing else changes.  Outside the read range, src holds noise and the map
    holds CTU rows of a second legal map."""
    name, depth, W, H, ctu, st, pk, luma_only, content, mk = case
    luma, cb, cr, units, prm = D.case_inputs(case)
    frame = device_deblock(cu, depth, luma, cb, cr, units, prm)
    assert_planes_equal(frame, D.oracle_deblock(depth, luma, cb, cr, units, prm), name)
    rng = np.random.default_rng([5, sum(map(ord, name))])
    other = D.make_map(rng, W, H, ctu, depth, st, **mk)
    u, p = ctu // 4, dparams(prm)
    odd = sum(map(ord, name)) % 2 == 1
    for r0, r1 in bands((H + ctu - 1) // ctu):
        (y0, y1), (c0, c1) = shard.filter_halo(r0, r1, ctu, H)
        rows = [(y0, y1), (c0, c1), (c0, c1)]
        m = other.copy()
        m[max(0, (r0 - 1) * u):(r1 + 1) * u] = units[max(0, (r0 - 1) * u):(r1 + 1) * u]
        ubuf = cu.to_device(m)
        src = [noise_outside(rng, img, a, b, depth) if img is not None else None for img, (a, b) in zip((luma, cb, cr), rows)]
        Sp = Planes(cu, src, odd)
        Dp = Planes(cu, [sentinel_like(img) if img is not None else None for img in src], not odd)
        cu.deblock_rows(depth, W, H, ctu, r0, r1, Sp.ptrs, Sp.stride, Sp.cs, Dp.ptrs, Dp.stride, Dp.cs, ubuf, p)
        cu.sync()
        Dp.check(rows, frame, (name, r0, r1, "out of place"))
        Sp.check([(0, 0)] * 3, frame, (name, r0, r1, "src unchanged"))
        cu.deblock_rows(depth, W, H, ctu, r0, r1, Sp.ptrs, Sp.stride, Sp.cs, Sp.ptrs, Sp.stride, Sp.cs, ubuf, p)
        cu.sync()
        Sp.check(rows, frame, (name, r0, r1, "in place"))
        for b in (Sp, Dp, ubuf):
            b.free()


# ---- SAO ----

@pytest.mark.parametrize("case", SAO_CASES, ids=[c[0] for c in SAO_CASES])
def test_sao_stats_rows_match_frame(cu, case):
    name, depth, W, H, ctu = case[:5]
    rec, fenc, params, merge, units = S.case_inputs(case)
    frame = device_stats(cu, depth, rec, fenc, ctu)
    assert np.array_equal(frame, S.oracle_stats(depth, rec, fenc, ctu))
    rng = np.random.default_rng([6, sum(map(ord, name))])
    cols, n, per = (W + ctu - 1) // ctu, S.num_ctus(W, H, ctu), SAO_STATS_PER_CTU * 4
    for r0, r1 in bands((H + ctu - 1) // ctu):
        Y0, Y1 = r0 * ctu, min(H, r1 * ctu)
        lo = [(Y0, Y1)] + [(Y0 // 2, Y1 // 2)] * 2
        R = Planes(cu, [noise_outside(rng, q, a - 1, b, depth) if q is not None else None for q, (a, b) in zip(rec, lo)], True)
        F = Planes(cu, [noise_outside(rng, q, a, b, depth) if q is not None else None for q, (a, b) in zip(fenc, lo)])
        buf = cu.to_device(np.full(n * per, GARBAGE, np.uint8))
        cu.sao_stats_rows(depth, W, H, ctu, r0, r1, F.ptrs, F.stride, F.cs, R.ptrs, R.stride, R.cs, buf)
        cu.sync()
        raw = buf.download(np.uint8)
        got = raw.view(np.int32).reshape((n,) + S.STATS_SHAPE)
        assert np.array_equal(got[r0 * cols:r1 * cols], frame[r0 * cols:r1 * cols]), (name, r0, r1)
        assert (raw[:r0 * cols * per] == GARBAGE).all() and (raw[r1 * cols * per:] == GARBAGE).all(), (name, r0, r1, "other records")
        for b in (R, F, buf):
            b.free()


SAO_APPLY = [(c, None) for c in SAO_CASES] + [(c, (0, 0)) for c in S.cases() if c[0] in ("d8_bypass", "d10_ctu32_208x104")]


@pytest.mark.parametrize("case,flags", SAO_APPLY, ids=[c[0] + ("" if f is None else "_sao_off") for c, f in SAO_APPLY])
def test_sao_apply_rows_match_frame(cu, case, flags):
    """Band rows equal the in-place frame call; rows outside the band keep their sentinel; src is not written.  src holds
    noise outside rows [Y0 - 1, Y1 + 1), the source outside [Y0, Y1), and the records of other CTUs are another decision's.
    With flags (0, 0) SAO is off on every plane and the call still copies the band (restoring bypass units)."""
    name, depth, W, H, ctu = case[:5]
    sl, sc = case[7] if flags is None else flags
    rec, fenc, params, merge, units = S.case_inputs(case)
    frame = device_apply(cu, depth, rec, ctu, params, sl, sc, units, fenc)
    assert_planes_equal(frame, S.oracle_apply(depth, rec, ctu, params, sl, sc, units, fenc), name)
    rng = np.random.default_rng([7, sum(map(ord, name))])
    other, _ = S.make_params(rng, W, H, ctu, depth)
    cols = (W + ctu - 1) // ctu
    ubuf = cu.to_device(units) if units is not None else None
    odd = sum(map(ord, name)) % 2 == 1
    for r0, r1 in bands((H + ctu - 1) // ctu):
        Y0, Y1 = r0 * ctu, min(H, r1 * ctu)
        lo = [(Y0, Y1)] + [(Y0 // 2, Y1 // 2)] * 2
        src = [noise_outside(rng, q, a - 1, b + 1, depth) if q is not None else None for q, (a, b) in zip(rec, lo)]
        Sp = Planes(cu, src, odd)
        Dp = Planes(cu, [sentinel_like(q) if q is not None else None for q in src], not odd)
        F = Planes(cu, [noise_outside(rng, q, a, b, depth) if q is not None else None for q, (a, b) in zip(fenc, lo)])
        pp = other.copy()
        pp[:, r0 * cols:r1 * cols] = params[:, r0 * cols:r1 * cols]
        pbuf = cu.to_device(pp)
        fa = (F.ptrs, F.stride, F.cs) if units is not None else ((None, None, None), 0, 0)
        cu.sao_apply_rows(depth, W, H, ctu, r0, r1, Sp.ptrs, Sp.stride, Sp.cs, Dp.ptrs, Dp.stride, Dp.cs, pbuf, sl, sc, ubuf, *fa)
        cu.sync()
        Dp.check(lo, frame, (name, r0, r1))
        Sp.check([(0, 0)] * 3, frame, (name, r0, r1, "src unchanged"))
        assert pbuf.download(np.uint8).tobytes() == pp.tobytes()
        for b in (Sp, Dp, F, pbuf):
            b.free()
    if ubuf is not None:
        ubuf.free()


def test_sao_apply_rows_out_of_range_records(cu):
    """Any byte values in the records give, band by band, what the frame call gives for the same bytes."""
    depth, W, H, ctu = 8, 200, 136, 32
    rng = np.random.default_rng(78)
    rec, fenc = S.make_pictures(rng, W, H, depth)
    n = S.num_ctus(W, H, ctu)
    params = rng.integers(0, 256, (3, n, 8)).astype(np.uint8).view(S.SAO_CTU).reshape(3, n)
    frame = device_apply(cu, depth, rec, ctu, params, 1, 1, None, fenc)
    pbuf = cu.to_device(params)
    Sp = Planes(cu, rec)
    Dp = Planes(cu, [sentinel_like(q) for q in rec])
    for r0, r1 in shard.row_blocks(5, 0, 2) + shard.row_blocks(5, 1, 2):
        cu.sao_apply_rows(depth, W, H, ctu, r0, r1, Sp.ptrs, Sp.stride, Sp.cs, Dp.ptrs, Dp.stride, Dp.cs, pbuf, 1, 1)
    cu.sync()
    Dp.check([(0, H), (0, H // 2), (0, H // 2)], frame, "records")
    for b in (Sp, Dp, pbuf):
        b.free()


# ---- whole chains ----

class Chain:
    """One picture's inputs on the device: the pre-deblock picture, the source, the map and the deblocking parameters."""

    def __init__(self, cu, depth, W, H, ctu, rec, fenc, units, prm):
        self.cu, self.depth, self.W, self.H, self.ctu = cu, depth, W, H, ctu
        self.rec, self.fenc = rec, fenc
        self.R, self.F = Planes(cu, rec), Planes(cu, fenc)
        self.ubuf, self.p = cu.to_device(units), dparams(prm)
        self.rows = (H + ctu - 1) // ctu
        self.n = S.num_ctus(W, H, ctu)

    def scratch(self):
        return Planes(self.cu, [sentinel_like(q) for q in self.rec])

    def frame(self):
        """deblock_frame in place on a copy, sao_stats_frame, the stand-in decision, sao_apply_frame: (planes, stats, params)"""
        cu, d, W, H, ctu = self.cu, self.depth, self.W, self.H, self.ctu
        P = Planes(cu, self.rec)
        cu.deblock_frame(d, P.ptrs[0], P.stride, P.ptrs[1], P.ptrs[2], P.cs, W, H, self.ubuf, self.p)
        sbuf = cu.alloc(self.n * SAO_STATS_PER_CTU * 4)
        cu.sao_stats_frame(d, W, H, ctu, self.F.ptrs, self.F.stride, self.F.cs, P.ptrs, P.stride, P.cs, sbuf)
        stats = sbuf.download(np.int32).reshape((self.n,) + S.STATS_SHAPE)
        params = decide(stats, d)
        pbuf = cu.to_device(params)
        cu.sao_apply_frame(d, W, H, ctu, P.ptrs, P.stride, P.cs, pbuf, 1, 1, self.ubuf, self.F.ptrs, self.F.stride, self.F.cs)
        cu.sync()
        out = [g.picture(g.download()) for g in P.g]
        for b in (P, sbuf, pbuf):
            b.free()
        return out, stats, params

    def deblock(self, r0, r1, src, dst):
        self.cu.deblock_rows(self.depth, self.W, self.H, self.ctu, r0, r1, src.ptrs, src.stride, src.cs, dst.ptrs, dst.stride,
                             dst.cs, self.ubuf, self.p)

    def stats(self, r0, r1, dbk, sbuf):
        self.cu.sao_stats_rows(self.depth, self.W, self.H, self.ctu, r0, r1, self.F.ptrs, self.F.stride, self.F.cs, dbk.ptrs,
                               dbk.stride, dbk.cs, sbuf)

    def apply(self, r0, r1, dbk, ref, pbuf):
        self.cu.sao_apply_rows(self.depth, self.W, self.H, self.ctu, r0, r1, dbk.ptrs, dbk.stride, dbk.cs, ref.ptrs, ref.stride,
                               ref.cs, pbuf, 1, 1, self.ubuf, self.F.ptrs, self.F.stride, self.F.cs)

    def free(self):
        for b in (self.R, self.F, self.ubuf):
            b.free()


def chain_inputs(rng, W, H, ctu, depth, split=None):
    units = D.make_map(rng, W, H, ctu, depth, B_SLICE, p_intra=0.1, p_bypass=0.01, split=split)
    luma, cb, cr = D.make_planes(rng, W, H, depth)
    rec = [luma, cb, cr]
    fenc = [np.clip(q.astype(np.int32) + rng.integers(-3, 4, q.shape) * (1 << (depth - 8)), 0, (1 << depth) - 1).astype(q.dtype)
            for q in rec]
    return rec, fenc, units, D.params_array(B_SLICE, 1, -1, 2, -3, bypass=1)


def run_bands(ch, nbands, params):
    """deblock_rows, sao_stats_rows and sao_apply_rows band by band (block partition into nbands), through one deblocked
    scratch; returns (planes, stats)."""
    cu = ch.cu
    Sc, Ref = ch.scratch(), ch.scratch()
    sbuf = cu.to_device(np.full(ch.n * SAO_STATS_PER_CTU, -1, np.int32))
    pbuf = cu.to_device(params)
    parts = [b for g in range(nbands) for b in shard.row_blocks(ch.rows, g, nbands)]
    for r0, r1 in parts:
        ch.deblock(r0, r1, ch.R, Sc)
    for r0, r1 in parts:
        ch.stats(r0, r1, Sc, sbuf)
    for r0, r1 in parts:
        ch.apply(r0, r1, Sc, Ref, pbuf)
    cu.sync()
    got = [g.picture(g.download()) for g in Ref.g]
    stats = sbuf.download(np.int32).reshape((ch.n,) + S.STATS_SHAPE)
    for b in (Sc, Ref, sbuf, pbuf):
        b.free()
    return got, stats


@pytest.mark.timeout(900)
@pytest.mark.parametrize("depth", [8, 10])
def test_filter_rows_2160p(cu, depth):
    rng = np.random.default_rng(3840 + depth)
    W, H = 3840, 2160
    rec, fenc, units, prm = chain_inputs(rng, W, H, 64, depth, split={6: 0.85, 5: 0.6, 4: 0.35})
    ch = Chain(cu, depth, W, H, 64, rec, fenc, units, prm)
    want, wstats, params = ch.frame()
    for nb in (1, 2, 4, 8):
        got, stats = run_bands(ch, nb, params)
        assert np.array_equal(stats, wstats), nb
        assert_planes_equal(got, want, "2160p %d bands" % nb)
    ch.free()


@pytest.mark.timeout(900)
def test_filter_rows_4320p_8_bands(cu):
    """The geometry of a 7680x4320 10-bit picture over 8 row shards."""
    rng = np.random.default_rng(4320)
    W, H, depth = 7680, 4320, 10
    rec, fenc, units, prm = chain_inputs(rng, W, H, 64, depth, split={6: 0.6, 5: 0.4, 4: 0.3})
    ch = Chain(cu, depth, W, H, 64, rec, fenc, units, prm)
    want, wstats, params = ch.frame()
    got, stats = run_bands(ch, 8, params)
    assert np.array_equal(stats, wstats)
    assert_planes_equal(got, want, "4320p 8 bands")
    ch.free()


ROW_BY_ROW = [(8, 200, 136, 64), (10, 208, 104, 32), (8, 200, 72, 16), (10, 120, 56, 16), (8, 1920, 1080, 64)]


@pytest.mark.timeout(300)
@pytest.mark.parametrize("depth,W,H,ctu", ROW_BY_ROW, ids=["%d-%dx%d-ctu%d" % g for g in ROW_BY_ROW])
def test_filter_rows_row_by_row_lag_order(cu, depth, W, H, ctu):
    """FrameFilter's order on one GPU, one CTU row at a time into a single deblocked scratch and a single reference: deblock
    row r as soon as it is reconstructed, statistics of row r, apply row r - 1; then apply the last row.  When row r is
    deblocked, the reconstruction and the map below it are not there yet (noise and another map's rows here).  Equal to the
    frame chain byte for byte."""
    rng = np.random.default_rng([depth, W, H, ctu])
    rec, fenc, units, prm = chain_inputs(rng, W, H, ctu, depth)
    other = D.make_map(rng, W, H, ctu, depth, B_SLICE)
    ch = Chain(cu, depth, W, H, ctu, rec, fenc, units, prm)
    want, wstats, params = ch.frame()
    Sc, Ref = ch.scratch(), ch.scratch()
    sbuf = cu.to_device(np.full(ch.n * SAO_STATS_PER_CTU, -1, np.int32))
    pbuf = cu.to_device(params)
    for r in range(ch.rows):
        Y1 = min(H, (r + 1) * ctu)
        m = other.copy()
        m[:Y1 // 4] = units[:Y1 // 4]
        R = Planes(cu, [noise_outside(rng, q, 0, b, depth) for q, b in zip(rec, (Y1, Y1 // 2, Y1 // 2))])
        mbuf = cu.to_device(m)
        cu.deblock_rows(depth, W, H, ctu, r, r + 1, R.ptrs, R.stride, R.cs, Sc.ptrs, Sc.stride, Sc.cs, mbuf, ch.p)
        cu.sync()
        R.free()
        mbuf.free()
        ch.stats(r, r + 1, Sc, sbuf)
        if r:
            ch.apply(r - 1, r, Sc, Ref, pbuf)
    ch.apply(ch.rows - 1, ch.rows, Sc, Ref, pbuf)
    cu.sync()
    assert np.array_equal(sbuf.download(np.int32).reshape((ch.n,) + S.STATS_SHAPE), wstats)
    assert_planes_equal([g.picture(g.download()) for g in Ref.g], want, "row by row")
    for b in (Sc, Ref, sbuf, pbuf):
        b.free()
    ch.free()


# ---- emulated row shards on the frame analyser ----

@pytest.mark.timeout(600)
@pytest.mark.parametrize("depth", [8, 10])
def test_filter_rows_shards_on_analyser(cu, depth):
    """World 2 and 3, block and cyclic.  Each rank starts from its own copy of the CU-64 reconstruction holding only its
    bands and the halo rows exchange_halos would give it (noise elsewhere), deblocks its bands into its own scratch, writes
    the statistics of its CTUs and applies the decision into its bands of reference 1; after ref_updated /
    ref_chroma_updated the reference allocations, margins included, equal reference 0's, made by recon_to_ref,
    deblock_frame, sao_stats_frame, sao_apply_frame and ref_updated."""
    from frame_helpers import Workload, MARGIN_X, MARGIN_Y
    from chroma_helpers import chroma_inner
    from test_gpu_x_chroma_residual import open_analyser, source
    W, H, ctu = 200, 136, 64
    wl = Workload(W, H, depth=depth, numRefs=2, method=3, subme=3, merange=57, rect=1, qp=30, chroma=True)
    a = open_analyser(cu, wl)
    a.analyse(source(wl), wl.field, stages=15)
    rows = a.ctu_rows
    rng = np.random.default_rng(99 + depth)
    units = D.make_map(rng, W, H, ctu, depth, B_SLICE, p_bypass=0.05)
    ubuf, p = cu.to_device(units), dparams(D.params_array(B_SLICE, 0, 1, 0, 0, 1))
    src = [a.src_plane(k) for k in range(3)]
    fen, fs, fcs = [s[0] for s in src], src[0][1], src[1][1]
    n = S.num_ctus(W, H, ctu)

    # reference 0: the frame chain
    a.recon_to_ref(0, 0, 0, rows)
    a.recon_to_ref_chroma(0, 0, 0, rows)
    y, ys = a.ref_plane_ptr(0)
    (u, cs), (v, _) = a.ref_plane_chroma(0, 0), a.ref_plane_chroma(0, 1)
    cu.deblock_frame(depth, y, ys, u, v, cs, W, H, ubuf, p)
    sbuf = cu.alloc(n * SAO_STATS_PER_CTU * 4)
    cu.sao_stats_frame(depth, W, H, ctu, fen, fs, fcs, (y, u, v), ys, cs, sbuf)
    stats = sbuf.download(np.int32).reshape((n,) + S.STATS_SHAPE)
    params = decide(stats, depth)
    pbuf = cu.to_device(params)
    cu.sao_apply_frame(depth, W, H, ctu, (y, u, v), ys, cs, pbuf, 1, 1, ubuf, fen, fs, fcs)
    a.ref_updated(0)
    a.ref_chroma_updated(0)
    want_y, want_c = a.fetch(("plane", 0, 0)), [a.fetch_chroma(("ref", 0, k)) for k in range(2)]

    recon = [np.ascontiguousarray(a.fetch("recon0").reshape(wl.fenc.shape)[MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W])] + \
            [np.ascontiguousarray(chroma_inner(wl, a.fetch_chroma(("recon", 0, k)))) for k in range(2)]
    y1, ys1 = a.ref_plane_ptr(1)
    (u1, cs1), (v1, _) = a.ref_plane_chroma(1, 0), a.ref_plane_chroma(1, 1)
    for world in (2, 3):
        for mode in ("block", "cyclic"):
            sends = shard.halo_sends(rows, world, H, ctu, mode)
            st = cu.to_device(np.full(n * SAO_STATS_PER_CTU, -1, np.int32))
            for g in range(world):
                mine = shard.row_blocks(rows, g, world, mode)
                have = [np.zeros(H, bool), np.zeros(H // 2, bool)]
                for r0, r1 in mine:
                    have[0][r0 * ctu:min(H, r1 * ctu)] = True
                    have[1][r0 * ctu // 2:min(H, r1 * ctu) // 2] = True
                for _, (a0, a1), (c0, c1) in sends:                 # what exchange_halos gives every rank
                    have[0][a0:a1] = True
                    have[1][c0:c1] = True
                copy = [np.where(have[min(k, 1)][:, None], q, rng.integers(0, 1 << depth, q.shape).astype(q.dtype))
                        for k, q in enumerate(recon)]
                Rg = Planes(cu, copy)
                Sg = Planes(cu, [sentinel_like(q) for q in copy])
                for r0, r1 in mine:
                    cu.deblock_rows(depth, W, H, ctu, r0, r1, Rg.ptrs, Rg.stride, Rg.cs, Sg.ptrs, Sg.stride, Sg.cs, ubuf, p)
                    cu.sao_stats_rows(depth, W, H, ctu, r0, r1, fen, fs, fcs, Sg.ptrs, Sg.stride, Sg.cs, st)
                    cu.sao_apply_rows(depth, W, H, ctu, r0, r1, Sg.ptrs, Sg.stride, Sg.cs, (y1, u1, v1), ys1, cs1, pbuf, 1, 1,
                                      ubuf, fen, fs, fcs)
                cu.sync()
                Rg.free()
                Sg.free()
            assert np.array_equal(st.download(np.int32).reshape((n,) + S.STATS_SHAPE), stats), (world, mode, "statistics")
            st.free()
            a.ref_updated(1)
            a.ref_chroma_updated(1)
            assert np.array_equal(a.fetch(("plane", 1, 0)), want_y), (world, mode, "luma reference allocation")
            for k in range(2):
                assert np.array_equal(a.fetch_chroma(("ref", 1, k)), want_c[k]), (world, mode, "chroma reference allocation", k)
    for b in (ubuf, sbuf, pbuf):
        b.free()
    a.close()


# ---- refusals ----

def test_filter_rows_refusals(cu):
    """One refusal per argument rule of the band calls: -1 with a message, no launch, no buffer written."""
    depth, W, H, ctu = 8, 64, 48, 16
    rng = np.random.default_rng(8)
    rec, fenc = S.make_pictures(rng, W, H, depth)
    params, _ = S.make_params(rng, W, H, ctu, depth)
    units = D.make_map(rng, W, H, ctu, depth, B_SLICE, p_bypass=0.2)
    SY, SU, SV = [cu.to_device(q) for q in rec]
    DY, DU, DV = [cu.to_device(sentinel_like(q)) for q in rec]
    FY, FU, FV = [cu.to_device(q) for q in fenc]
    n = S.num_ctus(W, H, ctu)
    ST = cu.to_device(np.full(n * SAO_STATS_PER_CTU, 7, np.int32))
    PR, UN = cu.to_device(params), cu.to_device(units)
    prm = DeblockParams(*[int(x) for x in D.params_array(B_SLICE)])
    L = cu.L
    base = dict(depth=8, W=W, H=H, ctu=ctu, r0=0, r1=3)
    dgood = dict(base, sy=SY.ptr, scb=SU.ptr, scr=SV.ptr, ss=W, scs=W // 2, y=DY.ptr, cb=DU.ptr, cr=DV.ptr, s=W, cs=W // 2, units=UN.ptr)
    sgood = dict(base, fy=FY.ptr, fcb=FU.ptr, fcr=FV.ptr, fs=W, fcs=W // 2, y=SY.ptr, cb=SU.ptr, cr=SV.ptr, s=W, cs=W // 2, stats=ST.ptr)
    agood = dict(dgood, params=PR.ptr, sl=1, sc=1, fy=FY.ptr, fcb=FU.ptr, fcr=FV.ptr, fs=W, fcs=W // 2)

    def deblock(**kw):
        a = dict(dgood, **kw)
        return L.x265cu_deblock_rows(cu.ctx, a["depth"], a["W"], a["H"], a["ctu"], a["r0"], a["r1"], a["sy"], a["scb"], a["scr"],
                                     a["ss"], a["scs"], a["y"], a["cb"], a["cr"], a["s"], a["cs"], a["units"], C.byref(prm))

    def stats(**kw):
        a = dict(sgood, **kw)
        return L.x265cu_sao_stats_rows(cu.ctx, a["depth"], a["W"], a["H"], a["ctu"], a["r0"], a["r1"], a["fy"], a["fcb"], a["fcr"],
                                       a["fs"], a["fcs"], a["y"], a["cb"], a["cr"], a["s"], a["cs"], a["stats"])

    def apply(**kw):
        a = dict(agood, **kw)
        return L.x265cu_sao_apply_rows(cu.ctx, a["depth"], a["W"], a["H"], a["ctu"], a["r0"], a["r1"], a["sy"], a["scb"], a["scr"],
                                       a["ss"], a["scs"], a["y"], a["cb"], a["cr"], a["s"], a["cs"], a["params"], a["sl"], a["sc"],
                                       a["units"], a["fy"], a["fcb"], a["fcr"], a["fs"], a["fcs"])

    rows = [dict(ctu=8), dict(ctu=128), dict(ctu=48), dict(r0=-1), dict(r0=2, r1=2), dict(r0=2, r1=1), dict(r1=4)]
    bad = [(f, kw) for f in (deblock, stats, apply) for kw in rows]
    bad += [(f, kw) for f in (deblock, apply) for kw in (dict(sy=None), dict(ss=W - 1), dict(scs=W // 2 - 1), dict(scb=None, scr=None),
                                                         dict(y=None), dict(depth=9), dict(H=44))]
    bad += [(deblock, dict(units=None)), (stats, dict(stats=None)), (stats, dict(y=None)), (stats, dict(fcb=None, fcr=None))]
    bad += [(apply, dict(sy=DY.ptr)), (apply, dict(scb=DU.ptr)), (apply, dict(params=None)), (apply, dict(sc=2))]
    for f, kw in bad:
        k = cu.launch_count()
        assert f(**kw) == -1 and cu.last_error(), (f.__name__, kw)
        assert cu.launch_count() == k, (f.__name__, kw)
    cu.sync()
    for buf, img in ((SY, rec[0]), (SU, rec[1]), (SV, rec[2])):
        assert np.array_equal(buf.download(pixel_dtype(depth)).reshape(img.shape), img)
    for buf, img in ((DY, rec[0]), (DU, rec[1]), (DV, rec[2])):
        assert np.array_equal(buf.download(pixel_dtype(depth)).reshape(img.shape), sentinel_like(img))
    assert (ST.download(np.int32) == 7).all()
    assert deblock() == 0 and stats() == 0 and apply() == 0 and deblock(r0=2, r1=3, cb=None, cr=None, scb=None, scr=None) == 0
    cu.sync()
    for b in (SY, SU, SV, DY, DU, DV, FY, FU, FV, ST, PR, UN):
        b.free()
