"""The band contract of x265cu_deblock_rows / x265cu_sao_stats_rows / x265cu_sao_apply_rows, pinned on the restatements
(oracle/oracle_deblock.c, oracle/oracle_sao.c, which tests/test_deblock_oracle_vs_ref.py and tests/test_sao_oracle_vs_ref.py
pin to the real Deblock / SAO): for a band of CTU rows [r0, r1), whatever lies outside the rows a call reads does not change
the rows it writes.  The inputs outside the read range are replaced by noise (pixels, and whole CTU rows of the deblocking map
taken from a second legal map; SAO records of the CTUs outside the band from a second decision), and the whole-picture
oracle's output in the write range must stay byte-identical.  Bands: row_blocks of worlds 1, 2 and 3 in both modes, and every
one-row band; CTU 16, 32 and 64; heights that end in a partial CTU row.  Also the shard plumbing: filter_halo, halo_sends and
exchange_halos under gloo."""
import os
import socket

import numpy as np
import pytest

import deblock_helpers as D
import sao_helpers as S
from common import pixel_dtype
from x265_b200 import shard
from x265_b200.lib import B_SLICE, P_SLICE

# deblock_helpers.cases() has CTU 64 / 32 only: CTU 16 with H % 16 == 8, and CTU 32 with a one-CTU-row band of 8 rows
EXTRA_DEBLOCK = [("B%d_ctu16_h72" % d, d, 200, 72, 16, B_SLICE, dict(beta=1, tc=2, cb=-3, cr=4), False, "blocky", {}) for d in (8, 10)] + \
                [("P8_ctu32_h104", 8, 136, 104, 32, P_SLICE, {}, False, "blocky", {}),
                 ("B10_ctu16_luma_only", 10, 120, 56, 16, B_SLICE, {}, True, "blocky", dict(p_bypass=0.1))]
DEBLOCK_CASES = D.cases() + EXTRA_DEBLOCK


def bands(nrows):
    """Every band of row_blocks for worlds 1..3 in both modes, and every one-row band."""
    out = {(r, r + 1) for r in range(nrows)}
    for world in (1, 2, 3):
        for mode in ("block", "cyclic"):
            for g in range(world):
                out.update(shard.row_blocks(nrows, g, world, mode))
    return sorted(out)


def noise_outside(rng, img, y0, y1, depth):
    """img with rows outside [y0, y1) replaced by uniform noise"""
    out = rng.integers(0, 1 << depth, img.shape).astype(img.dtype)
    out[max(y0, 0):y1] = img[max(y0, 0):y1]
    return out


@pytest.mark.parametrize("case", DEBLOCK_CASES, ids=[c[0] for c in DEBLOCK_CASES])
def test_deblock_band_depends_only_on_its_read_range(case):
    name, depth, W, H, ctu, st, pk, luma_only, content, mk = case
    luma, cb, cr, units, prm = D.case_inputs(case)
    want = D.oracle_deblock(depth, luma, cb, cr, units, prm)
    rng = np.random.default_rng([99, sum(map(ord, name))])
    other = D.make_map(rng, W, H, ctu, depth, st, **mk)
    nrows = (H + ctu - 1) // ctu
    u = ctu // 4
    for r0, r1 in bands(nrows):
        (y0, y1), (c0, c1) = shard.filter_halo(r0, r1, ctu, H)
        m = other.copy()
        m[max(0, (r0 - 1) * u):(r1 + 1) * u] = units[max(0, (r0 - 1) * u):(r1 + 1) * u]
        py = noise_outside(rng, luma, y0, y1, depth)
        pu = noise_outside(rng, cb, c0, c1, depth) if cb is not None else None
        pv = noise_outside(rng, cr, c0, c1, depth) if cr is not None else None
        got = D.oracle_deblock(depth, py, pu, pv, m, prm)
        assert np.array_equal(got[0][y0:y1], want[0][y0:y1]), (name, r0, r1, "luma")
        for k in (1, 2):
            if want[k] is not None:
                assert np.array_equal(got[k][c0:c1], want[k][c0:c1]), (name, r0, r1, "chroma", k)


EXTRA_SAO = [("d10_ctu16_h56", 10, 120, 56, 16, True, {}, (1, 1), True), ("d8_ctu32_h104_merge", 8, 136, 104, 32, True,
             dict(p_merge=0.5), (1, 1), False)]
SAO_CASES = S.cases() + EXTRA_SAO


def _band_rows(r0, r1, ctu, H):
    Y0, Y1 = r0 * ctu, min(H, r1 * ctu)
    return Y0, Y1, Y0 // 2, Y1 // 2


@pytest.mark.parametrize("case", SAO_CASES, ids=[c[0] for c in SAO_CASES])
def test_sao_band_depends_only_on_its_read_range(case):
    name, depth, W, H, ctu = case[:5]
    sl, sc = case[7]
    rec, fenc, params, merge, units = S.case_inputs(case)
    want_st = S.oracle_stats(depth, rec, fenc, ctu)
    want_ap = S.oracle_apply(depth, rec, ctu, params, sl, sc, units, fenc)
    rng = np.random.default_rng([77, sum(map(ord, name))])
    other, _ = S.make_params(rng, W, H, ctu, depth)
    cols, nrows = (W + ctu - 1) // ctu, (H + ctu - 1) // ctu
    for r0, r1 in bands(nrows):
        Y0, Y1, C0, C1 = _band_rows(r0, r1, ctu, H)
        lo = [(Y0, Y1)] + [(C0, C1)] * 2
        # statistics: deblocked rows [Y0 - 1, Y1), source rows [Y0, Y1)
        pr = [noise_outside(rng, p, a - 1, b, depth) if p is not None else None for p, (a, b) in zip(rec, lo)]
        pf = [noise_outside(rng, p, a, b, depth) if p is not None else None for p, (a, b) in zip(fenc, lo)]
        got = S.oracle_stats(depth, pr, pf, ctu)
        sel = slice(r0 * cols, r1 * cols)
        assert np.array_equal(got[sel], want_st[sel]), (name, r0, r1, "stats")
        # apply: deblocked rows [Y0 - 1, Y1 + 1), source rows [Y0, Y1), the records of the band's CTUs
        pr = [noise_outside(rng, p, a - 1, b + 1, depth) if p is not None else None for p, (a, b) in zip(rec, lo)]
        pp = other.copy()
        pp[:, sel] = params[:, sel]
        got = S.oracle_apply(depth, pr, ctu, pp, sl, sc, units, pf)
        for k, (a, b) in enumerate(lo):
            if want_ap[k] is not None:
                assert np.array_equal(got[k][a:b], want_ap[k][a:b]), (name, r0, r1, "apply", k)


def test_filter_halo():
    assert shard.filter_halo(0, 1, 64, 136) == ((0, 68), (0, 36))
    assert shard.filter_halo(1, 2, 64, 136) == ((60, 132), (28, 68))
    assert shard.filter_halo(2, 3, 64, 136) == ((124, 136), (60, 68))      # last band: 8 rows, clipped below
    assert shard.filter_halo(0, 3, 64, 136) == ((0, 136), (0, 68))         # the whole picture
    assert shard.filter_halo(4, 5, 16, 72) == ((60, 72), (28, 36))
    assert shard.filter_halo(1, 3, 32, 104) == ((28, 100), (12, 52))


GEOMS = [(136, 64), (104, 32), (72, 16), (2160, 64), (4320, 64), (64, 64), (200, 16)]


@pytest.mark.parametrize("H,ctu", GEOMS)
def test_halo_sends_cover_every_band(H, ctu):
    """After the halo exchange, every rank holds, for each of its bands, every pre-deblock row x265cu_deblock_rows reads."""
    nrows = (H + ctu - 1) // ctu
    for world in (1, 2, 3, 8):
        for mode in ("block", "cyclic"):
            sends = shard.halo_sends(nrows, world, H, ctu, mode)
            for src, (y0, y1), (c0, c1) in sends:
                assert 0 <= y0 < y1 <= H and 0 <= c0 < c1 <= H // 2 and y1 - y0 <= 4 and c1 - c0 <= 4
                assert all(shard.row_owner(y // ctu, nrows, world, mode) == src for y in (y0, y1 - 1)), "a rank sends its own rows"
            for g in range(world):
                have_y, have_c = np.zeros(H, bool), np.zeros(H // 2, bool)
                for r0, r1 in shard.row_blocks(nrows, g, world, mode):
                    have_y[r0 * ctu:min(H, r1 * ctu)] = True
                    have_c[r0 * ctu // 2:min(H, r1 * ctu) // 2] = True
                for _, (y0, y1), (c0, c1) in sends:
                    have_y[y0:y1] = True
                    have_c[c0:c1] = True
                for r0, r1 in shard.row_blocks(nrows, g, world, mode):
                    (y0, y1), (c0, c1) = shard.filter_halo(r0, r1, ctu, H)
                    assert have_y[y0:y1].all() and have_c[c0:c1].all(), (world, mode, g, r0, r1)
            if world == 1:
                assert sends == []


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close()
    return p


def _halo_worker(rank, world, port, ret):
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    ok = True
    for (W, H, ctu, depth, mode) in ((96, 136, 64, 8, "block"), (96, 136, 64, 10, "cyclic"), (64, 72, 16, 8, "cyclic"),
                                     (64, 104, 32, 10, "block")):
        es, my, cmy = (1 if depth == 8 else 2), 5, 3
        stride, cstride = W + 24, W // 2 + 12
        nrows = (H + ctu - 1) // ctu
        rng = np.random.default_rng([W, H, ctu, depth])
        truth = [rng.integers(0, 1 << depth, (H + 2 * my, stride)).astype(pixel_dtype(depth))] + \
                [rng.integers(0, 1 << depth, (H // 2 + 2 * cmy, cstride)).astype(pixel_dtype(depth)) for _ in range(2)]
        mine = [np.full_like(t, 7) for t in truth]
        for r0, r1 in shard.row_blocks(nrows, rank, world, mode):      # this rank reconstructed only its own bands
            y0, y1 = r0 * ctu, min(H, r1 * ctu)
            mine[0][my + y0:my + y1] = truth[0][my + y0:my + y1]
            for k in (1, 2):
                mine[k][cmy + y0 // 2:cmy + y1 // 2] = truth[k][cmy + y0 // 2:cmy + y1 // 2]
        ts = [torch.from_numpy(m.view(np.uint8).reshape(-1)) for m in mine]
        n = shard.exchange_halos(dist, ts[0], ts[1:], nrows, world, H, ctu, stride, cstride, my, cmy, es, mode)
        sends = shard.halo_sends(nrows, world, H, ctu, mode)
        ok = ok and n == sum(((y1 - y0) * stride + 2 * (c1 - c0) * cstride) * es for _, (y0, y1), (c0, c1) in sends)
        for r0, r1 in shard.row_blocks(nrows, rank, world, mode):
            (y0, y1), (c0, c1) = shard.filter_halo(r0, r1, ctu, H)
            ok = ok and np.array_equal(mine[0][my + y0:my + y1], truth[0][my + y0:my + y1])
            for k in (1, 2):
                ok = ok and np.array_equal(mine[k][cmy + c0:cmy + c1], truth[k][cmy + c0:cmy + c1])
    t = torch.tensor([1 if ok else 0]); dist.all_reduce(t, op=dist.ReduceOp.MIN)
    ret[rank] = int(t.item())
    dist.destroy_process_group()


def test_exchange_halos_gloo():
    import torch.multiprocessing as mp
    world = 2
    mgr = mp.Manager(); ret = mgr.dict()
    mp.spawn(_halo_worker, args=(world, _free_port(), ret), nprocs=world, join=True)
    assert all(ret[r] == 1 for r in range(world))
