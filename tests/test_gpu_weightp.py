"""k_weightp_costs and x265cu_weightp_analyse on the device against the restatement (oracle/oracle_weightp.c), and the
Lookahead mirror's weight_analyse against the reference's stored result."""
import ctypes as C

import numpy as np
import pytest

import weightp_helpers as WH
from common import ptr
from x265_b200.lib import WpFrame, WpCand

pytestmark = pytest.mark.gpu


def _device_records(cu, c):
    """the case's planes uploaded; returns (records, keep-alive buffers, intraCost buffer, mvs buffers)"""
    keep = []
    es = np.dtype(c.pics[0][0].dtype).itemsize

    def up(a):
        b = cu.to_device(np.ascontiguousarray(a)); keep.append(b); return b.ptr
    recs = []
    for i in range(3):
        r = WpFrame()
        C.memmove(C.byref(r), C.byref(c.recs[i]), C.sizeof(WpFrame))
        la = c.la.fr[i]
        for k in range(4):
            r.lowres[k] = up(la["planes"][k]) + c.la.org * es
        if c.chroma[i] is not None:
            cs = c.chroma[i][0].shape[1]
            r.cb, r.cr = [up(p) + (WH.CMY * cs + WH.CMX) * es for p in c.chroma[i]]
        recs.append(r)
    intra = up(c.intraCost)
    mvs = [up(m) if m is not None else None for m in c.mvs]
    return recs, keep, intra, mvs


def _cands(depth):
    """the unweighted reference, then every w0 0..127 with each denominator 0..7 and each offset -128 / 0 / 127 in turn"""
    return [WpCand(0, 0, 0, 0)] + [WpCand(1, w0, w0 % 8, (-128, 0, 127)[w0 % 3]) for w0 in range(128)]


@pytest.fixture(scope="module")
def cu():
    import x265_b200
    return x265_b200.load()


COST_CASES = [c for c in WH.CASES if c[8] in ("edge", "la", "none", "rand") and
              (c[2] >= 1920 or c[1] in ("fade_up", "motion_fade") or c[1] in WH.NOISE_KINDS)]


@pytest.mark.parametrize("case", COST_CASES, ids=[c[0] for c in COST_CASES])
def test_costs_equal_restatement(cu, case):
    """every candidate's weightCost, luma with and without motion fields and both chroma planes, equals the restatement"""
    c = WH.Case(case)
    recs, keep, intra, mvs = _device_records(cu, c)
    O = WH.load_oracle_wp()
    cands = _cands(c.depth)
    for chunk in (cands[:48], cands[48:96], cands[96:]):
        if not chunk:
            continue
        arr = (WpCand * len(chunk))(*chunk)
        for plane in range(3 if c.csp else 1):
            for lst in range(c.nl):
                for use in ([False, True] if c.mvs[lst] is not None else [False]):
                    want = np.zeros(len(chunk), np.uint32)
                    O.orc_wp_costs(c.depth, C.byref(c.params), C.byref(c.recs[1]), C.byref(c.recs[2 * lst]), ptr(c.intraCost),
                                   c.mvs[lst].ctypes.data if use else None, plane, arr, len(chunk), ptr(want))
                    got = np.zeros(len(chunk), np.uint32)
                    cu.check(cu.L.x265cu_weightp_costs(cu.ctx, c.depth, C.byref(c.params), C.byref(recs[1]), C.byref(recs[2 * lst]),
                                                       intra, mvs[lst] if use else None, plane, arr, len(chunk), got.ctypes.data))
                    assert np.array_equal(got, want), (plane, lst, use)


def test_chroma_paths(cu):
    """synthetic vectors through all four chroma filter paths and both sides of mcChroma's pixel-vs-CU test"""
    c = WH.Case(WH._case("fade_up", 1920, 1080, 10, 1, "P", 1, "none"))
    ncu = c.la.w8 * c.la.h8
    rng = np.random.default_rng(5)
    c.mvs[0] = rng.integers(-40, 41, (ncu, 2)).astype(np.int32)
    recs, keep, intra, mvs = _device_records(cu, c)
    cands = _cands(10)[:48]
    arr = (WpCand * 48)(*cands)
    WH.oracle_counters(reset=True)
    for plane in (1, 2):
        want = np.zeros(48, np.uint32)
        WH.load_oracle_wp().orc_wp_costs(c.depth, C.byref(c.params), C.byref(c.recs[1]), C.byref(c.recs[0]), ptr(c.intraCost),
                                         c.mvs[0].ctypes.data, plane, arr, 48, ptr(want))
        got = np.zeros(48, np.uint32)
        cu.check(cu.L.x265cu_weightp_costs(cu.ctx, c.depth, C.byref(c.params), C.byref(recs[1]), C.byref(recs[0]), intra,
                                           mvs[0], plane, arr, 48, got.ctypes.data))
        assert np.array_equal(got, want), plane
    k = WH.oracle_counters(reset=True)
    assert all(k[n] > 0 for n in ("path_copy", "path_hpp", "path_vpp", "path_hv", "mc_block", "copy_block")), k


def _bent_block():
    """an 8x8 sign pattern whose every 4x4 quarter is a bent function, (-1)^(x0 y0 + x1 y1): all 16 Hadamard coefficients
    of a quarter have the same magnitude, so a +-1023 difference gives the largest 10-bit SATD, 2 * 4 * 16 * 1023 / 2"""
    y, x = np.mgrid[0:8, 0:8]
    return ((x & 1) * (y & 1) + ((x >> 1) & 1) * ((y >> 1) & 1)) & 1


def test_chroma_sum_wraps(cu):
    """10-bit 4096x2160 chroma of maximal SATD in every 8x8 block: 34560 blocks x 130944 passes 2^32, and the device sum
    wraps to the restatement's (and the reference's, whose sum is uint32) value"""
    W, H, depth = 4096, 2160, 10
    cw, ch = W // 2, H // 2
    sign = np.tile(_bent_block(), (ch // 8, cw // 8))
    ref = np.where(sign == 1, 1023, 0).astype(np.uint16)
    fenc = np.where(sign == 1, 0, 1023).astype(np.uint16)
    planes = [np.pad(p, ((WH.CMY, WH.CMY), (WH.CMX, WH.CMX)), mode="edge") for p in (fenc, ref)]
    cs = planes[0].shape[1]
    org = (WH.CMY * cs + WH.CMX) * 2
    from x265_b200.lib import WpParams
    prm = WpParams(1, (C.c_int32 * 2)(1, 0), 3, W, H, 1)
    host, dev = [], []
    keep = []
    for p in planes:
        hr, dr = WpFrame(), WpFrame()
        hr.cb = hr.cr = p.ctypes.data + org
        b = cu.to_device(p); keep.append(b)
        dr.cb = dr.cr = b.ptr + org
        for r in (hr, dr):
            r.chromaStride = cs
        host.append(hr); dev.append(dr)
    arr = (WpCand * 2)(WpCand(0, 0, 0, 0), WpCand(1, 64, 6, 0))
    want = np.zeros(2, np.uint32)
    WH.load_oracle_wp().orc_wp_costs(depth, C.byref(prm), C.byref(host[0]), C.byref(host[1]), None, None, 1, arr, 2, ptr(want))
    assert int(want[0]) == (34560 * 130944) % (1 << 32)
    got = np.zeros(2, np.uint32)
    cu.check(cu.L.x265cu_weightp_costs(cu.ctx, depth, C.byref(prm), C.byref(dev[0]), C.byref(dev[1]), None, None, 1, arr, 2,
                                       got.ctypes.data))
    assert np.array_equal(got, want)


@pytest.mark.parametrize("case", WH.CASES, ids=[c[0] for c in WH.CASES])
def test_analysis_equals_restatement(cu, case):
    c = WH.Case(case)
    recs, keep, intra, mvs = _device_records(cu, c)
    want = WH.oracle_table(c, fill=-7)
    got = np.full((2, 16, 3, 4), -7, np.int32)
    refs = (C.POINTER(WpFrame) * 2)(C.pointer(recs[0]), C.pointer(recs[2]) if c.nl == 2 else C.POINTER(WpFrame)())
    n0 = cu.launch_count()
    cu.check(cu.L.x265cu_weightp_analyse(cu.ctx, c.depth, C.byref(c.params), C.byref(recs[1]), intra, refs,
                                         (C.c_void_p * 2)(*mvs), got.ctypes.data))
    assert cu.launch_count() - n0 <= c.nl * (3 if c.csp else 1)
    assert np.array_equal(got, want)
    assert c.written(got) == WH.stored(c.name)


E2E_CASES = [c for c in WH.CASES if c[2] == 328 and c[8] == "la" and c[5] and c[1] != "noise_flat_chroma"]
E2E_CASES = E2E_CASES[:4] + [c for c in E2E_CASES if c[1] in WH.NOISE_KINDS]


@pytest.mark.parametrize("case", E2E_CASES, ids=[c[0] for c in E2E_CASES])
def test_lookahead_end_to_end(cu, case):
    """init_frame(aq=..., keep_chroma=True), intra_batch and the estimates, then weight_analyse equals the reference"""
    from x265_b200.lookahead import Lookahead
    c = WH.Case(case)
    la = Lookahead(cu, c.W, c.H, c.depth, 3)
    try:
        for i, (y, cb, cr) in enumerate(c.pics):
            la.init_frame(i, y, cb=cb, cr=cr, aq={"mode": 2, "weightp": True}, keep_chroma=True)
        la.intra_batch([0, 1, 2])
        if c.nl == 1:
            la.cost(0, 1, 1)
        else:
            la.cost(0, 2, 1)
        for i in range(3):
            assert np.array_equal(la.fr[i]["wp_sum"], c.stats[i][0]) and np.array_equal(la.fr[i]["wp_ssd"], c.stats[i][1])
        t = la.weight_analyse(1, "P" if c.nl == 1 else "B", [0, 2][:c.nl], WH.BFRAMES, [c.params.numRefIdx[l] for l in range(c.nl)])
        assert c.written(t) == WH.stored(c.name)
    finally:
        la.close()


def test_reinit_drops_chroma_and_statistics(cu):
    """a window slot re-initialised without keep_chroma / aq does not keep the previous frame's chroma or statistics"""
    from x265_b200.lookahead import Lookahead
    c = WH.Case(WH.CASES[1])
    la = Lookahead(cu, c.W, c.H, c.depth, 3)
    try:
        for i, (y, cb, cr) in enumerate(c.pics):
            la.init_frame(i, y, cb=cb, cr=cr, aq={"mode": 2, "weightp": True}, keep_chroma=True)
        la.intra_batch([0, 1, 2])
        la.init_frame(1, c.pics[1][0])
        assert la.fr[1].get("chroma") is None
        with pytest.raises(ValueError):
            la.weight_analyse(1, "P", [0], WH.BFRAMES, [1])
        la.init_frame(1, c.pics[1][0], aq={"mode": 2, "weightp": True})
        la.fr[1]["has_intra"] = False
        la.intra_batch([1])
        la.cost(0, 1, 1)
        t = la.weight_analyse(1, "P", [0], WH.BFRAMES, [1])         # 4:0:0 now: the luma entry is the 4:2:0 case's
        assert t[0, 0, 0].tolist() == WH.stored(c.name)[0]
    finally:
        la.close()


def test_refusals(cu):
    c = WH.Case(WH.CASES[0])
    arr = (WpCand * 1)(WpCand(1, 200, 0, 0))
    got = np.zeros(1, np.uint32)
    assert cu.L.x265cu_weightp_costs(cu.ctx, 8, C.byref(c.params), C.byref(c.recs[1]), C.byref(c.recs[0]), None, None, 1,
                                     arr, 1, got.ctypes.data) == -1
    assert "x265cu_weightp_costs" in cu.last_error()
