"""GPU: x265cu_sao_stats_frame / x265cu_sao_apply_frame against the plain-C restatement (oracle/oracle_sao.c, which
tests/test_sao_oracle_vs_ref.py pins to the real SAO classes), byte-exact: the pin's cases, planes and stats inside guard
bands, 3840x2160 at 8 and 10 bit, luma-only calls, stats over garbage, the deblock -> stats -> apply recon loop on the frame
analyser, and the refusals."""
import numpy as np
import pytest

import deblock_helpers as D
import sao_helpers as S
from common import pixel_dtype
from test_gpu_deblock import GuardedPlane, dparams
from x265_b200.lib import B_SLICE, SAO_STATS_PER_CTU

pytestmark = pytest.mark.gpu
GARBAGE = 0x5A


@pytest.fixture(scope="module")
def cu():
    import x265_b200
    return x265_b200.load()


def upload_planes(cu, planes, stride=None, cstride=None, shift=0):
    """GuardedPlanes of (y, cb, cr) (None stays None)"""
    W = planes[0].shape[1]
    out = [GuardedPlane(cu, planes[0], stride or W, shift=shift)]
    for p in planes[1:]:
        out.append(GuardedPlane(cu, p, cstride or W // 2, shift=shift) if p is not None else None)
    return out


def ptrs(gp):
    return [g.ptr if g is not None else None for g in gp]


def free_all(gp):
    for g in gp:
        if g is not None:
            g.free()


def device_stats(cu, depth, rec, fenc, ctu, stride=None, cstride=None, shift=0, guard=0):
    """x265cu_sao_stats_frame on guarded copies; the stats buffer starts as garbage, with `guard` garbage records around it."""
    H, W = rec[0].shape
    n = S.num_ctus(W, H, ctu)
    R, F = upload_planes(cu, rec, stride, cstride, shift), upload_planes(cu, fenc, stride, cstride, shift)
    per = SAO_STATS_PER_CTU * 4
    buf = cu.to_device(np.full((n + 2 * guard) * per, GARBAGE, np.uint8))
    cu.sao_stats_frame(depth, W, H, ctu, ptrs(F), F[0].stride, F[1].stride if F[1] else 0, ptrs(R), R[0].stride,
                       R[1].stride if R[1] else 0, buf.ptr + guard * per)
    cu.sync()
    raw = buf.download(np.uint8)
    if guard:
        assert (raw[:guard * per] == GARBAGE).all() and (raw[guard * per + n * per:] == GARBAGE).all(), "stats guard changed"
    for g in R + F:
        if g is not None:
            whole = g.download()
            got, want = g.outside(whole)
            assert np.array_equal(got, want)
            assert np.array_equal(g.picture(whole), g.picture(g.expect_outside)), "stats changed a plane"
    buf.free()
    free_all(R)
    free_all(F)
    return raw[guard * per:guard * per + n * per].view(np.int32).reshape((n,) + S.STATS_SHAPE)


def device_apply(cu, depth, rec, ctu, params, sl, sc, units, fenc, stride=None, cstride=None, shift=0, check_guards=False):
    H, W = rec[0].shape
    R = upload_planes(cu, rec, stride, cstride, shift)
    F = upload_planes(cu, fenc, None, None) if units is not None else [None, None, None]
    pbuf = cu.to_device(params)
    ubuf = cu.to_device(units) if units is not None else None
    cu.sao_apply_frame(depth, W, H, ctu, ptrs(R), R[0].stride, R[1].stride if R[1] else 0, pbuf, sl, sc, ubuf,
                       ptrs(F), F[0].stride if F[0] else 0, F[1].stride if F[1] else 0)
    cu.sync()
    out = []
    for g in R:
        if g is None:
            out.append(None)
            continue
        whole = g.download()
        if check_guards:
            got, want = g.outside(whole)
            assert np.array_equal(got, want), "samples outside the picture changed"
        out.append(g.picture(whole))
    if check_guards:
        assert pbuf.download(np.uint8).tobytes() == params.tobytes(), "the parameters changed"
    free_all(R)
    free_all(F)
    pbuf.free()
    if ubuf is not None:
        ubuf.free()
    return out


def assert_planes_equal(got, want, what):
    for k, (g, w) in enumerate(zip(got, want)):
        if w is None:
            assert g is None
            continue
        assert np.array_equal(g, w), (what, "plane %d" % k, int(np.count_nonzero(g != w)))


CASES = S.cases()


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_sao_stats_matches_oracle(cu, case):
    depth, ctu = case[1], case[4]
    rec, fenc, params, merge, units = S.case_inputs(case)
    want = S.oracle_stats(depth, rec, fenc, ctu)
    got = device_stats(cu, depth, rec, fenc, ctu)
    assert np.array_equal(got, want), int(np.count_nonzero(got != want))


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_sao_apply_matches_oracle(cu, case):
    depth, ctu, (sl, sc) = case[1], case[4], case[7]
    rec, fenc, params, merge, units = S.case_inputs(case)
    want = S.oracle_apply(depth, rec, ctu, params, sl, sc, units, fenc)
    assert_planes_equal(device_apply(cu, depth, rec, ctu, params, sl, sc, units, fenc), want, case[0])


GUARDS = [(8, 200, 136, 64, 216, 112, 0), (10, 208, 104, 32, 256, 128, 0), (8, 200, 136, 16, 203, 109, 1), (10, 120, 72, 64, 141, 75, 1)]


@pytest.mark.parametrize("depth,W,H,ctu,stride,cstride,shift", GUARDS, ids=["%d-%dx%d-ctu%d-s%d-c%d-o%d" % g for g in GUARDS])
def test_sao_guard_bands(cu, depth, W, H, ctu, stride, cstride, shift):
    """Planes inside sentinel-filled allocations (the third and fourth with strides that are not multiples of 16 bytes and a
    base one pixel past an aligned address) and a stats array between garbage records: only the picture and the record
    array change, and the parameters are not written."""
    rng = np.random.default_rng([depth, W, stride])
    rec, fenc = S.make_pictures(rng, W, H, depth)
    params, _ = S.make_params(rng, W, H, ctu, depth)
    units = D.make_map(rng, W, H, ctu, depth, B_SLICE, p_bypass=0.1)
    got = device_stats(cu, depth, rec, fenc, ctu, stride, cstride, shift, guard=2)
    assert np.array_equal(got, S.oracle_stats(depth, rec, fenc, ctu))
    want = S.oracle_apply(depth, rec, ctu, params, 1, 1, units, fenc)
    assert_planes_equal(device_apply(cu, depth, rec, ctu, params, 1, 1, units, fenc, stride, cstride, shift, True), want, "guards")


@pytest.mark.timeout(600)
@pytest.mark.parametrize("depth", [8, 10])
def test_sao_2160p(cu, depth):
    """3840x2160, CTU 64, deblocked with a preset-slow-shaped map first; rare bypass units."""
    rng = np.random.default_rng(2160 + depth)
    W, H = 3840, 2160
    units = D.make_map(rng, W, H, 64, depth, B_SLICE, p_intra=0.1, p_bypass=0.01, split={6: 0.85, 5: 0.6, 4: 0.35})
    luma, cb, cr = D.make_planes(rng, W, H, depth)
    rec = list(D.oracle_deblock(depth, luma, cb, cr, units, D.params_array(B_SLICE, bypass=1)))
    fenc = [np.clip(p.astype(np.int32) + rng.integers(-3, 4, p.shape) * (1 << (depth - 8)), 0, (1 << depth) - 1).astype(p.dtype)
            for p in rec]
    params, _ = S.make_params(rng, W, H, 64, depth)
    assert np.array_equal(device_stats(cu, depth, rec, fenc, 64), S.oracle_stats(depth, rec, fenc, 64))
    want = S.oracle_apply(depth, rec, 64, params, 1, 1, units, fenc)
    assert_planes_equal(device_apply(cu, depth, rec, 64, params, 1, 1, units, fenc), want, "2160p")


@pytest.mark.parametrize("depth", [8, 10])
def test_sao_luma_only_equals_luma_of_three_planes(cu, depth):
    rng = np.random.default_rng(500 + depth)
    rec, fenc = S.make_pictures(rng, 200, 136, depth)
    params, _ = S.make_params(rng, 200, 136, 32, depth)
    st3 = device_stats(cu, depth, rec, fenc, 32)
    st1 = device_stats(cu, depth, [rec[0], None, None], [fenc[0], None, None], 32)
    assert np.array_equal(st1[:, :, 0], st3[:, :, 0]) and not st1[:, :, 1:].any()
    both = device_apply(cu, depth, rec, 32, params, 1, 1, None, fenc)
    alone = device_apply(cu, depth, [rec[0], None, None], 32, params, 1, 0, None, [fenc[0], None, None])
    assert np.array_equal(alone[0], both[0]) and alone[1] is None


def test_sao_out_of_range_records(cu):
    """Any byte values in the records: types outside -1..4 are off, bandPos is read & 31, offsets of any int8 are clipped."""
    depth = 8
    rng = np.random.default_rng(77)
    rec, fenc = S.make_pictures(rng, 200, 136, depth)
    n = S.num_ctus(200, 136, 32)
    raw = rng.integers(0, 256, (3, n, 8)).astype(np.uint8)
    params = raw.view(S.SAO_CTU).reshape(3, n)
    fixed = params.copy()
    t = fixed["typeIdx"]
    fixed["typeIdx"] = np.where((t < -1) | (t > 4), -1, t)
    fixed["bandPos"] &= 31
    got = device_apply(cu, depth, rec, 32, params, 1, 1, None, fenc)
    assert_planes_equal(got[:2], S.oracle_apply(depth, rec, 32, fixed, 1, 1, None, fenc)[:2], "records")


@pytest.mark.timeout(300)
@pytest.mark.parametrize("depth", [8, 10])
def test_sao_recon_loop_on_analyser(cu, depth):
    """recon_to_ref / recon_to_ref_chroma, x265cu_deblock_frame, x265cu_sao_stats_frame on src_plane and the reference, a
    decision the test derives from the device statistics, x265cu_sao_apply_frame, ref_updated / ref_chroma_updated: the
    reference allocations, margins included, equal those of a second analyser set from the host with the oracle's picture,
    and the next analysis run gives identical outputs on both."""
    from frame_helpers import Workload, MARGIN_X, MARGIN_Y
    from chroma_helpers import chroma_inner
    from test_gpu_x_chroma_residual import open_analyser, source
    W, H, ctu = 200, 136, 64
    wl = Workload(W, H, depth=depth, numRefs=2, method=3, subme=3, merange=57, rect=1, qp=30, chroma=True)
    a = open_analyser(cu, wl)
    a.analyse(source(wl), wl.field, stages=15)
    rows = a.ctu_rows
    a.recon_to_ref(3, 0, 0, rows)
    a.recon_to_ref_chroma(3, 0, 0, rows)
    luma = np.ascontiguousarray(a.fetch("recon3").reshape(wl.fenc.shape)[MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W])
    chroma = [np.ascontiguousarray(chroma_inner(wl, a.fetch_chroma(("recon", 3, k)))) for k in range(2)]
    fenc = [np.ascontiguousarray(wl.fenc[MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W])] + \
           [np.ascontiguousarray(chroma_inner(wl, wl.fencC[k])) for k in range(2)]
    rng = np.random.default_rng(88 + depth)
    units = D.make_map(rng, W, H, 64, depth, B_SLICE, p_bypass=0.05)
    prm = D.params_array(B_SLICE, 0, 1, 0, 0, 1)
    dbk = list(D.oracle_deblock(depth, luma, chroma[0], chroma[1], units, prm))
    ostats = S.oracle_stats(depth, dbk, fenc, ctu)

    ubuf = cu.to_device(units)
    y, ys = a.ref_plane_ptr(0)
    (u, cs), (v, _) = a.ref_plane_chroma(0, 0), a.ref_plane_chroma(0, 1)
    cu.deblock_frame(depth, y, ys, u, v, cs, W, H, ubuf, dparams(prm))
    src = [a.src_plane(k) for k in range(3)]
    n = S.num_ctus(W, H, ctu)
    sbuf = cu.to_device(np.full(n * SAO_STATS_PER_CTU, -1, np.int32))
    cu.sao_stats_frame(depth, W, H, ctu, [s[0] for s in src], src[0][1], src[1][1], (y, u, v), ys, cs, sbuf)
    dstats = sbuf.download(np.int32).reshape((n,) + S.STATS_SHAPE)
    assert np.array_equal(dstats, ostats), "device statistics"
    params = decide(dstats, depth)
    pbuf = cu.to_device(params)
    cu.sao_apply_frame(depth, W, H, ctu, (y, u, v), ys, cs, pbuf, 1, 1, ubuf, [s[0] for s in src], src[0][1], src[1][1])
    a.ref_updated(0)
    a.ref_chroma_updated(0)
    want = S.oracle_apply(depth, dbk, ctu, params, 1, 1, units, fenc)

    b = open_analyser(cu, wl)
    b.set_ref(0, want[0])
    b.set_ref_chroma(0, want[1], want[2])
    assert np.array_equal(a.fetch(("plane", 0, 0)), b.fetch(("plane", 0, 0))), "luma reference allocation"
    for k in range(2):
        assert np.array_equal(a.fetch_chroma(("ref", 0, k)), b.fetch_chroma(("ref", 0, k))), ("chroma reference allocation", k)

    nxt = Workload(W, H, depth=depth, numRefs=2, method=3, subme=3, merange=57, rect=1, qp=30, chroma=True, seed=266)
    res = []
    for an in (a, b):
        an.load_inputs(source(nxt), wl.field)
        an.run_resident(7)
        cu.sync()
        r = dict(me=an.fetch("me_out"), coef=an.fetch("coef"), recon=[an.fetch("recon%d" % d) for d in range(4)])
        an.analyse(source(nxt), wl.field, stages=7)
        r.update(sse=an.cu_sse.copy(), numsig=an.cu_numsig.copy(), ref=an.cu_ref.copy(), intra=an.intra_cost.copy(), packed=an.me_packed.copy())
        res.append(r)
    for k in res[0]:
        x, z = res[0][k], res[1][k]
        assert all(np.array_equal(p, q) for p, q in zip(x, z)) if k == "recon" else np.array_equal(x, z), k
    for buf in (ubuf, sbuf, pbuf):
        buf.free()
    a.close()
    b.close()


def decide(stats, depth):
    """A deterministic stand-in for the host's decision: per CTU and plane, the type with the most samples whose class
    offsets are the rounded mean differences (clipped to OFFSET_THRESH - 1); BO takes the 4 bands from the fullest one."""
    n = stats.shape[0]
    t = S.offset_thresh(depth) - 1
    out = np.zeros((3, n), S.SAO_CTU)
    for a in range(n):
        for p in range(3):
            cnt, org = stats[a, 0, p].astype(np.int64), stats[a, 1, p].astype(np.int64)
            ty = int(np.argmax(cnt.sum(axis=1)))
            if p == 2:
                ty = int(out[1, a]["typeIdx"])
            if ty == 4:
                band = int(np.argmax(cnt[4]))
                cls = [(band + i) & 31 for i in range(4)]
            else:
                cls = [1, 2, 3, 4]
            off = [int(np.clip(np.rint(org[ty, k] / cnt[ty, k]) if cnt[ty, k] else 0, -t, t)) for k in cls]
            out[p, a]["typeIdx"] = ty
            out[p, a]["bandPos"] = cls[0] if ty == 4 else 0
            out[p, a]["offset"] = off
    return out


def test_sao_refusals(cu):
    """Each argument rule returns -1 with a message before any launch and leaves the buffers alone."""
    depth, W, H, ctu = 8, 64, 32, 32
    rng = np.random.default_rng(6)
    rec, fenc = S.make_pictures(rng, W, H, depth)
    params, _ = S.make_params(rng, W, H, ctu, depth)
    units = D.make_map(rng, W, H, ctu, depth, B_SLICE, p_bypass=0.2)
    Y, U, V = [cu.to_device(p) for p in rec]
    FY, FU, FV = [cu.to_device(p) for p in fenc]
    n = S.num_ctus(W, H, ctu)
    ST = cu.to_device(np.full(n * SAO_STATS_PER_CTU, 7, np.int32))
    PR, UN = cu.to_device(params), cu.to_device(units)
    L = cu.L
    sgood = dict(depth=8, width=W, height=H, ctu=ctu, fy=FY.ptr, fcb=FU.ptr, fcr=FV.ptr, fs=W, fcs=W // 2, y=Y.ptr, cb=U.ptr,
                 cr=V.ptr, s=W, cs=W // 2, stats=ST.ptr)
    agood = dict(depth=8, width=W, height=H, ctu=ctu, y=Y.ptr, cb=U.ptr, cr=V.ptr, s=W, cs=W // 2, params=PR.ptr, sl=1, sc=1,
                 units=UN.ptr, fy=FY.ptr, fcb=FU.ptr, fcr=FV.ptr, fs=W, fcs=W // 2)

    def stats(**kw):
        a = dict(sgood, **kw)
        return L.x265cu_sao_stats_frame(cu.ctx, a["depth"], a["width"], a["height"], a["ctu"], a["fy"], a["fcb"], a["fcr"], a["fs"],
                                        a["fcs"], a["y"], a["cb"], a["cr"], a["s"], a["cs"], a["stats"])

    def apply(**kw):
        a = dict(agood, **kw)
        return L.x265cu_sao_apply_frame(cu.ctx, a["depth"], a["width"], a["height"], a["ctu"], a["y"], a["cb"], a["cr"], a["s"],
                                        a["cs"], a["params"], a["sl"], a["sc"], a["units"], a["fy"], a["fcb"], a["fcr"], a["fs"], a["fcs"])

    common = [dict(depth=9), dict(width=0), dict(width=68), dict(height=-8), dict(height=36), dict(ctu=8), dict(ctu=128),
              dict(s=W - 1), dict(cs=W // 2 - 1), dict(y=None), dict(cb=None), dict(cr=None)]
    bad = [(stats, kw) for kw in common + [dict(stats=None), dict(fy=None), dict(fcb=None), dict(fs=W - 1), dict(fcs=W // 2 - 1),
                                           dict(fcb=None, fcr=None)]]
    bad += [(apply, kw) for kw in common + [dict(params=None), dict(sl=2), dict(sc=-1), dict(cb=None, cr=None),
                                            dict(fy=None), dict(fcb=None), dict(fcb=None, fcr=None), dict(fs=W - 1)]]
    for f, kw in bad:
        k = cu.launch_count()
        assert f(**kw) == -1 and cu.last_error(), (f.__name__, kw)
        assert cu.launch_count() == k, (f.__name__, kw)
    cu.sync()
    for buf, img in ((Y, rec[0]), (U, rec[1]), (V, rec[2])):
        assert np.array_equal(buf.download(pixel_dtype(depth)).reshape(img.shape), img)
    assert (ST.download(np.int32) == 7).all()
    assert stats() == 0 and apply() == 0 and apply(cb=None, cr=None, sc=0, fcb=None, fcr=None) == 0 and apply(units=None, fy=None, fcb=None, fcr=None) == 0
    cu.sync()
    for b in (Y, U, V, FY, FU, FV, ST, PR, UN):
        b.free()
