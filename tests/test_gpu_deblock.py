"""GPU: x265cu_deblock_frame against the plain-C restatement (oracle/oracle_deblock.c, which tests/test_deblock_oracle_vs_ref.py
pins to the real Deblock class), byte-exact: the pin's geometries and parameters, planes inside guard bands, 3840x2160 at 8 and
10 bit, luma-only calls, the recon -> deblock -> reference loop on the frame analyser, and the refusals."""
import ctypes as C

import numpy as np
import pytest

import deblock_helpers as D
from common import pixel_dtype
from x265_b200.lib import DEBLOCK_UNIT, DeblockParams, B_SLICE

pytestmark = pytest.mark.gpu
SENTINEL = 0xA5


@pytest.fixture(scope="module")
def cu():
    import x265_b200
    return x265_b200.load()


def dparams(prm):
    return DeblockParams(*[int(x) for x in prm])


class GuardedPlane:
    """A picture inside a larger device allocation filled with a sentinel: `rows_above` rows above, `cols_left` + `shift`
    pixels left of pixel (0,0), the same below / right; `stride` in pixels."""

    def __init__(self, cu, img, stride, rows_above=4, cols_left=8, shift=0):
        self.cu, self.h, self.w = cu, img.shape[0], img.shape[1]
        self.dtype, self.es = img.dtype, img.dtype.itemsize
        self.stride, self.rows = stride, self.h + 2 * rows_above
        self.total = self.stride * self.rows + 2 * cols_left + shift
        self.org = rows_above * stride + cols_left + shift
        host = np.full(self.total * self.es, SENTINEL, np.uint8).view(self.dtype).copy()
        view = host[self.org:self.org + (self.h - 1) * stride + self.w]
        for y in range(self.h):
            view[y * stride:y * stride + self.w] = img[y]
        self.expect_outside = host.copy()
        self.buf = cu.to_device(host)

    @property
    def ptr(self):
        return self.buf.ptr + self.org * self.es

    def download(self):
        return self.buf.download(self.dtype)

    def picture(self, whole):
        return np.stack([whole[self.org + y * self.stride:self.org + y * self.stride + self.w] for y in range(self.h)])

    def outside(self, whole):
        mask = np.ones(self.total, bool)
        for y in range(self.h):
            mask[self.org + y * self.stride:self.org + y * self.stride + self.w] = False
        return whole[mask], self.expect_outside[mask]

    def free(self):
        self.buf.free()


def device_deblock(cu, depth, luma, cb, cr, units, prm, stride=None, cstride=None, shift=0, check_guards=False):
    """Runs x265cu_deblock_frame on copies of the planes placed in guarded allocations; returns the host planes."""
    H, W = luma.shape
    stride = stride or W
    cstride = cstride or W // 2
    planes = [GuardedPlane(cu, luma, stride, shift=shift)]
    if cb is not None:
        planes += [GuardedPlane(cu, cb, cstride, shift=shift), GuardedPlane(cu, cr, cstride, shift=shift)]
    ubuf = cu.to_device(units)
    cu.deblock_frame(depth, planes[0].ptr, stride, planes[1].ptr if cb is not None else None, planes[2].ptr if cb is not None else None,
                     cstride, W, H, ubuf, dparams(prm))
    cu.sync()
    out = []
    for p in planes:
        whole = p.download()
        if check_guards:
            got, want = p.outside(whole)
            assert np.array_equal(got, want), "samples outside the picture changed"
        out.append(p.picture(whole))
        p.free()
    if check_guards:
        assert ubuf.download(np.uint8).tobytes() == units.tobytes(), "the unit map changed"
    ubuf.free()
    return out + [None] * (3 - len(out))


def assert_planes_equal(got, want, what):
    for k, (g, w) in enumerate(zip(got, want)):
        if w is None:
            assert g is None
            continue
        assert np.array_equal(g, w), (what, "plane %d" % k, int(np.count_nonzero(g != w)))


@pytest.mark.parametrize("case", D.cases(), ids=[c[0] for c in D.cases()])
def test_deblock_matches_oracle(cu, case):
    depth = case[1]
    luma, cb, cr, units, prm = D.case_inputs(case)
    want = D.oracle_deblock(depth, luma, cb, cr, units, prm)
    assert_planes_equal(device_deblock(cu, depth, luma, cb, cr, units, prm), want, case[0])


GUARDS = [(8, 200, 136, 216, 112, 0), (10, 200, 136, 256, 128, 0), (8, 200, 136, 203, 109, 1), (10, 136, 104, 141, 75, 1)]


@pytest.mark.parametrize("depth,W,H,stride,cstride,shift", GUARDS, ids=["%d-%dx%d-s%d-c%d-o%d" % g for g in GUARDS])
def test_deblock_guard_bands(cu, depth, W, H, stride, cstride, shift):
    """Planes inside larger sentinel-filled allocations: only the picture area changes, and the map is not written.  The
    third and fourth cases use strides that are not multiples of 16 bytes and a base one pixel past an aligned address."""
    rng = np.random.default_rng([depth, W, stride])
    units = D.make_map(rng, W, H, 64, depth, B_SLICE)
    luma, cb, cr = D.make_planes(rng, W, H, depth)
    prm = D.params_array(B_SLICE, 1, -1, 2, -3)
    want = D.oracle_deblock(depth, luma, cb, cr, units, prm)
    got = device_deblock(cu, depth, luma, cb, cr, units, prm, stride, cstride, shift, check_guards=True)
    assert_planes_equal(got, want, "guards")


def slow_map(rng, W, H, depth, slice_type):
    """A map shaped like preset slow's CU mix: CTU 64, mostly 16..32 CUs, rect and AMP PUs, some intra."""
    return D.make_map(rng, W, H, 64, depth, slice_type, p_intra=0.1, split={6: 0.85, 5: 0.6, 4: 0.35})


@pytest.mark.timeout(600)
@pytest.mark.parametrize("depth", [8, 10])
def test_deblock_2160p(cu, depth):
    rng = np.random.default_rng(2160 + depth)
    W, H = 3840, 2160
    units = slow_map(rng, W, H, depth, B_SLICE)
    luma, cb, cr = D.make_planes(rng, W, H, depth)
    prm = D.params_array(B_SLICE)
    want = D.oracle_deblock(depth, luma, cb, cr, units, prm)
    assert_planes_equal(device_deblock(cu, depth, luma, cb, cr, units, prm), want, "2160p")


@pytest.mark.parametrize("depth", [8, 10])
def test_deblock_luma_only_equals_luma_of_three_planes(cu, depth):
    rng = np.random.default_rng(400 + depth)
    units = D.make_map(rng, 200, 136, 32, depth, B_SLICE)
    luma, cb, cr = D.make_planes(rng, 200, 136, depth)
    prm = D.params_array(B_SLICE, -2, 3, 5, -5)
    both = device_deblock(cu, depth, luma, cb, cr, units, prm)
    alone = device_deblock(cu, depth, luma, None, None, units, prm)
    assert np.array_equal(alone[0], both[0]) and alone[1] is None


@pytest.mark.timeout(300)
@pytest.mark.parametrize("depth", [8, 10])
def test_deblock_recon_loop_on_analyser(cu, depth):
    """recon_to_ref / recon_to_ref_chroma, x265cu_deblock_frame on ref_plane / ref_plane_chroma, ref_updated /
    ref_chroma_updated: the whole reference allocations, margins included, equal those of a second analyser whose reference
    was set from the host with the oracle-deblocked picture, and the next analysis run gives identical outputs on both."""
    from frame_helpers import Workload, MARGIN_X, MARGIN_Y
    from chroma_helpers import chroma_inner
    from test_gpu_x_chroma_residual import open_analyser, source
    W, H = 200, 136
    wl = Workload(W, H, depth=depth, numRefs=2, method=3, subme=3, merange=57, rect=1, qp=30, chroma=True)
    a = open_analyser(cu, wl)
    a.analyse(source(wl), wl.field, stages=15)
    rows = a.ctu_rows
    a.recon_to_ref(3, 0, 0, rows)
    a.recon_to_ref_chroma(3, 0, 0, rows)
    luma = np.ascontiguousarray(a.fetch("recon3").reshape(wl.fenc.shape)[MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W])
    chroma = [np.ascontiguousarray(chroma_inner(wl, a.fetch_chroma(("recon", 3, k)))) for k in range(2)]
    rng = np.random.default_rng(77 + depth)
    units = D.make_map(rng, W, H, 64, depth, B_SLICE)
    prm = D.params_array(B_SLICE, 0, 1, 0, 0)
    want = D.oracle_deblock(depth, luma, chroma[0], chroma[1], units, prm)

    ubuf = cu.to_device(units)
    y, ys = a.ref_plane_ptr(0)
    (u, cs), (v, _) = a.ref_plane_chroma(0, 0), a.ref_plane_chroma(0, 1)
    cu.deblock_frame(depth, y, ys, u, v, cs, W, H, ubuf, dparams(prm))
    a.ref_updated(0)
    a.ref_chroma_updated(0)

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
    ubuf.free()
    a.close()
    b.close()


def test_deblock_refusals(cu):
    """Each argument rule returns -1 with a message before any launch and leaves the planes alone."""
    depth, W, H = 8, 64, 32
    rng = np.random.default_rng(5)
    units = D.make_map(rng, W, H, 64, depth, B_SLICE)
    luma, cb, cr = D.make_planes(rng, W, H, depth)
    Y, U, V, M = cu.to_device(luma), cu.to_device(cb), cu.to_device(cr), cu.to_device(units)
    L = cu.L
    good = dict(depth=8, luma=Y.ptr, stride=W, cb=U.ptr, cr=V.ptr, cstride=W // 2, width=W, height=H, units=M.ptr,
                prm=list(D.params_array(B_SLICE)))

    def call(**kw):
        a = dict(good)
        a.update(kw)
        prm = DeblockParams(*a["prm"])
        return L.x265cu_deblock_frame(cu.ctx, a["depth"], a["luma"], a["stride"], a["cb"], a["cr"], a["cstride"], a["width"],
                                      a["height"], a["units"], C.byref(prm))

    def prm_with(i, v):
        p = list(good["prm"])
        p[i] = v
        return p

    bad = [dict(depth=9), dict(width=0), dict(width=68), dict(height=-8), dict(height=36), dict(stride=W - 1), dict(cstride=W // 2 - 1),
           dict(prm=prm_with(0, 3)), dict(prm=prm_with(1, 7)), dict(prm=prm_with(2, -7)), dict(prm=prm_with(3, 13)),
           dict(prm=prm_with(4, -13)), dict(prm=prm_with(5, 2)), dict(luma=None), dict(units=None), dict(cb=None), dict(cr=None)]
    for kw in bad:
        n = cu.launch_count()
        assert call(**kw) == -1 and cu.last_error(), kw
        assert cu.launch_count() == n, kw
    cu.sync()
    for buf, img in ((Y, luma), (U, cb), (V, cr)):
        assert np.array_equal(buf.download(pixel_dtype(depth)).reshape(img.shape), img)
    assert call() == 0 and call(cb=None, cr=None) == 0
    cu.sync()
    for b in (Y, U, V, M):
        b.free()
