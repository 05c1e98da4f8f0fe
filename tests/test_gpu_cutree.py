"""x265cu_cutree (cuTree's propagation chain on the device) against the restatement oracle/oracle_cutree.c, which
tests/test_cutree_oracle_vs_ref.py pins to the real Lookahead::cuTree: every frame's whole propagateCost array and the
finish list, bit for bit, over the pin's windows (saturation and the int32 wrap included), the launch shapes of 1080p and
2160p with a 40-frame window, and one end-to-end window on the device lookahead (Lookahead.cu_tree) finished on the host."""
import ctypes as C

import numpy as np
import pytest

import cutree_helpers as T
from x265_b200.lib import CutreeFrame, CutreeParams

pytestmark = pytest.mark.gpu
CASES = T.cases()


@pytest.fixture(scope="module")
def cu():
    import x265_b200
    return x265_b200.load()


class DeviceWindow:
    """The window's arrays on the device, propagateCost filled with the shim's pattern."""

    def __init__(self, cu, win):
        self.cu, self.win, self.bufs = cu, win, []
        self.recs = (CutreeFrame * win.n)()
        self.prop = {}
        for f in range(win.n):
            r = self.recs[f]
            r.intraCost = self._put(win.intra[f], np.int32)
            r.invQscale = self._put(win.invq[f], np.int32)
            r.propagateCost = self._put(T.pattern(f, win.ncu), np.uint16)
            self.prop[r.propagateCost] = self.bufs[-1]
            r.sliceType = win.types[f]
        for (b, d0, d1), a in win.costs.items():
            self.recs[b].lowresCosts[d0][d1] = self._put(a, np.uint16)
        for (b, lst, dist), a in win.mvs.items():
            self.recs[b].mvs[lst][dist] = self._put(a, np.int32)
        p = win.prm
        self.prm = CutreeParams(p["bIntra"], p["lookaheadDepth"], p["bBPyramid"], p["bEnableWeightedBiPred"], p["vbv"], p["fpsNum"], p["fpsDenom"])

    def _put(self, a, dt):
        a = np.ascontiguousarray(a, dt)
        b = self.cu.alloc(max(a.nbytes, 4))
        b.upload(a)
        self.bufs.append(b)
        return b.ptr

    def reset(self):
        for f in range(self.win.n):
            self.prop[self.recs[f].propagateCost].upload(T.pattern(f, self.win.ncu))

    def run(self):
        fin = np.zeros(2 * (self.win.n + 2), np.int32)
        nf = self.cu.L.x265cu_cutree(self.cu.ctx, self.recs, self.win.n - 1, C.byref(self.prm), self.win.w8, self.win.h8,
                                     fin.ctypes.data, self.win.n + 2)
        assert nf >= 0, self.cu.last_error()
        self.cu.sync()
        props = [self.prop[self.recs[f].propagateCost].download(np.uint16, self.win.ncu) for f in range(self.win.n)]
        return props, [(int(fin[2 * k]), int(fin[2 * k + 1])) for k in range(nf)]

    def close(self):
        for b in self.bufs:
            b.free()


def _check(cu, win, runs=1):
    want, _, want_fin = win.oracle()
    d = DeviceWindow(cu, win)
    try:
        for r in range(runs):
            if r:
                d.reset()
            got, fin = d.run()
            assert fin == want_fin
            for f in range(win.n):
                assert np.array_equal(got[f], want[f]), "frame %d: %d words differ" % (f, int(np.sum(got[f] != want[f])))
    finally:
        d.close()


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_cutree_device_matches_oracle(cu, case):
    name, w8, h8, types, prm, kw = case
    _check(cu, T.synth_window(cu, name, w8, h8, types, prm, **kw))


@pytest.mark.parametrize("name,prm", [("pyr0", T.params(bBPyramid=0)), ("pyr1", T.params(bBPyramid=1)),
                                      ("vbv", T.params(vbv=1, bBPyramid=1))])
def test_cutree_device_matches_oracle_clip(cu, name, prm):
    _check(cu, T.clip_window(prm, T.CLIP_TYPES))


SHAPES = [("1080p_bf4_pyr", 120, 68, 4, 1, {}), ("2160p_bf4_pyr", 240, 135, 4, 1, {}), ("2160p_bf8", 240, 135, 8, 0, {}),
          ("2160p_one_cu", 240, 135, 4, 1, dict(mv="one_cu")), ("1080p_overflow", 120, 68, 3, 1, dict(amount="overflow"))]


@pytest.mark.parametrize("name,w8,h8,bf,pyr,kw", SHAPES, ids=[s[0] for s in SHAPES])
def test_cutree_device_shapes(cu, name, w8, h8, bf, pyr, kw):
    """A 40-frame window (41 frames) at the lowres CU grids of 1080p and 2160p; run twice, identical both times."""
    win = T.synth_window(cu, name, w8, h8, T.slice_types(41, bf), T.params(bBPyramid=pyr), **kw)
    _check(cu, win, runs=2)


def test_cutree_device_refusals(cu):
    win = T.synth_window(cu, "refusal", 9, 6, T.slice_types(9, 3), T.params())
    d = DeviceWindow(cu, win)
    try:
        fin = np.zeros(64, np.int32)
        run = lambda: cu.L.x265cu_cutree(cu.ctx, d.recs, win.n - 1, C.byref(d.prm), win.w8, win.h8, fin.ctypes.data, 32)
        # the chain reads the mini-GOP (4, 8) only (frame 0 is an earlier anchor): its middle B is (4, 8, 6)
        keep = d.recs[6].lowresCosts[2][2]
        d.recs[6].lowresCosts[2][2] = None
        assert run() == -1 and "not supplied" in cu.last_error()
        d.recs[6].lowresCosts[2][2] = keep
        keep = d.recs[6].invQscale
        d.recs[6].invQscale = None
        assert run() == -1 and "invQscale" in cu.last_error()
        d.recs[6].invQscale = keep
        assert cu.L.x265cu_cutree(cu.ctx, d.recs, win.n - 1, C.byref(d.prm), win.w8, win.h8, fin.ctypes.data, 0) == -1
        p0 = CutreeParams(0, 0, 0, 0, 0, 25, 1)               # lookaheadDepth 0, nothing after frame 0: the reference divides by 0
        one = (CutreeFrame * 1)(d.recs[0])
        assert cu.L.x265cu_cutree(cu.ctx, one, 0, C.byref(p0), win.w8, win.h8, fin.ctypes.data, 32) == -1
        got, f = d.run()                                          # nothing was launched by the refusals
        assert f
    finally:
        d.close()


def test_cutree_end_to_end_lookahead(cu):
    """The device lookahead's own estimates of the clip, then Lookahead.cu_tree; the host finishes the listed frames (the
    reference's real cuTreeFinish where oracle/_ref is built, else the restated one) and gets the reference's
    qpCuTreeOffset."""
    from frame_helpers import gen_luma
    from x265_b200.lookahead import Lookahead
    prm = T.params(bBPyramid=1)
    win = T.clip_window(prm, T.CLIP_TYPES)
    W, H = T.CLIP_SIZE
    la = Lookahead(cu, W, H, 8, len(T.CLIP_TYPES), keep_costs=True)
    try:
        assert (la.w8, la.h8) == (win.w8, win.h8)
        for i in range(win.n):
            la.init_frame(i, gen_luma(W, H, i, s1=17.0, s2=11.0, bits=8, noise=False))
            la.set_invqscale(i, win.invq[i])
        la.intra_batch(range(win.n))
        for i in range(win.n):
            assert np.array_equal(la.fr[i]["intraCost"].download(np.int32, la.ncu), win.intra[i])
        finish, costs = la.cu_tree(T.CLIP_TYPES, b_pyramid=True)
        want_prop, want_qp, want_fin = win.oracle()
        assert finish == want_fin and finish
        ref = T.load_ref_cutree(8)
        ref_qp = win.reference()[1] if ref is not None else want_qp
        for f, d in finish:
            assert np.array_equal(costs[f], want_prop[f]), f
            qp = win.reference_finish(f, d, costs[f]) if ref is not None else win.oracle_finish(f, d, costs[f])
            assert np.array_equal(qp, ref_qp[f], equal_nan=True), f
        with pytest.raises(ValueError, match="lives on rank"):
            la.cu_tree(T.CLIP_TYPES, world=2, rank=0)
    finally:
        la.close()
