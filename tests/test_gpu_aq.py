"""Adaptive quantisation on the device: x265cu_aq_energy's energies and plane totals equal the restatement
(oracle/oracle_aq.c, pinned to the real calcAdaptiveQuantFrame by tests/test_aq_oracle_vs_ref.py) on every picture of the
pin, on the largest grid and on padded strides; the refusals come before any launch; and the lookahead with
init_frame(aq=...) reproduces the reference's invQscaleFactor and the costs that follow from it."""
import ctypes as C

import numpy as np
import pytest

import aq_helpers as A

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cu():
    import x265_b200
    return x265_b200.load()


def _device_energy(cu, pic, W, H, depth, qg, pad=0):
    """x265cu_aq_energy on the planes uploaded with `pad` extra elements per row (noise in the padding)."""
    rng = np.random.default_rng(pad)
    ptrs, keep = [], []
    for k, pl in enumerate(pic):
        if pl is None:
            ptrs.append(None)
            continue
        h, w = pl.shape
        buf = rng.integers(0, 1 << depth, (h, w + pad)).astype(pl.dtype)
        buf[:, :w] = pl
        d = cu.to_device(buf)
        keep.append(d)
        ptrs.append(d.ptr)
    nb, _, _ = A.geometry(W, H, qg)
    e, t = cu.alloc(4 * nb), cu.alloc(48)
    rc = cu.L.x265cu_aq_energy(cu.ctx, depth, ptrs[0], W + pad, ptrs[1], ptrs[2], W // 2 + pad, W, H, qg, e.ptr, t.ptr)
    assert rc == 0, cu.last_error()
    cu.sync()
    return e.download(np.uint32, nb), t.download(np.uint64, 6)


@pytest.mark.parametrize("case", A.PICTURES, ids=[c[0] for c in A.PICTURES])
@pytest.mark.parametrize("qg", [8, 16])
def test_aq_energy_matches_oracle(cu, case, qg):
    name, W, H, depth, c420, content = case
    pic = A.make_picture(case)
    e, t = _device_energy(cu, pic, W, H, depth, qg)
    oe, ot = A.oracle_energy(pic, W, H, depth, qg)
    assert np.array_equal(e, oe) and np.array_equal(t, ot)


@pytest.mark.parametrize("depth,qg", [(10, 8), (8, 16)])
def test_aq_energy_2160p(cu, depth, qg):
    """3840x2160: at 10 bit and qgSize 8 the largest grid (480 x 270 blocks); both runs give the same result."""
    W, H = 3840, 2160
    pic = A.picture(W, H, depth, "fullrange")
    e, t = _device_energy(cu, pic, W, H, depth, qg)
    oe, ot = A.oracle_energy(pic, W, H, depth, qg)
    assert np.array_equal(e, oe) and np.array_equal(t, ot)
    e2, t2 = _device_energy(cu, pic, W, H, depth, qg)
    assert np.array_equal(e, e2) and np.array_equal(t, t2)


@pytest.mark.parametrize("pad", [6, 96])
def test_aq_energy_padded_strides(cu, pad):
    """Strides above the row, with noise past the picture: reads clamp to the picture, never into the padding."""
    W, H, depth = 328, 184, 10
    pic = A.picture(W, H, depth, "noise")
    for qg in (8, 32):
        e, t = _device_energy(cu, pic, W, H, depth, qg, pad)
        oe, ot = A.oracle_energy(pic, W, H, depth, qg)
        assert np.array_equal(e, oe) and np.array_equal(t, ot)


@pytest.mark.parametrize("what", ["aq-mode 4", "qgSize 12", "odd width", "one chroma", "depth 12", "narrow stride", "NULL out"])
def test_aq_refusals_before_launch(cu, what):
    from x265_b200.lib import AqOut, AqParams
    W, H, depth, qg = 64, 64, 8, 32
    y, cb, cr = (cu.to_device(p) for p in A.picture(W, H, 8, "noise"))
    e, t = cu.alloc(4 * 64), cu.alloc(48)
    args = dict(depth=depth, y=y.ptr, stride=W, cb=cb.ptr, cr=cr.ptr, cstride=W // 2, W=W, H=H, qg=qg, e=e.ptr, t=t.ptr)
    if what == "qgSize 12": args["qg"] = 12
    if what == "odd width": args["W"] = 63
    if what == "one chroma": args["cr"] = None
    if what == "depth 12": args["depth"] = 12
    if what == "narrow stride": args["stride"] = W - 2
    if what == "NULL out": args["t"] = None
    before = cu.launch_count()
    if what == "aq-mode 4":
        p = AqParams(aqMode=4, qgSize=qg, aqStrength=1.0)
        invq = cu.alloc(4 * 16)
        rc = cu.L.x265cu_aq_frame(cu.ctx, depth, y.ptr, W, cb.ptr, cr.ptr, W // 2, W, H, C.byref(p), invq.ptr, C.byref(AqOut()))
    else:
        a = args
        rc = cu.L.x265cu_aq_energy(cu.ctx, a["depth"], a["y"], a["stride"], a["cb"], a["cr"], a["cstride"], a["W"], a["H"], a["qg"],
                                   a["e"], a["t"])
    assert rc == -1 and cu.launch_count() == before, what
    assert "x265cu_aq_" in cu.last_error()


@pytest.mark.parametrize("depth,lslices", [(8, 8), (10, 0)])
def test_lookahead_init_frame_aq(cu, depth, lslices, request):
    """Lookahead.init_frame(..., aq=...) on the clip of test_gpu_lookahead.py's AQ case: every frame's resident invQscale
    equals the reference's invQscaleFactor, and costEstAq / rowSatds equal the oracle's (pinned to the reference) with no
    set_invqscale call."""
    from frame_helpers import gen_chroma
    from lookahead_helpers import OracleLookahead
    from test_lookahead_oracle_vs_ref import aq_inputs
    from x265_b200.lookahead import Lookahead, coop_slices
    from common import load_oracle
    W, H = 1280, 720
    frames, ref, _, invq = aq_inputs(request, depth, lslices, W, H)
    sl = coop_slices(H, lslices)
    la = Lookahead(cu, W, H, depth, len(frames), lookahead_slices=lslices)
    for i, img in enumerate(frames):
        la.init_frame(i, img, cb=gen_chroma(W, H, i, 1, bits=depth), cr=gen_chroma(W, H, i, 2, bits=depth),
                      aq=dict(mode=2, strength=1.0, qg_size=32))
        assert np.array_equal(la.fr[i]["invq"].download(np.int32), invq[i]), i
        assert la.fr[i]["qpAqOffset"].shape == (la.ncu,) and la.fr[i]["wp_sum"][0] > 0
    la.intra_batch(range(len(frames)))
    orc = OracleLookahead(load_oracle(depth), frames, depth, slices=sl if sl[0] > 1 else None, invq=invq)
    for (p0, p1, b) in [(0, 1, 1), (0, 2, 1), (0, 2, 2)]:
        a, c = la.cost(p0, p1, b), orc.cost(p0, p1, b)
        d0, d1 = b - p0, p1 - b
        r = la.fr[b]["res"][(d0, d1)]
        assert a == c and r["costEstAq"] == orc.fr[b]["costEst"][(d0, d1)][1], (p0, p1, b)
        assert np.array_equal(r["rowSatds"], orc.fr[b]["rowSatds"][(d0, d1)])
    la.close()


def test_lookahead_init_frame_aq_qg8_weightp(cu):
    """qgSize 8 with weightp and variance on a 4:2:0 frame: the resident invQscale is the restatement's invQscaleFactor8x8
    and the frame record holds its qpAqOffset, wp_sum / wp_ssd, blockVariance and frameVariance."""
    from x265_b200.lookahead import Lookahead
    W, H, depth = 640, 368, 8
    y, cb, cr = A.picture(W, H, depth, "smooth")
    la = Lookahead(cu, W, H, depth, 1)
    la.init_frame(0, y, cb=cb, cr=cr, aq=dict(mode=3, strength=1.0, qg_size=8, weightp=True, variance=True))
    want = A.oracle((y, cb, cr), W, H, depth, (3, 1.0, 8, 1, 1, 0))
    f = la.fr[0]
    assert np.array_equal(f["invq"].download(np.int32), want["invQscaleFactor8x8"])
    nb = A.geometry(W, H, 8)[0]
    assert np.array_equal(f["qpAqOffset"][:nb].view(np.uint64), want["qpAqOffset"][:nb].view(np.uint64))
    assert np.array_equal(f["wp_sum"], want["wp_sum"]) and np.array_equal(f["wp_ssd"], want["wp_ssd"])
    assert np.array_equal(f["blockVariance"][:nb], want["blockVariance"][:nb]) and f["frameVariance"] == want["frameVariance"]
    la.close()
