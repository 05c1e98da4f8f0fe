"""GPU parity of the frame-level CTU-analysis pipeline (x265cu_analyser_*: job build -> batched
motionEstimate -> fused MC/residual/DCT/quant/IDCT/recon -> intra search) against the oracle driver,
which test_frame_oracle_vs_ref.py pins to the real reference code.  Every output array is compared
bit-exactly; full-size (2160p) runs are checked through size-independent properties in bench.py."""
import numpy as np
import pytest

from common import load_oracle
from frame_helpers import Workload, cpu_analyse, lambda_for, run_analyser, assert_frame_equal, MARGIN_X, MARGIN_Y
from me_helpers import mvcost_table

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cu():
    import x265_b200
    return x265_b200.load()


@pytest.mark.parametrize("depth", [8, 10])
@pytest.mark.parametrize("noise", [False, True])
@pytest.mark.parametrize("size", [(200, 136), (256, 128)])
def test_frame_analysis(cu, depth, noise, size):
    O = load_oracle(depth)
    qp = 30
    W, H = size
    wl = Workload(W, H, depth=depth, numRefs=2, method=3, subme=3, merange=57, rect=1, qp=qp, noise=noise)
    tab = mvcost_table(O, lambda_for(qp, depth))
    want = cpu_analyse(O, "orc_analyse_frame", wl, tab, threads=8)
    an = run_analyser(cu, wl)
    assert an.stride == wl.stride
    assert_frame_equal(an, want, wl)
    # border extension of the uploaded source plane
    vw = W + 2 * MARGIN_X      # columns past the right margin are stride padding
    assert np.array_equal(an.fetch("fenc").reshape(wl.fenc.shape)[:, :vw], wl.fenc[:, :vw])
    # packed D2H form
    assert np.array_equal(an.me_packed[:, 0], want["me_out"][:, 0])
    assert np.array_equal(an.me_packed[:, 1].view(np.uint32) & 0xffff, want["me_out"][:, 1].astype(np.uint32) & 0xffff)
    assert np.array_equal(an.me_packed[:, 1].view(np.uint32) >> 16, want["me_out"][:, 2].astype(np.uint32) & 0xffff)
    an.close()


@pytest.mark.parametrize("depth", [8, 10])
@pytest.mark.parametrize("mode,world", [("block", 2), ("cyclic", 2), ("block", 3)])
def test_row_shards_equal_full_frame(cu, depth, mode, world):
    """CTU-row shards (x265cu_analyser_*_rows): the shards' slices, computed by separate launches in any order,
    are bit-identical to the same entries of a full-frame run, and the recon rows promoted to a reference
    reproduce the full-frame reconstruction (sharding changes placement, never arithmetic; SURVEY 8(e))."""
    from x265_b200 import shard
    qp = 30
    W, H = 200, 200                                   # 4 CTU rows, the last one 8 pixels high
    wl = Workload(W, H, depth=depth, numRefs=2, method=3, subme=3, merange=57, rect=1, qp=qp, noise=True)
    full = run_analyser(cu, wl)
    want = {k: np.array(getattr(full, k)) for k in ("me_packed", "cu_sse", "cu_numsig", "cu_ref", "intra_cost")}
    want_coef = full.fetch("coef")
    want_recon = [full.fetch("recon%d" % d) for d in range(4)]
    nrows = full.ctu_rows
    assert nrows == 4
    full.close()

    import x265_b200
    p = wl.params
    an = x265_b200.Analyser(cu, W, H, depth=depth, numRefs=p["numRefs"], method=p["method"], subme=p["subme"],
                            merange=p["merange"], rect=p["rect"], qp=qp, lam=lambda_for(qp, depth))
    for r, ref in enumerate(wl.refs):
        an.set_ref(r, ref[MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W])
    fenc = np.ascontiguousarray(wl.fenc[MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W])
    for k in want:
        getattr(an, k)[...] = 0
    # the shards of all "ranks", highest rank first (order must not matter)
    seen_jobs = 0
    for g in reversed(range(world)):
        for r0, r1 in shard.row_blocks(nrows, g, world, mode):
            an.analyse_rows(fenc, wl.field, r0, r1)
            j0, nj, c0, nc = an.row_range(r0, r1)
            seen_jobs += nj
            assert np.array_equal(an.me_packed[j0:j0 + nj], want["me_packed"][j0:j0 + nj]), (g, r0, r1)
            assert an.d2h_bytes_rows(r0, r1) == nj * 8 + nc * 160
    assert seen_jobs == an.njobs
    for k in want:
        assert np.array_equal(getattr(an, k), want[k]), k
    assert np.array_equal(an.fetch("coef"), want_coef)
    for d in range(4):
        got = an.fetch("recon%d" % d).reshape(wl.fenc.shape)[MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W]
        exp = want_recon[d].reshape(wl.fenc.shape)[MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W]
        assert np.array_equal(got, exp), "recon depth %d" % d
    # promote the reconstructed rows (CU size 16 plane) to reference 1, row block by row block, then re-extend
    for g in range(world):
        for r0, r1 in shard.row_blocks(nrows, g, world, mode):
            an.recon_to_ref(2, 1, r0, r1)
    an.ref_updated(1)
    ptr, stride = an.ref_plane_ptr(1)
    assert stride == wl.stride
    es = 1 if depth == 8 else 2
    buf = np.zeros(stride * (H + 2 * MARGIN_Y), an.dtype)
    base = ptr - (MARGIN_Y * stride + MARGIN_X) * es
    cu.check(cu.L.x265cu_d2h(cu.ctx, buf.ctypes.data, base, buf.nbytes)); cu.sync()
    newref = buf.reshape(wl.fenc.shape)
    rec = want_recon[2].reshape(wl.fenc.shape)[MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W]
    assert np.array_equal(newref[MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W], rec)
    # borders replicated like extendPicBorder (pixel.cpp:1027-1041)
    vw = W + 2 * MARGIN_X
    padded = np.pad(rec, ((MARGIN_Y, MARGIN_Y), (MARGIN_X, MARGIN_X)), mode="edge")
    assert np.array_equal(newref[:, :vw], padded)
    an.close()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("depth,amp,noise", [(8, 0, False), (8, 0, True), (10, 1, False), (10, 1, True), (8, 1, True)])
def test_window_search_equals_global_search(cu, depth, amp, noise, monkeypatch):
    """The shared-memory-window integer search (me_window.cuh: TMA-staged window per CU group, column-walk raster) against
    the global-memory kernel (X265CU_ME_WINDOW=0) on the same frame: every motionEstimate result identical.  1024x576
    leaves most search windows unclipped by the picture edge (the small frames above are clipped almost everywhere)."""
    import x265_b200
    qp = 30
    W, H = 1024, 576
    nrefs = 3
    wl = Workload(W, H, depth=depth, numRefs=nrefs, method=3, subme=3, merange=57, rect=1, qp=qp, noise=noise, amp=amp)
    res = {}
    for mode in ("0", "1"):
        monkeypatch.setenv("X265CU_ME_WINDOW", mode)
        an = x265_b200.Analyser(cu, W, H, depth=depth, numRefs=nrefs, method=3, subme=3, merange=57, rect=1, qp=qp, lam=lambda_for(qp, depth), amp=amp)
        for r, ref in enumerate(wl.refs):
            an.set_ref(r, ref[MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W])
        fenc = np.ascontiguousarray(wl.fenc[MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W])
        an.analyse(fenc, wl.field, stages=1)
        res[mode] = (an.fetch("me_out").reshape(-1, 4).copy(), an.fetch("jobs"))
        an.close()
    a, b = res["0"][0], res["1"][0]
    bad = np.nonzero((a[:, :3] != b[:, :3]).any(axis=1))[0]
    assert len(bad) == 0, (len(bad), len(a), res["0"][1][bad[:4]].tolist(), a[bad[:4]].tolist(), b[bad[:4]].tolist())
