"""GPU parity of the frame analyser's 4:2:0 chroma residual stage (stage bit 3, x265_b200/csrc/resid.cuh) against the
oracle's frame driver, which tests/test_chroma_residual_oracle_vs_ref.py pins to the real reference code: chroma levels, chroma
recon planes and per-CU chroma SSE / numSig, with the luma outputs of the same run.  Row shards, promotion of the chroma recon
to a reference, a second frame searched on the device-reconstructed references, and the refusals.  Kept in a file that sorts
last so that a fault here cannot disturb the verified tests."""
import ctypes as C

import numpy as np
import pytest

from chroma_helpers import cpu_analyse_chroma, chroma_inner, load_oracle_chroma
from frame_helpers import Workload, lambda_for, assert_frame_equal, pad_plane, pad_plane_c, MARGIN_X, MARGIN_Y
from me_helpers import mvcost_table

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cu():
    import x265_b200
    return x265_b200.load()


def inner(c, W, H):
    mx, my = MARGIN_X // 2, MARGIN_Y // 2
    return np.ascontiguousarray(c[my:my + H // 2, mx:mx + W // 2])


def open_analyser(cu, wl, offsets=(0, 0)):
    """An analyser with the workload's references and source chroma resident and the chroma residual enabled."""
    import x265_b200
    p, W, H = wl.params, wl.W, wl.H
    an = x265_b200.Analyser(cu, W, H, depth=wl.depth, numRefs=p["numRefs"], method=p["method"], subme=p["subme"],
                            merange=p["merange"], rect=p["rect"], qp=p["qp"], lam=lambda_for(p["qp"], wl.depth), amp=p["amp"])
    an.enable_chroma()
    an.enable_chroma_residual(*offsets)
    for r, ref in enumerate(wl.refs):
        an.set_ref(r, ref[MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W])
        an.set_ref_chroma(r, inner(wl.refC[r][0], W, H), inner(wl.refC[r][1], W, H))
    an.load_chroma(inner(wl.fencC[0], W, H), inner(wl.fencC[1], W, H))
    return an


def source(wl):
    return np.ascontiguousarray(wl.fenc[MARGIN_Y:MARGIN_Y + wl.H, MARGIN_X:MARGIN_X + wl.W])


def oracle(wl, offsets=(0, 0), max_ctu_rows=0):
    O = load_oracle_chroma(wl.depth)
    tab = mvcost_table(O, lambda_for(wl.params["qp"], wl.depth))
    return cpu_analyse_chroma(O, "orc_analyse_frame_chroma", wl, tab, offsets=offsets, threads=8, max_ctu_rows=max_ctu_rows)


def assert_chroma_equal(an, want, wl, ncu=None, rows=None):
    """The device's chroma outputs against the CPU driver's (CUs [0, ncu) and chroma rows [0, rows) when given)."""
    ncu = an.ncu if ncu is None else ncu
    assert an.chroma_qp() == tuple(want["qpc"])
    sse, numsig = an.chroma_results()
    assert np.array_equal(numsig[:ncu], want["cu_numsig_c"][:ncu]), "chroma numSig"
    assert np.array_equal(sse[:ncu], want["cu_sse_c"][:ncu]), "chroma SSE"
    nlev = an.ncoef // 4 if ncu == an.ncu else int(want["cu_coef_off"][ncu]) // 4
    for k, name in enumerate(("coef_cb", "coef_cr")):
        assert np.array_equal(an.fetch_chroma(name)[:nlev], want["coef_c"][k][:nlev]), name
    for d in range(4):
        for k in range(2):
            got = chroma_inner(wl, an.fetch_chroma(("recon", d, k)))
            exp = chroma_inner(wl, want["recon_c"][d][k])
            if rows is not None:
                got, exp = got[:rows], exp[:rows]
            assert np.array_equal(got, exp), ("chroma recon", d, k)


PARITY = [(W, H, d, noise) for W, H in ((200, 136), (256, 128)) for d in (8, 10) for noise in (False, True)]


@pytest.mark.timeout(300)
@pytest.mark.parametrize("W,H,depth,noise", PARITY, ids=["%dx%d-%d-%s" % (c[0], c[1], c[2], "noise" if c[3] else "smooth") for c in PARITY])
def test_chroma_residual_parity(cu, W, H, depth, noise):
    wl = Workload(W, H, depth=depth, numRefs=2, method=3, subme=3, merange=57, rect=1, qp=30, noise=noise, chroma=True)
    want = oracle(wl)
    an = open_analyser(cu, wl)
    an.analyse(source(wl), wl.field, stages=15)
    assert_frame_equal(an, want, wl)
    assert_chroma_equal(an, want, wl)
    an.close()


CASES = [("amp10_offsets", 10, dict(amp=1, subme=4, noise=True), (-12, 12)), ("offsets8", 8, dict(noise=True), (12, -12)),
         ("far8", 8, dict(field="far", motion=(0, 0)), (0, 0)), ("far10", 10, dict(field="far"), (0, 0)),
         ("mixed8", 8, dict(field="mixed"), (0, 0)), ("cut10", 10, dict(content="cut", qp=3), (0, 0))]


@pytest.mark.timeout(300)
@pytest.mark.parametrize("name,depth,opts,offsets", CASES, ids=[c[0] for c in CASES])
def test_chroma_residual_cases(cu, name, depth, opts, offsets):
    """10-bit rect + AMP, the chroma QP offsets at both ends of their range, vectors at the search clamps ("far") and mixed
    vectors, and a cut from black at a low QP (DC-only TUs, the recon clip)."""
    kw = dict(numRefs=2, method=3, subme=3, merange=57, rect=1, qp=30, chroma=True)
    kw.update(opts)
    wl = Workload(200, 136, depth=depth, **kw)
    want = oracle(wl, offsets)
    an = open_analyser(cu, wl, offsets)
    an.analyse(source(wl), wl.field, stages=15)
    assert_frame_equal(an, want, wl)
    assert_chroma_equal(an, want, wl)
    an.close()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("depth", [8, 10])
def test_chroma_residual_leaves_luma(cu, depth):
    """Stages 1|2|4 give the same luma outputs and ME results with bit 3 as without it."""
    wl = Workload(200, 136, depth=depth, numRefs=2, method=3, subme=3, merange=57, rect=1, qp=30, noise=True, chroma=True)
    res = []
    for stages in (7, 15):
        an = open_analyser(cu, wl)
        an.analyse(source(wl), wl.field, stages=stages)
        res.append(dict(me=an.fetch("me_out"), coef=an.fetch("coef"), sse=an.cu_sse.copy(), ns=an.cu_numsig.copy(), ref=an.cu_ref.copy(),
                        intra=an.intra_cost.copy(), packed=an.me_packed.copy(), recon=[an.fetch("recon%d" % d) for d in range(4)]))
        an.close()
    for k in res[0]:
        a, b = res[0][k], res[1][k]
        assert all(np.array_equal(x, y) for x, y in zip(a, b)) if k == "recon" else np.array_equal(a, b), k


@pytest.mark.timeout(900)
def test_chroma_residual_full_size(cu):
    """3840x2160 8-bit, 4 references, chroma on (bench.py c3 geometry): the first 2 CTU rows against the CPU driver."""
    wl = Workload(3840, 2160, depth=8, numRefs=4, method=3, subme=3, merange=57, rect=1, qp=30, chroma=True)
    want = oracle(wl, max_ctu_rows=2)
    an = open_analyser(cu, wl)
    an.analyse_rows(source(wl), wl.field, 0, 2, stages=15)
    assert_chroma_equal(an, want, wl, ncu=want["ncu_run"], rows=64)
    an.close()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("depth", [8, 10])
def test_chroma_residual_shards_and_promotion(cu, depth):
    """Row shards reproduce a full-frame run; recon_to_ref_chroma + ref_chroma_updated make a reference of the chroma recon with
    its borders replicated as extendPicBorder does."""
    W, H = 200, 200
    wl = Workload(W, H, depth=depth, numRefs=2, method=3, subme=3, merange=57, rect=1, qp=30, noise=True, chroma=True)
    full = open_analyser(cu, wl)
    full.analyse(source(wl), wl.field, stages=15)
    want_sse, want_ns = full.chroma_results()
    shard = open_analyser(cu, wl)
    rows = shard.ctu_rows
    assert rows == 4
    sse, ns = np.zeros((shard.ncu, 2), np.uint64), np.zeros((shard.ncu, 2), np.uint32)
    for r0, r1 in ((0, 1), (1, 3), (3, 4)):
        shard.analyse_rows(source(wl), wl.field, r0, r1, stages=15)
        shard.chroma_results(r0, r1, sse, ns)
    assert np.array_equal(sse, want_sse) and np.array_equal(ns, want_ns)
    for name in ("coef_cb", "coef_cr"):
        assert np.array_equal(shard.fetch_chroma(name), full.fetch_chroma(name)), name
    for d in range(4):
        for k in range(2):
            assert np.array_equal(shard.fetch_chroma(("recon", d, k)), full.fetch_chroma(("recon", d, k))), (d, k)
    # promote depth 3 (8x8 CUs, which tile the picture) to reference 1, shard by shard, then extend the borders
    for r0, r1 in ((0, 2), (2, 4)):
        shard.recon_to_ref_chroma(3, 1, r0, r1)
    shard.ref_chroma_updated(1)
    for k in range(2):
        rec = chroma_inner(wl, shard.fetch_chroma(("recon", 3, k)))
        want, _, _ = pad_plane_c(rec, depth, shard.stride)
        assert np.array_equal(shard.fetch_chroma(("ref", 1, k)), want), k
    full.close()
    shard.close()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("depth", [8, 10])
def test_chroma_residual_closed_loop(cu, depth):
    """A second frame whose motion search (chroma-SATD term on) reads reference 0 = the device's 8x8-CU reconstruction of the
    first frame, luma and chroma, against the CPU driver fed the same planes."""
    W, H = 200, 136
    wl = Workload(W, H, depth=depth, numRefs=2, method=3, subme=3, merange=57, rect=1, qp=30, chroma=True)
    an = open_analyser(cu, wl)
    an.analyse(source(wl), wl.field, stages=15)
    rows = an.ctu_rows
    an.recon_to_ref(3, 0, 0, rows)
    an.ref_updated(0)
    an.recon_to_ref_chroma(3, 0, 0, rows)
    an.ref_chroma_updated(0)
    luma = an.fetch("recon3").reshape(wl.fenc.shape)[MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W]
    chroma = [chroma_inner(wl, an.fetch_chroma(("recon", 3, k))) for k in range(2)]
    # the next frame: the source moves on, reference 0 is the reconstruction
    nxt = Workload(W, H, depth=depth, numRefs=2, method=3, subme=3, merange=57, rect=1, qp=30, chroma=True, seed=266)
    wl.fenc, wl.fencC = nxt.fenc, nxt.fencC
    wl.refs[0] = pad_plane(np.ascontiguousarray(luma), depth)[0]
    wl.refC[0] = [pad_plane_c(np.ascontiguousarray(c), depth, wl.stride)[0] for c in chroma]
    want = oracle(wl)
    an.load_chroma(inner(wl.fencC[0], W, H), inner(wl.fencC[1], W, H))
    an.analyse(source(wl), wl.field, stages=15)
    assert_frame_equal(an, want, wl)
    assert_chroma_equal(an, want, wl)
    an.close()


def test_chroma_residual_refusals(cu):
    """Bit 3 without enable_chroma_residual, enable_chroma_residual before enable_chroma and an offset of 13: each returns -1
    with a message and launches nothing."""
    import x265_b200
    wl = Workload(200, 136, depth=8, numRefs=2, method=3, subme=3, merange=57, rect=1, qp=30, chroma=True)
    an = x265_b200.Analyser(cu, 200, 136, depth=8, numRefs=2, qp=30)
    L = cu.L

    def refused(call):
        n = cu.launch_count()
        assert call() == -1 and cu.last_error()
        assert cu.launch_count() == n
    refused(lambda: L.x265cu_analyser_enable_chroma_residual(an.h, 0, 0))
    an.load_inputs(source(wl), wl.field)
    refused(lambda: L.x265cu_analyser_run_resident(an.h, 15))
    an.enable_chroma()
    refused(lambda: L.x265cu_analyser_run_resident(an.h, 8))
    refused(lambda: L.x265cu_analyser_enable_chroma_residual(an.h, 13, 0))
    refused(lambda: L.x265cu_analyser_enable_chroma_residual(an.h, 0, -13))
    refused(lambda: L.x265cu_analyser_run_rows(an.h, 15, 0, 1))
    an.enable_chroma_residual(0, 0)
    an.run_resident(8)                     # before any search: vector 0 of every CU
    cu.sync()
    an.close()
