"""GPU parity of the frame analyser's weighted P-slice references (x265cu_analyser_set_ref_weights) against the oracle's frame
driver with weights, which tests/test_wref_oracle_vs_ref.py pins to the real reference code: the weighted search planes, every
ME result, the luma and chroma residual outputs, at 8 and 10 bit and at the c3 geometry; the Lookahead's weight table end to
end; row shards; reference updates; clearing and the identity entry; the refusals.  Kept in a file that sorts last."""
import numpy as np
import pytest

from chroma_helpers import chroma_inner
from frame_helpers import assert_frame_equal, lambda_for, MARGIN_X, MARGIN_Y, pad_plane, pad_plane_c
from wref_helpers import (load_oracle_wref, fade_workload, cpu_analyse_wref, table, entry, identity, plane_area, MIXES)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cu():
    import x265_b200
    return x265_b200.load()


def inner(c, W, H):
    mx, my = MARGIN_X // 2, MARGIN_Y // 2
    return np.ascontiguousarray(c[my:my + H // 2, mx:mx + W // 2])


def source(wl):
    return np.ascontiguousarray(wl.fenc[MARGIN_Y:MARGIN_Y + wl.H, MARGIN_X:MARGIN_X + wl.W])


def open_analyser(cu, wl, tab=None):
    """An analyser with the workload's (unweighted) references and source chroma resident, chroma residual on, and the weights."""
    import x265_b200
    p, W, H = wl.params, wl.W, wl.H
    an = x265_b200.Analyser(cu, W, H, depth=wl.depth, numRefs=p["numRefs"], method=p["method"], subme=p["subme"],
                            merange=p["merange"], rect=p["rect"], qp=p["qp"], lam=lambda_for(p["qp"], wl.depth), amp=p["amp"])
    an.enable_chroma()
    an.enable_chroma_residual(0, 0)
    for r, ref in enumerate(wl.refs):
        an.set_ref(r, ref[MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W])
        an.set_ref_chroma(r, inner(wl.refC[r][0], W, H), inner(wl.refC[r][1], W, H))
        if tab is not None:
            an.set_ref_weights(r, tab[r])
    an.load_chroma(inner(wl.fencC[0], W, H), inner(wl.fencC[1], W, H))
    return an


def oracle(wl, tab, max_ctu_rows=0):
    return cpu_analyse_wref(load_oracle_wref(wl.depth), "orc", wl, tab, threads=8, max_ctu_rows=max_ctu_rows)


def assert_chroma_equal(an, want, wl, ncu=None, rows=None):
    ncu = an.ncu if ncu is None else ncu
    sse, numsig = an.chroma_results()
    assert np.array_equal(numsig[:ncu], want["cu_numsig_c"][:ncu]), "chroma numSig"
    assert np.array_equal(sse[:ncu], want["cu_sse_c"][:ncu]), "chroma SSE"
    nlev = an.ncoef // 4 if ncu == an.ncu else int(want["cu_coef_off"][ncu]) // 4
    for k, name in enumerate(("coef_cb", "coef_cr")):
        assert np.array_equal(an.fetch_chroma(name)[:nlev], want["coef_c"][k][:nlev]), name
    for d in range(4):
        for k in range(2):
            got, exp = chroma_inner(wl, an.fetch_chroma(("recon", d, k))), chroma_inner(wl, want["recon_c"][d][k])
            if rows is not None:
                got, exp = got[:rows], exp[:rows]
            assert np.array_equal(got, exp), ("chroma recon", d, k)


def assert_planes_equal(an, want, wl):
    """What the search reads for every reference: luma phase 0 and both chroma planes, margins included."""
    for r in range(wl.params["numRefs"]):
        assert np.array_equal(plane_area(wl, an.fetch(("plane", r, 0))), plane_area(wl, want["planes"][0][r])), ("luma", r)
        for k in range(2):
            assert np.array_equal(plane_area(wl, an.fetch_search_chroma(r, k), True), plane_area(wl, want["planes"][1][r][k], True)), ("chroma", r, k)


PARITY = [(d, noise, mix) for d in (8, 10) for noise in (False, True) for mix in ("one", "two", "three")]


@pytest.mark.timeout(300)
@pytest.mark.parametrize("depth,noise,mix", PARITY, ids=["%d-%s-%s" % (c[0], "noise" if c[1] else "smooth", c[2]) for c in PARITY])
def test_weighted_parity(cu, depth, noise, mix):
    rows = MIXES[mix](depth)
    wl = fade_workload(200, 136, depth, numRefs=len(rows), noise=noise)
    tab = table(rows)
    want = oracle(wl, tab)
    an = open_analyser(cu, wl, tab)
    an.analyse(source(wl), wl.field, stages=15)
    assert_frame_equal(an, want, wl)
    assert_chroma_equal(an, want, wl)
    assert_planes_equal(an, want, wl)
    an.close()


@pytest.mark.timeout(900)
def test_weighted_c3_geometry(cu):
    """3840x2160 8-bit, 4 references (two weighted), STAR, subme 3: the first 2 CTU rows against the oracle."""
    rows = MIXES["three"](8) + [None]
    wl = fade_workload(3840, 2160, 8, numRefs=4, gains=(0.62, 0.7, 0.78, 0.9))
    tab = table(rows)
    want = oracle(wl, tab, max_ctu_rows=2)
    an = open_analyser(cu, wl, tab)
    an.analyse_rows(source(wl), wl.field, 0, 2, stages=15)
    nj, nc = want["njobs_run"], want["ncu_run"]
    me = an.fetch("me_out").reshape(-1, 4)[:nj, :3]
    assert np.array_equal(me, want["me_out"][:nj, :3])
    assert np.array_equal(an.cu_ref[:nc], want["cu_ref"][:nc])
    assert np.array_equal(an.cu_sse[:nc], want["cu_sse"][:nc]) and np.array_equal(an.cu_numsig[:nc], want["cu_numsig"][:nc])
    assert_chroma_equal(an, want, wl, ncu=nc, rows=64)
    an.close()


@pytest.mark.timeout(300)
def test_weighted_lookahead_end_to_end(cu):
    """Lookahead.weight_analyse of a noisy fade (the weights tests' "noise_fade", P slice) gives a table with luma and chroma
    weighted; the analyser with that table equals the oracle with it."""
    from x265_b200.lookahead import Lookahead
    import weightp_helpers as WH
    W, H, depth = 328, 184, 8
    pics = WH.pictures("noise_fade", W, H, depth)
    la = Lookahead(cu, W, H, depth, 3)
    try:
        for i, (y, cb, cr) in enumerate(pics):
            la.init_frame(i, y, cb=cb, cr=cr, aq={"mode": 2, "weightp": True}, keep_chroma=True)
        la.intra_batch([0, 1, 2])
        la.cost(0, 1, 1)
        t = la.weight_analyse(1, "P", [0], WH.BFRAMES, [1])
    finally:
        la.close()
    assert t[0][0][0][0] == 1 and t[0][0][1][0] == 1, t[0][0]
    tab = t[0][:1]
    wl = fade_workload(W, H, depth, numRefs=1)
    wl.fenc = pad_plane(pics[1][0], depth)[0]
    wl.fencC = [pad_plane_c(pics[1][k], depth, wl.stride)[0] for k in (1, 2)]
    wl.refs = [pad_plane(pics[0][0], depth)[0]]
    wl.refC = [[pad_plane_c(pics[0][k], depth, wl.stride)[0] for k in (1, 2)]]
    want = oracle(wl, tab)
    an = open_analyser(cu, wl, tab)
    an.analyse(source(wl), wl.field, stages=15)
    assert_frame_equal(an, want, wl)
    assert_chroma_equal(an, want, wl)
    assert_planes_equal(an, want, wl)
    an.close()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("depth", [8, 10])
def test_weighted_row_shards(cu, depth):
    wl = fade_workload(200, 200, depth, numRefs=2, noise=True)
    tab = table(MIXES["two"](depth))
    full = open_analyser(cu, wl, tab)
    full.analyse(source(wl), wl.field, stages=15)
    shard = open_analyser(cu, wl, tab)
    sse, ns = np.zeros((shard.ncu, 2), np.uint64), np.zeros((shard.ncu, 2), np.uint32)
    for r0, r1 in ((2, 4), (0, 1), (1, 2)):
        shard.analyse_rows(source(wl), wl.field, r0, r1, stages=15)
        shard.chroma_results(r0, r1, sse, ns)
    assert np.array_equal(shard.me_packed, full.me_packed) and np.array_equal(shard.cu_ref, full.cu_ref)
    assert np.array_equal(shard.cu_sse, full.cu_sse) and np.array_equal(shard.cu_numsig, full.cu_numsig)
    assert np.array_equal(shard.fetch("coef"), full.fetch("coef"))
    want_sse, want_ns = full.chroma_results()
    assert np.array_equal(sse, want_sse) and np.array_equal(ns, want_ns)
    full.close()
    shard.close()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("depth", [8, 10])
def test_weighted_reference_updates(cu, depth):
    """After recon_to_ref + ref_updated (luma and chroma) and after set_ref with new pixels, the next run searches the weighted
    version of the new pixels."""
    W, H = 200, 136
    wl = fade_workload(W, H, depth, numRefs=2, noise=True)
    tab = table(MIXES["two"](depth))
    an = open_analyser(cu, wl, tab)
    an.analyse(source(wl), wl.field, stages=15)
    rows = an.ctu_rows
    an.recon_to_ref(3, 0, 0, rows)
    an.ref_updated(0)
    an.recon_to_ref_chroma(3, 0, 0, rows)
    an.ref_chroma_updated(0)
    luma = an.fetch("recon3").reshape(wl.fenc.shape)[MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W]
    chroma = [chroma_inner(wl, an.fetch_chroma(("recon", 3, k))) for k in range(2)]
    wl.refs[0] = pad_plane(np.ascontiguousarray(luma), depth)[0]
    wl.refC[0] = [pad_plane_c(np.ascontiguousarray(c), depth, wl.stride)[0] for c in chroma]
    want = oracle(wl, tab)
    an.analyse(source(wl), wl.field, stages=15)
    assert_frame_equal(an, want, wl)
    assert_chroma_equal(an, want, wl)
    assert_planes_equal(an, want, wl)
    # set_ref with other pixels: reference 0 becomes the source itself, faded
    other = fade_workload(W, H, depth, numRefs=2, noise=False, seed=300)
    wl.refs[0], wl.refC[0] = other.refs[0], other.refC[0]
    an.set_ref(0, wl.refs[0][MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W])
    an.set_ref_chroma(0, inner(wl.refC[0][0], W, H), inner(wl.refC[0][1], W, H))
    want = oracle(wl, tab)
    an.analyse(source(wl), wl.field, stages=15)
    assert_frame_equal(an, want, wl)
    assert_chroma_equal(an, want, wl)
    an.close()


def results(an):
    return dict(me=an.fetch("me_out"), coef=an.fetch("coef"), sse=an.cu_sse.copy(), ns=an.cu_numsig.copy(), ref=an.cu_ref.copy(),
                intra=an.intra_cost.copy(), packed=an.me_packed.copy(), coef_c=[an.fetch_chroma(n) for n in ("coef_cb", "coef_cr")],
                chroma=an.chroma_results(), recon=[an.fetch("recon%d" % d) for d in range(4)],
                recon_c=[an.fetch_chroma(("recon", d, k)) for d in range(4) for k in range(2)])


def same_results(a, b):
    for k in a:
        x, y = a[k], b[k]
        assert all(np.array_equal(p, q) for p, q in zip(x, y)) if isinstance(x, (list, tuple)) else np.array_equal(x, y), k


@pytest.mark.timeout(300)
@pytest.mark.parametrize("depth", [8, 10])
def test_weighted_clear_and_identity(cu, depth):
    """Set then clear gives a never-weighted analyser's results bit for bit; an identity entry leaves the search unchanged and
    matches the oracle, whose residual takes the 14-bit path."""
    wl = fade_workload(200, 136, depth, numRefs=2, noise=True)
    plain = open_analyser(cu, wl)
    plain.analyse(source(wl), wl.field, stages=15)
    base = results(plain)
    an = open_analyser(cu, wl, table(MIXES["two"](depth)))
    an.analyse(source(wl), wl.field, stages=15)
    weighted = results(an)
    assert not np.array_equal(weighted["me"], base["me"])
    an.set_ref_weights(0, None)
    an.analyse(source(wl), wl.field, stages=15)
    same_results(results(an), base)
    tab = table([[entry(64, 6, 0), identity(6), identity(6)], None])
    an.set_ref_weights(0, tab[0])
    an.analyse(source(wl), wl.field, stages=15)
    ident = results(an)
    assert np.array_equal(ident["me"], base["me"])
    want = oracle(wl, tab)
    assert_frame_equal(an, want, wl)
    assert_chroma_equal(an, want, wl)
    plain.close()
    an.close()


def test_weighted_refusals(cu):
    """Each bad argument returns -1 with a reason, launches nothing and changes nothing: the next run reproduces the last."""
    import ctypes as C
    wl = fade_workload(200, 136, 8, numRefs=2, noise=True)
    an = open_analyser(cu, wl, table(MIXES["two"](8)))
    an.analyse(source(wl), wl.field, stages=15)
    before = results(an)
    L = cu.L
    good = [1, 40, 5, 3]
    bad_entries = [[2, 40, 5, 3], [-1, 40, 5, 3], [1, 40, 8, 3], [1, 40, -1, 3], [1, 256, 5, 3], [1, -129, 5, 3], [1, 40, 5, 128],
                   [1, 40, 5, -129]]
    for bad in bad_entries:
        for k in range(3):
            e = np.array([good] * 3, np.int32)
            e[k] = bad
            n = cu.launch_count()
            assert L.x265cu_analyser_set_ref_weights(an.h, 1, e.ctypes.data) == -1 and cu.last_error()
            assert cu.launch_count() == n
    e = np.array([good] * 3, np.int32)
    for idx in (-1, 2, 16):
        assert L.x265cu_analyser_set_ref_weights(an.h, idx, e.ctypes.data) == -1 and cu.last_error()
    an.analyse(source(wl), wl.field, stages=15)
    same_results(results(an), before)
    an.close()
