"""GPU parity of the frame analyser's B slices (x265cu_analyser_set_lists, stage bit 4) against the oracle's B-slice driver,
which tests/test_bidir_oracle_vs_ref.py pins to the real reference code: the BIDIR record of every CU and the luma and chroma
residual outputs, bi-predicted CUs included, on every CPU case and at 3840x2160 with 2+2 references; row shards; the return to
a P slice; the refusals; the record layout.  Kept in a file that sorts last."""
import ctypes as C

import numpy as np
import pytest

from bidir_helpers import (load_oracle_bidir, bidir_workload, cpu_analyse_bidir, stages_for, BidirCu, CASES, case_id)
from frame_helpers import assert_frame_equal, lambda_for, MARGIN_X, MARGIN_Y

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


def open_analyser(cu, wl, lists, chroma):
    """An analyser with the workload's references resident, the lists set, and with chroma: the chroma planes and residual."""
    import x265_b200
    p, W, H = wl.params, wl.W, wl.H
    an = x265_b200.Analyser(cu, W, H, depth=wl.depth, numRefs=p["numRefs"], method=p["method"], subme=p["subme"],
                            merange=p["merange"], rect=p["rect"], qp=p["qp"], lam=lambda_for(p["qp"], wl.depth), amp=p["amp"])
    if chroma:
        an.enable_chroma()
        an.enable_chroma_residual(0, 0)
    for r, ref in enumerate(wl.refs):
        an.set_ref(r, ref[MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W])
        if chroma:
            an.set_ref_chroma(r, inner(wl.refC[r][0], W, H), inner(wl.refC[r][1], W, H))
    if chroma:
        an.load_chroma(inner(wl.fencC[0], W, H), inner(wl.fencC[1], W, H))
    if lists is not None:
        an.set_lists(*lists)
    return an


def oracle(wl, n0, chroma, max_ctu_rows=0):
    return cpu_analyse_bidir(load_oracle_bidir(wl.depth), "orc", wl, n0, chroma, threads=8, max_ctu_rows=max_ctu_rows)


def assert_chroma_equal(an, want, wl, ncu=None, rows=None):
    from chroma_helpers import chroma_inner
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


def assert_bidir_equal(got, want):
    """Every BIDIR record byte for byte."""
    n = len(want)
    bad = np.nonzero((got.view(np.uint8).reshape(n, -1) != want.view(np.uint8).reshape(n, -1)).any(axis=1))[0]
    assert len(bad) == 0, (len(bad), got[bad[:4]].tolist(), want[bad[:4]].tolist())


@pytest.mark.timeout(300)
@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_bidir_parity(cu, case):
    depth, (n0, n1), chroma, (W, H), qp, kind = case
    wl = bidir_workload(W, H, depth, n0, n1, kind, qp=qp)
    want = oracle(wl, n0, chroma)
    an = open_analyser(cu, wl, (n0, n1), chroma)
    an.analyse(source(wl), wl.field, stages=stages_for(chroma))
    assert_bidir_equal(an.bidir_results(), want["bidir"])
    assert_frame_equal(an, want, wl)
    if chroma:
        assert_chroma_equal(an, want, wl)
    an.close()


@pytest.mark.timeout(900)
def test_bidir_c3_geometry(cu):
    """3840x2160 8-bit, 2+2 references, chroma on: the first 2 CTU rows against the oracle."""
    wl = bidir_workload(3840, 2160, 8, 2, 2, "between", qp=30)
    want = oracle(wl, 2, True, max_ctu_rows=2)
    an = open_analyser(cu, wl, (2, 2), True)
    an.analyse_rows(source(wl), wl.field, 0, 2, stages=stages_for(True))
    nj, nc = want["njobs_run"], want["ncu_run"]
    assert np.array_equal(an.fetch("me_out").reshape(-1, 4)[:nj, :3], want["me_out"][:nj, :3])
    assert_bidir_equal(an.bidir_results(0, 2)[:nc], want["bidir"][:nc])
    assert (want["bidir"][:nc]["interDir"] == 3).mean() > 0.5
    assert np.array_equal(an.cu_ref[:nc], want["cu_ref"][:nc])
    assert np.array_equal(an.cu_sse[:nc], want["cu_sse"][:nc]) and np.array_equal(an.cu_numsig[:nc], want["cu_numsig"][:nc])
    assert_chroma_equal(an, want, wl, ncu=nc, rows=64)
    an.close()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("depth", [8, 10])
def test_bidir_row_shards(cu, depth):
    """analyse_rows over a band partition gives the full-frame records and residual results."""
    wl = bidir_workload(200, 256, depth, 2, 2, "between")
    st = stages_for(True)
    full = open_analyser(cu, wl, (2, 2), True)
    full.analyse(source(wl), wl.field, stages=st)
    shard = open_analyser(cu, wl, (2, 2), True)
    rec = np.zeros_like(full.bidir_results())
    sse, ns = np.zeros((shard.ncu, 2), np.uint64), np.zeros((shard.ncu, 2), np.uint32)
    for r0, r1 in ((2, 4), (0, 1), (1, 2)):
        shard.analyse_rows(source(wl), wl.field, r0, r1, stages=st)
        shard.bidir_results(r0, r1, rec)
        shard.chroma_results(r0, r1, sse, ns)
    assert rec.tobytes() == full.bidir_results().tobytes()
    assert np.array_equal(shard.fetch("coef"), full.fetch("coef")) and np.array_equal(shard.cu_ref, full.cu_ref)
    assert np.array_equal(shard.cu_sse, full.cu_sse) and np.array_equal(shard.cu_numsig, full.cu_numsig)
    want_sse, want_ns = full.chroma_results()
    assert np.array_equal(sse, want_sse) and np.array_equal(ns, want_ns)
    full.close()
    shard.close()


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
def test_bidir_back_to_p(cu, depth):
    """After B runs, set_lists(numRefs, 0) gives results byte-identical to a never-B analyser on the same inputs."""
    wl = bidir_workload(200, 136, depth, 2, 2, "between")
    plain = open_analyser(cu, wl, None, True)
    plain.analyse(source(wl), wl.field, stages=15)
    base = results(plain)
    an = open_analyser(cu, wl, (2, 2), True)
    an.analyse(source(wl), wl.field, stages=stages_for(True))
    assert (an.bidir_results()["interDir"] == 3).any()
    assert not np.array_equal(an.cu_sse, base["sse"])
    an.set_lists(4, 0)
    an.analyse(source(wl), wl.field, stages=15)
    same_results(results(an), base)
    plain.close()
    an.close()


def test_bidir_refusals(cu):
    """Each refusal returns -1 with a reason, launches nothing and changes nothing: the next run reproduces the last."""
    from wref_helpers import entry
    wl = bidir_workload(200, 136, 8, 1, 1, "between")
    L = cu.L
    an = open_analyser(cu, wl, None, True)
    n = cu.launch_count()
    assert L.x265cu_analyser_run_resident(an.h, 16) == -1 and cu.last_error()       # value 16 on a P slice
    assert cu.launch_count() == n
    for n0, n1 in ((0, 2), (1, -1), (1, 2), (3, 0), (2, 1)):
        assert L.x265cu_analyser_set_lists(an.h, n0, n1) == -1 and cu.last_error()
    an.set_lists(1, 1)
    an.analyse(source(wl), wl.field, stages=stages_for(True))
    before = results(an)
    rec = an.bidir_results().copy()
    an.load_inputs(source(wl), wl.field)
    for st in (2, 8, 10, 1 | 2, 1 | 8):                              # B-slice residuals without value 16
        n = cu.launch_count()
        assert L.x265cu_analyser_run_resident(an.h, st) == -1 and cu.last_error()
        assert cu.launch_count() == n
    an.set_ref_weights(0, np.array([entry(40, 5, 3)] * 3, np.int32))
    n = cu.launch_count()
    for st in (1, 16 | 2, 4):                                       # any B-slice run while a slot is weighted
        assert L.x265cu_analyser_run_resident(an.h, st) == -1 and cu.last_error()
    assert cu.launch_count() == n
    an.set_ref_weights(0, None)
    an.analyse(source(wl), wl.field, stages=stages_for(True))
    same_results(results(an), before)
    assert an.bidir_results().tobytes() == rec.tobytes()
    an.close()


def test_bidir_record_layout(cu):
    """x265cu_bidir_cu as ctypes sees it, and the numpy record of Analyser.bidir_results."""
    from x265_b200.lib import BIDIR_CU
    assert C.sizeof(BidirCu) == BIDIR_CU.itemsize == 20
    for name in ("uniCost", "biCost", "interDir", "ref", "zero", "mv"):
        assert getattr(BidirCu, name).offset == BIDIR_CU.fields[name][1], name
