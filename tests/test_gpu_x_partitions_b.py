"""GPU parity of the frame analyser's PART_B stage (stage bit 6: the inter estimate of every partition of a B slice's CUs) against
the oracle's PART_B driver, which tests/test_part_b_oracle_vs_ref.py pins to the real reference code: every PART_B record byte
for byte on every CPU case and at 3840x2160; row bands; a PART_B-only run after an ME run; that the stage changes no other
output; the refusals; the record layout."""
import ctypes as C

import numpy as np
import pytest

from frame_helpers import Workload, lambda_for, MARGIN_X, MARGIN_Y
from part_b_helpers import load_oracle_part_b, cpu_analyse_part_b, case_workload, PartBCu, STAGES, CASES, case_id

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


def open_analyser(cu, wl, n0, chroma, chroma_residual=False):
    """An analyser of a B slice (list 0 = slots [0, n0)) with the workload's references resident and, with chroma, the chroma
    planes (and, with chroma_residual, the chroma residual stage)."""
    import x265_b200
    p, W, H = wl.params, wl.W, wl.H
    an = x265_b200.Analyser(cu, W, H, depth=wl.depth, numRefs=p["numRefs"], method=p["method"], subme=p["subme"],
                            merange=p["merange"], rect=p["rect"], qp=p["qp"], lam=lambda_for(p["qp"], wl.depth), amp=p["amp"])
    if chroma:
        an.enable_chroma()
        if chroma_residual:
            an.enable_chroma_residual(0, 0)
    for r, ref in enumerate(wl.refs):
        an.set_ref(r, ref[MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W])
        if chroma:
            an.set_ref_chroma(r, inner(wl.refC[r][0], W, H), inner(wl.refC[r][1], W, H))
    if chroma:
        an.load_chroma(inner(wl.fencC[0], W, H), inner(wl.fencC[1], W, H))
    an.set_lists(n0, p["numRefs"] - n0)
    return an


def oracle(wl, n0, chroma, max_ctu_rows=0):
    return cpu_analyse_part_b(load_oracle_part_b(wl.depth), "orc", wl, n0, chroma, threads=8, max_ctu_rows=max_ctu_rows)


def assert_part_b_equal(got, want):
    """Every PART_B record byte for byte."""
    n = len(want)
    bad = np.nonzero((got.view(np.uint8).reshape(n, -1) != want.view(np.uint8).reshape(n, -1)).any(axis=1))[0]
    assert len(bad) == 0, (len(bad), bad[:2].tolist(), got[bad[:2]].tolist(), want[bad[:2]].tolist())


@pytest.mark.timeout(300)
@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_part_b_parity(cu, case):
    wl, n0, chroma = case_workload(case)
    want = oracle(wl, n0, chroma)
    an = open_analyser(cu, wl, n0, chroma)
    an.analyse(source(wl), wl.field, stages=STAGES)
    assert np.array_equal(an.fetch("me_out").reshape(-1, 4)[:, :3], want["me_out"][:, :3])
    assert_part_b_equal(an.part_b_results(), want["part_b"])
    an.close()


@pytest.mark.timeout(900)
@pytest.mark.parametrize("depth, n0, n1, amp, subme, rows", [(8, 2, 2, 0, 3, 2), (10, 3, 2, 1, 4, 1)],
                         ids=["c3-8bit-2+2-rect", "c4-10bit-3+2-amp"])
def test_part_b_2160p(cu, depth, n0, n1, amp, subme, rows):
    """3840x2160 against the oracle on the first CTU rows: 8-bit, lists 2+2, rect, chroma on, 2 rows; 10-bit, lists 3+2,
    rect + AMP, subme 4, chroma on, 1 row."""
    wl = Workload(3840, 2160, depth=depth, numRefs=n0 + n1, subme=subme, rect=1, amp=amp, qp=30, chroma=True)
    want = oracle(wl, n0, True, max_ctu_rows=rows)
    an = open_analyser(cu, wl, n0, True)
    an.analyse_rows(source(wl), wl.field, 0, rows, stages=STAGES)
    nj, nc = want["njobs_run"], want["ncu_run"]
    assert np.array_equal(an.fetch("me_out").reshape(-1, 4)[:nj, :3], want["me_out"][:nj, :3])
    got = an.part_b_results(0, rows)[:nc]
    assert_part_b_equal(got, want["part_b"][:nc])
    an.close()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("depth", [8, 10])
def test_part_b_row_bands(cu, depth):
    """analyse_rows over a band partition gives the full-frame records."""
    wl, n0, chroma = case_workload((depth, (2, 2), (1, 1), "s3", (328, 200), 22, "occlusion"))
    full = open_analyser(cu, wl, n0, chroma)
    full.analyse(source(wl), wl.field, stages=STAGES)
    shard = open_analyser(cu, wl, n0, chroma)
    rec = np.zeros_like(full.part_b_results())
    for r0, r1 in ((2, 4), (0, 1), (1, 2)):
        shard.analyse_rows(source(wl), wl.field, r0, r1, stages=STAGES)
        shard.part_b_results(r0, r1, rec)
    assert rec.tobytes() == full.part_b_results().tobytes()
    full.close()
    shard.close()


@pytest.mark.timeout(300)
def test_part_b_alone_after_me(cu):
    """Stage value 64 alone after a value-1 run gives the records of a combined run."""
    wl, n0, chroma = case_workload((8, (1, 1), (1, 1), "s3", (200, 136), 22, "static"))
    both = open_analyser(cu, wl, n0, chroma)
    both.analyse(source(wl), wl.field, stages=1 | 64)
    alone = open_analyser(cu, wl, n0, chroma)
    alone.analyse(source(wl), wl.field, stages=1)
    alone.run_resident(64)
    assert alone.part_b_results().tobytes() == both.part_b_results().tobytes()
    both.close()
    alone.close()


def results(an):
    return dict(me=an.fetch("me_out"), coef=an.fetch("coef"), sse=an.cu_sse.copy(), ns=an.cu_numsig.copy(), ref=an.cu_ref.copy(),
                intra=an.intra_cost.copy(), packed=an.me_packed.copy(), bidir=an.bidir_results(),
                coef_c=[an.fetch_chroma(n) for n in ("coef_cb", "coef_cr")], chroma=an.chroma_results(),
                recon=[an.fetch("recon%d" % d) for d in range(4)],
                recon_c=[an.fetch_chroma(("recon", d, k)) for d in range(4) for k in range(2)])


@pytest.mark.timeout(300)
@pytest.mark.parametrize("kind", ["average", "occlusion"])
def test_part_b_changes_nothing_else(cu, kind):
    """Adding value 64 to a B-slice run leaves the ME, BIDIR, luma and chroma residual, and intra outputs byte-identical."""
    wl, n0, chroma = case_workload((10, (2, 2), (1, 1), "s3", (328, 200), 22, kind))
    plain = open_analyser(cu, wl, n0, chroma, chroma_residual=True)
    plain.analyse(source(wl), wl.field, stages=31)
    an = open_analyser(cu, wl, n0, chroma, chroma_residual=True)
    an.analyse(source(wl), wl.field, stages=31 | 64)
    a, b = results(plain), results(an)
    for k in a:
        x, y = a[k], b[k]
        assert all(np.array_equal(p, q) for p, q in zip(x, y)) if isinstance(x, (list, tuple)) else np.array_equal(x, y), k
    plain.close()
    an.close()


def test_part_b_refusals(cu):
    """part_b_results before any value-64 run and with a bad row range; value 64 on a P slice and while a reference is
    weighted: each refused before any launch, with the records untouched.  The plane-reach checks hold for every picture
    the analyser accepts, so their refusal is not reached here."""
    from x265_b200.lib import PART_B_CU
    from wref_helpers import entry, identity
    wl, n0, chroma = case_workload((8, (1, 1), (1, 0), "s3", (200, 136), 22, "average"))
    L = cu.L
    an = open_analyser(cu, wl, n0, chroma)
    rec = np.zeros(an.ncu, PART_B_CU)
    assert L.x265cu_analyser_part_b_results(an.h, 0, an.ctu_rows, rec.ctypes.data) == -1 and cu.last_error()
    an.analyse(source(wl), wl.field, stages=STAGES)
    before = an.part_b_results().copy()
    for r0, r1 in ((-1, 1), (0, an.ctu_rows + 1), (2, 1)):
        assert L.x265cu_analyser_part_b_results(an.h, r0, r1, rec.ctypes.data) == -1 and cu.last_error()

    def refused(stages_list):
        for st in stages_list:
            n = cu.launch_count()
            assert L.x265cu_analyser_run_resident(an.h, st) == -1 and cu.last_error()
            assert cu.launch_count() == n
        assert an.part_b_results().tobytes() == before.tobytes()
    # a P slice
    an.set_lists(2, 0)
    refused((64, 1 | 64, 32 | 64))
    # a weighted reference
    an.set_lists(1, 1)
    an.set_ref_weights(0, [entry(40, 5, 3), identity(6), identity(6)])
    refused((64, 1 | 64))
    an.set_ref_weights(0, None)
    # the B slice again: the same records
    an.analyse(source(wl), wl.field, stages=STAGES)
    assert an.part_b_results().tobytes() == before.tobytes()
    an.close()


def test_part_b_record_layout(cu):
    """x265cu_part_b_cu as ctypes sees it, the numpy record of Analyser.part_b_results, and the C sizeof / offsetof."""
    from x265_b200.lib import PART_B_CU
    assert C.sizeof(PartBCu) == PART_B_CU.itemsize == 320
    offs = dict(cost=0, sa8d=32, biCost=64, interDir=128, ref=144, zero=176, mv=192)      # offsetof in include/x265_b200.h
    for name, off in offs.items():
        assert getattr(PartBCu, name).offset == PART_B_CU.fields[name][1] == off, name
