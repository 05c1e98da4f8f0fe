"""GPU parity of the frame analyser's PART stage (stage bit 5: the inter estimate of every partition of a P slice's CUs) against
the oracle's PART driver, which tests/test_part_oracle_vs_ref.py pins to the real reference code: every PART record byte for
byte on every CPU case and at 3840x2160; row bands; a PART-only run after an ME run; that the stage changes no other output;
the refusals; the record layout."""
import ctypes as C

import numpy as np
import pytest

from frame_helpers import Workload, lambda_for, MARGIN_X, MARGIN_Y
from part_helpers import load_oracle_part, cpu_analyse_part, case_workload, PartCu, STAGES, CASES, case_id

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


def open_analyser(cu, wl, chroma, tab=None, chroma_residual=False):
    """An analyser with the workload's references resident, the weights of `tab` set, and with chroma: the chroma planes (and,
    with chroma_residual, the chroma residual stage)."""
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
    if tab is not None:
        for r in range(p["numRefs"]):
            an.set_ref_weights(r, tab[r] if tab[r][0][0] else None)
    return an


def oracle(wl, chroma, tab=None, max_ctu_rows=0):
    return cpu_analyse_part(load_oracle_part(wl.depth), "orc", wl, chroma, tab, threads=8, max_ctu_rows=max_ctu_rows)


def assert_part_equal(got, want):
    """Every PART record byte for byte."""
    n = len(want)
    bad = np.nonzero((got.view(np.uint8).reshape(n, -1) != want.view(np.uint8).reshape(n, -1)).any(axis=1))[0]
    assert len(bad) == 0, (len(bad), got[bad[:2]].tolist(), want[bad[:2]].tolist())


@pytest.mark.timeout(300)
@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_part_parity(cu, case):
    depth, nr, geo, chroma, size, kind = case
    wl, tab = case_workload(case)
    want = oracle(wl, chroma, tab)
    an = open_analyser(cu, wl, chroma, tab)
    an.analyse(source(wl), wl.field, stages=STAGES)
    assert np.array_equal(an.fetch("me_out").reshape(-1, 4)[:, :3], want["me_out"][:, :3])
    assert np.array_equal(an.cu_ref, want["cu_ref"])
    assert_part_equal(an.part_results(), want["part"])
    an.close()


@pytest.mark.timeout(900)
@pytest.mark.parametrize("depth, nr, amp, subme, rows", [(8, 4, 0, 3, 2), (10, 5, 1, 4, 1)], ids=["c3-8bit-4ref-rect", "c4-10bit-5ref-amp"])
def test_part_2160p(cu, depth, nr, amp, subme, rows):
    """3840x2160 against the oracle on the first CTU rows: 8-bit, 4 references, rect, chroma on, 2 rows; 10-bit, 5 references,
    rect + AMP, subme 4, chroma on, 1 row."""
    wl = Workload(3840, 2160, depth=depth, numRefs=nr, subme=subme, rect=1, amp=amp, qp=30, chroma=True)
    want = oracle(wl, True, max_ctu_rows=rows)
    an = open_analyser(cu, wl, True)
    an.analyse_rows(source(wl), wl.field, 0, rows, stages=STAGES)
    nj, nc = want["njobs_run"], want["ncu_run"]
    assert np.array_equal(an.fetch("me_out").reshape(-1, 4)[:nj, :3], want["me_out"][:nj, :3])
    got = an.part_results(0, rows)[:nc]
    assert_part_equal(got, want["part"][:nc])
    wins = set(np.argmin(got["cost"], axis=1).tolist())
    assert wins > {0}, wins
    an.close()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("depth", [8, 10])
def test_part_row_bands(cu, depth):
    """analyse_rows over a band partition gives the full-frame records."""
    wl, tab = case_workload((depth, 2, (1, 1), True, (328, 200), "split"))
    full = open_analyser(cu, wl, True)
    full.analyse(source(wl), wl.field, stages=STAGES)
    shard = open_analyser(cu, wl, True)
    rec = np.zeros_like(full.part_results())
    for r0, r1 in ((2, 4), (0, 1), (1, 2)):
        shard.analyse_rows(source(wl), wl.field, r0, r1, stages=STAGES)
        shard.part_results(r0, r1, rec)
    assert rec.tobytes() == full.part_results().tobytes()
    full.close()
    shard.close()


@pytest.mark.timeout(300)
def test_part_alone_after_me(cu):
    """Stage value 32 alone after a value-1 run gives the records of a combined run."""
    wl, tab = case_workload((8, 2, (1, 1), True, (328, 200), "fade"))
    both = open_analyser(cu, wl, True, tab)
    both.analyse(source(wl), wl.field, stages=1 | 32)
    alone = open_analyser(cu, wl, True, tab)
    alone.analyse(source(wl), wl.field, stages=1)
    alone.run_resident(32)
    assert alone.part_results().tobytes() == both.part_results().tobytes()
    both.close()
    alone.close()


def results(an):
    return dict(me=an.fetch("me_out"), coef=an.fetch("coef"), sse=an.cu_sse.copy(), ns=an.cu_numsig.copy(), ref=an.cu_ref.copy(),
                intra=an.intra_cost.copy(), packed=an.me_packed.copy(), coef_c=[an.fetch_chroma(n) for n in ("coef_cb", "coef_cr")],
                chroma=an.chroma_results(), recon=[an.fetch("recon%d" % d) for d in range(4)],
                recon_c=[an.fetch_chroma(("recon", d, k)) for d in range(4) for k in range(2)])


@pytest.mark.timeout(300)
@pytest.mark.parametrize("kind", ["split", "fade"])
def test_part_changes_nothing_else(cu, kind):
    """Adding value 32 to a run leaves the ME, luma and chroma residual, and intra outputs byte-identical."""
    wl, tab = case_workload((10, 2, (1, 1), True, (328, 200), kind))
    plain = open_analyser(cu, wl, True, tab, chroma_residual=True)
    plain.analyse(source(wl), wl.field, stages=15)
    an = open_analyser(cu, wl, True, tab, chroma_residual=True)
    an.analyse(source(wl), wl.field, stages=15 | 32)
    a, b = results(plain), results(an)
    for k in a:
        x, y = a[k], b[k]
        assert all(np.array_equal(p, q) for p, q in zip(x, y)) if isinstance(x, (list, tuple)) else np.array_equal(x, y), k
    plain.close()
    an.close()


def test_part_refusals(cu):
    """part_results before any value-32 run and with a bad row range; value 32 on a B slice, refused before any launch with the
    records untouched."""
    wl, tab = case_workload((8, 2, (1, 0), True, (200, 136), "motion"))
    L = cu.L
    an = open_analyser(cu, wl, True)
    from x265_b200.lib import PART_CU
    rec = np.zeros(an.ncu, PART_CU)
    assert L.x265cu_analyser_part_results(an.h, 0, an.ctu_rows, rec.ctypes.data) == -1 and cu.last_error()
    an.analyse(source(wl), wl.field, stages=STAGES)
    before = an.part_results().copy()
    for r0, r1 in ((-1, 1), (0, an.ctu_rows + 1), (2, 1)):
        assert L.x265cu_analyser_part_results(an.h, r0, r1, rec.ctypes.data) == -1 and cu.last_error()
    an.set_lists(1, 1)
    an.load_inputs(source(wl), wl.field)
    for st in (32, 1 | 32, 16 | 32):
        n = cu.launch_count()
        assert L.x265cu_analyser_run_resident(an.h, st) == -1 and cu.last_error()
        assert cu.launch_count() == n
    assert an.part_results().tobytes() == before.tobytes()
    an.set_lists(2, 0)
    an.analyse(source(wl), wl.field, stages=STAGES)
    assert an.part_results().tobytes() == before.tobytes()
    an.close()


def test_part_record_layout(cu):
    """x265cu_part_cu as ctypes sees it, and the numpy record of Analyser.part_results."""
    from x265_b200.lib import PART_CU
    assert C.sizeof(PartCu) == PART_CU.itemsize == 144
    for name in ("cost", "sa8d", "ref", "mv"):
        assert getattr(PartCu, name).offset == PART_CU.fields[name][1], name
