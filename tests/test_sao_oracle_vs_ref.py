"""Frame-level SAO: the plain-C restatement (oracle/oracle_sao.c: statistics of every CTU, then apply as a stencil of the
deblocked picture and the transquant-bypass restoration) against the REAL SAO / Deblock / FrameFilter::ParallelFilter
classes (oracle/ref_shim_sao.cpp), whole arrays and planes compared.  Where oracle/_ref is absent the reference's stored
results (tests/golden/sao_ref.json) stand in for it.

The decomposition pin: FrameFilter's interleaved order (deblocking, the statistics of CTU c - 2, the apply of the previous
row three columns behind) equals deblocking the whole picture, then the statistics of every CTU, then the apply.  Also:
every decision counter of the restatement is reached, and the SAO record layout matches include/x265_b200.h."""
import numpy as np
import pytest

import deblock_helpers as D
import sao_helpers as S
from x265_b200.lib import B_SLICE, SAO_CTU

CASES = S.cases()


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_sao_oracle_matches_reference(request, case):
    """Each step alone on a picture taken as deblocked: the statistics of every CTU, and the applied planes."""
    name, depth, W, H, ctu, chroma, pk, (sl, sc), bypass = case
    rec, fenc, params, merge, units = S.case_inputs(case)
    stats = S.oracle_stats(depth, rec, fenc, ctu)
    out = S.oracle_apply(depth, rec, ctu, params, sl, sc, units, fenc)
    if sl:
        assert not np.array_equal(out[0], rec[0])
    R = S.SaoRefResults(request, depth)
    R.same("stats", lambda: S.ref_stats(depth, rec, fenc, ctu), stats)
    R.same("planes", lambda: [p for p in S.ref_apply(depth, rec, ctu, params, merge, sl, sc, units, fenc) if p is not None],
           [p for p in out if p is not None])


def test_sao_cr_follows_cb_off():
    """Cr with a type >= 0 and Cb off stays untouched (generateChromaOffsets filters Cr with Cb's type)."""
    case = [c for c in CASES if c[0] == "d8_ctu64_200x136"][0]
    rec, fenc, params, merge, units = S.case_inputs(case)
    params[1]["typeIdx"] = -1
    params[2]["typeIdx"] = 1
    out = S.oracle_apply(8, rec, 64, params, 1, 1, None, fenc)
    assert np.array_equal(out[2], rec[2]) and np.array_equal(out[1], rec[1])


PIN = [("d8_ctu64", 8, 200, 136, 64, True, False), ("d10_ctu64", 10, 224, 136, 64, True, False),
       ("d8_ctu32", 8, 208, 104, 32, True, False), ("d10_ctu16", 10, 200, 72, 16, True, False),
       ("d8_luma_only", 8, 200, 136, 64, False, False), ("d10_one_ctu_wide", 10, 48, 136, 64, True, False),
       ("d8_two_ctus_wide", 8, 120, 136, 64, True, False), ("d10_one_row", 10, 224, 40, 64, True, False),
       ("d8_bypass", 8, 200, 136, 64, True, True), ("d10_bypass", 10, 208, 104, 32, True, True)]


def pin_inputs(case, seed=99):
    name, depth, W, H, ctu, chroma, bypass = case
    rng = np.random.default_rng([seed, sum(map(ord, name))])
    units = D.make_map(rng, W, H, ctu, depth, B_SLICE, p_bypass=0.15 if bypass else 0.0)
    luma, cb, cr = D.make_planes(rng, W, H, depth, "blocky", chroma)
    _, fenc = S.make_pictures(rng, W, H, depth, chroma)
    fenc = [np.clip(p.astype(np.int64) + (q.astype(np.int64) - p.astype(np.int64)) // 8, 0, (1 << depth) - 1).astype(p.dtype)
            if p is not None else None for p, q in zip([luma, cb, cr], fenc)]
    params, merge = S.make_params(rng, W, H, ctu, depth)
    dprm = D.params_array(B_SLICE, 1, -1, 2, -2, 1 if bypass else 0)
    return [luma, cb, cr], fenc, units, dprm, params, merge


@pytest.mark.parametrize("case", PIN, ids=[c[0] for c in PIN])
def test_sao_decomposition_matches_interleaved_reference(request, case):
    """oracle deblock -> oracle statistics -> oracle apply (+ bypass restoration) equals the reference's interleaved
    FrameFilter order, for the statistics of every CTU and the final planes."""
    name, depth, W, H, ctu, chroma, bypass = case
    rec, fenc, units, dprm, params, merge = pin_inputs(case)
    dbk = list(D.oracle_deblock(depth, rec[0], rec[1], rec[2], units, dprm))
    stats = S.oracle_stats(depth, dbk, fenc, ctu)
    out = S.oracle_apply(depth, dbk, ctu, params, 1, 1 if chroma else 0, units if bypass else None, fenc)
    R = S.SaoRefResults(request, depth)

    def ref():
        planes, st = S.ref_frame(depth, rec, fenc, ctu, units, dprm, params, merge, 1, 1 if chroma else 0)
        return [st] + [p for p in planes if p is not None]
    R.same("stats_and_planes", ref, [stats] + [p for p in out if p is not None])


def test_sao_cases_reach_every_decision():
    cnt = np.zeros(len(S.COUNTERS), np.int64)
    for case in CASES:
        rec, fenc, params, merge, units = S.case_inputs(case)
        S.oracle_stats(case[1], rec, fenc, case[4], cnt)
        S.oracle_apply(case[1], rec, case[4], params, case[7][0], case[7][1], units, fenc, cnt)
    missing = [n for n, v in zip(S.COUNTERS, cnt) if v == 0]
    assert not missing, dict(zip(S.COUNTERS, cnt.tolist()))


def test_sao_record_matches_header():
    """x265cu_sao_ctu: field order, types and offsets of the host mirror against the header."""
    from test_deblock_oracle_vs_ref import _header_struct
    sizes = {"int8_t": 1, "uint8_t": 1}
    fields = _header_struct("x265cu_sao_ctu")
    names = [n.split("[")[0] for _, n in fields]
    assert names == list(SAO_CTU.names)
    off = 0
    for (ctype, n), name in zip(fields, names):
        count = int(n.split("[")[1].rstrip("]")) if "[" in n else 1
        f = SAO_CTU.fields[name]
        assert f[1] == off and f[0].itemsize == sizes[ctype] * count, (n, f)
        assert f[0].base.kind == ("u" if ctype.startswith("u") else "i"), n
        off += sizes[ctype] * count
    assert SAO_CTU.itemsize == off == 8
