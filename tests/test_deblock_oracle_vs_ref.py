"""Frame-level deblocking: the plain-C restatement (oracle/oracle_deblock.c, vertical pass then horizontal pass over the whole
picture) against the REAL Deblock::deblockCTU run over real CUData CTUs in FrameFilter's CTU order (oracle/ref_shim_deblock.cpp:
x265ref_deblock_frame), whole planes compared.  This pins the restated arithmetic and the claim that the reference's CTU order
equals the two-pass order.  Where oracle/_ref is absent the reference's stored results (tests/golden/deblock_ref.json) stand
in for it.  Also: the layouts of the decision map and parameter records against include/x265_b200.h."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import deblock_helpers as D
from common import ROOT

CASES = D.cases()


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_deblock_oracle_matches_reference(request, case):
    depth, ctu = case[1], case[4]
    luma, cb, cr, units, prm = D.case_inputs(case)
    out = D.oracle_deblock(depth, luma, cb, cr, units, prm)
    assert not np.array_equal(out[0], luma) or case[8] == "noise"
    R = D.DeblockRefResults(request, depth)
    planes = [p for p in out if p is not None]
    R.same("planes", lambda: [p for p in D.ref_deblock(depth, luma, cb, cr, units, prm, ctu) if p is not None], planes)


def test_deblock_cases_reach_every_decision():
    """Over the cases above, every decision of the restatement is taken: BS 0 / 1 / 2, the d >= beta skip, the strong filter,
    the normal filter with both / one / neither side-2 sample modified, and chroma segments."""
    cnt = np.zeros(len(D.COUNTERS), np.int64)
    for case in CASES:
        luma, cb, cr, units, prm = D.case_inputs(case)
        D.oracle_deblock(case[1], luma, cb, cr, units, prm, cnt)
    missing = [n for n, v in zip(D.COUNTERS, cnt) if v == 0]
    assert not missing, dict(zip(D.COUNTERS, cnt.tolist()))


def _header_struct(name):
    txt = open(os.path.join(ROOT, "include", "x265_b200.h")).read()
    body = re.search(r"typedef struct \{([^{}]*)\}\s*%s;" % name, txt, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = []
    for decl in body.split(";"):
        decl = decl.strip()
        if decl:
            ctype, names = decl.split(None, 1)
            fields += [(ctype, n.strip()) for n in names.split(",")]
    return fields


def test_deblock_records_match_header():
    """x265cu_deblock_unit / x265cu_deblock_params: field order, types and offsets of the host mirror against the header."""
    from x265_b200.lib import DEBLOCK_UNIT, DeblockParams
    sizes = {"int8_t": 1, "uint8_t": 1, "int16_t": 2, "int32_t": 4}
    unit = _header_struct("x265cu_deblock_unit")
    assert [re.sub(r"\[.*", "", n) for _, n in unit] == list(DEBLOCK_UNIT.names)
    off = 0
    for ctype, n in unit:
        count = int(np.prod([int(d) for d in re.findall(r"\[(\d+)\]", n)] or [1]))
        sz = sizes[ctype]
        off = (off + sz - 1) // sz * sz
        f = DEBLOCK_UNIT.fields[re.sub(r"\[.*", "", n)]
        assert f[1] == off and f[0].itemsize == sz * count and f[0].base.itemsize == sz, (n, f)
        assert f[0].base.kind == ("u" if ctype.startswith("u") else "i"), n
        off += sz * count
    assert DEBLOCK_UNIT.itemsize == off == 16
    prm = _header_struct("x265cu_deblock_params")
    assert [n for _, n in prm] == [n for n, _ in DeblockParams._fields_]
    assert all(t == "int32_t" for t, _ in prm) and C.sizeof(DeblockParams) == 24
