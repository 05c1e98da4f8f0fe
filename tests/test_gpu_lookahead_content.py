"""GPU parity of the lookahead (x265cu_frame_init_lowres -> x265cu_lowres_intra_batch -> x265cu_lookahead_cost_batch) on
content other than the moving clip: lookahead_helpers.content_frames' static, constant, flat, fast, cut, fading and
full-range pictures, which take the branches the clip never does -- the bidir zero-MV skip and the bidir tie
(lookahead.cuh:209-219, 266), vectors on their CU's search bound and far predictors (:161-162, :186-211), the full-tie
intra search (:80-97) and saturated per-CU costs.  test_lookahead_oracle_vs_ref.py pins the oracle to the reference on the
same kinds.

Every case runs one window the way tests/test_gpu_lookahead_shapes.py does: init_frame for every frame, one intra_batch,
then every batch of conflict_free_batches(window_triples(n, bframes)) prepared and launched before a single sync.  Lowres
planes, intra estimates, every estimate and every motion field must equal the oracle's bit for bit."""
from types import SimpleNamespace

import numpy as np
import pytest

from common import load_oracle, pixel_dtype
from frame_helpers import MARGIN_X, MARGIN_Y
from lookahead_helpers import OracleLookahead, CONTENT_KINDS, content_frames
from test_gpu_lookahead_shapes import check_window
from test_lookahead_oracle_vs_ref import AQ_PARAMS, assert_content_reaches, content_invq
from x265_b200.lookahead import Lookahead, coop_slices, window_triples, conflict_free_batches

pytestmark = pytest.mark.gpu

NFRAMES, BFRAMES = 6, 3

# name: (kind, W, H, depth, lookahead slices, AQ)
CASES = {}
for _kind in CONTENT_KINDS:
    for _W, _H in ((416, 240), (200, 136)):                 # 200x136: partial lowres CUs on the right and at the bottom
        for _d in (8, 10):
            if _kind != "full10" or _d == 10:
                CASES["%s-%dx%d-%d" % (_kind, _W, _H, _d)] = (_kind, _W, _H, _d, 0, False)
for _kind in ("static", "fast", "cut"):                     # 120x68 CUs: 4-CTA clusters
    CASES["%s-1080p" % _kind] = (_kind, 1920, 1080, 8, 0, False)
for _kind in ("static", "fast"):
    for _ls in (4, 8):
        CASES["%s-720p-slices%d" % (_kind, _ls)] = (_kind, 1280, 720, 8, _ls, False)
for _kind in ("flat", "static", "cut"):
    for _d in (8, 10):
        CASES["%s-aq-%d" % (_kind, _d)] = (_kind, 416, 240, _d, 0, True)

AQ = dict(mode=AQ_PARAMS[0], strength=AQ_PARAMS[1], qg_size=AQ_PARAMS[2])


def assert_reads_inside_margins(orc):
    """Every block the window's vectors make the device read stays inside the lowres planes' extended margins: the vector
    applied to its own CU and to the CUs that take it as a predictor (left, above-left, above, above-right), the 8x8 block,
    and one more pixel right and down for the second plane of a quarter-pel average."""
    lw, lh = orc.w8 * 8, orc.h8 * 8
    cx = np.arange(orc.w8 * orc.h8) % orc.w8
    cy = np.arange(orc.w8 * orc.h8) // orc.w8
    for b, f in enumerate(orc.fr):
        for key, m in f["mvs"].items():
            for dx in (-1, 0, 1):
                for dy in (-1, 0):
                    x0 = 8 * (cx + dx) + (m[:, 0] >> 2)
                    y0 = 8 * (cy + dy) + (m[:, 1] >> 2)
                    assert (x0 >= -MARGIN_X).all() and (x0 + 9 <= lw + MARGIN_X).all(), (b, key, "x", int(x0.min()), int(x0.max()))
                    assert (y0 >= -MARGIN_Y).all() and (y0 + 9 <= lh + MARGIN_Y).all(), (b, key, "y", int(y0.min()), int(y0.max()))


def oracle_window(name):
    """The case's frames, window triples and launch batches, and the oracle run in window order."""
    kind, W, H, depth, lslices, aq = CASES[name]
    frames = content_frames(kind, W, H, depth, NFRAMES)
    triples = window_triples(NFRAMES, BFRAMES)
    batches = conflict_free_batches(triples)
    check_window(triples, batches)
    chroma, invq = content_invq(kind, W, H, depth, frames) if aq else (None, None)
    sl = coop_slices(H, lslices)
    assert (sl[0] > 1) == (lslices > 0), (name, sl)
    orc = OracleLookahead(load_oracle(depth), frames, depth, slices=sl if sl[0] > 1 else None, invq=invq)
    for t in triples:
        orc.cost(*t)
    return SimpleNamespace(name=name, kind=kind, depth=depth, lslices=lslices, frames=frames, chroma=chroma, invq=invq,
                           triples=triples, batches=batches, orc=orc)


@pytest.fixture(scope="module")
def cu():
    import x265_b200
    return x265_b200.load()


@pytest.fixture(scope="module", params=list(CASES))
def window(request, cu):
    """One case's window on the device and in the oracle; computed once for the tests of the case."""
    w = oracle_window(request.param)
    assert_content_reaches(w.kind, w.depth, w.orc, w.triples)
    assert_reads_inside_margins(w.orc)                    # before any launch: the device run reads inside its planes
    H, W = w.frames[0].shape
    la = Lookahead(cu, W, H, w.depth, NFRAMES, lookahead_slices=w.lslices)
    w.invq_dev = []
    for i, img in enumerate(w.frames):
        if w.invq is not None:
            la.init_frame(i, img, cb=w.chroma[i][0], cr=w.chroma[i][1], aq=AQ)
            w.invq_dev.append(la.fr[i]["invq"].download(np.int32))
        else:
            la.init_frame(i, img)
    la.intra_batch(range(NFRAMES))
    preps = [la.prepare_batch(bt) for bt in w.batches]
    for p in preps:
        la.launch_batch(p)
    cu.sync()
    for p in preps:
        la.collect_batch(p, full=True)
    w.la = la
    yield w
    la.close()


def test_lowres_and_intra(window):
    """Lowres::init planes and lowresIntraEstimate of every frame of the window; with init_frame(aq=...), every frame's
    resident invQscale equals the AQ restatement's invQscaleFactor."""
    orc, la, depth = window.orc, window.la, window.depth
    if window.invq is not None:
        assert any((q != 256).any() for q in window.invq)
        for i in range(NFRAMES):
            assert np.array_equal(window.invq_dev[i], window.invq[i]), ("invQscale", i)
    vw = orc.w8 * 8 + 2 * MARGIN_X
    for i in range(NFRAMES):
        for k in range(4):
            want = orc.fr[i]["planes"][k]
            got = la.fr[i]["planes"][k].download(pixel_dtype(depth)).reshape(want.shape)
            assert np.array_equal(got[:, :vw], want[:, :vw]), ("lowres plane", i, k)
        f, g = orc.fr[i], la.fr[i]
        assert np.array_equal(g["intraCost"].download(np.int32), f["intraCost"]), ("intraCost", i)
        assert np.array_equal(g["intraMode"].download(np.uint8), f["intraMode"]), ("intraMode", i)
        assert np.array_equal(g["lc0"].download(np.uint16), f["lowresCosts"][(0, 0)]), ("intra lowresCosts", i)
        assert np.array_equal(g["rs0"].download(np.int32), f["rowSatds"][(0, 0)]), ("intra rowSatds", i)
        assert tuple(int(x) for x in g["out0"].download(np.int64)) == f["costEst"][(0, 0)], ("intra costEst", i)


def test_window_estimates(window):
    """Every (p0, p1, b) estimate of the window: frame cost, costEstAq, intraMbs, per-CU costs (with their list bits) and
    row sums."""
    orc, la = window.orc, window.la
    for (p0, p1, b) in window.triples:
        d0, d1 = b - p0, p1 - b
        r, f = la.fr[b]["res"][(d0, d1)], orc.fr[b]
        t = (p0, p1, b)
        assert (r["score"], r["costEstAq"]) == f["costEst"][(d0, d1)], (t, r["score"], r["costEstAq"], f["costEst"][(d0, d1)])
        assert r["intraMbs"] == f["estIntraMbs"][(d0, d1)], (t, r["intraMbs"], f["estIntraMbs"][(d0, d1)])
        bad = np.nonzero(r["lowresCosts"] != f["lowresCosts"][(d0, d1)])[0]
        assert bad.size == 0, (t, "lowresCosts differ at %d CUs, first %s" % (bad.size, bad[:6]),
                               r["lowresCosts"][bad[:6]], f["lowresCosts"][(d0, d1)][bad[:6]])
        bad = np.nonzero(r["rowSatds"] != f["rowSatds"][(d0, d1)])[0]
        assert bad.size == 0, (t, "rowSatds differ at rows %s" % bad[:6])


def test_window_motion_fields(window):
    """Every motion field the window created, (b, list, distance) -> vectors and costs, both lists."""
    orc, la = window.orc, window.la
    for b in range(NFRAMES):
        assert set(la.fr[b]["mvs"]) == set(orc.fr[b]["mvs"]) == set(la.fr[b]["mvcosts"]), b
        for key in orc.fr[b]["mvs"]:
            mvs = la.fr[b]["mvs"][key].download(np.int32).reshape(-1, 2)
            bad = np.nonzero((mvs != orc.fr[b]["mvs"][key]).any(axis=1))[0]
            assert bad.size == 0, ((b,) + key, "mvs differ at %d CUs, first %s" % (bad.size, bad[:6]),
                                   mvs[bad[:6]], orc.fr[b]["mvs"][key][bad[:6]])
            costs = la.fr[b]["mvcosts"][key].download(np.int32)
            bad = np.nonzero(costs != orc.fr[b]["mvcosts"][key])[0]
            assert bad.size == 0, ((b,) + key, "mvcosts differ at %d CUs, first %s" % (bad.size, bad[:6]),
                                   costs[bad[:6]], orc.fr[b]["mvcosts"][key][bad[:6]])
