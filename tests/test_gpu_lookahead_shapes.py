"""GPU parity of the lookahead (x265cu_frame_init_lowres -> x265cu_lowres_intra_batch -> x265cu_lookahead_cost_batch) at the
launch shapes of the 1080p and 2160p configurations, which the frame sizes of tests/test_gpu_lookahead.py never reach.

k_lookahead_cost runs every wavefront job (a triple, or one cooperative slice of it) on a thread-block cluster of 1, 2 or 4
CTAs of LA_WARPS warps, sized from the frame's longest anti-diagonal; a diagonal longer than the cluster's warps takes several
rounds.  k_lowres_intra caps its grid at 4 x SMs CTAs of 32 CUs and grid-strides past that.  Each case names the shapes it
targets (SHAPES: one entry per launch shape, with the C lines that choose it).  The mirror below restates the launch's shape
rules; every case asserts on the host that it lands where it says, test_every_shape_is_targeted keeps SHAPES and CASES in
step, and test_launch_grid checks the cluster-size rule against the grid torch.profiler records.

Every case runs one lookahead window the way the c2 benchmark step does: init_frame for every frame, one intra_batch, then
every batch of conflict_free_batches(window_triples(n, bframes)) prepared and launched before a single sync, so later
launches read motion fields that earlier launches of the same stream searched.  The oracle (lookahead_helpers.OracleLookahead,
which test_lookahead_oracle_vs_ref.py pins to the reference at these geometries) runs the same triples in window order.
Lowres planes, intra costs, every estimate (cost, costEstAq, intraMbs, per-CU costs, row sums) and every motion field the
window created must match bit for bit.
"""
import json
from types import SimpleNamespace

import numpy as np
import pytest

from common import load_oracle, pixel_dtype
from frame_helpers import gen_luma, MARGIN_X
from lookahead_helpers import OracleLookahead
from x265_b200.lookahead import Lookahead, coop_slices, lowres_geometry, window_triples, conflict_free_batches

pytestmark = pytest.mark.gpu

LA_WARPS = 16                                             # warps per CTA of k_lookahead_cost (lookahead.cuh:119)

SHAPES = {
    "cluster4_one_round": "4-CTA cluster, every diagonal in one round of its 64 warps: x265cu.cu:363-366, lookahead.cuh:151-152",
    "cluster4_full_round": "4-CTA cluster whose longest diagonal fills all 64 warps exactly: lookahead.cuh:152",
    "cluster4_two_rounds": "4-CTA cluster, diagonals longer than 64 CUs take a second round (k += nwarps): lookahead.cuh:152",
    "cluster4_single_cu_round": "longest diagonal of 65 CUs on a 4-CTA cluster: its 65th CU is the only work of round 2",
    "cluster2_width_bound": "longest diagonal bound by the width ((w8 + 1) / 2 < h8), 3 CTAs rounded down to 2, so 2 rounds: "
                            "x265cu.cu:364-366",
    "cluster1_strip": "1-CTA cluster on a grid 4 CUs wide or high (the narrowest legal picture): hundreds of diagonals of <= 4 CUs",
    "intra_grid_stride": "k_lowres_intra past its cap of 4 x SMs CTAs: the grid-stride loop, x265cu.cu:339, lookahead.cuh:51",
    "sliced_cluster4": "cooperative slices on a 4-CTA cluster sized from h8 while each slice's diagonals are shorter; the slice jobs "
                       "of a triple accumulate into one set of totals: lookahead.cuh:141-145, x265cu.cu:347-354",
}

# name: (W, H, depth, lookahead slices, window frames, bframes, shapes targeted).  w8 x h8 is the lowres CU grid.
CASES = {
    "c2": (1920, 1080, 8, 0, 10, 4, {"cluster4_one_round"}),                         # 120x68: diagonals of 60 CUs
    "medium": (1920, 1080, 8, 8, 10, 4, {"sliced_cluster4"}),                        # 6 slices of 10 rows, the last of 18
    "slow_2160": (3840, 2160, 8, 4, 5, 2, {"sliced_cluster4", "intra_grid_stride"}),  # 240x135, slices of 33 / 33 / 33 / 36 rows
    "slower_2160": (3840, 2160, 10, 0, 5, 2, {"cluster4_two_rounds", "intra_grid_stride"}),   # diagonals of 120 CUs
    "round_edge": (2080, 1040, 8, 0, 10, 4, {"cluster4_single_cu_round"}),           # 130x65
    "round_full": (2048, 1024, 8, 0, 10, 4, {"cluster4_full_round"}),                # 128x64
    "portrait": (1080, 1920, 8, 0, 10, 4, {"cluster2_width_bound"}),                 # 68x120: diagonals of 34 CUs
    "wide_strip": (3840, 64, 8, 0, 10, 4, {"cluster1_strip"}),                       # 240x4: 246 diagonals
    "tall_strip": (64, 2160, 8, 0, 10, 4, {"cluster1_strip"}),                       # 4x135: 272 diagonals
}


# ---------------------------------------------------------------------------------------------------------------------
# the mirror of the launch's shape rules
def launch_shape(W, H, lslices):
    """Cluster size of x265cu_lookahead_cost_batch and, per wavefront job of a triple, its rows, diagonals and rounds."""
    w8, h8, _ = lowres_geometry(W, H)
    maxdiag = min(h8, (w8 + 1) // 2)                                       # x265cu.cu:364, from the whole frame's h8
    csize = (maxdiag + LA_WARPS - 1) // LA_WARPS                           # :365
    csize = 4 if csize >= 4 else (2 if csize >= 2 else 1)                  # :366
    nwarps = csize * LA_WARPS                                              # lookahead.cuh:135
    nsl, rps = coop_slices(H, lslices)
    jobs = []
    for sl in range(nsl):                                                  # one job per slice (x265_b200/lookahead.py prepare_batch)
        y0, y1 = rps * sl, (h8 if sl == nsl - 1 else rps * (sl + 1))
        hs = y1 - y0
        ndiag = (w8 - 1) + 2 * (hs - 1) + 1                                # lookahead.cuh:145
        lens = [min(hs - 1, t >> 1) - max(0, (t - (w8 - 1) + 1) >> 1) + 1 for t in range(ndiag)]   # :151
        longest = max(lens)
        assert longest == min(hs, (w8 + 1) // 2), (W, H, sl, longest)
        rounds = (longest + nwarps - 1) // nwarps                          # :152, k += nwarps
        jobs.append(dict(hs=hs, ndiag=ndiag, longest=longest, rounds=rounds, last=longest - (rounds - 1) * nwarps))
    return dict(w8=w8, h8=h8, maxdiag=maxdiag, csize=csize, nwarps=nwarps, jobs=jobs)


def intra_passes(ncu, sms):
    """Grid-stride passes of k_lowres_intra: 32 CUs per CTA, at most 4 x SMs CTAs (x265cu.cu:339, lookahead.cuh:51)."""
    bx = min((ncu + 31) // 32, 4 * sms)
    return (ncu + 32 * bx - 1) // (32 * bx)


def shapes_of(case, sms):
    """The SHAPES a case's launches land on, according to the mirror."""
    W, H, _, lslices = CASES[case][:4]
    s = launch_shape(W, H, lslices)
    jobs, cs, nw = s["jobs"], s["csize"], s["nwarps"]
    got = set()
    if cs == 4 and len(jobs) == 1:
        j = jobs[0]
        if j["rounds"] == 1:
            got.add("cluster4_one_round")
            if j["longest"] == nw:
                got.add("cluster4_full_round")
        if j["rounds"] == 2:
            got.add("cluster4_two_rounds")
            if j["last"] == 1:
                got.add("cluster4_single_cu_round")
    if cs == 2 and s["maxdiag"] < s["h8"] and (s["maxdiag"] + LA_WARPS - 1) // LA_WARPS == 3 and jobs[0]["rounds"] == 2:
        got.add("cluster2_width_bound")
    if cs == 1 and min(s["w8"], s["h8"]) == 4 and jobs[0]["ndiag"] > 200:
        got.add("cluster1_strip")
    if intra_passes(s["w8"] * s["h8"], sms) > 1:
        got.add("intra_grid_stride")
    if cs == 4 and len(jobs) > 1 and all(j["rounds"] == 1 and j["longest"] < s["maxdiag"] for j in jobs):
        got.add("sliced_cluster4")
    return got


def searchers(order):
    """Motion field (b, list, distance) -> the triple that searches it when the triples run in `order` (the first to use
    it; list 1 is searched only by B triples)."""
    out = {}
    for (p0, p1, b) in order:
        out.setdefault((b, 0, b - p0), (p0, p1, b))
        if p1 > b:
            out.setdefault((b, 1, p1 - b), (p0, p1, b))
    return out


def check_window(triples, batches):
    """The batches launch the triples in an order that lets the same kind of triple search every motion field as in window
    order, and the window reuses fields: a B triple reads a list-0 field a P triple searched, another a list-1 field an
    earlier B triple searched.
    A field's search depends on b, its list and distance, and on whether the searching triple is bidirectional (the zero-MV
    skip rule, lookahead.cuh:209, 219), not on the triple's other reference.  The batches do hand some list-1 fields to a
    different B triple than window order does (at n = 10, bframes = 4: (2, 1, 2) goes to (1, 4, 2) instead of (0, 4, 2)),
    which gives the same field.  A field that window order gives to a P triple and the batches to a B triple would not."""
    flat = [t for bt in batches for t in bt]
    assert sorted(flat) == sorted(triples)
    who = searchers(triples)
    kind = lambda order: {k: t[1] > t[2] for k, t in searchers(order).items()}
    assert kind(flat) == kind(triples)
    bs = [(p0, p1, b) for (p0, p1, b) in triples if p1 > b]
    p_searched = [who[(b, 0, b - p0)] for (p0, p1, b) in bs]
    assert any(s[1] == s[2] for s in p_searched), "no B triple reads a list-0 field a P triple searched"
    assert any(who[(b, 1, p1 - b)] != (p0, p1, b) for (p0, p1, b) in bs), "no B triple reads a list-1 field another B triple searched"


# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def cu():
    import x265_b200
    return x265_b200.load()


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _frames(W, H, depth, n):
    return [gen_luma(W, H, i, s1=17.0, s2=11.0, bits=depth) for i in range(n)]


def _gpu_lookahead(cu, frames, depth, lslices):
    H, W = frames[0].shape
    la = Lookahead(cu, W, H, depth, len(frames), lookahead_slices=lslices)
    for i, img in enumerate(frames):
        la.init_frame(i, img)
    la.intra_batch(range(len(frames)))
    return la


@pytest.fixture(scope="module", params=list(CASES))
def window(request, cu, sms):
    """One case's window on the device and in the oracle; computed once for the tests of the case."""
    name = request.param
    W, H, depth, lslices, n, bframes, targets = CASES[name]
    assert targets <= shapes_of(name, sms), (name, targets, shapes_of(name, sms))
    triples = window_triples(n, bframes)
    batches = conflict_free_batches(triples)
    check_window(triples, batches)
    frames = _frames(W, H, depth, n)
    sl = coop_slices(H, lslices)
    orc = OracleLookahead(load_oracle(depth), frames, depth, slices=sl if sl[0] > 1 else None)
    for t in triples:
        orc.cost(*t)
    la = _gpu_lookahead(cu, frames, depth, lslices)
    preps = [la.prepare_batch(bt) for bt in batches]
    assert [p["njobs"] for p in preps] == [len(bt) * len(launch_shape(W, H, lslices)["jobs"]) for bt in batches]
    for p in preps:
        la.launch_batch(p)
    cu.sync()
    for p in preps:
        la.collect_batch(p, full=True)
    yield SimpleNamespace(name=name, depth=depth, n=n, triples=triples, orc=orc, la=la)
    la.close()


def test_lowres_and_intra(window):
    """Lowres::init planes and lowresIntraEstimate of every frame of the window."""
    orc, la, depth = window.orc, window.la, window.depth
    vw = orc.w8 * 8 + 2 * MARGIN_X
    for i in range(window.n):
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
    """Every (p0, p1, b) estimate of the window: frame cost, costEstAq, intraMbs, per-CU costs and row sums."""
    orc, la = window.orc, window.la
    for (p0, p1, b) in window.triples:
        d0, d1 = b - p0, p1 - b
        r, f = la.fr[b]["res"][(d0, d1)], orc.fr[b]
        t = (p0, p1, b)
        assert (r["score"], r["costEstAq"]) == f["costEst"][(d0, d1)], (t, r["score"], r["costEstAq"], f["costEst"][(d0, d1)])
        assert r["intraMbs"] == f["estIntraMbs"][(d0, d1)], (t, r["intraMbs"], f["estIntraMbs"][(d0, d1)])
        bad = np.nonzero(r["lowresCosts"] != f["lowresCosts"][(d0, d1)])[0]
        assert bad.size == 0, (t, "lowresCosts differ at %d CUs, first %s" % (bad.size, bad[:6]))
        bad = np.nonzero(r["rowSatds"] != f["rowSatds"][(d0, d1)])[0]
        assert bad.size == 0, (t, "rowSatds differ at rows %s" % bad[:6])
    # the content has intra-coded CUs in the P estimates, so a lost intraMbs count would show
    assert any(orc.fr[b]["estIntraMbs"][(b - p0, 0)] for (p0, p1, b) in window.triples if p1 == b)


def test_window_motion_fields(window):
    """Every motion field the window created, (b, list, distance) -> vectors and costs, both lists."""
    orc, la = window.orc, window.la
    for b in range(window.n):
        assert set(la.fr[b]["mvs"]) == set(orc.fr[b]["mvs"]) == set(la.fr[b]["mvcosts"]), b
        for key in orc.fr[b]["mvs"]:
            mvs = la.fr[b]["mvs"][key].download(np.int32).reshape(-1, 2)
            bad = np.nonzero((mvs != orc.fr[b]["mvs"][key]).any(axis=1))[0]
            assert bad.size == 0, ((b,) + key, "mvs differ at %d CUs, first %s" % (bad.size, bad[:6]))
            bad = np.nonzero(la.fr[b]["mvcosts"][key].download(np.int32) != orc.fr[b]["mvcosts"][key])[0]
            assert bad.size == 0, ((b,) + key, "mvcosts differ at %d CUs, first %s" % (bad.size, bad[:6]))
    assert any(lst == 1 and d > 0 for f in orc.fr for (lst, d) in f["mvs"])


# ---------------------------------------------------------------------------------------------------------------------
def test_every_shape_is_targeted(sms):
    targeted = set().union(*(c[-1] for c in CASES.values()))
    assert targeted == set(SHAPES), (set(SHAPES) - targeted, targeted - set(SHAPES))
    for name, case in CASES.items():
        assert case[-1] <= shapes_of(name, sms), (name, case[-1], shapes_of(name, sms))


GRID_CASES = ["wide_strip", "portrait", "c2", "medium"]              # cluster sizes 1, 2, 4, and a sliced launch
GRID_TRIPLES = [(0, 1, 1), (0, 2, 2), (1, 2, 2)]                      # one conflict-free batch


def record_grid_traces(out_dir):
    """One launch of GRID_TRIPLES per GRID_CASES entry under torch.profiler, each trace saved as out_dir/<case>.json.
    test_launch_grid runs this in a fresh process: inside a long pytest process that has profiled and launched much
    before, the profiler was seen to record no kernel at all."""
    import os
    import torch
    import x265_b200
    from torch.profiler import profile, ProfilerActivity
    cu = x265_b200.load()
    for case in GRID_CASES:
        W, H, depth, lslices = CASES[case][:4]
        la = _gpu_lookahead(cu, _frames(W, H, depth, 3), depth, lslices)
        prep = la.prepare_batch(GRID_TRIPLES)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            la.launch_batch(prep)
            cu.sync()
            torch.cuda.synchronize()
        la.collect_batch(prep)
        la.close()
        prof.export_chrome_trace(os.path.join(out_dir, case + ".json"))


@pytest.fixture(scope="module")
def grid_traces(tmp_path_factory):
    import os
    import subprocess
    import sys
    out = tmp_path_factory.mktemp("grid_traces")
    here = os.path.dirname(os.path.abspath(__file__))
    code = ("import sys; sys.path[:0] = [%r, %r]; import test_gpu_lookahead_shapes as T; T.record_grid_traces(%r)"
            % (os.path.dirname(here), here, str(out)))
    r = subprocess.run([sys.executable, "-c", code], cwd=os.path.dirname(here), stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:]
    return out


@pytest.mark.parametrize("case", GRID_CASES)
def test_launch_grid(grid_traces, case):
    """The cluster-size rule of the mirror against the launch grid of k_lookahead_cost that torch.profiler records:
    grid.x = jobs x cluster size, jobs = triples x slices."""
    W, H, depth, lslices = CASES[case][:4]
    s = launch_shape(W, H, lslices)
    assert conflict_free_batches(GRID_TRIPLES) == [GRID_TRIPLES]
    kernels = [e for e in json.load(open(grid_traces / (case + ".json"))).get("traceEvents", []) if e.get("cat") == "kernel"]
    events = [e for e in kernels if "k_lookahead_cost" in e.get("name", "")]
    if not events:
        pytest.skip("torch.profiler recorded no k_lookahead_cost launch on this host (kernels recorded: %s)"
                    % sorted({e.get("name", "")[:40] for e in kernels}))
    grids = [e.get("args", {}).get("grid") for e in events]
    if any(g is None for g in grids):
        pytest.skip("torch.profiler's trace has no launch grid field on this host")
    assert [g[0] for g in grids] == [len(GRID_TRIPLES) * len(s["jobs"]) * s["csize"]], (case, grids, s["csize"])
