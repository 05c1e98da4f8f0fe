"""GPU parity of x265cu_pred_cost_batch on every kernel route and staged sub-path, at the states tests/test_gpu_predcost.py never
reaches: every phase pair of each list on every route, vectors at CUData::clipMv's limits on guarded pictures, 0 / maxv content,
row pitches and PU positions of every alignment, lists past one grid of the staged launches, and the properties of a list
(every entry written once, order and repetition independent, one job per route).

Each case names the paths it targets (PATHS: one entry per route and staged sub-path, with the lines it lives at).
pred_route mirrors the dispatch predicates of k_pred_uni / k_pred_cost line by line; every case asserts on the host that its
jobs reach what it names, and test_every_path_is_targeted keeps PATHS and the cases in step.  Grid caps come from the
device's SM count.

Outputs are sentinel-filled and compared bit-exactly with the oracle's orc_pred_cost_batch (pinned to the reference by
tests/test_pred_oracle_vs_ref.py) and, where oracle/_ref is built, with the reference's x265ref_pred_cost_batch.  Every plane
sits inside a poison-filled guard band (pred_helpers.Pics), so a read past PicYuv's margins changes a result."""
import numpy as np
import pytest

import pred_helpers as ph
from common import load_oracle, load_ref, pixel_dtype

pytestmark = pytest.mark.gpu

DEPTHS = [8, 10]
SENTINEL = -1431655766            # 0xAAAAAAAA: no cost is negative

# ---------------------------------------------------------------------------------------------------------------------
# the path table (lines of x265_b200/csrc/predcost.cuh unless named)
PATHS = {
    "uni_small": "one list, power-of-two PU with both sides <= 16: k_pred_uni<P, 0>, me_subpel_batch<P, 0> at :398-399; class at :378 (me.cuh:694)",
    "uni_big": "one list, every other PU (12x16 / 16x12 and AMP sizes included): k_pred_uni<P, 1>, me_subpel_batch<P, 1> at :398-399",
    "uni_chroma": "one list, SATD + chroma term: me_set_chroma / me_chroma_batch<P, CLS> at :400-405 (cc.on: me.cuh:970)",
    "bi_small_luma8": "two lists, power-of-two PU <= 16x16 with w >= 8: pb_bi_luma<P, 8> at :384, :259-289",
    "bi_small_luma4": "two lists, power-of-two PU with w = 4: pb_bi_luma<P, 4> at :385",
    "bi_small_avgpp": "two lists, small PU, pixelavg_pp of the pixel predictions: pb_bi_luma avgpp at :268, :279",
    "bi_small_chroma": "two lists, small PU, addAvg SATD + chroma: pb_bi_chroma at :386-393, :295-344",
    "bi_warp": "two lists, 12x16 / 16x12: k_pred_cost<P, 32, 16>, one warp per PU, at :185-192, launch :434",
    "bi_cta": "two lists, a side > 16: k_pred_cost<P, 128, 64>, one CTA per PU, launch :436",
    "staged_luma_pixel_copy": "pc_predict<P, TPJ, MAXS, 8, false> copy at :37-46 (pixelavg_pp lists, :108-119)",
    "staged_luma_pixel_h": "pc_predict 8-tap hpp at :59-70",
    "staged_luma_pixel_v": "pc_predict 8-tap vpp at :59-70",
    "staged_luma_pixel_hv": "pc_predict 8-tap hps + vsp at :72-90",
    "staged_luma_short_copy": "pc_predict<.., 8, true> p2s at :37-46 (addAvg lists, :121-134)",
    "staged_luma_short_h": "pc_predict 8-tap hps at :59-70",
    "staged_luma_short_v": "pc_predict 8-tap vps at :59-70",
    "staged_luma_short_hv": "pc_predict 8-tap hps + vss at :72-90",
    "staged_chroma_short_copy": "pc_predict<.., 4, true> p2s of a chroma plane at :37-46, called at :199-210",
    "staged_chroma_short_h": "pc_predict 4-tap eighth-pel hps at :59-70",
    "staged_chroma_short_v": "pc_predict 4-tap eighth-pel vps at :59-70",
    "staged_chroma_short_hv": "pc_predict 4-tap eighth-pel hps + vss at :72-90",
    "staged_satd8x4": "pc_cost 8x4 tiles (width a multiple of 8) at :150-159",
    "staged_satd4x4": "pc_cost 4x4 tiles at :160-168",
    "staged_chroma_w4": "chroma SATD of a 4-wide block (4x4 tiles) at :209",
    "staged_chroma_w8": "chroma SATD of an 8-wide block at :209",
    "staged_chroma_w12": "chroma SATD of a 12-wide block (4x4 tiles) at :209",
    "staged_chroma_w16": "chroma SATD of a 16-wide block at :209",
    "staged_chroma_w24": "chroma SATD of a 24-wide block at :209",
    "staged_chroma_w32": "chroma SATD of a 32-wide block at :209",
    "lgsegw2": "k_pred_uni job with 16-byte fenc segments: me_set_shape me.cuh:68 (source block and row pitch 16-byte aligned)",
    "lgsegw1": "k_pred_uni job with 8-byte fenc segments: me.cuh:68",
    "lgsegw0": "k_pred_uni job with 4-byte fenc segments: me.cuh:68",
    "rstride_override": "k_pred_uni job whose reference row pitch is not a multiple of 8 bytes: me.cuh:1644",
    "warp_trips": "k_pred_cost<P, 32, 16> job on the second or a later grid-stride trip (grid capped at 16 x SMs CTAs, :431-432)",
    "cta_trips": "k_pred_cost<P, 128, 64> job on the second or a later grid-stride trip (:431, :433)",
}


# ---------------------------------------------------------------------------------------------------------------------
# mirror of the dispatch
def pred_route(jb):
    """(launch, route) of one job: k_pred_uni's `bi && CLS != 0` (:367) and me_subpel_class (:378, me.cuh:694);
    k_pred_cost's `small != (MAXS == 16)` (:189-190) and its uniElsewhere skips (:191-192)"""
    w, h = int(jb["pw"]), int(jb["ph"])
    bi = jb["ref0"] >= 0 and jb["ref1"] >= 0
    pow2 = not ((w & (w - 1)) | (h & (h - 1)))
    small = w <= 16 and h <= 16
    if not bi:
        return ("k_pred_uni<P, 0>", "uni_small") if pow2 and small else ("k_pred_uni<P, 1>", "uni_big")
    if small and pow2:
        return "k_pred_uni<P, 0>", "bi_small"
    return ("k_pred_cost<P, 32, 16>", "bi_warp") if small else ("k_pred_cost<P, 128, 64>", "bi_cta")


def _phase(mv, fb):
    xf, yf = mv[0] & ((1 << fb) - 1), mv[1] & ((1 << fb) - 1)
    return "copy" if not (xf | yf) else "h" if not yf else "v" if not xf else "hv"


def pred_paths(jb, chroma, fenc_addr, fstride, es):
    """every path of PATHS one job reaches (trips excepted: they depend on the job's index).  chroma: planes given.
    fenc_addr: device address of the source plane's pixel (0, 0)."""
    launch, route = pred_route(jb)
    w, h = int(jb["pw"]), int(jb["ph"])
    satd, cflag, avgpp = jb["cost"] == 1, bool(jb["flags"] & 1), bool(jb["flags"] & 2)
    out = set()
    if route.startswith("uni") or route == "bi_small":
        wpr = (w * es) >> 2                                                         # me_set_shape (me.cuh:61-69)
        fal = (fenc_addr + int(jb["offset"]) * es) | (fstride * es)
        lgsegw = min(wpr.bit_length() - 1, 2 if fal & 15 == 0 else 1 if fal & 7 == 0 else 0)
        if (fstride * es) & 7:                                                      # me.cuh:1644
            out.add("rstride_override")
            lgsegw = 0
        out.add("lgsegw%d" % lgsegw)
    if route.startswith("uni"):
        out.add(route)
        if satd and chroma and cflag and w % 8 == 0 and h % 8 == 0:                 # :400, me.cuh:970
            out.add("uni_chroma")
        return out
    if route == "bi_small":
        out.add("bi_small_luma8" if w >= 8 else "bi_small_luma4")
        if avgpp:
            out.add("bi_small_avgpp")
        if satd and not avgpp and chroma and cflag and w % 8 == 0 and h % 8 == 0:  # :386, me.cuh:970
            out.add("bi_small_chroma")
        return out
    out.add(route)
    kind = "pixel" if avgpp else "short"                                           # :108-134
    for l in (0, 1):
        out.add("staged_luma_%s_%s" % (kind, _phase([int(v) for v in jb["mv%d" % l]], 2)))
    assert satd, "two-list SAD: outside the API (SAD jobs are Search::selectMVP's, one list)"
    out.add("staged_satd8x4" if w % 8 == 0 else "staged_satd4x4")                # :150-168
    cw, chh = w >> 1, h >> 1
    if satd and cflag and not avgpp and chroma and cw % 4 == 0 and chh % 4 == 0:   # :199
        out.add("staged_chroma_w%d" % cw)
        for l in (0, 1):
            out.add("staged_chroma_short_%s" % _phase([int(v) for v in jb["mv%d" % l]], 3))
    return out


def trip_paths(jobs, sms):
    """warp_trips / cta_trips: a job of that launch at an index past the first grid-stride trip (:431-436)"""
    n = len(jobs)
    per_warp = 4 * min((n + 3) // 4, 16 * sms)
    per_cta = min(n, 16 * sms)
    out = set()
    for i in range(per_cta, n):
        r = pred_route(jobs[i])[1]
        if r == "bi_cta":
            out.add("cta_trips")
        elif r == "bi_warp" and i >= per_warp:
            out.add("warp_trips")
        if len(out) == 2:
            break
    return out


# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def cu():
    import x265_b200
    return x265_b200.load()


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


class DevPics:
    """Device copies of a Pics; the tables point at each plane's pixel (0, 0)"""

    def __init__(self, cu, pics):
        self.cu, self.pics = cu, pics
        es = self.es = np.dtype(pixel_dtype(pics.depth)).itemsize
        self.bufs = []

        def up(a):
            b = cu.to_device(a)
            self.bufs.append(b)
            return b
        self.fenc = up(pics.fenc)
        refs = [up(r) for r in pics.refs]
        fc = [up(c) for c in pics.fc]
        rc = [[up(c) for c in pair] for pair in pics.rc]
        self.tab = up(np.array([r.ptr + pics.org * es for r in refs], np.uint64))
        self.tcb = up(np.array([p[0].ptr + pics.corg * es for p in rc], np.uint64))
        self.tcr = up(np.array([p[1].ptr + pics.corg * es for p in rc], np.uint64))
        self.fenc_at = self.fenc.ptr + pics.org * es
        self.fc_at = [c.ptr + pics.corg * es for c in fc]

    def run(self, jobs, chroma=True):
        """x265cu_pred_cost_batch of the list into a sentinel-filled output; returns the output"""
        cu, pics = self.cu, self.pics

        class At:
            def __init__(self, p): self.ptr = p
        dj = cu.to_device(np.ascontiguousarray(jobs))
        do = cu.to_device(np.full(len(jobs), SENTINEL, np.int32))
        ch = (At(self.fc_at[0]), At(self.fc_at[1]), self.tcb, self.tcr, pics.cstride) if chroma else None
        cu.pred_cost_batch(pics.depth, At(self.fenc_at), pics.stride, self.tab, pics.stride, ch, dj, len(jobs), do)
        got = do.download(np.int32)
        dj.free(); do.free()
        return got

    def paths(self, jobs, chroma=True):
        out = set()
        for jb in jobs:
            out |= pred_paths(jb, chroma, self.fenc_at, self.pics.stride, self.es)
        return out

    def free(self):
        for b in self.bufs:
            b.free()


def assert_costs(dp, jobs, got, chroma, what):
    """every entry written, and equal to the oracle's (and the reference's, where oracle/_ref is built)"""
    pics = dp.pics
    unwritten = np.nonzero(got == SENTINEL)[0]
    assert unwritten.size == 0, "%s: %d entries not written, first %s (routes %s)" % (
        what, unwritten.size, unwritten[:6].tolist(), [pred_route(jobs[i])[1] for i in unwritten[:6]])
    want = ph.oracle_batch(load_oracle(pics.depth), pics, jobs, chroma)
    R = load_ref(pics.depth)
    for who, w in (("oracle", want), ("reference", ph.ref_batch(R, pics, jobs, chroma) if R is not None else None)):
        if w is None:
            continue
        bad = np.nonzero(got != w)[0]
        assert bad.size == 0, "%s: %d costs differ from the %s's, first: %s" % (
            what, bad.size, who, [(int(i), pred_route(jobs[i])[1], jobs[i].tolist(), int(got[i]), int(w[i])) for i in bad[:6]])


def run_case(cu, pics, jobs, targets, what):
    """targets: {chroma planes given: the paths the list must reach}; runs the list with chroma planes and with NULL"""
    assert ph.reads_in_margins(pics, jobs).all(), "%s: a job reads past the margins (outside the API's contract)" % what
    dp = DevPics(cu, pics)
    try:
        for chroma in (True, False):
            missing = set(targets[chroma]) - dp.paths(jobs, chroma)
            assert not missing, "%s (chroma planes %s) does not reach %s" % (what, chroma, sorted(missing))
            assert_costs(dp, jobs, dp.run(jobs, chroma), chroma, "%s, chroma planes %s" % (what, chroma))
    finally:
        dp.free()


# ---------------------------------------------------------------------------------------------------------------------
ROUTES = ("uni_small", "uni_big", "uni_chroma", "bi_small_luma8", "bi_small_luma4", "bi_small_avgpp", "bi_small_chroma", "bi_warp", "bi_cta")
STAGED = tuple(p for p in PATHS if p.startswith("staged_"))
SWEEP_TARGETS = set(ROUTES) | set(STAGED)


@pytest.mark.parametrize("depth", DEPTHS)
@pytest.mark.parametrize("content", ["sweep_smooth", "sweep_random"])
def test_route_phase_sweep(cu, depth, content):
    """Every PU shape x every kind of job (pred_helpers.SWEEP_KINDS: one list L0 / L1, two lists with addAvg and with
    pixelavg_pp, SAD and SATD, chroma flag on and off, ref0 == ref1 with equal vectors) x every luma phase pair of each list,
    every eighth-pel pair for shapes with a chroma SATD; with chroma planes and with NULL"""
    pics, jobs, kinds = ph.family(content, depth)
    luma_only = {p for p in SWEEP_TARGETS if "chroma" not in p}
    run_case(cu, pics, jobs, {True: SWEEP_TARGETS, False: luma_only}, content)
    same = [jb for jb, k in zip(jobs, kinds) if k == "bi_same_ref"]
    assert all(jb["ref0"] == jb["ref1"] and tuple(jb["mv0"]) == tuple(jb["mv1"]) for jb in same) and len(same) > 100


@pytest.mark.parametrize("depth", DEPTHS)
def test_clip_limits(cu, depth):
    """PUs of CUs 64 / 32 / 16 / 8 (AMP parts included) at the corners and edge midpoints of a 192x128 picture, vectors at and
    just inside CUData::clipMv's box with every fraction it allows, planes in a poison-filled guard band"""
    pics, jobs, _ = ph.family("clip", depth)
    targets = {"uni_small", "uni_big", "uni_chroma", "bi_small_luma8", "bi_small_luma4", "bi_small_avgpp", "bi_small_chroma", "bi_warp", "bi_cta"}
    run_case(cu, pics, jobs, {True: targets, False: targets - {"uni_chroma", "bi_small_chroma"}}, "clip limits")


@pytest.mark.parametrize("depth", DEPTHS)
def test_saturated_content(cu, depth):
    """0 / maxv blocks and edges: the pixel-path interpolation and the addAvg clips engage at both ends (the share is asserted
    by test_pred_oracle_vs_ref.py::test_saturated_content_engages_the_clips on the same list)"""
    pics, jobs, _ = ph.family("saturated", depth)
    targets = {"uni_small", "uni_big", "uni_chroma", "bi_small_luma8", "bi_small_chroma", "bi_warp", "bi_cta", "staged_luma_short_hv", "staged_luma_pixel_hv"}
    run_case(cu, pics, jobs, {True: targets, False: targets - {"uni_chroma", "bi_small_chroma"}}, "saturated")


STRIDE_TARGETS = {(8, "stride16"): {"lgsegw2", "lgsegw1", "lgsegw0"}, (8, "stride8"): {"lgsegw1", "lgsegw0"},
                  (8, "stride4"): {"lgsegw0", "rstride_override"}, (10, "stride16"): {"lgsegw2", "lgsegw1"},
                  (10, "stride8"): {"lgsegw1"}, (10, "stride4"): {"lgsegw0", "rstride_override"}}


@pytest.mark.parametrize("depth", DEPTHS)
@pytest.mark.parametrize("name", ["stride16", "stride8", "stride4"])
def test_strides_and_bases(cu, depth, name):
    """Luma row pitches of a multiple of 16 bytes, of 8 and of 4 only (pred_helpers.STRIDES), PU x positions of every
    multiple-of-4 residue mod 16: every fenc segment width of me_set_shape and the row-pitch override"""
    pics, jobs, _ = ph.family(name, depth)
    t = STRIDE_TARGETS[(depth, name)] | {"uni_small", "uni_big", "bi_small_luma8", "bi_warp", "bi_cta"}
    run_case(cu, pics, jobs, {True: t, False: t}, name)


FRAME_CASES = [(8, True, "against", 57), (8, False, "against", 57), (10, True, "against", 57), (8, True, "far", 92)]


@pytest.mark.parametrize("case", FRAME_CASES, ids=["8-chroma", "8-avgpp", "10-chroma", "8-far-merange92"])
def test_past_one_grid(cu, sms, case):
    """bench.pred_jobs_of over the oracle frame driver's motion-search jobs and results of a 512x320 frame (rect + AMP, 2
    references): more jobs than 4 x 16 x SMs, so that both k_pred_cost launches take two or more grid-stride trips.  Chroma off
    makes the bi jobs pixelavg_pp; the far field with merange 92 clamps the windows at the picture edges."""
    depth, chroma, field, merange = case
    pics, jobs = ph.frame_jobs(depth, chroma, field, merange)
    assert len(jobs) > 4 * 16 * sms, (len(jobs), sms)
    t = {"warp_trips", "cta_trips", "uni_small", "uni_big", "bi_small_luma8", "bi_small_luma4", "bi_warp", "bi_cta"}
    t |= {"uni_chroma", "bi_small_chroma"} if chroma else {"bi_small_avgpp"}
    reached = trip_paths(jobs, sms)
    assert {"warp_trips", "cta_trips"} <= reached, reached
    dp = DevPics(cu, pics)
    try:
        missing = t - (dp.paths(jobs) | reached)
        assert not missing, missing
        assert ph.reads_in_margins(pics, jobs).all()
        assert_costs(dp, jobs, dp.run(jobs), True, "frame list %s" % (case,))
    finally:
        dp.free()


def _grid_plus_one(pics, jobs, sms, rng):
    """a list of exactly 4 x 16 x SMs + 1 jobs drawn from `jobs`, whose last job (the only one on the warp launch's second
    trip) is a 12x16 / 16x12 two-list job and whose CTA-launch jobs reach the later trips"""
    n = 4 * 16 * sms + 1
    pick = jobs[rng.integers(0, len(jobs), n)]
    warp = [jb for jb in jobs if pred_route(jb)[1] == "bi_warp"]
    pick[-1] = warp[int(rng.integers(0, len(warp)))]
    return pick


@pytest.mark.parametrize("depth", DEPTHS)
def test_grid_plus_one(cu, sms, depth):
    pics, jobs, _ = ph.family("sweep_random", depth)
    lst = _grid_plus_one(pics, jobs, sms, np.random.default_rng(depth))
    assert len(lst) == 4 * 16 * sms + 1
    assert trip_paths(lst, sms) == {"warp_trips", "cta_trips"}
    dp = DevPics(cu, pics)
    try:
        assert_costs(dp, lst, dp.run(lst), True, "4 x 16 x SMs + 1 jobs")
    finally:
        dp.free()


@pytest.mark.parametrize("depth", DEPTHS)
def test_list_properties(cu, depth):
    """A shuffled copy gives the same per-job costs, two calls give identical results, a call makes 4 launches; n = 1 on each
    route and a list of one route only give the costs of the same jobs in the whole list"""
    pics, jobs, _ = ph.family("sweep_random", depth)
    dp = DevPics(cu, pics)
    try:
        base = dp.run(jobs)
        assert_costs(dp, jobs, base, True, "whole list")
        assert np.array_equal(dp.run(jobs), base), "two calls differ"
        perm = np.random.default_rng(depth).permutation(len(jobs))
        assert np.array_equal(dp.run(jobs[perm]), base[perm]), "a shuffled list gives other costs"
        n0 = cu.launch_count()
        dp.run(jobs[:8])
        assert cu.launch_count() - n0 == 4
        routes = np.array([pred_route(jb)[1] for jb in jobs])
        for r in ("uni_small", "uni_big", "bi_small", "bi_warp", "bi_cta"):
            idx = np.nonzero(routes == r)[0]
            assert idx.size > 0, r
            one = dp.run(jobs[idx[:1]])
            assert one[0] == base[idx[0]], ("n = 1", r, int(one[0]), int(base[idx[0]]))
            assert np.array_equal(dp.run(jobs[idx]), base[idx]), ("one route only", r)
    finally:
        dp.free()


# ---------------------------------------------------------------------------------------------------------------------
def _targets():
    """the paths the cases above name"""
    t = set(SWEEP_TARGETS)
    for v in STRIDE_TARGETS.values():
        t |= v
    return t | {"warp_trips", "cta_trips"}


def test_every_path_is_targeted():
    assert _targets() == set(PATHS), (set(PATHS) - _targets(), _targets() - set(PATHS))
