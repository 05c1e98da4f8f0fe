"""GPU parity: batched motion estimation (x265cu_me_batch, one warp per MotionEstimate::motionEstimate
call, motion.cpp:739-1569) against the oracle restatement, which test_oracle_vs_ref.py pins to the
real reference MotionEstimate.  Bit-exact (cost, qmv.x, qmv.y) for DIA / HEX / STAR, all PU sizes,
all sub-pel levels, full-res and lowres planes, 8 and 10 bit."""
import ctypes as C
import numpy as np
import pytest

from common import load_oracle, ptr, pixel_dtype, make_plane, P, I, IP
from me_helpers import OrcMeJob, mvcost_table, lowres_planes, MVRANGE

pytestmark = pytest.mark.gpu

SIZES = [(8, 8), (16, 16), (32, 32), (64, 64), (16, 8), (8, 16), (32, 16), (16, 32), (64, 32), (32, 64), (16, 12), (12, 16),
         (16, 4), (4, 16), (32, 24), (24, 32), (32, 8), (8, 32), (64, 48), (48, 64), (64, 16), (16, 64), (8, 4), (4, 8)]


@pytest.fixture(scope="module")
def cu():
    import x265_b200
    return x265_b200.load()


def build_jobs(rng, W, H, margin, stride, org, n, method, lowres, merange):
    from x265_b200.lib import ME_JOB
    jobs = np.zeros(n, ME_JOB)
    for t in range(n):
        w, h = (8, 8) if lowres else SIZES[int(rng.integers(0, len(SIZES)))]
        bx = int(rng.integers(0, (W - w) // 4 + 1)) * 4
        by = int(rng.integers(0, (H - h) // 4 + 1)) * 4
        qmvp = (int(rng.integers(-40, 41)), int(rng.integers(-40, 41)))
        lim = margin - 12
        j = jobs[t]
        j["offset"] = org + by * stride + bx
        j["ref"] = 0
        j["pw"] = w; j["ph"] = h
        j["mvmin"] = (max(-bx - lim, (qmvp[0] >> 2) - merange), max(-by - lim, (qmvp[1] >> 2) - merange))
        j["mvmax"] = (min(W - w - bx + lim, (qmvp[0] >> 2) + merange), min(H - h - by + lim, (qmvp[1] >> 2) + merange))
        j["qmvp"] = qmvp
        nc = 0 if lowres else int(rng.integers(0, 4))
        j["numCand"] = nc
        j["mvc"] = rng.integers(-60, 61, 8)
        j["method"] = method
        j["subme"] = int(rng.integers(0, 8))
        j["merange"] = merange
    return jobs


def oracle_run(O, depth, fenc, refs, stride, jobs, lowres, tab):
    out = np.zeros((len(jobs), 4), np.int32)
    O.orc_motion_estimate.argtypes = [C.POINTER(OrcMeJob), P]
    for t, j in enumerate(jobs):
        job = OrcMeJob()
        job.fenc = fenc.ctypes.data; job.fencStride = stride; job.offset = int(j["offset"])
        for i in range(4):
            job.ref[i] = refs[i].ctypes.data
        job.refStride = stride; job.lowres = lowres; job.pw = int(j["pw"]); job.ph = int(j["ph"])
        job.method = int(j["method"]); job.subme = int(j["subme"])
        job.mvmin[0], job.mvmin[1] = int(j["mvmin"][0]), int(j["mvmin"][1])
        job.mvmax[0], job.mvmax[1] = int(j["mvmax"][0]), int(j["mvmax"][1])
        job.qmvp[0], job.qmvp[1] = int(j["qmvp"][0]), int(j["qmvp"][1])
        mvc = np.ascontiguousarray(j["mvc"].astype(np.int32))
        job.numCand = int(j["numCand"]); job.mvc = mvc.ctypes.data; job.merange = int(j["merange"])
        job.mvcost = tab.ctypes.data + MVRANGE * 2
        q = np.zeros(2, np.int32)
        out[t, 0] = O.orc_motion_estimate(C.byref(job), ptr(q))
        out[t, 1:3] = q
    return out


@pytest.mark.parametrize("depth", [8, 10])
@pytest.mark.parametrize("method", [0, 1, 3, 5])
@pytest.mark.parametrize("lowres", [0, 1])
@pytest.mark.parametrize("smooth", [True, False])
def test_me_batch(cu, depth, method, lowres, smooth, lam=None):
    """lam: the mv cost lambda, by default that of QP 33."""
    O = load_oracle(depth)
    rng = np.random.default_rng(100 + method * 7 + lowres * 3 + depth + smooth)
    W, H, margin = 256, 192, 96
    mx = (1 << depth) - 1
    merange = 57 if (method == 3 and not lowres) else (9 if method == 5 else 16)      # 5 = X265_FULL_SEARCH: exhaustive
    if lowres:
        yy, xx = np.mgrid[0:H * 2, 0:W * 2]
        def img(shift):
            if smooth:
                v = 128 + 60 * np.sin((xx + 3 * shift) / 37.0) + 40 * np.cos((yy - 2 * shift) / 29.0) + rng.integers(-6, 7, xx.shape)
                return (np.clip(v, 0, 255).astype(np.int64) << (depth - 8)).astype(pixel_dtype(depth))
            return rng.integers(0, mx + 1, xx.shape).astype(pixel_dtype(depth))
        fpl, stride, org, _, _ = lowres_planes(O, depth, img(0), W * 2, H * 2, margin)
        refs, _, _, _, _ = lowres_planes(O, depth, img(2), W * 2, H * 2, margin)
        fenc = fpl[0]
    else:
        fenc, stride, org = make_plane(rng, depth, W, H, margin, smooth=smooth)
        refb, _, _ = make_plane(rng, depth, W, H, margin, smooth=smooth)
        if smooth:
            sh = np.roll(np.roll(fenc, 5, axis=0), -7, axis=1)
            refb = np.clip(sh.astype(np.int64) + rng.integers(-3, 4, sh.shape), 0, mx).astype(fenc.dtype)
        refs = [refb] * 4
    n = 160 if method != 3 else 96
    jobs = build_jobs(rng, W, H, margin, stride, org, n, method, lowres, merange)
    if lam is None:
        lam = 11.3137 if depth == 8 else 45.2548
    tab = mvcost_table(O, lam)
    want = oracle_run(O, depth, fenc, refs, stride, jobs, lowres, tab)

    assert np.array_equal(cu.mvcost_table(lam, MVRANGE), tab)       # host table builder is bit-exact
    d_fenc = cu.to_device(fenc)
    d_refs = [cu.to_device(r) for r in (refs if lowres else refs[:1])]
    table = np.array([d.ptr for d in d_refs], np.uint64)
    d_table = cu.to_device(table)
    d_tab = cu.to_device(tab)
    d_jobs = cu.to_device(jobs)
    d_out = cu.alloc(n * 16)
    cu.me_batch(depth, d_fenc, stride, d_table, stride, lowres, d_tab, MVRANGE, d_jobs, n, d_out)
    got = d_out.download(np.int32).reshape(n, 4)
    bad = np.nonzero((got[:, :3] != want[:, :3]).any(axis=1))[0]
    assert len(bad) == 0, (len(bad), [(jobs[b].tolist(), got[b].tolist(), want[b].tolist()) for b in bad[:3]])
    for d in [d_fenc, d_table, d_tab, d_jobs, d_out] + d_refs:
        d.free()


@pytest.mark.parametrize("depth", [8, 10])
@pytest.mark.parametrize("method", [0, 1, 3, 5])
@pytest.mark.parametrize("lowres", [0, 1])
@pytest.mark.parametrize("smooth", [True, False])
@pytest.mark.parametrize("qp", ["0", "top"])
def test_me_batch_qp_extremes(cu, depth, method, lowres, smooth, qp):
    """The same jobs with the lambda of QP 0 (mv costs of 0 to 2 near the MVP: SAD ties decide the arg-mins) and of the
    top QP, 51 or 63 at 10 bit (the MVP dominates, and at 10 bit the cost table reaches its cap of 32767)."""
    from frame_helpers import lambda_for, qp_max
    test_me_batch(cu, depth, method, lowres, smooth, lam=lambda_for(0 if qp == "0" else qp_max(depth), depth))


FAR_RANGES = {0: 57, 1: 57, 3: 92, 5: 8}


@pytest.mark.parametrize("depth", [8, 10])
@pytest.mark.parametrize("method", [0, 1, 3, 5])
@pytest.mark.parametrize("chroma", [False, True])
def test_me_batch_far_predictor(cu, depth, method, chroma):
    """Predictors beyond the search range: MV 0 wins the pre-checks and the search starts outside [mvmin.x, mvmax.x]
    (test_oracle_vs_ref.py::test_motion_estimate_far_predictor pins the oracle to the reference there).  Reference 0 is the
    source itself (static), reference 1 the source moved by (2, -1) px, so that the search moves on from MV 0 in many jobs.
    x265cu_me_batch and x265cu_me_batch_chroma against the oracle, every PU size."""
    from me_helpers import far_window, mv0_wins, orc_chroma_job, shifted
    from x265_b200.lib import ME_JOB
    O = load_oracle(depth)
    rng = np.random.default_rng(700 + 11 * method + depth + chroma)
    W, H, margin = 256, 192, 96
    merange = FAR_RANGES[method]
    fenc, stride, org = make_plane(rng, depth, W, H, margin, smooth=True)
    fc = [make_plane(rng, depth, W // 2, H // 2, margin // 2, smooth=True)[0] for _ in range(2)]
    cstride = fc[0].shape[1]
    refs, refc = [fenc, shifted(fenc, (2, -1))], [fc, [shifted(c, (1, -1)) for c in fc]]
    n = 96
    jobs = np.zeros(n, ME_JOB)
    for t in range(n):
        w, h = SIZES[t % len(SIZES)]
        bx = int(rng.integers(0, (W - w) // 8 + 1)) * 8; by = int(rng.integers(0, (H - h) // 8 + 1)) * 8
        qmvp, mvmin, mvmax = far_window(rng, W, H, w, h, bx, by, margin, merange)
        j = jobs[t]
        j["offset"] = org + by * stride + bx
        j["ref"] = t & 1
        j["pw"] = w; j["ph"] = h
        j["mvmin"] = mvmin; j["mvmax"] = mvmax; j["qmvp"] = qmvp
        j["numCand"] = int(rng.integers(0, 4))
        j["mvc"] = rng.integers(-60, 61, 8)
        j["method"] = method
        j["subme"] = int(rng.integers(0, 8))
        j["merange"] = merange
    lam = 11.3137 if depth == 8 else 45.2548
    tab = mvcost_table(O, lam)
    want = np.zeros((n, 4), np.int32)
    O.orc_motion_estimate.argtypes = [C.POINTER(OrcMeJob), P]
    wins = moved = 0
    for t, j in enumerate(jobs):
        r = int(j["ref"])
        one = dict(fenc=fenc, ref=refs[r], stride=stride, fc=fc, rc=refc[r], cstride=cstride, offset=int(j["offset"]),
                   qmvp=tuple(int(v) for v in j["qmvp"]), mvmin=tuple(int(v) for v in j["mvmin"]),
                   mvmax=tuple(int(v) for v in j["mvmax"]), ncand=int(j["numCand"]),
                   mvc=np.ascontiguousarray(j["mvc"].astype(np.int32)), w=int(j["pw"]), h=int(j["ph"]))
        job = orc_chroma_job(O, one, method, int(j["subme"]), merange, tab)
        job.chroma = int(chroma)
        q = np.zeros(2, np.int32)
        want[t, 0] = O.orc_motion_estimate(C.byref(job), ptr(q))
        want[t, 1:3] = q
        wins += mv0_wins(fenc, refs[r], stride, one["offset"], one["w"], one["h"], one["qmvp"], one["mvmin"], one["mvmax"], tab)
        moved += abs(int(q[0])) >= 4 and not (4 * one["mvmin"][0] <= int(q[0]) <= 4 * one["mvmax"][0])
    # the state under test: 0 outside every job's x range, MV 0 the start of most searches, which often move on from there
    # while still outside the range (FULL scans only the range)
    assert ((jobs["mvmin"][:, 0] > 0) | (jobs["mvmax"][:, 0] < 0)).all() and wins > 0.7 * n, wins
    assert method == 5 or moved > 0.1 * n, moved

    bufs = []
    def dev(a):
        d = cu.to_device(a); bufs.append(d); return d
    d_fenc = dev(fenc)
    d_refs = [d_fenc, dev(refs[1])]
    d_table = dev(np.array([d.ptr for d in d_refs], np.uint64))
    d_tab = dev(tab); d_jobs = dev(jobs)
    d_out = cu.alloc(n * 16); bufs.append(d_out)
    if chroma:
        d_cb, d_cr = dev(fc[0]), dev(fc[1])
        d_rc = [(d_cb, d_cr), (dev(refc[1][0]), dev(refc[1][1]))]
        d_cbt, d_crt = dev(np.array([d[0].ptr for d in d_rc], np.uint64)), dev(np.array([d[1].ptr for d in d_rc], np.uint64))
        cu.me_batch_chroma(depth, d_fenc, stride, d_table, stride, d_cb, d_cr, d_cbt, d_crt, cstride, d_tab, MVRANGE, d_jobs, n, d_out)
    else:
        cu.me_batch(depth, d_fenc, stride, d_table, stride, 0, d_tab, MVRANGE, d_jobs, n, d_out)
    got = d_out.download(np.int32).reshape(n, 4)
    bad = np.nonzero((got[:, :3] != want[:, :3]).any(axis=1))[0]
    assert len(bad) == 0, (len(bad), [(jobs[b].tolist(), got[b].tolist(), want[b].tolist()) for b in bad[:3]])
    for d in bufs:
        d.free()


@pytest.mark.parametrize("depth", [8, 10])
@pytest.mark.parametrize("method", [1, 3])
@pytest.mark.parametrize("smooth", [True, False])
def test_me_batch_chroma(cu, depth, method, smooth):
    """x265cu_me_batch_chroma: the chroma-SATD term of subpelCompare (motion.cpp:1601-1661) for 4:2:0, bit-exact against
    the oracle (pinned to the real MotionEstimate by test_oracle_vs_ref.py::test_motion_estimate_chroma_satd).  The
    job list mixes PU sizes / sub-pel levels with and without the term, two references."""
    from me_helpers import chroma_case, orc_chroma_job
    from x265_b200.lib import ME_JOB
    O = load_oracle(depth)
    rng = np.random.default_rng(300 + method * 5 + depth + smooth)
    W, H, margin = 256, 192, 96
    merange = 57 if method == 3 else 16
    cs = [chroma_case(depth, rng, 8, 8, smooth, merange, W, H, margin) for _ in range(2)]     # two references (+ their chroma)
    stride, cstride = cs[0]["stride"], cs[0]["cstride"]
    org = margin * stride + margin
    fenc, fc = cs[0]["fenc"], cs[0]["fc"]
    n = 128 if method != 3 else 80
    jobs = np.zeros(n, ME_JOB)
    for t in range(n):
        w, h = SIZES[int(rng.integers(0, len(SIZES)))]
        bx = int(rng.integers(0, (W - w) // 8 + 1)) * 8; by = int(rng.integers(0, (H - h) // 8 + 1)) * 8
        qmvp = (int(rng.integers(-40, 41)), int(rng.integers(-40, 41)))
        lim = margin - 12
        j = jobs[t]
        j["offset"] = org + by * stride + bx
        j["ref"] = t & 1
        j["pw"] = w; j["ph"] = h
        j["mvmin"] = (max(-bx - lim, (qmvp[0] >> 2) - merange), max(-by - lim, (qmvp[1] >> 2) - merange))
        j["mvmax"] = (min(W - w - bx + lim, (qmvp[0] >> 2) + merange), min(H - h - by + lim, (qmvp[1] >> 2) + merange))
        j["qmvp"] = qmvp
        j["numCand"] = int(rng.integers(0, 4))
        j["mvc"] = rng.integers(-60, 61, 8)
        j["method"] = method
        j["subme"] = int(rng.integers(2, 8))
        j["merange"] = merange
    lam = 11.3137 if depth == 8 else 45.2548
    tab = mvcost_table(O, lam)
    want = np.zeros((n, 4), np.int32)
    O.orc_motion_estimate.argtypes = [C.POINTER(OrcMeJob), P]
    nchroma = 0
    for t, j in enumerate(jobs):
        r = int(j["ref"])
        one = dict(fenc=fenc, ref=cs[r]["ref"], stride=stride, fc=fc, rc=cs[r]["rc"], cstride=cstride, offset=int(j["offset"]),
                   qmvp=(int(j["qmvp"][0]), int(j["qmvp"][1])), mvmin=(int(j["mvmin"][0]), int(j["mvmin"][1])),
                   mvmax=(int(j["mvmax"][0]), int(j["mvmax"][1])), ncand=int(j["numCand"]),
                   mvc=np.ascontiguousarray(j["mvc"].astype(np.int32)), w=int(j["pw"]), h=int(j["ph"]))
        job = orc_chroma_job(O, one, method, int(j["subme"]), merange, tab)
        q = np.zeros(2, np.int32)
        want[t, 0] = O.orc_motion_estimate(C.byref(job), ptr(q))
        want[t, 1:3] = q
        nchroma += int(j["subme"]) > 2 and one["w"] % 8 == 0 and one["h"] % 8 == 0
    assert nchroma > n // 3

    bufs = []
    def dev(a):
        d = cu.to_device(a); bufs.append(d); return d
    d_fenc = dev(fenc)
    d_refs = [dev(c["ref"]) for c in cs]
    d_table = dev(np.array([d.ptr for d in d_refs], np.uint64))
    d_fcb, d_fcr = dev(fc[0]), dev(fc[1])
    d_rcb = [dev(c["rc"][0]) for c in cs]; d_rcr = [dev(c["rc"][1]) for c in cs]
    d_cbt = dev(np.array([d.ptr for d in d_rcb], np.uint64)); d_crt = dev(np.array([d.ptr for d in d_rcr], np.uint64))
    d_tab = dev(tab); d_jobs = dev(jobs)
    d_out = cu.alloc(n * 16); bufs.append(d_out)
    cu.me_batch_chroma(depth, d_fenc, stride, d_table, stride, d_fcb, d_fcr, d_cbt, d_crt, cstride, d_tab, MVRANGE, d_jobs, n, d_out)
    got = d_out.download(np.int32).reshape(n, 4)
    bad = np.nonzero((got[:, :3] != want[:, :3]).any(axis=1))[0]
    assert len(bad) == 0, (len(bad), [(jobs[b].tolist(), got[b].tolist(), want[b].tolist()) for b in bad[:3]])
    # the luma-only entry point on the same jobs must differ somewhere (the term is really active) ...
    cu.me_batch(depth, d_fenc, stride, d_table, stride, 0, d_tab, MVRANGE, d_jobs, n, d_out)
    luma = d_out.download(np.int32).reshape(n, 4)
    assert (luma[:, 0] != got[:, 0]).sum() > n // 4
    # ... and agree on every job for which the reference switches the term off
    off = np.array([not (int(j["subme"]) > 2 and int(j["pw"]) % 8 == 0 and int(j["ph"]) % 8 == 0) for j in jobs])
    assert np.array_equal(luma[off, :3], got[off, :3])
    for d in bufs:
        d.free()
