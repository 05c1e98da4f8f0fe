"""Frame-level workload helpers shared by tests and bench.py: synthetic frames (BASELINE.md
generator), margin-extended planes, the predictor field, and the ctypes view of the CPU drivers
(oracle/frame_driver.h instantiated by the oracle and by the reference shim)."""
import ctypes as C
import numpy as np

from common import P, I, ptr, pixel_dtype

MARGIN_X, MARGIN_Y = 96, 80          # picyuv.cpp:87-88 for CTU 64
MVRANGE = 65536


class FsParams(C.Structure):
    _fields_ = [("width", I), ("height", I), ("stride", I), ("numRefs", I), ("method", I), ("subme", I),
                ("merange", I), ("rect", I), ("qp", I), ("amp", I)]


class DrvFrame(C.Structure):
    _fields_ = [("p", FsParams), ("fenc", P), ("refs", P * 16), ("field", P), ("mvcost", P),
                ("njobs", I), ("jobs", P), ("me_out", P),
                ("ncu", I), ("cus", P), ("cu_jobs", P), ("cu_coef_off", P), ("coef", P), ("recon", P * 4),
                ("cu_sse", P), ("cu_numsig", P), ("cu_ref", P), ("intra_cost", P),
                ("threads", I), ("next", I), ("stage", I),
                ("chroma", I), ("cstride", I), ("fencC", P * 2), ("refC", (P * 2) * 16),
                ("maxCtuRows", I), ("njobs_run", I), ("ncu_run", I)]


def stride_for(width):
    return (width + 2 * MARGIN_X + 63) // 64 * 64


CONTENTS = ("smooth", "noise", "flat", "full10", "cut")
FIELDS = ("against", "true", "zero", "mixed", "far")
# content="cut" is a cut from black: its reference frames are black in every plane (Workload), so the prediction is 0 at
# every vector, sub-pel ones included, and every SAD of a block ties


def _cut_areas(img, maxv, s):
    """The source of content "cut": full-white rectangles and one black one over the smooth clip, at the luma positions
    divided by s.  The first white rectangle is CTU (1, 0), so it covers whole 32x32 TUs with a constant residual; the
    second and the black one have edges that cut through TUs, whose ringing overshoots 0 and maxv."""
    H, W = img.shape[0] * s, img.shape[1] * s
    img[0:64 // s, 64 // s:128 // s] = maxv
    for (fx, fy, fw, fh), v in (((0.62, 0.50, 0.25, 0.30), maxv), ((0.08, 0.60, 0.20, 0.25), 0)):
        x0, y0 = int(fx * W) + 5, int(fy * H) + 3
        img[y0 // s:(y0 + int(fh * H)) // s, x0 // s:(x0 + int(fw * W)) // s] = v
    return img


def _flat_areas(img, flat_value, scale):
    """Letterbox bars (top and bottom eighth) and four constant rectangles, at the same place in every frame: the SADs
    there tie, as over the bars and plain backgrounds of real video."""
    H, W = img.shape
    bar = max(H // 8, 1)
    img[:bar, :] = flat_value
    img[H - bar:, :] = flat_value
    for k, (fx, fy, fw, fh) in enumerate(((0.10, 0.25, 0.20, 0.20), (0.45, 0.30, 0.12, 0.35),
                                          (0.70, 0.55, 0.22, 0.18), (0.05, 0.60, 0.30, 0.10))):
        x0, y0 = int(fx * W), int(fy * H)
        img[y0:y0 + max(int(fh * H), 1), x0:x0 + max(int(fw * W), 1)] = (40 + 50 * k) * scale
    return img


def gen_luma(W, H, n, s1=37.0, s2=29.0, bits=8, seed=265, noise=False, content=None, motion=(3, -2)):
    """Luma of frame n of the BASELINE.md synthetic clip (global motion `motion` px/frame, default (3,-2)).
    content: "smooth" (the default), "noise" (same as noise=True), "flat" (smooth plus static flat areas), "full10"
    (10 bit only: smooth content generated at 10 bits, saturating at 0 and 1023, with noise in the two low bits) or "cut"
    (the source of a cut from black: smooth plus full-white and black rectangles, _cut_areas)."""
    content = content or ("noise" if noise else "smooth")
    assert content in CONTENTS and (content != "full10" or bits == 10), (content, bits)
    dx, dy = motion
    rng = np.random.default_rng(seed + n)
    if content == "noise":
        y = rng.integers(0, 256, (H, W))
    elif content == "full10":
        yy, xx = np.mgrid[0:H, 0:W]
        y = 512 + 700 * np.sin((xx + dx * n) / s1) + 480 * np.cos((yy + dy * n) / s2) + rng.integers(-24, 25, (H, W))
        return np.clip(y, 0, 1023).astype(pixel_dtype(bits))
    else:
        yy, xx = np.mgrid[0:H, 0:W]
        y = 128 + 60 * np.sin((xx + dx * n) / s1) + 40 * np.cos((yy + dy * n) / s2) + rng.integers(-6, 7, (H, W))
    y = np.clip(y, 0, 255).astype(np.int64) << (bits - 8)
    if content == "flat":
        y = _flat_areas(y, 16 << (bits - 8), 1 << (bits - 8))
    elif content == "cut":
        y = _cut_areas(y, (1 << bits) - 1, 1)
    return y.astype(pixel_dtype(bits))


def gen_chroma(W, H, n, plane, bits=8, seed=265, noise=False, content=None, motion=(3, -2)):
    """Cb (plane 1) / Cr (plane 2) of frame n, 4:2:0: smooth sinusoids moving with the clip's global motion (half the luma
    displacement), BASELINE.md generator; `content` as in gen_luma."""
    content = content or ("noise" if noise else "smooth")
    assert content in CONTENTS and (content != "full10" or bits == 10), (content, bits)
    dx, dy = motion
    cw, ch = W // 2, H // 2
    rng = np.random.default_rng(seed + 1000 * plane + n)
    if content == "noise":
        c = rng.integers(0, 256, (ch, cw))
    else:
        yy, xx = np.mgrid[0:ch, 0:cw]
        ph = 0.7 * plane
        if content == "full10":
            c = 512 + 650 * np.sin((xx + dx / 2 * n) / 23.0 + ph) + 450 * np.cos((yy + dy / 2 * n) / 19.0 - ph) + rng.integers(-16, 17, (ch, cw))
            return np.clip(c, 0, 1023).astype(pixel_dtype(bits))
        c = 128 + 30 * np.sin((xx + dx / 2 * n) / 23.0 + ph) + 25 * np.cos((yy + dy / 2 * n) / 19.0 - ph) + rng.integers(-4, 5, (ch, cw))
    c = np.clip(c, 0, 255).astype(np.int64) << (bits - 8)
    if content == "flat":
        c = _flat_areas(c, 128 << (bits - 8), 1 << (bits - 8))
    elif content == "cut":
        c = _cut_areas(c, (1 << bits) - 1, 2)
    return c.astype(pixel_dtype(bits))


def pad_plane_c(img, depth, luma_stride):
    """Margin-extended chroma plane: stride = luma stride / 2, margins = half the luma margins (picyuv.cpp:87-94)."""
    H, W = img.shape
    mx, my, stride = MARGIN_X // 2, MARGIN_Y // 2, luma_stride // 2
    buf = np.zeros((H + 2 * my, stride), pixel_dtype(depth))
    buf[my:my + H, mx:mx + W] = img
    buf[my:my + H, :mx] = img[:, :1]
    buf[my:my + H, mx + W:mx + W + mx] = img[:, -1:]
    buf[:my, :] = buf[my:my + 1, :]
    buf[my + H:, :] = buf[my + H - 1:my + H, :]
    return buf, stride, my * stride + mx


def pad_plane(img, depth):
    """Margin-extended plane (replicated borders, pixel.cpp:1027-1041); returns (buffer, stride, origin element offset)."""
    H, W = img.shape
    stride = stride_for(W)
    buf = np.zeros((H + 2 * MARGIN_Y, stride), pixel_dtype(depth))
    buf[MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W] = img
    buf[MARGIN_Y:MARGIN_Y + H, :MARGIN_X] = img[:, :1]
    buf[MARGIN_Y:MARGIN_Y + H, MARGIN_X + W:MARGIN_X + W + MARGIN_X] = img[:, -1:]
    buf[:MARGIN_Y, :] = buf[MARGIN_Y:MARGIN_Y + 1, :]
    buf[MARGIN_Y + H:, :] = buf[MARGIN_Y + H - 1:MARGIN_Y + H, :]
    return buf, stride, MARGIN_Y * stride + MARGIN_X


def make_field(W, H, numRefs, seed=7, kind="against", motion=(3, -2), merange=57):
    """16x16-granular qpel predictor field.  A job's MVP is its block's entry, its two candidates are the entries to the
    right and below (k_build_me_jobs).  kind:
      "against": the default: against the clip's global motion of (3,-2) px per frame, (-12, 8) qpel per reference
                 distance, plus +-6 qpel of jitter (every MVP within about 10 px of zero);
      "true":    the real displacement of reference r, (r + 1) * motion px, plus +-2 qpel: the search converges at once;
      "zero":    all zero: no MV 0 check and no candidates;
      "mixed":   independent vectors up to +-256 qpel per block, a mix of zero, full-pel and fractional ones, with blocks
                 equal to their left neighbour (candidate 0 == MVP) and right / lower neighbour pairs equal (candidate 0
                 == candidate 1);
      "far":     |MVP| between merange + 8 and merange + 150 px in x and in y, random signs: 0 lies outside the search
                 range, and some windows point past the picture and collapse against its clamps."""
    assert kind in FIELDS, kind
    rng = np.random.default_rng(seed)
    fw, fh = (W + 15) // 16, (H + 15) // 16
    f = np.zeros((numRefs, fh, fw, 2), np.int16)
    for r in range(numRefs):
        if kind == "against":
            f[r, :, :, 0] = -12 * (r + 1) + rng.integers(-6, 7, (fh, fw))
            f[r, :, :, 1] = 8 * (r + 1) + rng.integers(-6, 7, (fh, fw))
        elif kind == "true":
            for c in range(2):
                f[r, :, :, c] = 4 * motion[c] * (r + 1) + rng.integers(-2, 3, (fh, fw))
        elif kind == "mixed":
            v = rng.integers(-256, 257, (fh, fw, 2))
            sort = rng.integers(0, 3, (fh, fw))
            v[sort == 0] = 0
            v[sort == 1] &= ~3
            for _ in range(fw * fh // 6):
                y, x = int(rng.integers(0, fh)), int(rng.integers(1, fw))
                v[y, x] = v[y, x - 1]
            for _ in range(fw * fh // 6):
                y, x = int(rng.integers(0, fh - 1)), int(rng.integers(0, fw - 1))
                v[y + 1, x] = v[y, x + 1]
            f[r] = v
        elif kind == "far":
            for c in range(2):
                mag = 4 * (merange + rng.integers(8, 151, (fh, fw))) + rng.integers(0, 4, (fh, fw))
                f[r, :, :, c] = np.where(rng.integers(0, 2, (fh, fw)) == 1, mag, -mag)
    return f


class Workload:
    """Inputs of one analysed frame (host side)."""

    def __init__(self, W, H, depth=8, numRefs=4, method=3, subme=3, merange=57, rect=1, qp=30, noise=False, seed=265, chroma=False, amp=0,
                 field="against", motion=(3, -2), content=None):
        """field: the predictor field's kind (make_field); motion: the clip's displacement per frame in px; content:
        "smooth" / "noise" / "flat" / "full10" / "cut" (gen_luma; default from `noise`).  With "cut" every reference
        plane is black."""
        self.W, self.H, self.depth = W, H, depth
        self.chroma = chroma
        self.stride = stride_for(W)
        self.params = dict(width=W, height=H, stride=self.stride, numRefs=numRefs, method=method, subme=subme,
                           merange=merange, rect=rect, qp=qp, amp=amp)
        gen = dict(bits=depth, seed=seed, noise=noise, content=content, motion=motion)
        black = content == "cut"
        cur = gen_luma(W, H, numRefs, **gen)
        self.fenc, _, self.org = pad_plane(cur, depth)
        self.refs = []
        for r in range(numRefs):
            img = np.zeros_like(cur) if black else gen_luma(W, H, numRefs - 1 - r, **gen)
            self.refs.append(pad_plane(img, depth)[0])
        self.field = make_field(W, H, numRefs, kind=field, motion=motion, merange=merange)
        if chroma:
            # 4:2:0 planes for the chroma-SATD term of subpelCompare: [Cb, Cr] of the source and of every reference
            self.fencC, self.refC = [], []
            for pl in (1, 2):
                buf, self.cstride, self.corg = pad_plane_c(gen_chroma(W, H, numRefs, pl, **gen), depth, self.stride)
                self.fencC.append(buf)
            for r in range(numRefs):
                self.refC.append([np.zeros_like(self.fencC[0]) if black else
                                  pad_plane_c(gen_chroma(W, H, numRefs - 1 - r, pl, **gen), depth, self.stride)[0]
                                  for pl in (1, 2)])


def lambda_for(qp, depth):
    # x265_lambda_tab (constants.cpp:33-50): 2^(qp/6-2) * 2^(depth-8), rounded to 4 decimals like the table
    return round(2.0 ** (qp / 6.0 - 2.0) * (1 << (depth - 8)), 4)


def qp_max(depth):
    """Highest quantiser QP: 51 plus QP_BD_OFFSET, because the quantiser of a 10-bit encode runs at the slice QP + 12
    (quant.cpp:224)."""
    return 51 + 6 * (depth - 8)


def tus(res):
    """(x, y, T, CU size, T x T levels) of every TU of a frame result (cpu_analyse's layout: the levels of a CU are
    contiguous from its cu_coef_off, its TUs in raster order)."""
    for (x, y, S), off in zip(res["cus"].tolist(), res["cu_coef_off"].tolist()):
        T = min(S, 32)
        for t in range((S // T) ** 2):
            ty, tx = divmod(t, S // T)
            yield x + tx * T, y + ty * T, T, S, res["coef"][off + t * T * T:off + (t + 1) * T * T].reshape(T, T)


def tu_class(levels):
    """"zero" (every level 0), "dc" (the only nonzero level is the DC one: the DC-only inverse transform, quant.cpp:588),
    "ac1" (one nonzero level, not the DC one: the full inverse transform although numSig is 1) or "full"."""
    nz = np.count_nonzero(levels)
    return "zero" if nz == 0 else "full" if nz > 1 else "dc" if levels[0, 0] else "ac1"


def tu_classes(res):
    """Counts of a frame's TUs by tu_class."""
    n = dict(zero=0, dc=0, ac1=0, full=0)
    for *_, levels in tus(res):
        n[tu_class(levels)] += 1
    return n


def _clip16(a):
    return np.clip(a, -32768, 32767)


def recon_overshoot(O, res, wl):
    """Pixels of a frame predicted by 0 (content "cut": black references) whose reconstructed residual lies outside
    0..maxv, so that the clip of the reconstruction decides them.  The residual is recomputed from the levels in integers
    as the encoder does it (quant.cpp:543-605): dequantisation, then the DC-only shortcut or the two clipped inverse
    passes with the oracle's DCT matrix.  Asserts that the driver's reconstruction is that residual clipped, so the
    count is of the residual the driver really added."""
    depth, maxv = wl.depth, (1 << wl.depth) - 1
    per, rem = divmod(wl.params["qp"], 6)
    scale = (40, 45, 51, 57, 64, 72)[rem] << per           # scalinglist.cpp:130, quant.cpp:567
    mats = {T: np.ctypeslib.as_array(C.cast(O.orc_dct_matrix(T), C.POINTER(C.c_int16)), (T, T)).astype(np.int64)
            for T in (4, 8, 16, 32)}
    n = 0
    for x, y, T, S, levels in tus(res):
        kind = tu_class(levels)
        if kind == "zero":
            r = np.zeros((T, T), np.int64)
        else:
            dqshift = 6 - (15 - depth - (T.bit_length() - 1))
            d = _clip16((levels.astype(np.int64) * scale + (1 << (dqshift - 1))) >> dqshift)
            if kind == "dc":
                sh = 12 - (depth - 8) - 3
                r = np.full((T, T), (((int(d[0, 0]) + 1) >> 1) * 8 + (1 << (sh - 1))) >> sh, np.int64)
            else:
                M, sh = mats[T], 12 - (depth - 8)
                r = _clip16((_clip16((M.T @ d + 64) >> 7) @ M + (1 << (sh - 1))) >> sh)
        rec = res["recon"][{64: 0, 32: 1, 16: 2, 8: 3}[S]][MARGIN_Y + y:MARGIN_Y + y + T, MARGIN_X + x:MARGIN_X + x + T]
        assert np.array_equal(rec, np.clip(r, 0, maxv)), (x, y, T, S)
        n += int(((r < 0) | (r > maxv)).sum())
    return n


# QPs of the QP-range frame cases: together they take every rem = qp % 6 and per = qp / 6 from 0 to the top (8, or 10 at
# 10 bit), the quantiser's scale tables and shifts
QPS = {8: (0, 7, 20, 33, 41, 46, 51), 10: (0, 3, 13, 26, 40, 47, 58, 63)}
# (content, depth, qp, chroma): "cut" at every QP, "noise" and "flat" with chroma at the lowest and the highest
QP_CASES = ([("cut", d, qp, False) for d in QPS for qp in QPS[d]] +
            [(c, d, qp, c == "flat") for c in ("noise", "flat") for d in QPS for qp in (QPS[d][0], QPS[d][-1])])


def assert_qp_case_reaches(O, content, wl, res):
    """Asserts, on the CPU driver's frame `res` of a QP_CASES workload, that the case reaches the quantiser states it is
    there for, so that it cannot pass without running them."""
    qp, top = wl.params["qp"], wl.params["qp"] == qp_max(wl.depth)
    n = tu_classes(res)
    total = sum(n.values())
    if content == "cut":
        # black references: every SAD of a block ties; whole-white TUs take the DC-only shortcut at every QP
        assert not any(r.any() for r in wl.refs) and n["dc"] > 0, n
        over = recon_overshoot(O, res, wl)
        if qp == 0:
            assert over > 0, "no reconstruction reaches the clip"
            # a white 32x32 TU has the DC coefficient 32736 at 10 bit, which quantises to 52377 at QP 0
            assert wl.depth == 8 or (res["coef"] == 32767).any(), "no level reaches the int16 clip"
    elif content == "noise":
        # full TUs at QP 0; at the top QP all-zero TUs and TUs whose one level is not the DC one
        assert (n["full"] > 0.9 * total) if qp == 0 else (n["zero"] > 0 and n["ac1"] > 0), n
    elif content == "flat":
        # static flat areas: all-zero TUs at QP 0, and nearly only those at the top QP
        assert n["zero"] > (0.8 * total if top else 0), n


def run_analyser(cu, wl, lam=None):
    """The workload through x265cu_analyser at its QP, with lambda_for(qp) unless `lam` is given (luma, and chroma when
    the workload has it).  Returns the open Analyser."""
    import x265_b200
    p, H, W = wl.params, wl.H, wl.W
    an = x265_b200.Analyser(cu, W, H, depth=wl.depth, numRefs=p["numRefs"], method=p["method"], subme=p["subme"],
                            merange=p["merange"], rect=p["rect"], qp=p["qp"],
                            lam=lambda_for(p["qp"], wl.depth) if lam is None else lam, amp=p["amp"])
    for r, ref in enumerate(wl.refs):
        an.set_ref(r, ref[MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W])
    if wl.chroma:
        an.enable_chroma()
        mx, my = MARGIN_X // 2, MARGIN_Y // 2

        def inner(c):
            return np.ascontiguousarray(c[my:my + H // 2, mx:mx + W // 2])
        for r in range(len(wl.refs)):
            an.set_ref_chroma(r, inner(wl.refC[r][0]), inner(wl.refC[r][1]))
        an.load_chroma(inner(wl.fencC[0]), inner(wl.fencC[1]))
    an.analyse(np.ascontiguousarray(wl.fenc[MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W]), wl.field)
    return an


def assert_frame_equal(an, want, wl):
    """Every output of the analyser `an` bit for bit against the CPU driver's frame `want` (cpu_analyse) on the workload
    wl: job and CU lists, ME results, reference choice, levels, significant-level counts, SSE, the four reconstruction
    planes and the intra costs."""
    H, W = wl.H, wl.W
    assert an.njobs == want["njobs"] and an.ncu == want["ncu"] and an.ncoef == want["ncoef"]
    jobs = an.fetch("jobs")
    assert np.array_equal(jobs, want["jobs"]), "job lists differ"
    assert np.array_equal(an.fetch("cu_jobs").reshape(-1, wl.params["numRefs"]), want["cu_jobs"])
    me = an.fetch("me_out").reshape(-1, 4)
    bad = np.nonzero((me[:, :3] != want["me_out"][:, :3]).any(axis=1))[0]
    assert len(bad) == 0, (len(bad), len(me), jobs[bad[:4]].tolist(), me[bad[:4]].tolist(), want["me_out"][bad[:4]].tolist())
    assert np.array_equal(an.cu_ref, want["cu_ref"])
    assert np.array_equal(an.fetch("coef"), want["coef"])
    assert np.array_equal(an.cu_numsig, want["cu_numsig"]) and np.array_equal(an.cu_sse, want["cu_sse"])
    for d in range(4):
        got = an.fetch("recon%d" % d).reshape(wl.fenc.shape)[MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W]
        assert np.array_equal(got, want["recon"][d][MARGIN_Y:MARGIN_Y + H, MARGIN_X:MARGIN_X + W]), "recon depth %d" % d
    assert np.array_equal(an.intra_cost, want["intra_cost"])


def cpu_analyse(lib, fn_name, wl, mvcost_tab, threads=1, stages=7, max_ctu_rows=0):
    """Run the CPU driver (oracle: orc_analyse_frame, reference: x265ref_analyse_frame)."""
    dt = pixel_dtype(wl.depth)
    f = DrvFrame()
    for k, v in wl.params.items():
        setattr(f.p, k, v)
    es = np.dtype(dt).itemsize
    f.fenc = wl.fenc.ctypes.data + wl.org * es
    for r, ref in enumerate(wl.refs):
        f.refs[r] = ref.ctypes.data + wl.org * es
    f.field = wl.field.ctypes.data
    f.mvcost = mvcost_tab.ctypes.data + MVRANGE * 2
    if getattr(wl, "chroma", False):
        f.chroma, f.cstride = 1, wl.cstride
        for k in range(2):
            f.fencC[k] = wl.fencC[k].ctypes.data + wl.corg * es
            for r in range(len(wl.refs)):
                f.refC[r][k] = wl.refC[r][k].ctypes.data + wl.corg * es
    W, H, nref = wl.W, wl.H, wl.params["numRefs"]
    ctus = ((W + 63) // 64) * ((H + 63) // 64)
    maxjobs = ctus * nref * 593
    maxcu = ctus * 85
    from x265_b200.lib import ME_JOB
    out = dict(
        jobs=np.zeros(maxjobs, ME_JOB), me_out=np.zeros((maxjobs, 4), np.int32),
        cus=np.zeros((maxcu, 3), np.int16), cu_jobs=np.zeros((maxcu, nref), np.int32),
        cu_coef_off=np.zeros(maxcu, np.int64), coef=np.zeros(ctus * 4096 * 4, np.int16),
        recon=[np.zeros_like(wl.fenc) for _ in range(4)],
        cu_sse=np.zeros(maxcu, np.uint64), cu_numsig=np.zeros(maxcu, np.uint32), cu_ref=np.zeros(maxcu, np.int32),
        intra_cost=np.zeros((maxcu, 36), np.uint32))
    f.jobs = out["jobs"].ctypes.data; f.me_out = out["me_out"].ctypes.data
    f.cus = out["cus"].ctypes.data; f.cu_jobs = out["cu_jobs"].ctypes.data
    f.cu_coef_off = out["cu_coef_off"].ctypes.data; f.coef = out["coef"].ctypes.data
    for d in range(4):
        f.recon[d] = out["recon"][d].ctypes.data + wl.org * es
    f.cu_sse = out["cu_sse"].ctypes.data; f.cu_numsig = out["cu_numsig"].ctypes.data
    f.cu_ref = out["cu_ref"].ctypes.data; f.intra_cost = out["intra_cost"].ctypes.data
    f.threads = threads
    f.maxCtuRows = max_ctu_rows
    fn = getattr(lib, fn_name)
    fn.argtypes = [C.POINTER(DrvFrame), I]
    fn(C.byref(f), stages)
    nj, nc = f.njobs, f.ncu
    ncoef = int(out["cu_coef_off"][nc - 1] + int(out["cus"][nc - 1][2]) ** 2) if nc else 0
    res = dict(njobs_run=f.njobs_run, ncu_run=f.ncu_run, njobs=nj, ncu=nc, ncoef=ncoef, jobs=out["jobs"][:nj], me_out=out["me_out"][:nj], cus=out["cus"][:nc],
               cu_jobs=out["cu_jobs"][:nc], cu_coef_off=out["cu_coef_off"][:nc], coef=out["coef"][:ncoef],
               recon=out["recon"], cu_sse=out["cu_sse"][:nc], cu_numsig=out["cu_numsig"][:nc], cu_ref=out["cu_ref"][:nc],
               intra_cost=out["intra_cost"][:nc])
    return res
