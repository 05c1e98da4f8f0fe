"""Prediction-cost jobs (AMVP candidate SAD, merge candidate / bidir SATD: search.cpp:1901-2023, 2474-2607): the oracle's
job struct (oracle/oracle_pred.c), the reference shim call (oracle/ref_shim.cpp: x265ref_pred_cost) and a case generator
shared by the CPU pin test and the GPU parity test; guarded pictures, the batch calls of oracle and reference and the case
families of the path tests (tests/test_gpu_pred_paths.py, tests/test_pred_oracle_vs_ref.py)."""
import ctypes as C

import numpy as np

from common import P, I, IP, pixel_dtype
from me_helpers import make_plane

LUMA_PUS = [(8, 8), (16, 16), (32, 32), (64, 64), (16, 8), (8, 16), (32, 16), (16, 32), (64, 32), (32, 64), (8, 4), (4, 8),
            (16, 12), (12, 16), (16, 4), (4, 16), (32, 24), (24, 32), (32, 8), (8, 32), (64, 48), (48, 64), (64, 16), (16, 64)]


class OrcPredJob(C.Structure):
    _fields_ = [("fenc", P * 3), ("ref0", P * 3), ("ref1", P * 3), ("stride", IP), ("cstride", IP), ("w", I), ("h", I),
                ("mv0", I * 2), ("mv1", I * 2), ("cost", I), ("chroma", I), ("biAvgPP", I)]


def make_planes(depth, rng, smooth, nrefs=2, W=256, H=192, margin=96):
    """Source + `nrefs` reference pictures, 4:2:0 (chroma at half size with half the margin)."""
    mx = (1 << depth) - 1
    fenc, stride, org = make_plane(rng, depth, W, H, margin, smooth=smooth)

    def ref_of(src, dy, dx):
        if not smooth:
            return rng.integers(0, mx + 1, src.shape).astype(src.dtype)
        sh = np.roll(np.roll(src, dy, axis=0), dx, axis=1)
        return np.clip(sh.astype(np.int64) + rng.integers(-3, 4, sh.shape), 0, mx).astype(src.dtype)
    shifts = [(int(rng.integers(-5, 6)) * 2, int(rng.integers(-5, 6)) * 2) for _ in range(nrefs)]
    refs = [ref_of(fenc, *s) for s in shifts]
    fc, rc = [], [[] for _ in range(nrefs)]
    for _ in range(2):
        c, cstride, corg = make_plane(rng, depth, W // 2, H // 2, margin // 2, smooth=smooth)
        fc.append(c)
        for r in range(nrefs):
            rc[r].append(ref_of(c, shifts[r][0] // 2, shifts[r][1] // 2))
    return dict(fenc=fenc, refs=refs, fc=fc, rc=rc, stride=stride, cstride=cstride, org=org, corg=corg, W=W, H=H, margin=margin, depth=depth)


def random_job(pl, rng, w, h, kind):
    """kind: 'amvp' (SAD, one list), 'merge_uni', 'merge_bi' (SATD + chroma, addAvg), 'bidir_pp' (SATD, pixelavg_pp)."""
    W, H = pl["W"], pl["H"]
    bx = int(rng.integers(0, (W - w) // 4 + 1)) * 4; by = int(rng.integers(0, (H - h) // 4 + 1)) * 4
    bx &= ~1; by &= ~1
    mvs = [(int(rng.integers(-120, 121)), int(rng.integers(-120, 121))) for _ in range(2)]
    if rng.integers(0, 4) == 0:
        mvs[0] = (mvs[0][0] & ~3, mvs[0][1] & ~3)               # full-pel
    if rng.integers(0, 4) == 0:
        mvs[1] = (mvs[1][0] & ~3, mvs[1][1])                    # vertical only
    if rng.integers(0, 4) == 0:
        mvs[0] = (mvs[0][0], mvs[0][1] & ~3)                    # horizontal only
    lists = {"amvp": [int(rng.integers(0, 2))], "merge_uni": [int(rng.integers(0, 2))], "merge_bi": [0, 1], "bidir_pp": [0, 1]}[kind]
    return dict(bx=bx, by=by, w=w, h=h, mvs=mvs, lists=lists, cost=0 if kind == "amvp" else 1,
                chroma=int(kind in ("merge_uni", "merge_bi")), biAvgPP=int(kind == "bidir_pp"),
                ref=[int(rng.integers(0, len(pl["refs"]))), int(rng.integers(0, len(pl["refs"])))])


def plane_ptrs(pl, jb, es):
    """Pointers (ints) of source / list-0 / list-1 planes at the PU origin; an unused list is None."""
    off = pl["org"] + jb["by"] * pl["stride"] + jb["bx"]
    coff = pl["corg"] + (jb["by"] >> 1) * pl["cstride"] + (jb["bx"] >> 1)
    fenc = [pl["fenc"].ctypes.data + off * es, pl["fc"][0].ctypes.data + coff * es, pl["fc"][1].ctypes.data + coff * es]
    out = [fenc]
    for l in (0, 1):
        if l in jb["lists"]:
            r = jb["ref"][l]
            out.append([pl["refs"][r].ctypes.data + off * es, pl["rc"][r][0].ctypes.data + coff * es, pl["rc"][r][1].ctypes.data + coff * es])
        else:
            out.append(None)
    return out


def oracle_cost(O, pl, jb):
    es = np.dtype(pixel_dtype(pl["depth"])).itemsize
    fenc, r0, r1 = plane_ptrs(pl, jb, es)
    j = OrcPredJob()
    for k in range(3):
        j.fenc[k] = fenc[k]; j.ref0[k] = r0[k] if r0 else None; j.ref1[k] = r1[k] if r1 else None
    j.stride, j.cstride, j.w, j.h = pl["stride"], pl["cstride"], jb["w"], jb["h"]
    j.mv0[0], j.mv0[1] = jb["mvs"][0]; j.mv1[0], j.mv1[1] = jb["mvs"][1]
    j.cost, j.chroma, j.biAvgPP = jb["cost"], jb["chroma"], jb["biAvgPP"]
    O.orc_pred_cost.argtypes = [C.POINTER(OrcPredJob)]; O.orc_pred_cost.restype = C.c_int
    return int(O.orc_pred_cost(C.byref(j)))


# ---------------------------------------------------------------------------------------------------------------------
# Job lists in the batched entry point's layout (x265cu_pred_job) on guarded pictures: the case families of
# tests/test_gpu_pred_paths.py and tests/test_pred_oracle_vs_ref.py.
MARGIN_X, MARGIN_Y = 96, 80          # PicYuv's luma margins for CTU 64 (picyuv.cpp:87-88); chroma: half of each
GUARD_X, GUARD_Y = 64, 8             # poison-filled band around the margins, inside the allocation
POISON = {8: 0xA5, 10: 0x2A5}


class Pics:
    """A source picture and `nrefs` reference pictures, 4:2:0, each plane with PicYuv's replicated margins (extendPicBorder)
    inside an allocation whose remaining band (GUARD_X elements left and right, GUARD_Y rows above and below, at least) holds
    POISON.  fenc / refs / fc / rc are the flat allocations; org / corg the element offsets of pixel (0, 0)."""

    def __init__(self, depth, W, H, images, stride=None, cstride=None):
        self.depth, self.W, self.H = depth, W, H
        self.stride = stride or (W + 2 * (MARGIN_X + GUARD_X) + 63) // 64 * 64
        self.cstride = cstride or (W // 2 + MARGIN_X + 2 * GUARD_X + 31) // 32 * 32
        assert self.stride >= W + 2 * (MARGIN_X + GUARD_X) and self.cstride >= W // 2 + MARGIN_X + 2 * GUARD_X
        self.fenc2d, self.org = self._pad(images["fenc"], self.stride, MARGIN_X, MARGIN_Y)
        self.refs2d = [self._pad(im, self.stride, MARGIN_X, MARGIN_Y)[0] for im in images["refs"]]
        self.fc2d, self.corg = [], 0
        for im in images["fc"]:
            buf, self.corg = self._pad(im, self.cstride, MARGIN_X // 2, MARGIN_Y // 2)
            self.fc2d.append(buf)
        self.rc2d = [[self._pad(im, self.cstride, MARGIN_X // 2, MARGIN_Y // 2)[0] for im in pair] for pair in images["rc"]]
        self.fenc, self.refs = self.fenc2d.ravel(), [r.ravel() for r in self.refs2d]
        self.fc, self.rc = [c.ravel() for c in self.fc2d], [[c.ravel() for c in pair] for pair in self.rc2d]

    def _pad(self, img, stride, mx, my):
        h, w = img.shape
        gx = (GUARD_X + mx + 15) // 16 * 16 - mx                 # poison left of the margin, so that pixel (0, 0) is 16-element aligned
        assert stride - (gx + 2 * mx + w) >= GUARD_X
        buf = np.full((h + 2 * (my + GUARD_Y), stride), POISON[self.depth], pixel_dtype(self.depth))
        y0, x0 = GUARD_Y + my, gx + mx
        buf[y0:y0 + h, x0:x0 + w] = img
        buf[y0:y0 + h, gx:x0] = img[:, :1]
        buf[y0:y0 + h, x0 + w:x0 + w + mx] = img[:, -1:]
        buf[GUARD_Y:y0, gx:x0 + w + mx] = buf[y0, gx:x0 + w + mx]
        buf[y0 + h:y0 + h + my, gx:x0 + w + mx] = buf[y0 + h - 1, gx:x0 + w + mx]
        return buf, y0 * stride + x0

    def offset(self, x, y):
        return y * self.stride + x

    def reads_inside(self, reads):
        """whether every read rectangle (pred_numpy.pred_cost) lies inside the plane's picture + margins"""
        for (p, x0, y0, x1, y1) in reads:
            s = 1 if p == "luma" else 2
            W, H, mx, my = self.W // s, self.H // s, MARGIN_X // s, MARGIN_Y // s
            if x0 < -mx or y0 < -my or x1 > W - 1 + mx or y1 > H - 1 + my:
                return False
        return True


def content_images(depth, W, H, content, rng, nrefs):
    """Source and reference images (luma W x H, chroma half size) of one content kind:
    'smooth': the source plus a small shift and +-3 of noise per reference; 'random': independent uniform pixels;
    'saturated': independent patterns of 0 / maxv blocks, stripes and single-pixel edges (the interpolation overshoots
    past both ends of the pixel range, and the bi-prediction average of 0 / maxv pairs reaches the addAvg clips)."""
    mx = (1 << depth) - 1

    def one(w, h):
        if content == "random":
            return rng.integers(0, mx + 1, (h, w))
        if content == "smooth":
            yy, xx = np.mgrid[0:h, 0:w]
            img = 128 + 60 * np.sin(xx / 17.0 + rng.uniform(0, 6)) + 40 * np.cos(yy / 11.0) + rng.integers(-6, 7, (h, w))
            return np.clip(img, 0, 255).astype(np.int64) << (depth - 8)
        img = np.zeros((h, w), np.int64)
        for _ in range(w * h // 40):                             # 0 / maxv blocks of 1 to 12 px
            bw, bh = int(rng.integers(1, 13)), int(rng.integers(1, 13))
            x, y = int(rng.integers(0, w)), int(rng.integers(0, h))
            img[y:y + bh, x:x + bw] = mx if rng.integers(0, 2) else 0
        img[:, int(rng.integers(0, w)):][::3] ^= mx              # horizontal stripes over part of the plane
        return img

    def ref_of(src):
        if content != "smooth":
            return one(src.shape[1], src.shape[0])
        sh = np.roll(src, (int(rng.integers(-5, 6)), int(rng.integers(-5, 6))), axis=(0, 1))
        return np.clip(sh + rng.integers(-3, 4, sh.shape), 0, mx)
    fenc = one(W, H)
    fc = [one(W // 2, H // 2) for _ in range(2)]
    return dict(fenc=fenc, refs=[ref_of(fenc) for _ in range(nrefs)], fc=fc, rc=[[ref_of(c) for c in fc] for _ in range(nrefs)])


def reads_in_margins(pics, jobs):
    """Per job: whether every plane it reads (luma 8-tap at quarter-pel; with a chroma SATD, both chroma planes at
    eighth-pel) stays inside the picture + PicYuv margins -- pred_numpy.read_rect, over the whole list at once"""
    y, x = np.divmod(jobs["offset"].astype(np.int64), pics.stride)
    w, h = jobs["pw"].astype(np.int64), jobs["ph"].astype(np.int64)
    ok = np.ones(len(jobs), bool)
    for l in (0, 1):
        used = jobs["ref%d" % l] >= 0
        mv = jobs["mv%d" % l].astype(np.int64)
        for (s, taps, fb) in ((1, 8, 2), (2, 4, 3)):
            cx, cy, cw, ch = x >> (s - 1), y >> (s - 1), w >> (s - 1), h >> (s - 1)
            ix, iy = cx + (mv[:, 0] >> fb), cy + (mv[:, 1] >> fb)
            xf, yf = (mv[:, 0] & ((1 << fb) - 1)) != 0, (mv[:, 1] & ((1 << fb) - 1)) != 0
            x0, x1 = ix - np.where(xf, taps // 2 - 1, 0), ix + cw - 1 + np.where(xf, taps // 2, 0)
            y0, y1 = iy - np.where(yf, taps // 2 - 1, 0), iy + ch - 1 + np.where(yf, taps // 2, 0)
            W, H, mx, my = pics.W // s, pics.H // s, MARGIN_X // s, MARGIN_Y // s
            inside = (x0 >= -mx) & (y0 >= -my) & (x1 <= W - 1 + mx) & (y1 <= H - 1 + my)
            ok &= inside | ~used
    return ok


def make_pics(depth, W, H, content, rng, nrefs=3, stride=None, cstride=None):
    return Pics(depth, W, H, content_images(depth, W, H, content, rng, nrefs), stride, cstride)


def clip_box(W, H, cux, cuy):
    """CUData::clipMv's box (cudata.cpp:1915-1928) for a CU at (cux, cuy) with CTU 64, quarter-pel: (xmin, xmax, ymin, ymax)"""
    return (-(71 + cux) * 4, (W + 7 - cux) * 4, -(71 + cuy) * 4, (H + 7 - cuy) * 4)


def pred_job(pics, x, y, w, h, ref0=-1, ref1=-1, mv0=(0, 0), mv1=(0, 0), cost=1, flags=0):
    from x265_b200.lib import PRED_JOB
    j = np.zeros(1, PRED_JOB)[0]
    j["offset"] = pics.offset(x, y); j["pw"], j["ph"] = w, h
    j["ref0"], j["ref1"], j["cost"], j["flags"] = ref0, ref1, cost, flags
    j["mv0"], j["mv1"] = mv0, mv1
    return j


def job_list(jobs):
    from x265_b200.lib import PRED_JOB
    return np.array(jobs, PRED_JOB) if len(jobs) else np.zeros(0, PRED_JOB)


def _batch_args(pics, es, chroma):
    PA = C.c_void_p * len(pics.refs)
    at = lambda a, off: a.ctypes.data + off * es
    fc = [at(c, pics.corg) for c in pics.fc] if chroma else [None, None]
    return ([at(pics.fenc, pics.org), fc[0], fc[1], PA(*[at(r, pics.org) for r in pics.refs]),
             PA(*[at(rc[0], pics.corg) for rc in pics.rc]), PA(*[at(rc[1], pics.corg) for rc in pics.rc])], pics.stride, pics.cstride)


def oracle_batch(O, pics, jobs, chroma=True):
    """orc_pred_cost_batch of the list on the host copies of `pics`; chroma=False: no chroma planes (fencCb = NULL)"""
    es = np.dtype(pixel_dtype(pics.depth)).itemsize
    planes, stride, cstride = _batch_args(pics, es, chroma)
    jobs = np.ascontiguousarray(jobs)
    out = np.zeros(len(jobs), np.int32)
    O.orc_pred_cost_batch.restype = C.c_int
    O.orc_pred_cost_batch.argtypes = [C.c_void_p] * 6 + [IP, IP, C.c_void_p, I, C.c_void_p]
    O.orc_pred_cost_batch(*planes, stride, cstride, jobs.ctypes.data, len(jobs), out.ctypes.data)
    return out


def ref_batch(R, pics, jobs, chroma=True, threads=8):
    """x265ref_pred_cost_batch (the reference's Predict / MotionEstimate classes) of the list; it always takes chroma planes,
    so chroma=False clears the jobs' chroma flag instead"""
    es = np.dtype(pixel_dtype(pics.depth)).itemsize
    planes, stride, cstride = _batch_args(pics, es, True)
    jobs = np.array(jobs)
    if not chroma:
        jobs["flags"] &= 0xFE
    out = np.zeros(len(jobs), np.int32)
    R.x265ref_pred_cost_batch.restype = C.c_int
    R.x265ref_pred_cost_batch.argtypes = [C.c_void_p] * 6 + [IP, IP, C.c_void_p, I, C.c_void_p, I]
    R.x265ref_pred_cost_batch(*planes, stride, cstride, jobs.ctypes.data, len(jobs), out.ctypes.data, threads)
    return out


# ---- case families ----------------------------------------------------------------------------------------------------
def chroma_shape(w, h):
    """a chroma SATD exists for the PU (chroma block a multiple of 4x4: motion.cpp:204-212)"""
    return (w // 2) % 4 == 0 and (h // 2) % 4 == 0


# (name, lists, cost, flags): the kinds of job every PU shape is swept with.  SAD jobs have one list (Search::selectMVP;
# the API has no two-list SAD)
SWEEP_KINDS = [("l0_sad", "0", 0, 0), ("l1_sad", "1", 0, 0), ("l0_satd_chroma", "0", 1, 1), ("l1_satd", "1", 1, 0),
               ("l1_satd_chroma", "1", 1, 1), ("bi_addavg_chroma", "01", 1, 1), ("bi_addavg_satd", "01", 1, 0),
               ("bi_avgpp", "01", 1, 2), ("bi_avgpp_chroma_flag", "01", 1, 3), ("bi_same_ref", "=", 1, 1)]


def _phase_vectors(n, eighth):
    """n (>= 16 / 64) quarter-pel vectors whose phases run through every luma pair (eighth=False) or every eighth-pel chroma
    pair (eighth=True) of each list: list 1 takes the pairs in another order than list 0"""
    m = 64 if eighth else 16
    out = []
    for i in range(n):
        a, b = i % m, (i * 5 + 3) % m
        if eighth:
            out.append(((a & 7, a >> 3), (b & 7, b >> 3)))
        else:
            out.append(((a & 3, a >> 2), (b & 3, b >> 2)))
    return out


def phase_sweep(pics, rng, shapes=LUMA_PUS, kinds=SWEEP_KINDS):
    """Every PU shape x kind, with every luma phase pair of each list (16 jobs) or, for shapes with a chroma SATD, every
    eighth-pel pair (64 jobs); integer parts random within +-24 px, PUs anywhere in the picture on a 4-pel grid.
    Returns (jobs, kind name per job)."""
    jobs, kinds_of = [], []
    nref = len(pics.refs)
    for (w, h) in shapes:
        eighth = chroma_shape(w, h)
        for (name, lists, cost, flags) in kinds:
            for (p0, p1) in _phase_vectors(64 if eighth else 16, eighth):
                x = int(rng.integers(0, (pics.W - w) // 4 + 1)) * 4; y = int(rng.integers(0, (pics.H - h) // 4 + 1)) * 4
                vec = lambda p: tuple(int(rng.integers(-24, 25)) * (8 if eighth else 4) + p[c] for c in range(2))
                mv0, mv1 = vec(p0), vec(p1)
                r0, r1 = int(rng.integers(0, nref)), int(rng.integers(0, nref))
                if lists == "0":
                    j = pred_job(pics, x, y, w, h, ref0=r0, mv0=mv0, cost=cost, flags=flags)
                elif lists == "1":
                    j = pred_job(pics, x, y, w, h, ref1=r1, mv1=mv1, cost=cost, flags=flags)
                elif lists == "=":
                    j = pred_job(pics, x, y, w, h, ref0=r0, ref1=r0, mv0=mv0, mv1=mv0, cost=cost, flags=flags)
                else:
                    j = pred_job(pics, x, y, w, h, ref0=r0, ref1=r1, mv0=mv0, mv1=mv1, cost=cost, flags=flags)
                jobs.append(j); kinds_of.append(name)
    return job_list(jobs), kinds_of


def cu_parts(s):
    """(x, y, w, h) of the PUs of every inter partition of a CU of size s: 2Nx2N, 2NxN, Nx2N and, from CU 16, the four AMP
    shapes"""
    q, hs = s // 4, s // 2
    parts = [[(0, 0, s, s)], [(0, 0, s, hs), (0, hs, s, hs)], [(0, 0, hs, s), (hs, 0, hs, s)]]
    if s >= 16:
        parts += [[(0, 0, s, q), (0, q, s, s - q)], [(0, 0, s, s - q), (0, s - q, s, q)],
                  [(0, 0, q, s), (q, 0, s - q, s)], [(0, 0, s - q, s), (s - q, 0, q, s)]]
    return [pu for p in parts for pu in p]


def clip_limit_jobs(pics, rng):
    """PUs of CUs 64 / 32 / 16 / 8 (AMP parts included) at the four picture corners and the four edge midpoints, with
    vectors at and just inside CUData::clipMv's box: each component at the box's low end with every fraction (the
    full-pel value is the lowest allowed) and at its high end (fraction 0) and the full-pel position below it with every
    fraction.  Kinds rotate over one-list SAD, one-list SATD + chroma, two-list addAvg + chroma and two-list pixelavg_pp;
    the second list takes another vector of the box.  Returns (jobs, [(CU size, corner) per job])."""
    W, H = pics.W, pics.H
    nref = len(pics.refs)
    jobs, where = [], []
    k = 0
    for s in (64, 32, 16, 8):
        for (cx, cy) in ((0, 0), (W - s, 0), (0, H - s), (W - s, H - s),
                         ((W - s) // 2 // s * s, 0), ((W - s) // 2 // s * s, H - s), (0, (H - s) // 2 // s * s), (W - s, (H - s) // 2 // s * s)):
            xmin, xmax, ymin, ymax = clip_box(W, H, cx, cy)
            xs = [xmin, xmin + 1, xmin + 2, xmin + 3, xmax - 3, xmax - 2, xmax - 1, xmax]
            ys = [ymin, ymin + 1, ymin + 2, ymin + 3, ymax - 3, ymax - 2, ymax - 1, ymax]
            for (px, py, w, h) in cu_parts(s):
                for vx in xs:
                    for vy in ys:
                        kind = k % 4
                        k += 1
                        mv1 = (xs[int(rng.integers(0, 8))], ys[int(rng.integers(0, 8))])
                        r0, r1 = int(rng.integers(0, nref)), int(rng.integers(0, nref))
                        if kind == 0:
                            j = pred_job(pics, cx + px, cy + py, w, h, ref0=r0, mv0=(vx, vy), cost=0)
                        elif kind == 1:
                            j = pred_job(pics, cx + px, cy + py, w, h, ref1=r1, mv1=(vx, vy), cost=1, flags=1)
                        else:
                            j = pred_job(pics, cx + px, cy + py, w, h, ref0=r0, ref1=r1, mv0=(vx, vy), mv1=mv1, cost=1, flags=1 if kind == 2 else 2)
                        jobs.append(j); where.append((s, cx, cy))
    return job_list(jobs), where


def random_jobs(pics, rng, n, shapes=LUMA_PUS, xs=None, span=32):
    """n jobs of random shape, kind (SWEEP_KINDS), phases and integer parts within +-span px; x positions from `xs` if given"""
    jobs = []
    nref = len(pics.refs)
    for i in range(n):
        w, h = shapes[i % len(shapes)]
        name, lists, cost, flags = SWEEP_KINDS[int(rng.integers(0, len(SWEEP_KINDS)))]
        if xs is None:
            x = int(rng.integers(0, (pics.W - w) // 4 + 1)) * 4
        else:
            r = int(xs[i % len(xs)])
            x = int(rng.integers(0, (pics.W - w - r) // 16 + 1)) * 16 + r
        y = int(rng.integers(0, (pics.H - h) // 4 + 1)) * 4
        mv = lambda: tuple(int(rng.integers(-4 * span, 4 * span + 1)) for _ in range(2))
        mv0, mv1 = mv(), mv()
        r0, r1 = int(rng.integers(0, nref)), int(rng.integers(0, nref))
        if lists == "=":
            r1, mv1 = r0, mv0
        jobs.append(pred_job(pics, x, y, w, h, ref0=r0 if "0" in lists or "=" in lists else -1,
                             ref1=r1 if "1" in lists or "=" in lists else -1, mv0=mv0, mv1=mv1, cost=cost, flags=flags))
    return job_list(jobs)


# luma row pitch (elements) whose byte size is a multiple of 16, of 8 only, and of 4 only; the chroma pitch follows suit
STRIDES = {8: {"stride16": (448, 288), "stride8": (456, 296), "stride4": (452, 292)},
           10: {"stride16": (448, 288), "stride8": (452, 292), "stride4": (450, 290)}}
FAMILIES = ("sweep_smooth", "sweep_random", "clip", "saturated", "stride16", "stride8", "stride4")


def family(name, depth):
    """(pics, jobs, info) of one case family, the same on every call:
      sweep_*:   phase_sweep on a 256x192 picture (info: the kind of each job);
      clip:      clip_limit_jobs on a 192x128 picture (info: (CU size, cu x, cu y) of each job);
      saturated: 640 random jobs on 0 / maxv content (content_images);
      stride*:   480 random jobs on a 128x96 picture with the luma / chroma pitches of STRIDES, PU x positions of every
                 multiple-of-4 residue mod 16."""
    import zlib
    rng = np.random.default_rng(zlib.crc32(name.encode()) + depth)
    if name.startswith("sweep_"):
        pics = make_pics(depth, 256, 192, name[6:], rng)
        jobs, info = phase_sweep(pics, rng)
    elif name == "clip":
        pics = make_pics(depth, 192, 128, "random", rng)
        jobs, info = clip_limit_jobs(pics, rng)
    elif name == "saturated":
        pics = make_pics(depth, 192, 128, "saturated", rng)
        jobs, info = random_jobs(pics, rng, 640, span=16), None
    else:
        stride, cstride = STRIDES[depth][name]
        pics = make_pics(depth, 128, 96, "random", rng, stride=stride, cstride=cstride)
        jobs, info = random_jobs(pics, rng, 480, xs=(0, 4, 8, 12), span=16), None
    return pics, jobs, info


def frame_jobs(depth, chroma, field="against", merange=57, W=512, H=320):
    """(Pics, jobs): bench.pred_jobs_of over the motion-search jobs and results of the oracle's CPU frame driver on a W x H
    frame with rect + AMP partitions and 2 references (the planes are the workload's, repadded with guard bands)"""
    import os
    import sys
    from common import load_oracle
    from frame_helpers import Workload, cpu_analyse, lambda_for, MARGIN_X as MX, MARGIN_Y as MY
    from me_helpers import mvcost_table
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import bench
    O = load_oracle(depth)
    wl = Workload(W, H, depth=depth, numRefs=2, rect=1, amp=1, chroma=True, field=field, merange=merange)
    res = cpu_analyse(O, "orc_analyse_frame", wl, mvcost_table(O, lambda_for(wl.params["qp"], depth)), threads=8, stages=1)
    pj = bench.pred_jobs_of(res["jobs"], res["me_out"], 2, chroma)
    inner = lambda b, mx, my, s: np.ascontiguousarray(b[my:my + H // s, mx:mx + W // s])
    pics = Pics(depth, W, H, dict(fenc=inner(wl.fenc, MX, MY, 1), refs=[inner(r, MX, MY, 1) for r in wl.refs],
                                  fc=[inner(c, MX // 2, MY // 2, 2) for c in wl.fencC],
                                  rc=[[inner(c, MX // 2, MY // 2, 2) for c in rc] for rc in wl.refC]))
    # the workload's offsets are in its own stride: move them to the guarded pictures'
    y, x = np.divmod(pj["offset"].astype(np.int64), wl.stride)
    pj["offset"] = (y * pics.stride + x).astype(np.int32)
    return pics, pj


def ref_cost(R, pl, jb):
    es = np.dtype(pixel_dtype(pl["depth"])).itemsize
    fenc, r0, r1 = plane_ptrs(pl, jb, es)
    arr = lambda v: (P * 3)(*v) if v else None
    mv0 = (I * 2)(*jb["mvs"][0]); mv1 = (I * 2)(*jb["mvs"][1])
    R.x265ref_pred_cost.restype = C.c_int
    R.x265ref_pred_cost.argtypes = [C.POINTER(P), C.POINTER(P), C.POINTER(P), IP, IP, I, I, C.POINTER(I), C.POINTER(I), I, I, I]
    return int(R.x265ref_pred_cost(arr(fenc), arr(r0), arr(r1), pl["stride"], pl["cstride"], jb["w"], jb["h"], mv0, mv1,
                                   jb["cost"], jb["chroma"], jb["biAvgPP"]))
