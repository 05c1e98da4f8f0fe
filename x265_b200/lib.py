"""ctypes binding of libx265cu.so (include/x265_b200.h).  Host-side plumbing only: the arithmetic is
all in the CUDA library.  Raises CudaUnavailable instead of falling back when no GPU is present."""
import ctypes as C
import os

import numpy as np

from . import build as _build

P = C.c_void_p
I = C.c_int
I64 = C.c_int64
IP = C.c_ssize_t


class CudaUnavailable(RuntimeError):
    pass


class MeChroma(C.Structure):
    """x265cu_me_chroma (include/x265_b200.h)"""
    _fields_ = [("fencCb_dev", C.c_void_p), ("fencCr_dev", C.c_void_p), ("refCb_dev", C.c_void_p), ("refCr_dev", C.c_void_p),
                ("cstride", C.c_int)]


# job record layouts (must match include/x265_b200.h)
CMP_JOB = np.dtype([("a_off", "<i8"), ("b_off", "<i8"), ("a_stride", "<i4"), ("b_stride", "<i4"),
                    ("w", "<i2"), ("h", "<i2"), ("pad", "<i4")], align=True)
BLK_JOB = np.dtype([("d_off", "<i8"), ("a_off", "<i8"), ("b_off", "<i8"), ("d_stride", "<i4"), ("a_stride", "<i4"),
                    ("b_stride", "<i4"), ("w", "<i2"), ("h", "<i2"), ("p0", "<i4"), ("p1", "<i4"), ("p2", "<i4"), ("p3", "<i4")], align=True)
INTERP_JOB = np.dtype([("s_off", "<i8"), ("d_off", "<i8"), ("s_stride", "<i4"), ("d_stride", "<i4"), ("w", "<i2"), ("h", "<i2"),
                       ("idxX", "i1"), ("idxY", "i1"), ("rowExt", "i1"), ("ntaps", "i1")], align=True)
INTRA_JOB = np.dtype([("mode", "<i4"), ("bFilter", "<i4")], align=True)
PRED_JOB = np.dtype([("offset", "<i4"), ("pw", "<i2"), ("ph", "<i2"), ("ref0", "i1"), ("ref1", "i1"), ("cost", "u1"), ("flags", "u1"),
                     ("mv0", "<i2", 2), ("mv1", "<i2", 2)])
PRED_SAD, PRED_SATD, PRED_CHROMA, PRED_AVG_PP = 0, 1, 1, 2
ME_JOB = np.dtype([("offset", "<i4"), ("ref", "<i2"), ("pw", "i1"), ("ph", "i1"), ("mvmin", "<i2", 2), ("mvmax", "<i2", 2),
                   ("qmvp", "<i2", 2), ("mvc", "<i2", 8), ("numCand", "i1"), ("method", "i1"), ("subme", "i1"), ("merange", "i1")], align=True)
assert CMP_JOB.itemsize == 32 and BLK_JOB.itemsize == 56 and INTERP_JOB.itemsize == 32 and ME_JOB.itemsize == 40
# x265cu_deblock_unit: one record per 4x4 luma unit, raster order; flags bit 0 intra, bit 1 luma cbf, bit 2 tq-bypass
DEBLOCK_UNIT = np.dtype([("qp", "i1"), ("flags", "u1"), ("log2CuSize", "u1"), ("partSize", "u1"), ("tuDepth", "u1"),
                         ("refPic", "i1", 2), ("mv", "<i2", (2, 2))], align=True)
assert DEBLOCK_UNIT.itemsize == 16
B_SLICE, P_SLICE, I_SLICE = 0, 1, 2
# x265cu_sao_ctu: SaoCtuParam as the SAO decision leaves it; arrays [3][numCtus], CTU raster order
SAO_CTU = np.dtype([("typeIdx", "i1"), ("bandPos", "u1"), ("offset", "i1", 4), ("pad", "u1", 2)])
assert SAO_CTU.itemsize == 8
SAO_STATS_PER_CTU = 2 * 3 * 5 * 32      # int32: [count, offsetOrg][plane][SaoType][class], two SAO::PerPlane


class DeblockParams(C.Structure):
    """x265cu_deblock_params (include/x265_b200.h)"""
    _fields_ = [("sliceType", C.c_int32), ("betaOffsetDiv2", C.c_int32), ("tcOffsetDiv2", C.c_int32), ("cbQpOffset", C.c_int32),
                ("crQpOffset", C.c_int32), ("transquantBypass", C.c_int32)]

OPS_CMP = dict(sad=0, satd=1, sa8d=2, sse_pp=3, sse_ss=4, ssd_s=5, var=6, psy=7)
OPS_BLK = dict(copy_pp=0, copy_ss=1, copy_sp=2, copy_ps=3, sub_ps=4, add_ps=5, pixelavg_pp=6, addAvg=7, p2s=8, transpose=9,
               blockfill_s=10, cpy2Dto1D_shl=11, cpy2Dto1D_shr=12, cpy1Dto2D_shl=13, cpy1Dto2D_shr=14, weight_pp=15,
               weight_sp=16, scale2D_64to32=17, dequant_normal=18)
OPS_INTERP = dict(hpp=0, hps=1, vpp=2, vps=3, vsp=4, vss=5, hvpp=6)
OPS_TR = dict(dct=0, idct=1, dst4=2, idst4=3)

_PROTOS = {
    "x265cu_device_count": (I, []),
    "x265cu_create": (P, [I]),
    "x265cu_destroy": (None, [P]),
    "x265cu_last_error": (C.c_char_p, []),
    "x265cu_sync": (I, [P]),
    "x265cu_stream": (P, [P]),
    "x265cu_malloc": (P, [P, C.c_size_t]),
    "x265cu_free": (None, [P, P]),
    "x265cu_host_alloc": (P, [C.c_size_t]),
    "x265cu_host_free": (None, [P]),
    "x265cu_h2d": (I, [P, P, P, C.c_size_t]),
    "x265cu_d2h": (I, [P, P, P, C.c_size_t]),
    "x265cu_memset": (I, [P, P, I, C.c_size_t]),
    "x265cu_copy2d": (I, [P, P, C.c_size_t, P, C.c_size_t, C.c_size_t, C.c_size_t, I]),
    "x265cu_timer_begin": (I, [P]),
    "x265cu_timer_end": (C.c_float, [P]),
    "x265cu_launch_count": (C.c_uint64, [P]),
    "x265cu_me_phase_ms": (I, [P, C.POINTER(C.c_float)]),
    "x265cu_get_primitive": (P, [I, C.c_char_p, I, I, I]),
    "x265cu_primitive_error": (I, []),
    "x265cu_primitive_error_string": (C.c_char_p, []),
    "x265cu_primitive_error_clear": (None, []),
    "x265cu_primitive_calls": (C.c_uint64, []),
    "x265cu_pixelcmp_batch": (I, [P, I, I, P, P, P, I, P]),
    "x265cu_pixelcmp_grid": (I, [P, I, I, P, I64, P, I64, I, I, I, I, P]),
    "x265cu_blockop_batch": (I, [P, I, I, P, P, P, P, I]),
    "x265cu_interp_batch": (I, [P, I, I, P, P, P, I]),
    "x265cu_transform_batch": (I, [P, I, I, I, P, P, I, I64, I]),
    "x265cu_quant_batch": (I, [P, P, P, P, P, I, I, I, I, I, P]),
    "x265cu_dequant_normal_batch": (I, [P, P, P, I64, I, I]),
    "x265cu_dequant_scaling_batch": (I, [P, P, P, P, I, I, I, I]),
    "x265cu_intra_pred_batch": (I, [P, I, I, P, I64, P, I64, I, P, I]),
    "x265cu_intra_filter_batch": (I, [P, I, I, P, P, I64, I]),
    "x265cu_intra_allangs_batch": (I, [P, I, I, P, P, I64, P, I, I]),
    "x265cu_frame_init_lowres": (I, [P, I, P, I, P, P, P, P, I, I, I, I, I]),
    "x265cu_extend_border": (I, [P, I, P, I, I, I, I, I]),
    "x265cu_mvcost_table": (None, [C.c_double, I, P]),
    "x265cu_me_batch": (I, [P, I, P, I, P, I, I, P, I, P, I, P]),
    "x265cu_me_batch_chroma": (I, [P, I, P, I, P, I, P, P, I, P, I, P]),
    "x265cu_pred_cost_batch": (I, [P, I, P, I, P, I, P, P, I, P]),
    "x265cu_deblock_frame": (I, [P, I, P, I, P, P, I, I, I, P, P]),
    "x265cu_sao_stats_frame": (I, [P, I, I, I, I, P, P, P, I, I, P, P, P, I, I, P]),
    "x265cu_sao_apply_frame": (I, [P, I, I, I, I, P, P, P, I, I, P, I, I, P, P, P, P, I, I]),
    "x265cu_deblock_rows": (I, [P, I, I, I, I, I, I, P, P, P, I, I, P, P, P, I, I, P, P]),
    "x265cu_sao_stats_rows": (I, [P, I, I, I, I, I, I, P, P, P, I, I, P, P, P, I, I, P]),
    "x265cu_sao_apply_rows": (I, [P, I, I, I, I, I, I, P, P, P, I, I, P, P, P, I, I, P, I, I, P, P, P, P, I, I]),
}


class DeviceBuffer:
    """A device allocation owned by the Lib context."""

    def __init__(self, lib, nbytes):
        self.lib = lib
        self.nbytes = int(nbytes)
        self.ptr = lib.L.x265cu_malloc(lib.ctx, max(self.nbytes, 16))
        if not self.ptr:
            raise MemoryError("x265cu_malloc(%d) failed: %s" % (nbytes, lib.last_error()))

    def upload(self, arr, offset=0):
        arr = np.ascontiguousarray(arr)
        assert offset + arr.nbytes <= self.nbytes
        self.lib.check(self.lib.L.x265cu_h2d(self.lib.ctx, self.ptr + offset, arr.ctypes.data, arr.nbytes))
        self.lib.sync()          # pageable source: make the copy complete before numpy may free it
        return self

    def download(self, dtype, count=None, offset=0):
        dt = np.dtype(dtype)
        if count is None:
            count = (self.nbytes - offset) // dt.itemsize
        out = np.empty(count, dt)
        self.lib.check(self.lib.L.x265cu_d2h(self.lib.ctx, out.ctypes.data, self.ptr + offset, out.nbytes))
        self.lib.sync()
        return out

    def free(self):
        if self.ptr:
            self.lib.L.x265cu_free(self.lib.ctx, self.ptr)
            self.ptr = None


class Lib:
    def __init__(self, device=0, need_gpu=True):
        path = _build.build()
        self.path = path
        self.L = C.CDLL(path)
        for name, (res, args) in _PROTOS.items():
            f = getattr(self.L, name)       # AttributeError if the ABI lost a symbol
            f.restype = res
            f.argtypes = args
        self.ctx = None
        if need_gpu:
            if self.L.x265cu_device_count() <= 0:
                raise CudaUnavailable("libx265cu.so loaded but no CUDA device is visible; there is no CPU fallback")
            self.ctx = self.L.x265cu_create(device)
            if not self.ctx:
                raise CudaUnavailable("x265cu_create(%d) failed: %s" % (device, self.last_error()))

    # ---- plumbing ----
    def last_error(self):
        e = self.L.x265cu_last_error()
        return e.decode() if e else ""

    def check(self, rc):
        if rc != 0:
            raise RuntimeError("x265cu call failed: " + self.last_error())

    def sync(self):
        self.check(self.L.x265cu_sync(self.ctx))

    def alloc(self, nbytes):
        return DeviceBuffer(self, nbytes)

    def to_device(self, arr):
        arr = np.ascontiguousarray(arr)
        return DeviceBuffer(self, arr.nbytes).upload(arr)

    def timer_begin(self):
        self.check(self.L.x265cu_timer_begin(self.ctx))

    def timer_end(self):
        ms = self.L.x265cu_timer_end(self.ctx)
        if ms < 0:
            raise RuntimeError("timer failed: " + self.last_error())
        return ms

    def me_phase_ms(self):
        ms = (C.c_float * 3)()
        self.check(self.L.x265cu_me_phase_ms(self.ctx, ms))
        return [float(x) for x in ms]

    def launch_count(self):
        return int(self.L.x265cu_launch_count(self.ctx))

    def close(self):
        if self.ctx:
            self.L.x265cu_destroy(self.ctx)
            self.ctx = None

    # ---- per-call table ----
    def primitive(self, depth, name, restype, argtypes, i=0, j=0, k=0):
        p = self.L.x265cu_get_primitive(depth, name.encode(), i, j, k)
        if not p:
            return None
        return C.CFUNCTYPE(restype, *argtypes)(p)

    # ---- batched API (device buffers in, device buffers out) ----
    def pixelcmp_batch(self, depth, op, A, B, jobs_dev, n, out_dev):
        self.check(self.L.x265cu_pixelcmp_batch(self.ctx, depth, OPS_CMP[op], A.ptr, B.ptr, jobs_dev.ptr, n, out_dev.ptr))

    def pixelcmp_grid(self, depth, op, a_ptr, a_stride, b_ptr, b_stride, bw, bh, nbx, nby, out_dev):
        """a_ptr / b_ptr: device addresses of block (0,0) in each plane (ints); strides in pixels."""
        self.check(self.L.x265cu_pixelcmp_grid(self.ctx, depth, OPS_CMP[op], a_ptr, a_stride, b_ptr, b_stride, bw, bh, nbx, nby, out_dev.ptr))

    def blockop_batch(self, depth, op, D, A, B, jobs_dev, n):
        self.check(self.L.x265cu_blockop_batch(self.ctx, depth, OPS_BLK[op], D.ptr, A.ptr if A else None, B.ptr if B else None, jobs_dev.ptr, n))

    def interp_batch(self, depth, op, S, D, jobs_dev, n):
        self.check(self.L.x265cu_interp_batch(self.ctx, depth, OPS_INTERP[op], S.ptr, D.ptr, jobs_dev.ptr, n))

    def transform_batch(self, depth, op, size, S, D, stride, tu_pitch, n):
        self.check(self.L.x265cu_transform_batch(self.ctx, depth, OPS_TR[op], size, S.ptr, D.ptr, stride, tu_pitch, n))

    def me_batch(self, depth, fenc, fstride, refs_ptr_table, rstride, lowres, mvcost_dev, mvcost_range, jobs_dev, n, out_dev):
        centre = mvcost_dev.ptr + 2 * mvcost_range
        self.check(self.L.x265cu_me_batch(self.ctx, depth, fenc.ptr, fstride, refs_ptr_table.ptr, rstride, lowres, centre,
                                          mvcost_range, jobs_dev.ptr, n, out_dev.ptr))

    def me_batch_chroma(self, depth, fenc, fstride, refs_ptr_table, rstride, fenc_cb, fenc_cr, ref_cb_table, ref_cr_table, cstride,
                        mvcost_dev, mvcost_range, jobs_dev, n, out_dev):
        """x265cu_me_batch with the chroma-SATD term of subpelCompare (4:2:0 planes at half resolution)."""
        ch = MeChroma(fenc_cb.ptr, fenc_cr.ptr, ref_cb_table.ptr, ref_cr_table.ptr, cstride)
        self.check(self.L.x265cu_me_batch_chroma(self.ctx, depth, fenc.ptr, fstride, refs_ptr_table.ptr, rstride, C.byref(ch),
                                                 mvcost_dev.ptr + 2 * mvcost_range, mvcost_range, jobs_dev.ptr, n, out_dev.ptr))

    def pred_cost_batch(self, depth, fenc, fstride, refs_ptr_table, rstride, chroma, jobs_dev, n, out_dev):
        """x265cu_pred_cost_batch: AMVP candidate SADs, merge candidate / bidir SATDs (search.cpp:1901-2023, 2474-2607).
        chroma: None or (fenc_cb, fenc_cr, ref_cb_table, ref_cr_table, cstride) device buffers."""
        ch = MeChroma(chroma[0].ptr, chroma[1].ptr, chroma[2].ptr, chroma[3].ptr, chroma[4]) if chroma else None
        self.check(self.L.x265cu_pred_cost_batch(self.ctx, depth, fenc.ptr, fstride, refs_ptr_table.ptr, rstride,
                                                 C.byref(ch) if ch else None, jobs_dev.ptr, n, out_dev.ptr))

    def lookahead_weights_analyse(self, depth, fenc_buf, ref_bufs, wbuf, planesize, stride, width, lines, padoffset, intra_cost, stats):
        """x265cu_lookahead_weights_analyse: returns (isWeighted, scale, log2denom, offset); wbuf then holds the 4 weighted planes."""
        refs = (C.c_void_p * 4)(*[b.ptr for b in ref_bufs])
        intra = np.ascontiguousarray(intra_cost, np.int32)
        st = np.ascontiguousarray(stats, np.uint64)
        wp = np.zeros(4, np.int32)
        self.check(self.L.x265cu_lookahead_weights_analyse(self.ctx, depth, fenc_buf.ptr, refs, wbuf.ptr, planesize, stride, width, lines,
                                                           padoffset, intra.ctypes.data, st.ctypes.data, wp.ctypes.data))
        return tuple(int(x) for x in wp)

    def deblock_frame(self, depth, luma, stride, cb, cr, cstride, width, height, units, params):
        """x265cu_deblock_frame: deblocks a picture in place on the context's stream.  luma / cb / cr: device addresses (ints)
        of pixel (0,0), cb = cr = None for luma only; units: device buffer (or address) of (width / 4) x (height / 4)
        DEBLOCK_UNIT records; params: DeblockParams."""
        uptr = units.ptr if isinstance(units, DeviceBuffer) else units
        self.check(self.L.x265cu_deblock_frame(self.ctx, depth, luma, stride, cb, cr, cstride, width, height, uptr, C.byref(params)))

    def sao_stats_frame(self, depth, width, height, ctu, fenc, fstride, fcstride, rec, stride, cstride, stats):
        """x265cu_sao_stats_frame: fenc / rec: (y, cb, cr) device addresses of pixel (0,0), cb = cr = None for luma only;
        stats: device buffer (or address) of numCtus * SAO_STATS_PER_CTU int32."""
        sptr = stats.ptr if isinstance(stats, DeviceBuffer) else stats
        self.check(self.L.x265cu_sao_stats_frame(self.ctx, depth, width, height, ctu, fenc[0], fenc[1], fenc[2], fstride, fcstride,
                                                 rec[0], rec[1], rec[2], stride, cstride, sptr))

    def sao_apply_frame(self, depth, width, height, ctu, planes, stride, cstride, params, sao_luma, sao_chroma,
                        bypass_units=None, fenc=(None, None, None), fstride=0, fcstride=0):
        """x265cu_sao_apply_frame: applies the per-CTU SAO records (device buffer of [3][numCtus] SAO_CTU) to the planes (y,
        cb, cr device addresses) in place; bypass_units: None or the DEBLOCK_UNIT map whose tq-bypass units get the
        source samples (fenc) back."""
        def addr(b):
            return b.ptr if isinstance(b, DeviceBuffer) else b
        self.check(self.L.x265cu_sao_apply_frame(self.ctx, depth, width, height, ctu, planes[0], planes[1], planes[2], stride, cstride,
                                                 addr(params), sao_luma, sao_chroma, addr(bypass_units), fenc[0], fenc[1], fenc[2],
                                                 fstride, fcstride))

    # ---- the same filters over a band of CTU rows [r0, r1) (include/x265_b200.h, "the in-loop filters over a band") ----
    def deblock_rows(self, depth, width, height, ctu, r0, r1, src, sstride, scstride, dst, stride, cstride, units, params):
        """x265cu_deblock_rows: src / dst: (y, cb, cr) device addresses of pixel (0,0), cb = cr = None for luma only; writes dst
        luma rows [Y0 - 4, Y1 + 4) and chroma rows [C0 - 4, C1 + 4) with the whole-picture deblocked values."""
        uptr = units.ptr if isinstance(units, DeviceBuffer) else units
        self.check(self.L.x265cu_deblock_rows(self.ctx, depth, width, height, ctu, r0, r1, src[0], src[1], src[2], sstride, scstride,
                                              dst[0], dst[1], dst[2], stride, cstride, uptr, C.byref(params)))

    def sao_stats_rows(self, depth, width, height, ctu, r0, r1, fenc, fstride, fcstride, rec, stride, cstride, stats):
        """x265cu_sao_stats_rows: the records of the CTUs in rows [r0, r1) of the full-picture stats array."""
        sptr = stats.ptr if isinstance(stats, DeviceBuffer) else stats
        self.check(self.L.x265cu_sao_stats_rows(self.ctx, depth, width, height, ctu, r0, r1, fenc[0], fenc[1], fenc[2], fstride,
                                                fcstride, rec[0], rec[1], rec[2], stride, cstride, sptr))

    def sao_apply_rows(self, depth, width, height, ctu, r0, r1, src, sstride, scstride, dst, stride, cstride, params, sao_luma,
                       sao_chroma, bypass_units=None, fenc=(None, None, None), fstride=0, fcstride=0):
        """x265cu_sao_apply_rows: out of place, writes every sample of dst rows [Y0, Y1) / [C0, C1) from the deblocked src."""
        def addr(b):
            return b.ptr if isinstance(b, DeviceBuffer) else b
        self.check(self.L.x265cu_sao_apply_rows(self.ctx, depth, width, height, ctu, r0, r1, src[0], src[1], src[2], sstride, scstride,
                                                dst[0], dst[1], dst[2], stride, cstride, addr(params), sao_luma, sao_chroma,
                                                addr(bypass_units), fenc[0], fenc[1], fenc[2], fstride, fcstride))

    def mvcost_table(self, lam, rng):
        t = np.zeros(2 * rng + 1, np.uint16)
        self.L.x265cu_mvcost_table(C.c_double(lam), rng, t.ctypes.data)
        return t


_cached = {}


def load(device=0, need_gpu=True):
    key = (device, need_gpu)
    if key not in _cached:
        _cached[key] = Lib(device, need_gpu)
    return _cached[key]


LA_INTRA_JOB = np.dtype([("plane0", "<u8"), ("invQscale", "<u8"), ("intraCost", "<u8"), ("intraMode", "<u8"), ("lowresCosts", "<u8"),
                         ("rowSatds", "<u8"), ("out", "<u8")], align=True)
LA_JOB = np.dtype([("fenc", "<u8", 4), ("ref0", "<u8", 4), ("ref1", "<u8", 4), ("mvs", "<u8", 2), ("mvcosts", "<u8", 2), ("intraCost", "<u8"),
                   ("invQscale", "<u8"), ("lowresCosts", "<u8"), ("rowSatds", "<u8"), ("out", "<u8"), ("bidir", "<i4"), ("doSearch0", "<i4"),
                   ("doSearch1", "<i4"), ("rows", "<i4")], align=True)
assert LA_INTRA_JOB.itemsize == 56 and LA_JOB.itemsize == 184


# ---------------- cuTree's propagation chain (x265cu_cutree) ----------------
CUTREE_DIST = 18                          # X265CU_CUTREE_DIST = X265_BFRAME_MAX + 2
TYPE_I, TYPE_P, TYPE_B = 2, 3, 5          # X265_TYPE_* (x265.h)


class CutreeFrame(C.Structure):
    """x265cu_cutree_frame: device pointers of one frame's cuTree inputs (include/x265_b200.h)."""
    _fields_ = [("intraCost", P), ("invQscale", P), ("propagateCost", P), ("lowresCosts", P * CUTREE_DIST * CUTREE_DIST),
                ("mvs", P * CUTREE_DIST * 2), ("sliceType", C.c_int32), ("reserved", C.c_int32)]


class CutreeParams(C.Structure):
    _fields_ = [("bIntra", C.c_int32), ("lookaheadDepth", C.c_int32), ("bBPyramid", C.c_int32), ("bEnableWeightedBiPred", C.c_int32),
                ("vbv", C.c_int32), ("fpsNum", C.c_int32), ("fpsDenom", C.c_int32)]


# ---------------- frame-level analyser (x265cu_analyser_*) ----------------
class AnalysisParams(C.Structure):
    _fields_ = [("width", I), ("height", I), ("depth", I), ("numRefs", I), ("method", I), ("subme", I), ("merange", I),
                ("rect", I), ("qp", I), ("lam", C.c_double), ("amp", I)]


class AnalysisOut(C.Structure):
    _fields_ = [("me_packed", P), ("cu_sse", P), ("cu_numsig", P), ("cu_ref", P), ("intra_cost", P)]


_AN_PROTOS = {
    "x265cu_analyser_create": (P, [P, C.POINTER(AnalysisParams)]),
    "x265cu_analyser_destroy": (None, [P]),
    "x265cu_analyser_counts": (I, [P, C.POINTER(I), C.POINTER(I), C.POINTER(I), C.POINTER(I64), C.POINTER(I)]),
    "x265cu_analyser_set_ref": (I, [P, I, P, I]),
    "x265cu_analyser_load_inputs": (I, [P, P, I, P]),
    "x265cu_analyser_run_resident": (I, [P, I]),
    "x265cu_analyser_analyse": (I, [P, P, I, P, I, C.POINTER(AnalysisOut)]),
    "x265cu_analyser_fetch": (I, [P, I, P]),
    "x265cu_analyser_stage_ms": (I, [P, C.POINTER(C.c_float)]),
    "x265cu_analyser_ref_plane": (P, [P, I, C.POINTER(I)]),
    "x265cu_analyser_ref_updated": (I, [P, I]),
    "x265cu_analyser_ctu_rows": (I, [P]),
    "x265cu_analyser_row_range": (I, [P, I, I, C.POINTER(I), C.POINTER(I), C.POINTER(I), C.POINTER(I)]),
    "x265cu_analyser_run_rows": (I, [P, I, I, I]),
    "x265cu_analyser_analyse_rows": (I, [P, P, I, P, I, I, I, C.POINTER(AnalysisOut)]),
    "x265cu_analyser_recon_plane": (P, [P, I, C.POINTER(I)]),
    "x265cu_analyser_recon_to_ref": (I, [P, I, I, I, I]),
    "x265cu_analyser_enable_chroma": (I, [P]),
    "x265cu_analyser_set_ref_chroma": (I, [P, I, P, P, I]),
    "x265cu_analyser_load_chroma": (I, [P, P, P, I]),
    "x265cu_analyser_enable_chroma_residual": (I, [P, I, I]),
    "x265cu_analyser_chroma_qp": (I, [P, P]),
    "x265cu_analyser_chroma_results": (I, [P, I, I, P, P]),
    "x265cu_analyser_fetch_chroma": (I, [P, I, P]),
    "x265cu_analyser_recon_plane_chroma": (P, [P, I, I, C.POINTER(I)]),
    "x265cu_analyser_recon_to_ref_chroma": (I, [P, I, I, I, I]),
    "x265cu_analyser_ref_chroma_updated": (I, [P, I]),
    "x265cu_analyser_ref_plane_chroma": (P, [P, I, I, C.POINTER(I)]),
    "x265cu_analyser_src_plane": (P, [P, I, C.POINTER(I)]),
    "x265cu_analyser_set_ref_weights": (I, [P, I, P]),
}
STAGE_CHROMA_RESIDUAL = 8                 # analyser stage bit 3 (x265cu_analyser_enable_chroma_residual)
STAGE_BIDIR = 16                          # analyser stage bit 4: BIDIR of a B slice (x265cu_analyser_set_lists)
_AN_PROTOS["x265cu_analyser_set_lists"] = (I, [P, I, I])
_AN_PROTOS["x265cu_analyser_bidir_results"] = (I, [P, I, I, P])
# x265cu_bidir_cu (include/x265_b200.h)
BIDIR_CU = np.dtype([("uniCost", np.uint32), ("biCost", np.uint32), ("interDir", np.int8), ("ref", np.int8, 2), ("zero", np.uint8),
                     ("mv", np.int16, (2, 2))])
STAGE_PART = 32                           # analyser stage bit 5: the inter estimate of every partition of a P slice's CUs
_AN_PROTOS["x265cu_analyser_part_results"] = (I, [P, I, I, P])
# x265cu_part_cu (include/x265_b200.h): entries indexed by PartSize (2Nx2N 0, 2NxN 1, Nx2N 2, NxN 3, 2NxnU 4, 2NxnD 5,
# nLx2N 6, nRx2N 7)
PART_CU = np.dtype([("cost", np.uint32, 8), ("sa8d", np.uint32, 8), ("ref", np.int8, (8, 2)), ("mv", np.int16, (8, 2, 2))])
STAGE_PART_B = 64                         # analyser stage bit 6: the inter estimate of every partition of a B slice's CUs
_AN_PROTOS["x265cu_analyser_part_b_results"] = (I, [P, I, I, P])
# x265cu_part_b_cu (include/x265_b200.h): entries indexed by PartSize as PART_CU; per PU [pu], per list [pu][list]
PART_B_CU = np.dtype([("cost", np.uint32, 8), ("sa8d", np.uint32, 8), ("biCost", np.uint32, (8, 2)), ("interDir", np.int8, (8, 2)),
                      ("ref", np.int8, (8, 2, 2)), ("zero", np.uint8, (8, 2)), ("mv", np.int16, (8, 2, 2, 2))])
_AN_PROTOS["x265cu_propagate_cost_batch"] = (I, [P, P, P, P, P, P, C.c_double, I64])
_AN_PROTOS["x265cu_lowres_intra_batch"] = (I, [P, I, P, I, I, I, I, I])
_AN_PROTOS["x265cu_lookahead_cost_batch"] = (I, [P, I, P, I, I, I, I, P])
_AN_PROTOS["x265cu_lookahead_weights_analyse"] = (I, [P, I, P, P, P, I64, I, I, I, I64, P, P, P])
_AN_PROTOS["x265cu_cutree"] = (I, [P, P, I, P, I, I, P, I])
_AN_PROTOS["x265cu_cutree_estimates"] = (I, [P, I, P, P, I])


# ---------------- adaptive quantisation (x265cu_aq_energy / x265cu_aq_finish / x265cu_aq_frame) ----------------
class AqParams(C.Structure):
    """x265cu_aq_params (include/x265_b200.h)"""
    _fields_ = [("aqMode", C.c_int32), ("qgSize", C.c_int32), ("weightp", C.c_int32), ("variance", C.c_int32),
                ("hevcAq", C.c_int32), ("hdr10Opt", C.c_int32), ("aqMotion", C.c_int32), ("reserved", C.c_int32),
                ("aqStrength", C.c_double), ("quantOffsets", P)]


class AqOut(C.Structure):
    """x265cu_aq_out: host arrays, each may be NULL"""
    _fields_ = [("qpAqOffset", P), ("invQscaleFactor", P), ("invQscaleFactor8x8", P), ("wp_sum", P), ("wp_ssd", P),
                ("blockVariance", P), ("frameVariance", P)]


def aq_geometry(W, H, qg_size):
    """(energy grid blocks, blockCount, w8 * h8): the lengths of x265cu_aq_energy's energies, of qpAqOffset /
    invQscaleFactor / blockVariance / quantOffsets, and of invQscaleFactor8x8."""
    L = 8 if qg_size == 8 else 16
    w8, h8 = ((W // 2) + 7) >> 3, ((H // 2) + 7) >> 3
    return ((W + L - 1) // L) * ((H + L - 1) // L), (4 if qg_size == 8 else 1) * w8 * h8, w8 * h8


_AN_PROTOS["x265cu_aq_energy"] = (I, [P, I, P, I, P, P, I, I, I, I, P, P])
_AN_PROTOS["x265cu_aq_finish"] = (I, [I, I, I, C.POINTER(AqParams), P, P, C.POINTER(AqOut)])
_AN_PROTOS["x265cu_aq_frame"] = (I, [P, I, P, I, P, P, I, I, I, C.POINTER(AqParams), P, C.POINTER(AqOut)])
_PROTOS.update(_AN_PROTOS)


# ---------------- weighted-prediction analysis (x265cu_weightp_costs / _decide / _analyse) ----------------
class WpFrame(C.Structure):
    """x265cu_wp_frame (include/x265_b200.h): device planes at picture origin, the picture statistics and the poc"""
    _fields_ = [("lowres", P * 4), ("cb", P), ("cr", P), ("lowresStride", C.c_int32), ("chromaStride", C.c_int32),
                ("wp_sum", C.c_uint64 * 3), ("wp_ssd", C.c_uint64 * 3), ("poc", C.c_int32), ("reserved", C.c_int32)]


class WpParams(C.Structure):
    """x265cu_wp_params: sliceType 0 B / 1 P, csp 0 4:0:0 / 1 4:2:0"""
    _fields_ = [("sliceType", C.c_int32), ("numRefIdx", C.c_int32 * 2), ("bframes", C.c_int32), ("width", C.c_int32),
                ("height", C.c_int32), ("csp", C.c_int32)]


class WpCand(C.Structure):
    _fields_ = [("weighted", C.c_int32), ("w0", C.c_int32), ("denom", C.c_int32), ("offset", C.c_int32)]


class WpEntry(C.Structure):
    _fields_ = [("wtPresent", C.c_int32), ("inputWeight", C.c_int32), ("log2WeightDenom", C.c_int32), ("inputOffset", C.c_int32)]


WP_COST_FN = C.CFUNCTYPE(C.c_int, P, C.c_int, C.c_int, C.c_int, C.POINTER(WpCand), C.c_int, C.POINTER(C.c_uint32))

_WP_PROTOS = {
    "x265cu_weightp_costs": (I, [P, I, C.POINTER(WpParams), C.POINTER(WpFrame), C.POINTER(WpFrame), P, P, I,
                                 C.POINTER(WpCand), I, P]),
    "x265cu_weightp_decide": (I, [I, C.POINTER(WpParams), C.POINTER(WpFrame), C.POINTER(C.POINTER(WpFrame)), P,
                                  WP_COST_FN, P, P]),
    "x265cu_weightp_analyse": (I, [P, I, C.POINTER(WpParams), C.POINTER(WpFrame), P, C.POINTER(C.POINTER(WpFrame)),
                                   C.POINTER(P), P]),
}
_PROTOS.update(_WP_PROTOS)


class Analyser:
    """Host mirror of x265cu_analyser: the public call a user makes for one frame is analyse()."""

    def __init__(self, lib, width, height, depth=8, numRefs=4, method=3, subme=3, merange=57, rect=1, qp=30, lam=None, amp=0):
        self.lib = lib
        if lam is None:
            lam = round(2.0 ** (qp / 6.0 - 2.0) * (1 << (depth - 8)), 4)      # x265_lambda_tab (constants.cpp:33-50)
        self.params = AnalysisParams(width, height, depth, numRefs, method, subme, merange, rect, qp, lam, amp)
        self.h = lib.L.x265cu_analyser_create(lib.ctx, C.byref(self.params))
        if not self.h:
            raise RuntimeError("x265cu_analyser_create failed: " + lib.last_error())
        nj, nc, nt, st = I(), I(), I(), I()
        ncoef = I64()
        lib.L.x265cu_analyser_counts(self.h, C.byref(nj), C.byref(nc), C.byref(nt), C.byref(ncoef), C.byref(st))
        self.njobs, self.ncu, self.ntu, self.ncoef, self.stride = nj.value, nc.value, nt.value, ncoef.value, st.value
        self.depth, self.width, self.height, self.numRefs = depth, width, height, numRefs
        self.dtype = np.uint8 if depth == 8 else np.uint16
        # host result buffers (pinned so D2H is real DMA)
        self._pinned = []
        self.me_packed = self._pin((self.njobs, 2), np.int32)
        self.cu_sse = self._pin((self.ncu,), np.uint64)
        self.cu_numsig = self._pin((self.ncu,), np.uint32)
        self.cu_ref = self._pin((self.ncu,), np.int32)
        self.intra_cost = self._pin((self.ncu, 36), np.uint32)
        self.out = AnalysisOut(self.me_packed.ctypes.data, self.cu_sse.ctypes.data, self.cu_numsig.ctypes.data,
                               self.cu_ref.ctypes.data, self.intra_cost.ctypes.data)

    def _pin(self, shape, dtype):
        n = int(np.prod(shape)) * np.dtype(dtype).itemsize
        p = self.lib.L.x265cu_host_alloc(max(n, 16))
        if not p:
            raise MemoryError("pinned alloc failed")
        self._pinned.append(p)
        buf = (C.c_uint8 * n).from_address(p)
        return np.frombuffer(buf, dtype=dtype).reshape(shape)

    def set_ref(self, idx, img):
        img = np.ascontiguousarray(img, self.dtype)
        assert img.shape == (self.height, self.width)
        self.lib.check(self.lib.L.x265cu_analyser_set_ref(self.h, idx, img.ctypes.data, self.width))

    def load_inputs(self, fenc, field):
        fenc = np.ascontiguousarray(fenc, self.dtype)
        field = np.ascontiguousarray(field, np.int16)
        self.lib.check(self.lib.L.x265cu_analyser_load_inputs(self.h, fenc.ctypes.data, self.width, field.ctypes.data))

    def run_resident(self, stages=7):
        self.lib.check(self.lib.L.x265cu_analyser_run_resident(self.h, stages))

    def analyse(self, fenc, field, stages=7):
        """e2e: host frame + predictor field in, host results out (synchronous)."""
        self.lib.check(self.lib.L.x265cu_analyser_analyse(self.h, fenc.ctypes.data, self.width, field.ctypes.data, stages, C.byref(self.out)))
        return self

    # ---- CTU-row shards (x265cu_analyser_*_rows): rows [r0, r1) are one contiguous slice of every result array ----
    @property
    def ctu_rows(self):
        return int(self.lib.L.x265cu_analyser_ctu_rows(self.h))

    def row_range(self, r0, r1):
        """(job0, njobs, cu0, ncu) of the CTU rows [r0, r1)."""
        v = [I(), I(), I(), I()]
        self.lib.check(self.lib.L.x265cu_analyser_row_range(self.h, r0, r1, *[C.byref(x) for x in v]))
        return tuple(x.value for x in v)

    def run_rows(self, r0, r1, stages=7):
        self.lib.check(self.lib.L.x265cu_analyser_run_rows(self.h, stages, r0, r1))

    def analyse_rows(self, fenc, field, r0, r1, stages=7):
        """e2e for a row shard: host frame + field in, the shard's slice of the host result arrays out."""
        self.lib.check(self.lib.L.x265cu_analyser_analyse_rows(self.h, fenc.ctypes.data, self.width, field.ctypes.data, stages, r0, r1, C.byref(self.out)))
        return self

    def d2h_bytes_rows(self, r0, r1):
        _, nj, _, nc = self.row_range(r0, r1)
        return nj * 8 + nc * (8 + 4 + 4 + 36 * 4)

    def recon_plane_ptr(self, depth_idx):
        st = I()
        return self.lib.L.x265cu_analyser_recon_plane(self.h, depth_idx, C.byref(st)), st.value

    def recon_to_ref(self, depth_idx, ref_idx, r0, r1):
        self.lib.check(self.lib.L.x265cu_analyser_recon_to_ref(self.h, depth_idx, ref_idx, r0, r1))

    # ---- 4:2:0 chroma for the chroma-SATD term of subpelCompare ----
    def enable_chroma(self):
        self.lib.check(self.lib.L.x265cu_analyser_enable_chroma(self.h))

    def set_ref_chroma(self, idx, cb, cr):
        cb = np.ascontiguousarray(cb, self.dtype); cr = np.ascontiguousarray(cr, self.dtype)
        assert cb.shape == cr.shape == (self.height // 2, self.width // 2)
        self.lib.check(self.lib.L.x265cu_analyser_set_ref_chroma(self.h, idx, cb.ctypes.data, cr.ctypes.data, self.width // 2))

    def load_chroma(self, cb, cr):
        """Source chroma of the next analyse() / run_*() (pass pinned arrays for true async DMA)."""
        assert cb.shape == cr.shape == (self.height // 2, self.width // 2) and cb.dtype == self.dtype and cb.flags.c_contiguous and cr.flags.c_contiguous
        self.lib.check(self.lib.L.x265cu_analyser_load_chroma(self.h, cb.ctypes.data, cr.ctypes.data, self.width // 2))

    # ---- 4:2:0 chroma residual chain (stage bit 3) ----
    def enable_chroma_residual(self, cb_qp_offset=0, cr_qp_offset=0):
        """Allocates the chroma residual outputs and sets the planes' QP offsets (PPS + slice, -12..12); needs
        enable_chroma().  Afterwards runs may set stage bit 3 (STAGE_CHROMA_RESIDUAL)."""
        self.lib.check(self.lib.L.x265cu_analyser_enable_chroma_residual(self.h, cb_qp_offset, cr_qp_offset))

    def chroma_qp(self):
        """(Cb, Cr) quantiser QPs of the chroma residual stage."""
        q = (C.c_int * 2)()
        self.lib.check(self.lib.L.x265cu_analyser_chroma_qp(self.h, q))
        return q[0], q[1]

    def chroma_results(self, r0=0, r1=None, sse=None, numsig=None):
        """Per-CU [ncu][2] (Cb, Cr) SSE and number of nonzero levels of the CTU rows [r0, r1) (default: all), into the given
        full-frame arrays or new zeroed ones; returns (sse, numsig)."""
        r1 = self.ctu_rows if r1 is None else r1
        sse = np.zeros((self.ncu, 2), np.uint64) if sse is None else sse
        numsig = np.zeros((self.ncu, 2), np.uint32) if numsig is None else numsig
        assert sse.shape == numsig.shape == (self.ncu, 2) and sse.dtype == np.uint64 and numsig.dtype == np.uint32
        self.lib.check(self.lib.L.x265cu_analyser_chroma_results(self.h, r0, r1, sse.ctypes.data, numsig.ctypes.data))
        return sse, numsig

    # ---- B slices (x265cu_analyser_set_lists, stage bit 4) ----
    def set_lists(self, n0, n1):
        """Slots [0, n0) are list 0, [n0, n0 + n1) list 1 (n0 + n1 == numRefs); n1 == 0 is a P slice.  Afterwards runs may
        set stage bit 4 (STAGE_BIDIR), and a B slice's residual stages need it in the same call."""
        self.lib.check(self.lib.L.x265cu_analyser_set_lists(self.h, n0, n1))

    def bidir_results(self, r0=0, r1=None, out=None):
        """The BIDIR record (BIDIR_CU) of every CU of the CTU rows [r0, r1) (default: all) into the given full-frame array or
        a new zeroed one; returns it."""
        r1 = self.ctu_rows if r1 is None else r1
        out = np.zeros(self.ncu, BIDIR_CU) if out is None else out
        assert out.shape == (self.ncu,) and out.dtype == BIDIR_CU
        self.lib.check(self.lib.L.x265cu_analyser_bidir_results(self.h, r0, r1, out.ctypes.data))
        return out

    # ---- the inter estimate of every partition of a P slice's CUs (stage bit 5) ----
    def part_results(self, r0=0, r1=None, out=None):
        """The PART record (PART_CU) of every CU of the CTU rows [r0, r1) (default: all) into the given full-frame array or a
        new zeroed one; returns it.  Needs a run with stage bit 5 (STAGE_PART) first."""
        r1 = self.ctu_rows if r1 is None else r1
        out = np.zeros(self.ncu, PART_CU) if out is None else out
        assert out.shape == (self.ncu,) and out.dtype == PART_CU
        self.lib.check(self.lib.L.x265cu_analyser_part_results(self.h, r0, r1, out.ctypes.data))
        return out

    # ---- the inter estimate of every partition of a B slice's CUs (stage bit 6) ----
    def part_b_results(self, r0=0, r1=None, out=None):
        """The PART_B record (PART_B_CU) of every CU of the CTU rows [r0, r1) (default: all) into the given full-frame array or
        a new zeroed one; returns it.  Needs a run with stage bit 6 (STAGE_PART_B) first."""
        r1 = self.ctu_rows if r1 is None else r1
        out = np.zeros(self.ncu, PART_B_CU) if out is None else out
        assert out.shape == (self.ncu,) and out.dtype == PART_B_CU
        self.lib.check(self.lib.L.x265cu_analyser_part_b_results(self.h, r0, r1, out.ctypes.data))
        return out

    def chroma_plane_shape(self):
        """(rows, cstride) of a chroma plane allocation: the picture's origin is at row 40, column 48."""
        return self.height // 2 + 80, self.stride // 2

    def fetch_chroma(self, what):
        """"coef_cb" / "coef_cr": a plane's levels (ncoef / 4); ("recon", depthIdx, plane): the whole allocation of a chroma
        recon plane; ("ref", ref, plane): the whole allocation of a reference's chroma plane."""
        if what in ("coef_cb", "coef_cr"):
            out = np.zeros(self.ncoef // 4, np.int16)
            idx = 0 if what == "coef_cb" else 1
        else:
            kind, a, plane = what
            assert plane in (0, 1) and (kind == "recon" and 0 <= a < 4 or kind == "ref" and 0 <= a < self.numRefs), what
            out = np.zeros(self.chroma_plane_shape(), self.dtype)
            idx = (2 if kind == "recon" else 10) + 2 * a + plane
        self.lib.check(self.lib.L.x265cu_analyser_fetch_chroma(self.h, idx, out.ctypes.data))
        return out

    def recon_plane_chroma_ptr(self, depth_idx, plane):
        st = I()
        return self.lib.L.x265cu_analyser_recon_plane_chroma(self.h, depth_idx, plane, C.byref(st)), st.value

    # ---- weighted P-slice references (x265cu_analyser_set_ref_weights) ----
    def set_ref_weights(self, idx, entries):
        """Weights of reference idx: a (3, 4) int array {wtPresent, inputWeight, log2WeightDenom, inputOffset} for luma, Cb, Cr
        as Lookahead.weight_analyse()[0][idx] returns it, or None (unweighted)."""
        if entries is None:
            self.lib.check(self.lib.L.x265cu_analyser_set_ref_weights(self.h, idx, None))
            return
        e = np.ascontiguousarray(entries, np.int32)
        assert e.shape == (3, 4), e.shape
        self.lib.check(self.lib.L.x265cu_analyser_set_ref_weights(self.h, idx, e.ctypes.data))

    def fetch_search_chroma(self, ref, plane):
        """The whole allocation of the chroma plane (0 Cb, 1 Cr) that the chroma-SATD term of the search reads for reference
        ref: its weighted plane when it has one, else the reference's plane."""
        assert 0 <= ref < self.numRefs and plane in (0, 1)
        out = np.zeros(self.chroma_plane_shape(), self.dtype)
        self.lib.check(self.lib.L.x265cu_analyser_fetch_chroma(self.h, 10 + 2 * self.numRefs + 2 * ref + plane, out.ctypes.data))
        return out

    def recon_to_ref_chroma(self, depth_idx, ref_idx, r0, r1):
        self.lib.check(self.lib.L.x265cu_analyser_recon_to_ref_chroma(self.h, depth_idx, ref_idx, r0, r1))

    def ref_chroma_updated(self, idx):
        self.lib.check(self.lib.L.x265cu_analyser_ref_chroma_updated(self.h, idx))

    def ref_plane_chroma(self, idx, plane):
        """(device address of pixel (0,0), stride in elements) of chroma plane `plane` (0 Cb, 1 Cr) of reference idx."""
        st = I()
        p = self.lib.L.x265cu_analyser_ref_plane_chroma(self.h, idx, plane, C.byref(st))
        if not p:
            raise RuntimeError("x265cu_analyser_ref_plane_chroma(%d, %d): no such plane (enable_chroma() first)" % (idx, plane))
        return p, st.value

    def src_plane(self, plane):
        """(device address of pixel (0,0), stride in elements) of the resident source plane `plane` (0 luma, 1 Cb, 2 Cr)."""
        st = I()
        p = self.lib.L.x265cu_analyser_src_plane(self.h, plane, C.byref(st))
        if not p:
            raise RuntimeError("x265cu_analyser_src_plane(%d): no such plane (chroma: enable_chroma() first)" % plane)
        return p, st.value

    def h2d_bytes(self, field):
        return self.width * self.height * np.dtype(self.dtype).itemsize + field.nbytes

    def d2h_bytes(self):
        return self.me_packed.nbytes + self.cu_sse.nbytes + self.cu_numsig.nbytes + self.cu_ref.nbytes + self.intra_cost.nbytes

    def stage_ms(self):
        ms = (C.c_float * 4)()
        self.lib.check(self.lib.L.x265cu_analyser_stage_ms(self.h, ms))
        return [float(x) for x in ms]

    def ref_plane_ptr(self, idx):
        st = I()
        return self.lib.L.x265cu_analyser_ref_plane(self.h, idx, C.byref(st)), st.value

    def ref_updated(self, idx):
        self.lib.check(self.lib.L.x265cu_analyser_ref_updated(self.h, idx))

    def fetch(self, what):
        """A device-resident array by name, or ("plane", ref, phase): the whole allocation (stride x (height + 160)) of
        reference ref's phase plane yf * 4 + xf (phase 0 = the reference plane itself; for a weighted reference, of its weighted
        plane: what the search reads)."""
        es = np.dtype(self.dtype).itemsize
        rows = self.height + 160
        if isinstance(what, tuple):
            _, ref, phase = what
            assert 0 <= ref < self.numRefs and 0 <= phase < 16, what
            out = np.zeros((rows, self.stride), self.dtype)
            self.lib.check(self.lib.L.x265cu_analyser_fetch(self.h, 16 + 16 * ref + phase, out.ctypes.data))
            return out
        spec = {"jobs": (0, ME_JOB, self.njobs), "me_out": (1, np.int32, self.njobs * 4), "coef": (2, np.int16, self.ncoef),
                "recon0": (3, self.dtype, self.stride * rows), "recon1": (4, self.dtype, self.stride * rows),
                "recon2": (5, self.dtype, self.stride * rows), "recon3": (6, self.dtype, self.stride * rows),
                "cu_jobs": (7, np.int32, self.ncu * self.numRefs), "fenc": (8, self.dtype, self.stride * rows)}[what]
        out = np.zeros(spec[2], spec[1])
        self.lib.check(self.lib.L.x265cu_analyser_fetch(self.h, spec[0], out.ctypes.data))
        return out

    def close(self):
        if self.h:
            self.lib.L.x265cu_analyser_destroy(self.h)
            self.h = None
        for p in self._pinned:
            self.lib.L.x265cu_host_free(p)
        self._pinned = []
