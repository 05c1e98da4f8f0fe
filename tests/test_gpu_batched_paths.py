"""GPU parity of the batched C-ABI entry points (include/x265_b200.h section 2) on the dispatch paths the per-call table never
reaches.  Every per-call thunk stages its blocks compactly at a 64-byte-aligned arena offset with stride == width and a batch of
one (thunks.cuh, Stage::reserve / put), so a branch that depends on a misaligned base, an odd or padded stride, a 4-tap job or
more jobs than one grid holds runs only when a caller hands the batched entry points such a job list.

Each case names the path it targets (PATHS: one entry per dispatch branch, with the C lines it lives at).  The `*_path`
functions mirror the dispatch predicates line by line; every case asserts that the mirror sends it where it says, and
test_every_path_is_targeted keeps PATHS and the cases in step.  test_dispatch_kernel_names confirms the mirrors against the
kernel names torch.profiler records.  Grid caps come from the device's SM count.

Results are compared bit-exactly with the oracle (the plain-C restatement test_oracle_vs_ref.py pins to the reference), at 8
and 10 bit.  Every destination is sentinel-filled around and between the job rectangles (row padding, TU padding, the
elements before and after a misaligned base) and compared whole: a guard-band element that changed fails on its own
message.  The large-n cases draw inputs from a pool of POOL entries (a prime, so that TU t and TU t + one grid trip never
share an input); every job keeps its own destination.
"""
import ctypes as C
import zlib

import numpy as np
import pytest

from common import load_oracle, pixel_dtype, ptr, IP, LUMA_PU
from x265_b200.lib import BLK_JOB, INTERP_JOB, INTRA_JOB, OPS_BLK, OPS_INTERP

pytestmark = pytest.mark.gpu

DEPTHS = [8, 10]
POOL = 61
DCT, IDCT, DST4, IDST4 = 0, 1, 2, 3

# ---------------------------------------------------------------------------------------------------------------------
# the path table: every dispatch branch of the batched entry points this file targets, and where it is chosen
PATHS = {
    "mma_inv_swap": "IMMA inverse, role-swapped pass 2 with 4-byte stores (control): transform_mma.cuh:246-270, chosen at :319",
    "mma_inv_scatter": "IMMA inverse, scattered 2-byte stores (swapStore == 0): transform_mma.cuh:272-300, chosen at :319",
    "mma_inv_unaligned": "IMMA inverse, coefficient base not 16-byte aligned (in16 == false): transform_mma.cuh:80, 191-195",
    "mma_inv_trips": "IMMA inverse past one grid: 16x16 prefetch of the next TU, second grid-stride trip: transform_mma.cuh:142-149, 201-206, cap :316-317",
    "mma_fwd_contig": "IMMA forward on contiguous TUs (control): transform_mma.cuh:312-314",
    "mma_fwd_strided": "IMMA forward on strided rows (stride % 4 == 0, stride != N): transform_mma.cuh:314",
    "reg": "4x4 / 8x8 one-thread-per-TU kernel on contiguous aligned TUs (control): transform.cuh:277-278",
    "generic_transform": "k_transform: DST4 / IDST4, strided 4x4 / 8x8, misaligned 16x16 / 32x32, grid-stride loop: transform.cuh:295-307",
    "quant": "x265cu_quant_batch with many TUs and past one grid: x265cu.cu:144-153, transform.cuh:330-353",
    "dequant_normal": "x265cu_dequant_normal_batch, num not a multiple of 256, past one grid: x265cu.cu:155-163, transform.cuh:355-360",
    "dequant_scaling": "x265cu_dequant_scaling_batch, dq[i % numCoeff] across TUs, both shift branches: x265cu.cu:165-174, transform.cuh:363-375",
    "blockop_vector": "k_blockop vector path, 8 elements per thread (control): blockops.cuh:157-179",
    "blockop_scalar": "k_blockop scalar path: w % 8 != 0, or w % 8 == 0 rows that fail the alignment test: blockops.cuh:162-165, 181-185",
    "blockop_any_op": "k_blockop<P, -1> instantiation for the non-hot ops: blockops.cuh:206",
    "blockop_trips": "k_blockop grid-stride over jobs (n > 16 x SMs): blockops.cuh:151, cap :192",
    "intra_pred": "x265cu_intra_pred_batch, padded dst_stride / dst_pitch, n > 8 x SMs: x265cu.cu:176-187, intra.cuh:119-134",
    "allangs_packed": "k_intra_allangs_packed, dst 16-byte aligned (control): x265cu.cu:207-224",
    "allangs_cta": "k_intra_allangs_cta, dst 8- but not 16-byte aligned, n > 16 x SMs: x265cu.cu:204-206, 225-226",
    "allangs_generic": "k_intra_allangs, dst not 8-byte aligned, n > grid.y = 4096: x265cu.cu:230-233",
    "lowres_fast": "k_lowres_init_u8x8 / _u16x4 (control): x265cu.cu:251-260",
    "lowres_generic": "generic k_lowres_init: width not a multiple of 8 / 4, or src rows that fail the alignment test: x265cu.cu:261-264, blockops.cuh:215-250",
    "extend_padding": "k_extend_border margin rows copying the stride padding past width + mx: blockops.cuh:347-354",
    "propagate_trips": "x265cu_propagate_cost_batch past one grid, odd tail: x265cu.cu:387-396",
    "interp_4tap": "4-tap (chroma) jobs in x265cu_interp_batch, alone and mixed with 8-tap jobs: interp.cuh:310-397, 523-540",
}


def _ctype(depth):
    return "unsigned char" if depth == 8 else "unsigned short"


# ---------------------------------------------------------------------------------------------------------------------
# mirrors of the dispatch predicates; addresses are device byte addresses.  Each returns (kernel name prefix, path).
def transform_path(depth, op, N, src, dst, stride, pitch, n, sms):
    if op in (DST4, IDST4):
        N = 4                                                                        # transform.cuh:313
    if N in (16, 32) and op in (DCT, IDCT):                                          # transform_mma.cuh:309-311
        fwd = op == DCT
        if not fwd or not ((src & 7) or (stride & 3) or (pitch & 3) or (dst & 3)):   # :314
            kern = "k_transform_mma<%d, %d, %s>" % (depth, N, "true" if fwd else "false")
            warps = 8 * min((n + 7) // 8, 8 * sms)                                   # :316-317
            if not fwd and n > warps:
                return kern, "mma_inv_trips"
            if fwd:
                return kern, "mma_fwd_contig" if (stride == N and pitch == N * N) else "mma_fwd_strided"
            if src & 15:                                                             # :80
                return kern, "mma_inv_unaligned"
            vec = not (dst & 3) and not (stride & 1) and not (pitch & 1)             # :319
            return kern, "mma_inv_swap" if vec else "mma_inv_scatter"
    if op in (DCT, IDCT) and N in (4, 8) and stride == N and pitch == N * N and not ((src | dst) & 15):   # transform.cuh:277-278
        return "k_transform_reg<%d, %d, %s>" % (depth, N, "true" if op == DCT else "false"), "reg"
    return "k_transform<%d, %d>" % (depth, N), "generic_transform"


BLK_HOT = ("sub_ps", "add_ps", "pixelavg_pp", "addAvg", "copy_pp", "copy_ss", "copy_ps", "copy_sp", "p2s")   # blockops.cuh:197-205
# element types of (dst, a, b): "p" pixel, "s" int16, "-" unused (blockops.cuh:61-82); transpose and scale2D have no vector path
BLK_TYPES = {"copy_pp": "pp-", "copy_ss": "ss-", "copy_sp": "ps-", "copy_ps": "sp-", "sub_ps": "spp", "add_ps": "pps",
             "pixelavg_pp": "ppp", "addAvg": "pss", "p2s": "sp-", "transpose": "pp-", "blockfill_s": "s--",
             "cpy2Dto1D_shl": "ss-", "cpy2Dto1D_shr": "ss-", "cpy1Dto2D_shl": "ss-", "cpy1Dto2D_shr": "ss-",
             "weight_pp": "pp-", "weight_sp": "ps-", "scale2D_64to32": "pp-", "dequant_normal": "ss-"}
BLK_SCALAR_ONLY = ("transpose", "scale2D_64to32")


def blockop_kernel(depth, op):
    return "k_blockop<%s, %d>" % (_ctype(depth), OPS_BLK[op] if op in BLK_HOT else -1)        # blockops.cuh:195-206


def blockop_path(depth, op, jb, D, A, B):
    """blockops.cuh:157-165: the vector path needs w % 8 == 0 and every used operand's base and row pitch 8-element aligned"""
    if op in BLK_SCALAR_ONLY or jb["w"] % 8:
        return "blockop_scalar"
    es = 1 if depth == 8 else 2
    ok = True
    for base, off, stride, t in ((D, jb["d_off"], jb["d_stride"], BLK_TYPES[op][0]), (A, jb["a_off"], jb["a_stride"], BLK_TYPES[op][1]),
                                 (B, jb["b_off"], jb["b_stride"], BLK_TYPES[op][2])):
        if t == "-":
            continue
        s = es if t == "p" else 2
        ok = ok and ((base + int(off) * s) | (int(stride) * s)) % (8 * s) == 0
    return "blockop_vector" if ok else "blockop_scalar"


def allangs_path(depth, N, dst):
    """x265cu.cu:204-233"""
    if dst & 7 == 0 and 4 <= N <= 32:
        if dst & 15 == 0:
            uw = min(N * (1 if depth == 8 else 2), 16) // 4
            return "k_intra_allangs_packed<%s, %d>" % (_ctype(depth), uw), "allangs_packed"
        return "k_intra_allangs_cta<%s>" % _ctype(depth), "allangs_cta"
    return "k_intra_allangs<%s>" % _ctype(depth), "allangs_generic"


def lowres_path(depth, width, src, sstride, planes, dstride):
    """x265cu.cu:250-264"""
    dal = planes[0] | planes[1] | planes[2] | planes[3]
    if depth == 8 and width & 7 == 0 and (src | sstride) & 15 == 0 and (dal | dstride) & 7 == 0:
        return "k_lowres_init_u8x8", "lowres_fast"
    if depth != 8 and width & 3 == 0 and (src | (sstride * 2)) & 15 == 0 and (dal | (dstride * 2)) & 7 == 0:
        return "k_lowres_init_u16x4", "lowres_fast"
    return "k_lowres_init<%s>" % _ctype(depth), "lowres_generic"


def interp_kernel(depth, op, jb):
    """interp.cuh:310-314 (interp_fast_eligible): the row-segment kernel takes 8-tap pixel-source jobs of width % 8 == 0 up to 64"""
    fast = (jb["ntaps"] == 8 and jb["w"] % 8 == 0 and jb["w"] <= 64 and jb["h"] > 0 and op in ("hpp", "hps", "vpp", "vps", "hvpp"))
    if fast:
        group = 2 if op == "hvpp" else (1 if op in ("vpp", "vps") else 0)                     # interp.cuh:516-521
        return "k_interp_rows<%s, %d>" % (_ctype(depth), group)
    return "k_interp<%s>" % _ctype(depth)


# ---------------------------------------------------------------------------------------------------------------------
# helpers
def sentinel(dtype):
    """guard-band fill: outside the 10-bit pixel range for uint16, an unlikely value otherwise"""
    return {np.dtype(np.uint8): 0xA5, np.dtype(np.uint16): 0xFFFF, np.dtype(np.int16): -21846,
            np.dtype(np.int32): -1431655766, np.dtype(np.uint32): 0xAAAAAAAA}[np.dtype(dtype)]


def guarded(size, dtype):
    return np.full(size, sentinel(dtype), dtype)


def rect_index(off, stride, rows, cols, pitch=0, count=1):
    """element indices of `count` rectangles of rows x cols (row stride `stride`), the k-th at off + k * pitch: (count, rows, cols)"""
    t = np.arange(count, dtype=np.int64)[:, None, None]
    r = np.arange(rows, dtype=np.int64)[None, :, None]
    c = np.arange(cols, dtype=np.int64)[None, None, :]
    return off + t * pitch + r * stride + c


def check_guarded(got, want, written, what):
    """`written`: mask of the elements the jobs own; every other element must still hold the sentinel"""
    got, want, written = got.ravel(), want.ravel(), written.ravel()
    assert got.shape == want.shape
    bad = np.nonzero((got != want) & ~written)[0]
    assert bad.size == 0, "%s: guard band changed at %d elements, first %s: %s" % (what, bad.size, bad[:6], got[bad[:6]])
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, "%s: %d mismatches, first at %s: got %s want %s" % (what, bad.size, bad[:6], got[bad[:6]], want[bad[:6]])


def mask_of(size, idx):
    m = np.zeros(size, bool)
    m[np.asarray(idx).ravel()] = True
    return m


def span_mask(size, a, b):
    m = np.zeros(size, bool)
    m[a:b] = True
    return m


@pytest.fixture(scope="module")
def cu():
    import x265_b200
    return x265_b200.load()


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


class Dev:
    """A device copy of a host array; at(k) is the device address of element k."""

    def __init__(self, cu, arr):
        self.arr = np.ascontiguousarray(arr)
        self.buf = cu.to_device(self.arr)

    def at(self, k=0):
        return self.buf.ptr + int(k) * self.arr.itemsize

    def get(self):
        return self.buf.download(self.arr.dtype, self.arr.size).reshape(self.arr.shape)


@pytest.fixture
def dev(cu):
    held = []

    def make(arr):
        d = Dev(cu, arr)
        held.append(d)
        return d
    yield make
    for d in held:
        d.buf.free()


# ---------------------------------------------------------------------------------------------------------------------
# transforms (x265cu_transform_batch)
def coef_pool(rng, N):
    """IDCT / IDST inputs that are not forward-transform outputs: full-range int16, all 32767, all -32768, DC-only, last-only"""
    p = rng.integers(-32768, 32768, (POOL, N, N)).astype(np.int16)
    for k in range(POOL):
        kind = k % 6
        if kind == 2:
            p[k] = 32767
        elif kind == 3:
            p[k] = -32768
        elif kind == 4:
            dc = p[k, 0, 0] if k % 4 else (-32768 if k % 8 else 32767)
            p[k] = 0
            p[k, 0, 0] = dc
        elif kind == 5:
            last = p[k, N - 1, N - 1] if k % 4 else -32768
            p[k] = 0
            p[k, N - 1, N - 1] = last
    return p


def resid_pool(rng, N, depth):
    """forward inputs: residuals in +-(2^depth - 1), all +max, all -max, a +-max checkerboard"""
    mx = (1 << depth) - 1
    p = (rng.integers(0, mx + 1, (POOL, N, N)) - rng.integers(0, mx + 1, (POOL, N, N))).astype(np.int16)
    chk = np.where((np.arange(N)[:, None] + np.arange(N)[None, :]) % 2 == 0, mx, -mx).astype(np.int16)
    for k in range(POOL):
        if k % 5 == 2:
            p[k] = mx
        elif k % 5 == 3:
            p[k] = -mx
        elif k % 5 == 4:
            p[k] = chk if k % 2 else -chk
    return p


# (case id, op, N, src element offset, dst element offset, stride - N, tu_pitch - stride * N, TU count: "few" / "trips", path)
# DCT / DST4: stride and tu_pitch describe the source rows; IDCT / IDST4: the destination rows.
TRANSFORM_CASES = [
    ("idct16-swap", IDCT, 16, 0, 0, 2, 4, "few", "mma_inv_swap"),
    ("idct32-swap", IDCT, 32, 0, 0, 0, 0, "few", "mma_inv_swap"),
    ("idct16-odd-stride", IDCT, 16, 0, 0, 1, 3, "few", "mma_inv_scatter"),
    ("idct32-odd-stride", IDCT, 32, 0, 0, 3, 0, "few", "mma_inv_scatter"),
    ("idct16-odd-pitch", IDCT, 16, 0, 0, 2, 1, "few", "mma_inv_scatter"),
    ("idct32-odd-pitch", IDCT, 32, 0, 0, 0, 7, "few", "mma_inv_scatter"),
    ("idct16-dst-2byte", IDCT, 16, 0, 1, 4, 2, "few", "mma_inv_scatter"),
    ("idct32-dst-2byte", IDCT, 32, 0, 3, 2, 0, "few", "mma_inv_scatter"),
    ("idct16-src-2byte", IDCT, 16, 1, 0, 2, 2, "few", "mma_inv_unaligned"),
    ("idct32-src-8byte", IDCT, 32, 4, 0, 0, 0, "few", "mma_inv_unaligned"),
    ("idct16-src-8byte-scatter", IDCT, 16, 4, 1, 1, 0, "few", "mma_inv_unaligned"),
    ("idct32-src-2byte-scatter", IDCT, 32, 1, 0, 1, 1, "few", "mma_inv_unaligned"),
    ("idct16-trips", IDCT, 16, 0, 0, 0, 0, "trips", "mma_inv_trips"),
    ("idct32-trips", IDCT, 32, 0, 0, 2, 2, "trips", "mma_inv_trips"),
    ("idct16-trips-scatter", IDCT, 16, 0, 1, 1, 1, "trips", "mma_inv_trips"),
    ("idct16-trips-src-8byte", IDCT, 16, 4, 0, 0, 0, "trips", "mma_inv_trips"),
    ("dct16-contig", DCT, 16, 0, 0, 0, 0, "few", "mma_fwd_contig"),
    ("dct32-contig", DCT, 32, 0, 0, 0, 0, "few", "mma_fwd_contig"),
    ("dct16-strided", DCT, 16, 4, 2, 4, 8, "few", "mma_fwd_strided"),
    ("dct32-strided", DCT, 32, 4, 2, 8, 4, "few", "mma_fwd_strided"),
    ("dct16-strided-trips", DCT, 16, 0, 0, 4, 0, "trips", "mma_fwd_strided"),
    ("dct32-src-2byte", DCT, 32, 1, 0, 0, 0, "few", "generic_transform"),
    ("dct16-dst-2byte", DCT, 16, 0, 1, 4, 4, "few", "generic_transform"),
    ("dct4-contig", DCT, 4, 0, 0, 0, 0, "few", "reg"),
    ("idct8-contig", IDCT, 8, 0, 0, 0, 0, "few", "reg"),
    ("dct4-strided-trips", DCT, 4, 0, 0, 3, 5, "trips", "generic_transform"),
    ("idct4-strided-trips", IDCT, 4, 0, 0, 3, 5, "trips", "generic_transform"),
    ("dct8-strided-trips", DCT, 8, 0, 0, 1, 2, "trips", "generic_transform"),
    ("idct8-dst-2byte-trips", IDCT, 8, 0, 1, 0, 0, "trips", "generic_transform"),
    ("dst4", DST4, 4, 0, 0, 0, 0, "few", "generic_transform"),
    ("dst4-strided-trips", DST4, 4, 1, 0, 2, 3, "trips", "generic_transform"),
    ("idst4", IDST4, 4, 0, 0, 0, 0, "few", "generic_transform"),
    ("idst4-strided-trips", IDST4, 4, 1, 0, 2, 3, "trips", "generic_transform"),
]


def _transform_count(kind, op, N, sms):
    if kind == "few":
        return 333
    if op in (DST4, IDST4) or N in (4, 8):
        trip = 8 * sms * min(max(1024 // (N * N), 1), 16)            # k_transform: blocks x TUs per block (transform.cuh:297-299)
    else:
        trip = 64 * sms                                                # k_transform_mma: 8 x SMs CTAs of 8 warps (transform_mma.cuh:316-317)
    assert trip % POOL, "TU t and TU t + one trip would share an input"
    return 2 * trip + 37


@pytest.mark.parametrize("depth", DEPTHS)
@pytest.mark.parametrize("case", TRANSFORM_CASES, ids=[c[0] for c in TRANSFORM_CASES])
def test_transform_batch_paths(cu, dev, sms, depth, case):
    name, op, N, soff, doff, sd, pd, count, path = case
    O = load_oracle(depth)
    rng = np.random.default_rng(zlib.crc32(name.encode()) + depth)
    n = _transform_count(count, op, N, sms)
    NN = N * N
    stride = N + sd
    pitch = stride * N + pd
    fwd = op in (DCT, DST4)
    pool = resid_pool(rng, N, depth) if fwd else coef_pool(rng, N)
    out = np.zeros((POOL, N, N), np.int16)
    for k in range(POOL):
        if op == DCT:
            O.orc_dct(ptr(pool[k]), ptr(out[k]), IP(N), N)
        elif op == DST4:
            O.orc_dst4(ptr(pool[k]), ptr(out[k]), IP(N))
        elif op == IDCT:
            O.orc_idct(ptr(pool[k]), ptr(out[k]), IP(N), N)
        else:
            O.orc_idst4(ptr(pool[k]), ptr(out[k]), IP(N))
    sel = np.arange(n) % POOL
    G = 16                                                             # guard elements after the last TU
    if fwd:
        # strided source rows (noise in the padding: a kernel that reads it computes something else), contiguous coefficients
        src = rng.integers(-32768, 32768, soff + (n - 1) * pitch + (N - 1) * stride + N + G).astype(np.int16)
        src[rect_index(soff, stride, N, N, pitch, n)] = pool[sel]
        dst_idx = rect_index(doff, N, N, N, NN, n)
        want = guarded(doff + n * NN + G, np.int16)
    else:
        src = rng.integers(-32768, 32768, soff + n * NN + G).astype(np.int16)
        src[rect_index(soff, N, N, N, NN, n)] = pool[sel]
        dst_idx = rect_index(doff, stride, N, N, pitch, n)
        want = guarded(doff + (n - 1) * pitch + (N - 1) * stride + N + G, np.int16)
    want[dst_idx] = out[sel]
    dS, dD = dev(src), dev(guarded(want.size, np.int16))
    kern, got_path = transform_path(depth, op, N, dS.at(soff), dD.at(doff), stride, pitch, n, sms)
    assert got_path == path, (name, kern, got_path)
    cu.check(cu.L.x265cu_transform_batch(cu.ctx, depth, op, N, dS.at(soff), dD.at(doff), stride, pitch, n))
    check_guarded(dD.get(), want, mask_of(want.size, dst_idx), "%s n=%d" % (name, n))


# ---------------------------------------------------------------------------------------------------------------------
# quant family
QUANT_CASES = [(nc, du, nq) for nc in (16, 64, 256, 1024) for du in (0, 1) for nq in (0, 1)]


@pytest.mark.parametrize("depth", DEPTHS)
@pytest.mark.parametrize("numCoeff,withDeltaU,nquant", QUANT_CASES, ids=["%d-%s-%s" % (c, "deltaU" if d else "noDeltaU", "nquant" if q else "quant") for c, d, q in QUANT_CASES])
def test_quant_batch(cu, dev, sms, depth, numCoeff, withDeltaU, nquant):
    """More TUs than one grid holds (8 x SMs CTAs of 8 warps, x265cu.cu:149); per-TU numSig; qBits from the encoder's range at
    this depth (QUANT_SHIFT + per + transformShift, transformShift = 15 - depth - log2 N) plus the table tests' wider range."""
    O = load_oracle(depth)
    rng = np.random.default_rng(1000 + numCoeff + 10 * withDeltaU + 100 * nquant + depth)
    n = 64 * sms + 37
    log2n = int(np.log2(numCoeff)) // 2
    pool = rng.integers(-32768, 32768, (POOL, numCoeff)).astype(np.int16)
    for k in range(POOL):
        if k % 5 == 1:
            pool[k] = 32767
        elif k % 5 == 2:
            pool[k] = -32768
        elif k % 5 == 3:
            pool[k, rng.random(numCoeff) < 0.8] = 0                  # sparse: numSig far from numCoeff
    qc = rng.integers(1, 65024, numCoeff).astype(np.int32)          # |coef| * qc + add (< 2^24) stays below 2^31
    sel = np.arange(n) % POOL
    for qbits in (14 + int(rng.integers(0, 7)) + max(15 - depth - log2n, 0), int(rng.integers(8, 24))):
        add = int(rng.integers(0, 1 << (qbits - 1)))
        q_o = np.zeros((POOL, numCoeff), np.int16); du_o = np.zeros((POOL, numCoeff), np.int32); ns_o = np.zeros(POOL, np.uint32)
        for k in range(POOL):
            ns_o[k] = O.orc_quant(ptr(pool[k]), ptr(qc), ptr(du_o[k]), ptr(q_o[k]), qbits, add, numCoeff)
            if nquant:
                assert O.orc_nquant(ptr(pool[k]), ptr(qc), ptr(q_o[k]), qbits, add, numCoeff) == ns_o[k]
        G = 8
        coef = np.zeros(G + n * numCoeff, np.int16)
        coef[G:] = pool[sel].ravel()                                 # base 2 x G bytes past the allocation start
        want_q = guarded(2 * G + n * numCoeff, np.int16); want_q[G:G + n * numCoeff] = q_o[sel].ravel()
        want_du = guarded(2 * G + n * numCoeff, np.int32); want_du[G:G + n * numCoeff] = du_o[sel].ravel()
        want_ns = guarded(2 * G + n, np.uint32); want_ns[G:G + n] = ns_o[sel]
        dC, dQC = dev(coef), dev(qc)
        dQ, dDU, dNS = dev(guarded(want_q.size, np.int16)), dev(guarded(want_du.size, np.int32)), dev(guarded(want_ns.size, np.uint32))
        cu.check(cu.L.x265cu_quant_batch(cu.ctx, dC.at(G), dQC.at(), dDU.at(G) if withDeltaU else None, dQ.at(G), qbits, add,
                                         numCoeff, n, nquant, dNS.at(G)))
        what = "numCoeff %d qBits %d" % (numCoeff, qbits)
        check_guarded(dQ.get(), want_q, span_mask(want_q.size, G, G + n * numCoeff), what + " qCoef")
        check_guarded(dNS.get(), want_ns, span_mask(want_ns.size, G, G + n), what + " numSig")
        if withDeltaU:
            check_guarded(dDU.get(), want_du, span_mask(want_du.size, G, G + n * numCoeff), what + " deltaU")
        else:
            assert (dDU.get() == sentinel(np.int32)).all(), what + ": deltaU written although NULL was passed"


@pytest.mark.parametrize("depth", DEPTHS)
def test_dequant_normal_batch(cu, dev, sms, depth):
    """num past one grid (16 x SMs CTAs of 256, x265cu.cu:159) and not a multiple of 256; int16 extremes in."""
    O = load_oracle(depth)
    rng = np.random.default_rng(77 + depth)
    num = 2 * 16 * 256 * sms + 77
    q = rng.integers(-32768, 32768, num + 16).astype(np.int16)
    q[8:200] = 32767; q[200:400] = -32768
    for scale, shift in ((int(rng.integers(1, 32768)), int(rng.integers(1, 11))), (40 << 4, 6 - max(15 - depth - 5, 0) + 1), (32767, 1)):
        want = guarded(num + 16, np.int16)
        O.orc_dequant_normal(ptr(q, 8), ptr(want, 8), num, scale, shift)
        dQ, dC = dev(q), dev(guarded(num + 16, np.int16))
        cu.check(cu.L.x265cu_dequant_normal_batch(cu.ctx, dQ.at(8), dC.at(8), num, scale, shift))
        check_guarded(dC.get(), want, span_mask(want.size, 8, 8 + num), "scale %d shift %d" % (scale, shift))


@pytest.mark.parametrize("depth", DEPTHS)
@pytest.mark.parametrize("numCoeff", [16, 64, 256, 1024])
def test_dequant_scaling_batch(cu, dev, sms, depth, numCoeff):
    """dq[i % numCoeff] across TUs; per 0 / 3 / 9 with shifts on both sides of `shift + 4 > per` (transform.cuh:366-372);
    total past one grid.  dq reaches scaling-list magnitudes (up to 2^15), and per 9 with shift 0 / 1 shifts q * dq past 2^31,
    where the clip before the shift decides the result."""
    O = load_oracle(depth)
    rng = np.random.default_rng(300 + numCoeff + depth)
    n = (2 * 16 * 256 * sms) // numCoeff + 3
    pool = rng.integers(-32768, 32768, (POOL, numCoeff)).astype(np.int16)
    pool[1] = 32767; pool[2] = -32768
    dq = rng.integers(1, 1 << 15, numCoeff).astype(np.int32)
    dq[:4] = (1 << 15) - 1
    sel = np.arange(n) % POOL
    G = 8
    q = np.zeros(G + n * numCoeff, np.int16); q[G:] = pool[sel].ravel()
    dQ, dDQ = dev(q), dev(dq)
    for per, shift in ((0, 1), (0, int(rng.integers(2, 8))), (3, 0), (3, 5), (9, 0), (9, 1), (9, 2), (9, 5), (9, 6), (9, 8)):
        out = np.zeros((POOL, numCoeff), np.int16)
        for k in range(POOL):
            O.orc_dequant_scaling(ptr(pool[k]), ptr(dq), ptr(out[k]), numCoeff, per, shift)
        want = guarded(2 * G + n * numCoeff, np.int16); want[G:G + n * numCoeff] = out[sel].ravel()
        dC = dev(guarded(want.size, np.int16))
        cu.check(cu.L.x265cu_dequant_scaling_batch(cu.ctx, dQ.at(G), dDQ.at(), dC.at(G), numCoeff, n, per, shift))
        check_guarded(dC.get(), want, span_mask(want.size, G, G + n * numCoeff), "per %d shift %d" % (per, shift))


# ---------------------------------------------------------------------------------------------------------------------
# block ops (x265cu_blockop_batch)
AW, AH = 168, 72                      # source planes (AW % 8 == 0: row starts at 8-element multiples are vector-aligned)
SQUARE_OPS = ("transpose", "blockfill_s", "cpy2Dto1D_shl", "cpy2Dto1D_shr", "cpy1Dto2D_shl", "cpy1Dto2D_shr")


def _blk_sources(rng, depth):
    mx = (1 << depth) - 1
    pix = rng.integers(0, mx + 1, (AH, AW)).astype(pixel_dtype(depth))
    pix[3] = 0; pix[4] = mx; pix[5, ::2] = mx; pix[5, 1::2] = 0
    s16 = rng.integers(-32768, 32768, (AH, AW)).astype(np.int16)
    s16[3] = 32767; s16[4] = -32768; s16[5, ::2] = 32767; s16[5, 1::2] = -32768
    valid = rng.integers(0, mx + 1, (AH, AW)).astype(np.int16)       # copy_sp takes pixel values only
    valid[3] = mx; valid[4] = 0
    return pix.ravel(), s16.ravel(), valid.ravel()


def _blk_jobs(rng, op, depth, n):
    """n jobs cycling through: vector-eligible / w % 8 == 0 with one misaligned offset or stride / w % 8 != 0 / vector-eligible.
    Returns the job array, the destination size and each job's destination (offset, row pitch, rows, cols)."""
    jobs = np.zeros(n, BLK_JOB)
    ops_b = BLK_TYPES[op][2] != "-"
    cursor, places = 16, []
    corr = 14 - depth
    for k in range(n):
        cls = k % 4
        if op == "scale2D_64to32":
            w = h = 32
        elif op in SQUARE_OPS:
            w = h = 4 if cls == 2 else (8, 16, 32)[k % 3]
        elif cls == 2:
            w, h = [(4, 4), (12, 16), (6, 2), (2, 8), (20, 3), (4, 8), (1, 5)][k % 7]
        else:
            w, h = [(8, 4), (16, 4), (8, 8), (16, 16), (32, 8), (64, 2), (24, 3), (32, 32), (8, 1)][k % 9]
        rows_a = 2 * h if op == "scale2D_64to32" else h
        cols_a = 2 * w if op == "scale2D_64to32" else w
        a_stride = b_stride = AW
        d_stride = w + (0, 8, 16)[k % 3]
        mis = (k // 4) % 5 if cls == 1 else -1                       # which operand the misaligned job breaks
        if mis == 3:
            d_stride = w + 1 + 2 * (k % 3)
        if mis == 4:
            a_stride = AW - 1
        ar, ac = int(rng.integers(0, AH - rows_a + 1)), 8 * int(rng.integers(0, (AW - 4 - cols_a) // 8 + 1))
        br, bc = int(rng.integers(0, AH - h + 1)), 8 * int(rng.integers(0, (AW - 4 - w) // 8 + 1))
        a_off = ar * a_stride + ac + (1 if mis == 1 else 0)
        b_off = br * b_stride + bc + (1 if (mis == 2 and ops_b) else 0)
        if mis == 2 and not ops_b:
            a_off += 3
        if cls == 2:
            a_off += int(rng.integers(0, 3))
        pitch = 32 if op == "scale2D_64to32" else (w if op == "transpose" else d_stride)
        cursor = (cursor + 7) // 8 * 8
        d_off = cursor + (1 if mis == 0 else 0) + (int(rng.integers(0, 3)) if cls == 2 else 0)
        p = [0, 0, 0, 0]
        if op == "blockfill_s":
            p[0] = [-32768, 32767, int(rng.integers(-32768, 32768))][k % 3]
        elif op.startswith("cpy"):
            p[0] = int(rng.integers(1, 8))
        elif op in ("weight_pp", "weight_sp"):
            sh = corr + int(rng.integers(1, 7))
            p = [int(rng.integers(0, 128)), 1 << (sh - 1), sh, int(rng.integers(-128, 128)) << (depth - 8)]
        elif op == "dequant_normal":
            p = [int(rng.integers(1, 32768)), int(rng.integers(1, 11)), 0, 0]
        jobs[k] = (d_off, a_off, b_off, d_stride, a_stride, b_stride, w, h, *p)
        places.append((d_off, pitch, h, w))
        cursor = d_off + h * max(pitch, d_stride) + 5               # room for h rows at either pitch, then a gap
        assert a_off + (rows_a - 1) * a_stride + cols_a <= AW * AH and b_off + (h - 1) * b_stride + w <= AW * AH
    return jobs, cursor + 16, places


def _blk_oracle(O, op, jb, A, B, want):
    w, h = int(jb["w"]), int(jb["h"])
    do, ao, bo = int(jb["d_off"]), int(jb["a_off"]), int(jb["b_off"])
    ds, sa, sb = IP(int(jb["d_stride"])), IP(int(jb["a_stride"])), IP(int(jb["b_stride"]))
    p0, p1, p2, p3 = (int(jb[f]) for f in ("p0", "p1", "p2", "p3"))
    pd, pa, pb = ptr(want, do), ptr(A, ao), ptr(B, bo) if B is not None else None
    if op in ("copy_pp", "copy_ss", "copy_sp", "copy_ps"):
        getattr(O, "orc_" + op)(pd, ds, pa, sa, w, h)
    elif op == "sub_ps":
        O.orc_sub_ps(pd, ds, pa, pb, sa, sb, w, h)
    elif op == "add_ps":
        O.orc_add_ps(pd, ds, pa, pb, sa, sb, w, h)
    elif op == "pixelavg_pp":
        O.orc_pixelavg_pp(pd, ds, pa, sa, pb, sb, w, h)
    elif op == "addAvg":
        O.orc_addAvg(pa, pb, pd, sa, sb, ds, w, h)
    elif op == "p2s":
        O.orc_p2s(pa, sa, pd, ds, w, h)
    elif op == "transpose":
        O.orc_transpose(pd, pa, sa, w)                             # destination rows w apart whatever d_stride says (blockops.cuh:34)
    elif op == "blockfill_s":
        O.orc_blockfill_s(pd, ds, C.c_int16(p0), w)
    elif op.startswith("cpy2Dto1D"):
        tmp = np.zeros(w * w, np.int16)                            # the primitive's 1-D side is compact; the job places its rows
        getattr(O, "orc_" + op)(ptr(tmp), pa, sa, p0, w)
        want[rect_index(do, int(jb["d_stride"]), w, w)[0]] = tmp.reshape(w, w)
    elif op.startswith("cpy1Dto2D"):
        tmp = np.ascontiguousarray(A[rect_index(ao, int(jb["a_stride"]), w, w)[0]])
        getattr(O, "orc_" + op)(pd, ptr(tmp), ds, p0, w)
    elif op == "weight_pp":                                        # one stride for both planes: a call per row
        for y in range(h):
            O.orc_weight_pp(ptr(A, ao + y * int(jb["a_stride"])), ptr(want, do + y * int(jb["d_stride"])), IP(0), w, 1, p0, p1, p2, p3)
    elif op == "weight_sp":
        O.orc_weight_sp(pa, pd, sa, ds, w, h, p0, p1, p2, p3)
    elif op == "scale2D_64to32":
        O.orc_scale2D_64to32(pd, pa, sa)                           # destination rows 32 apart (blockops.cuh:51)
    elif op == "dequant_normal":
        for y in range(h):
            O.orc_dequant_normal(ptr(A, ao + y * int(jb["a_stride"])), ptr(want, do + y * int(jb["d_stride"])), w, p0, p1)
    else:
        raise AssertionError(op)


@pytest.mark.parametrize("depth", DEPTHS)
@pytest.mark.parametrize("op", list(OPS_BLK))
def test_blockop_batch_paths(cu, dev, sms, depth, op):
    """One list per op mixing vector-eligible jobs, w % 8 == 0 jobs with a misaligned d / a / b offset or stride, w % 8 != 0
    jobs, and more jobs than the 16 x SMs CTAs of one launch."""
    O = load_oracle(depth)
    rng = np.random.default_rng(500 + OPS_BLK[op] + 50 * depth)
    n = 16 * sms + 101
    jobs, dsize, places = _blk_jobs(rng, op, depth, n)
    pix, s16, valid = _blk_sources(rng, depth)
    t_d, t_a, t_b = BLK_TYPES[op]
    A = valid if op == "copy_sp" else (pix if t_a == "p" else s16)
    B = None if t_b == "-" else (pix if t_b == "p" else s16)
    ddt = pixel_dtype(depth) if t_d == "p" else np.int16
    want = guarded(dsize, ddt)
    for jb in jobs:
        _blk_oracle(O, op, jb, A, B, want)
    dA, dB, dJ = dev(A), dev(B if B is not None else np.zeros(8, np.int16)), dev(jobs)
    dD = dev(guarded(dsize, ddt))
    seen = {blockop_path(depth, op, jb, dD.at(), dA.at(), dB.at()) for jb in jobs}
    assert "blockop_scalar" in seen and (op in BLK_SCALAR_ONLY or "blockop_vector" in seen), seen
    cu.check(cu.L.x265cu_blockop_batch(cu.ctx, depth, OPS_BLK[op], dD.at(), dA.at(), dB.at() if B is not None else None, dJ.at(), n))
    written = np.zeros(dsize, bool)
    for (o, p, h, w) in places:
        written[rect_index(o, p, h, w).ravel()] = True
    check_guarded(dD.get(), want, written, op)


# ---------------------------------------------------------------------------------------------------------------------
# intra
def _nb_arrays(rng, depth, count, nbp):
    mx = (1 << depth) - 1
    nb = rng.integers(0, mx + 1, (count, nbp)).astype(pixel_dtype(depth))
    nb[1::7] = mx
    nb[2::7] = 0
    nb[3::7, ::2] = mx
    nb[3::7, 1::2] = 0
    return nb


@pytest.mark.parametrize("depth", DEPTHS)
@pytest.mark.parametrize("N", [4, 8, 16, 32])
def test_intra_pred_batch(cu, dev, sms, depth, N):
    """All 35 modes x bFilter in one list of more than 8 x SMs jobs (x265cu.cu:181), padded neighbour pitch, dst_stride and
    dst_pitch."""
    O = load_oracle(depth)
    rng = np.random.default_rng(600 + N + depth)
    dt = pixel_dtype(depth)
    n = 8 * sms + 141
    nbp = 4 * N + 1 + 6
    nb = _nb_arrays(rng, depth, n, nbp)
    stride, pitch, off = N + 3, (N + 3) * N + 5, 7
    jobs = np.zeros(n, INTRA_JOB)
    jobs["mode"] = np.arange(n) % 35
    jobs["bFilter"] = (np.arange(n) // 35) % 2
    size = off + (n - 1) * pitch + (N - 1) * stride + N + 9
    want = guarded(size, dt)
    for j in range(n):
        O.orc_intra_pred(ptr(want, off + j * pitch), IP(stride), ptr(nb, j * nbp), int(jobs["mode"][j]), int(jobs["bFilter"][j]), N)
    dNB, dJ, dD = dev(nb), dev(jobs), dev(guarded(size, dt))
    cu.check(cu.L.x265cu_intra_pred_batch(cu.ctx, depth, N, dNB.at(), nbp, dD.at(off), pitch, stride, dJ.at(), n))
    check_guarded(dD.get(), want, mask_of(size, rect_index(off, stride, N, N, pitch, n)), "N=%d" % N)


ALLANGS_CASES = [("packed", 0), ("cta", 8), ("generic", 1)]      # dst offset: 0, 8 bytes, 1 element


@pytest.mark.parametrize("depth", DEPTHS)
@pytest.mark.parametrize("N", [4, 8, 16, 32])
@pytest.mark.parametrize("kernel", [c[0] for c in ALLANGS_CASES])
def test_intra_allangs_batch_paths(cu, dev, sms, depth, N, kernel):
    """The three all-angs kernels by destination alignment, bLuma 0 and 1, with more jobs than each kernel's grid: 8 x SMs
    (packed), 16 x SMs (cta), grid.y = 4096 (generic)."""
    O = load_oracle(depth)
    rng = np.random.default_rng(700 + N + depth + len(kernel))
    dt = pixel_dtype(depth)
    es = np.dtype(dt).itemsize
    off = {"packed": 0, "cta": 8 // es, "generic": 1}[kernel]
    n = {"packed": 8 * sms, "cta": 16 * sms, "generic": 4096}[kernel] + 67
    nbp = 4 * N + 1 + 3
    pool = _nb_arrays(rng, depth, POOL, nbp)
    fpool = np.zeros_like(pool)
    for k in range(POOL):
        O.orc_intra_filter(ptr(pool[k]), ptr(fpool[k]), N)
    sel = np.arange(n) % POOL
    dNB, dF = dev(pool[sel]), dev(fpool[sel])
    blk = 33 * N * N
    size = off + n * blk + 32
    for bLuma in (0, 1):
        out = np.zeros((POOL, blk), dt)
        for k in range(POOL):
            O.orc_intra_pred_allangs(ptr(out[k]), ptr(pool[k]), ptr(fpool[k]), bLuma, N)
        want = guarded(size, dt)
        want[off:off + n * blk] = out[sel].ravel()
        dD = dev(guarded(size, dt))
        kern, path = allangs_path(depth, N, dD.at(off))
        assert path == "allangs_" + kernel, (kern, path)
        cu.check(cu.L.x265cu_intra_allangs_batch(cu.ctx, depth, N, dNB.at(), dF.at(), nbp, dD.at(off), bLuma, n))
        check_guarded(dD.get(), want, span_mask(size, off, off + n * blk), "%s bLuma %d" % (kernel, bLuma))


# ---------------------------------------------------------------------------------------------------------------------
# lowres and borders
LOWRES_CASES = [("fast", 200, 0), ("odd-width", 203, 0), ("width-mod8-4", 196, 0), ("src-misaligned", 200, 1)]


@pytest.mark.parametrize("depth", DEPTHS)
@pytest.mark.parametrize("case", LOWRES_CASES, ids=[c[0] for c in LOWRES_CASES])
def test_frame_init_lowres_paths(cu, dev, depth, case):
    """x265cu_frame_init_lowres with margins, so the one 4-plane border launch runs: the oracle's frame_init_lowres plus its
    extendPicBorder on each plane; margin rows copy whole strides, padding included."""
    name, width, soff = case
    O = load_oracle(depth)
    rng = np.random.default_rng(800 + width + soff + depth)
    dt = pixel_dtype(depth)
    height, mx, my = 37, 16, 11
    sstride, dstride = 448, 256                                    # dstride > width + 2 * mx: padding columns exist
    src = rng.integers(0, 1 << depth, soff + (2 * height + 2) * sstride).astype(dt)
    G = 64                                                          # guard elements before the top margin row and after the last row
    origin = G + my * dstride + mx
    size = origin + (height + my) * dstride + G
    planes = [guarded(size, dt) for _ in range(4)]
    O.orc_frame_init_lowres(ptr(src, soff), *[ptr(p, origin) for p in planes], IP(sstride), IP(dstride), width, height)
    for p in planes:
        O.orc_extend_pic_border(ptr(p, origin), IP(dstride), width, height, mx, my)
    dS = dev(src)
    dP = [dev(guarded(size, dt)) for _ in range(4)]
    kern, path = lowres_path(depth, width, dS.at(soff), sstride, [d.at(origin) for d in dP], dstride)
    assert path == ("lowres_fast" if name == "fast" or (name == "width-mod8-4" and depth == 10) else "lowres_generic"), (name, kern)
    cu.check(cu.L.x265cu_frame_init_lowres(cu.ctx, depth, dS.at(soff), sstride, *[d.at(origin) for d in dP], dstride, width, height, mx, my))
    written = mask_of(size, rect_index(origin - my * dstride - mx, dstride, height + 2 * my, width + 2 * mx))
    written[origin - my * dstride - mx:origin - mx] = True            # top margin rows: whole strides
    written[origin + height * dstride - mx:origin + (height + my) * dstride - mx] = True
    for k, (d, p) in enumerate(zip(dP, planes)):
        check_guarded(d.get(), p, written, "%s plane %d" % (name, k))


@pytest.mark.parametrize("depth", DEPTHS)
def test_extend_border_padding(cu, dev, depth):
    """x265cu_extend_border alone: odd width and height, stride > width + 2 * mx.  The margin rows are whole-stride copies of
    the first / last row from column -mx (pixel.cpp:1027-1041), so their padding columns take that row's padding."""
    O = load_oracle(depth)
    rng = np.random.default_rng(900 + depth)
    dt = pixel_dtype(depth)
    width, height, mx, my, stride = 77, 45, 13, 9, 115
    assert stride > width + 2 * mx
    G = 40
    origin = G + my * stride + mx
    size = origin + (height + my) * stride + G
    plane = rng.integers(0, 1 << depth, size).astype(dt)
    want = plane.copy()
    O.orc_extend_pic_border(ptr(want, origin), IP(stride), width, height, mx, my)
    dP = dev(plane)
    cu.check(cu.L.x265cu_extend_border(cu.ctx, depth, dP.at(origin), stride, width, height, mx, my))
    got = dP.get()
    np.testing.assert_array_equal(got, want)
    pad = slice(width + 2 * mx, stride)                             # padding columns width + mx .. stride - mx, counted from column -mx
    rows = got[origin - my * stride - mx:origin + (height + my) * stride - mx].reshape(height + 2 * my, stride)
    src_rows = plane[origin - mx:origin + height * stride - mx].reshape(height, stride)
    for y in range(my):
        np.testing.assert_array_equal(rows[y, pad], src_rows[0, pad], err_msg="top margin row %d padding" % y)
        np.testing.assert_array_equal(rows[my + height + y, pad], src_rows[-1, pad], err_msg="bottom margin row %d padding" % y)
    assert not np.array_equal(src_rows[0, pad], src_rows[1, pad])   # the rows' paddings differ, so the check sees which one was copied


# ---------------------------------------------------------------------------------------------------------------------
def test_propagate_cost_batch(cu, dev, sms):
    """Past one grid (16 x SMs CTAs of 256, x265cu.cu:392) with an odd tail, intraCost == 0 entries (0 / 0 -> INT_MIN) included.
    The entry point takes no bit depth: lowres costs are depth-independent."""
    O = load_oracle(8)
    rng = np.random.default_rng(1100)
    n = 2 * 16 * 256 * sms + 77
    pin = rng.integers(0, 65536, n).astype(np.uint16)
    intra = rng.integers(0, 1 << 15, n).astype(np.int32)
    intra[::97] = 0
    inter = rng.integers(0, 65536, n).astype(np.uint16)
    inter[::89] = 0
    invq = rng.integers(1, 1024, n).astype(np.int32)
    G = 8
    for fps in (256.0 * 0.34, 256.0):
        want = guarded(n + 2 * G, np.int32)
        O.orc_propagate_cost(ptr(want, G), ptr(pin), ptr(intra), ptr(inter), ptr(invq), ptr(np.array([fps])), n)
        dD = dev(guarded(n + 2 * G, np.int32))
        d = [dev(x) for x in (pin, intra, inter, invq)]
        cu.check(cu.L.x265cu_propagate_cost_batch(cu.ctx, dD.at(G), *[x.at() for x in d], C.c_double(fps), n))
        check_guarded(dD.get(), want, span_mask(want.size, G, G + n), "fps %g" % fps)
        assert (want[G:G + n] == np.iinfo(np.int32).min).any()


# ---------------------------------------------------------------------------------------------------------------------
# 4-tap (chroma) interpolation jobs
CHROMA_PU = sorted({(w // 2, h // 2) for (w, h) in LUMA_PU[1:]})   # the 4:2:0 chroma blocks of the inter luma PUs


@pytest.mark.parametrize("depth", DEPTHS)
@pytest.mark.parametrize("op", ["hpp", "hps", "vpp", "vps", "vsp", "vss"])
@pytest.mark.parametrize("mix", ["chroma", "mixed"])
def test_interp_batch_chroma(cu, dev, depth, op, mix):
    """ntaps = 4 jobs, fractions 0-7, every 4:2:0 block size; alone, and interleaved with 8-tap jobs of both kernels'
    kinds (width % 8 == 0 for the row-segment kernel, 12 / 4 for the generic one) in one list."""
    O = load_oracle(depth)
    rng = np.random.default_rng(1200 + OPS_INTERP[op] + depth + len(mix))
    dt = pixel_dtype(depth)
    SW, SH, DW = 320, 200, 112
    short_src, short_dst = op in ("vsp", "vss"), op in ("hps", "vps", "vss")
    if short_src:
        src = rng.integers(-(1 << 13), 1 << 13, (SH, SW)).astype(np.int16)
        src[7] = 16383; src[8] = -16384
    else:
        src = rng.integers(0, 1 << depth, (SH, SW)).astype(dt)
        src[7] = (1 << depth) - 1; src[8] = 0
    ddt = np.int16 if short_dst else dt
    luma = [(8, 8), (16, 4), (64, 16), (12, 16), (4, 8), (24, 32)]
    jobs, places, y = [], [], 2
    for k, (w, h) in enumerate(CHROMA_PU * 2):
        entries = [(w, h, 4, k % 8)]
        if mix == "mixed":
            lw, lh = luma[k % len(luma)]
            entries.append((lw, lh, 8, k % 4))
        for (bw, bh, nt, frac) in entries:
            ext = 1 if (op == "hps" and k % 2) else 0
            rows = bh + (nt - 1 if ext else 0)
            sx, sy = 8 + int(rng.integers(0, SW - 88)), 8 + int(rng.integers(0, SH - 88))
            dx = 1 + int(rng.integers(0, 8))
            jobs.append((sy * SW + sx, y * DW + dx, SW, DW, bw, bh, frac, 0, ext, nt))
            places.append((y * DW + dx, rows, bw))
            y += rows + 1
    j = np.zeros(len(jobs), INTERP_JOB)
    for i, t in enumerate(jobs):
        j[i] = t
    size = (y + 2) * DW
    want = guarded(size, ddt)
    fn = getattr(O, "orc_interp_" + op)
    for (s_off, d_off, ss, ds, w, h, ix, _, ext, nt) in jobs:
        if op == "hps":
            fn(ptr(src, s_off), IP(ss), ptr(want, d_off), IP(ds), ix, ext, nt, w, h)
        else:
            fn(ptr(src, s_off), IP(ss), ptr(want, d_off), IP(ds), ix, nt, w, h)
    kernels = {interp_kernel(depth, op, jb) for jb in j}
    assert "k_interp<%s>" % _ctype(depth) in kernels
    assert (j["ntaps"] == 4).any() and ((j["ntaps"] == 8).any() == (mix == "mixed"))
    dS, dD, dJ = dev(src), dev(guarded(size, ddt)), dev(j)
    cu.check(cu.L.x265cu_interp_batch(cu.ctx, depth, OPS_INTERP[op], dS.at(), dD.at(), dJ.at(), len(jobs)))
    written = np.zeros(size, bool)
    for (o, rows, w) in places:
        written[rect_index(o, DW, rows, w).ravel()] = True
    check_guarded(dD.get(), want, written, "%s %s" % (op, mix))


# ---------------------------------------------------------------------------------------------------------------------
def _targets():
    """the path every case of this file names"""
    t = {c[-1] for c in TRANSFORM_CASES}
    t |= {"quant", "dequant_normal", "dequant_scaling", "blockop_vector", "blockop_scalar", "blockop_any_op", "blockop_trips",
          "intra_pred", "lowres_fast", "lowres_generic", "extend_padding", "propagate_trips", "interp_4tap"}
    t |= {"allangs_" + c[0] for c in ALLANGS_CASES}
    return t


def test_every_path_is_targeted():
    assert _targets() == set(PATHS), (set(PATHS) - _targets(), _targets() - set(PATHS))
    assert any(op not in BLK_HOT for op in OPS_BLK)                # blockop_any_op: some op runs on k_blockop<P, -1>


def _kernel_names(run):
    """names of the device kernels `run` launches, from torch.profiler"""
    import torch
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    names = set()
    for e in prof.events():
        if str(getattr(e, "device_type", "")).endswith("CUDA") and e.name:
            names.add(e.name)
    return names


def _probes(cu, dev, sms, depth):
    """(kernel the mirror predicts, a small launch) for each branch whose choice shows in the kernel's name"""
    dt = pixel_dtype(depth)
    es = np.dtype(dt).itemsize
    buf, out = dev(np.zeros(1 << 16, np.int16)), dev(np.zeros(1 << 16, np.int16))
    probes = []

    def transform(op, N, soff, doff, stride, pitch):
        return lambda: cu.check(cu.L.x265cu_transform_batch(cu.ctx, depth, op, N, buf.at(soff), out.at(doff), stride, pitch, 4))
    for (op, N, soff, doff, stride, pitch) in ((IDCT, 16, 0, 0, 16, 256), (IDCT, 32, 4, 1, 33, 33 * 32), (DCT, 32, 4, 2, 40, 40 * 32),
                                               (DCT, 16, 1, 0, 16, 256), (IDST4, 4, 0, 0, 4, 16), (DCT, 4, 0, 0, 4, 16), (IDCT, 8, 0, 1, 8, 64)):
        probes.append((transform_path(depth, op, N, buf.at(soff), out.at(doff), stride, pitch, 4, sms)[0],
                       transform(op, N, soff, doff, stride, pitch)))
    nb, dst = dev(np.zeros(4 * 129, dt)), dev(np.zeros(2 * 33 * 16 * 16 + 64, dt))

    def allangs(N, off):
        return lambda: cu.check(cu.L.x265cu_intra_allangs_batch(cu.ctx, depth, N, nb.at(), nb.at(2 * 129), 129, dst.at(off), 1, 2))
    for N in (8, 16):
        for off in (0, 8 // es, 1):
            probes.append((allangs_path(depth, N, dst.at(off))[0], allangs(N, off)))
    src, pl = dev(np.zeros(8 * 448 + 16, dt)), [dev(np.zeros(64 * 32, dt)) for _ in range(4)]

    def lowres(w, so):
        return lambda: cu.check(cu.L.x265cu_frame_init_lowres(cu.ctx, depth, src.at(so), 448, *[p.at() for p in pl], 80, w, 2, 0, 0))
    for (w, so) in ((64, 0), (60, 0), (64, 1)):
        probes.append((lowres_path(depth, w, src.at(so), 448, [p.at() for p in pl], 80)[0], lowres(w, so)))
    jb = np.zeros(1, BLK_JOB)
    jb[0] = (0, 0, 0, 8, 8, 8, 8, 2, 1, 0, 1, 0)
    dj = dev(jb)

    def blockop(op):
        return lambda: cu.check(cu.L.x265cu_blockop_batch(cu.ctx, depth, OPS_BLK[op], out.at(), buf.at(), buf.at(), dj.at(), 1))
    for op in ("sub_ps", "weight_pp", "transpose"):
        probes.append((blockop_kernel(depth, op), blockop(op)))
    ij = np.zeros(2, INTERP_JOB)
    ij[0] = (8 * 64 + 8, 0, 64, 64, 8, 4, 1, 0, 0, 4)
    ij[1] = (8 * 64 + 8, 8 * 64, 64, 64, 8, 4, 1, 0, 0, 8)
    dij, isrc = dev(ij), dev(np.zeros(32 * 64, dt))
    run = lambda: cu.check(cu.L.x265cu_interp_batch(cu.ctx, depth, OPS_INTERP["hpp"], isrc.at(), out.at(), dij.at(), 2))
    for k in range(2):
        probes.append((interp_kernel(depth, "hpp", ij[k]), run))
    return probes


def test_dispatch_kernel_names(cu, dev, sms):
    """The mirrors above agree with the kernels the library launches: one small launch per branch whose choice shows in the
    kernel's name, checked against torch.profiler's record of the launch."""
    probes = _probes(cu, dev, sms, 8) + _probes(cu, dev, sms, 10)
    recorded = [(kern, _kernel_names(run)) for kern, run in probes]
    if not any(names for _, names in recorded):
        pytest.skip("torch.profiler recorded no kernel events on this host")
    missing = [(kern, sorted(names)) for kern, names in recorded if not any((" " + kern + "(") in (" " + nm) for nm in names)]
    assert not missing, missing
