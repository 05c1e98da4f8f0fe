// x265_b200/csrc/blockops.cuh -- elementwise block-op class.
// Semantics: /root/reference/source/common/pixel.cpp:393-491 (blockfill, cpy1D/2D, residual,
// transpose), :493-557 (weight, pixelavg), :584-602 (scale2D), :759-862 (copies, sub_ps, add_ps,
// addAvg), ipfilter.cpp:40-57 (p2s), dct.cpp:612-634 (dequant_normal).
#pragma once
#include "common.cuh"

template <typename P>
__device__ __forceinline__ void blockop_elem(int op, const x265cu_blk_job& jb, void* __restrict__ D, const void* __restrict__ A,
                                             const void* __restrict__ Bv, int x, int y)
{
    constexpr int depth = PixTraits<P>::depth;
    constexpr int maxv = PixTraits<P>::maxv;
    const int64_t di = jb.d_off + (int64_t)y * jb.d_stride + x;
    const int64_t ai = jb.a_off + (int64_t)y * jb.a_stride + x;
    const int64_t bi = jb.b_off + (int64_t)y * jb.b_stride + x;
    switch (op)
    {
    case X265CU_COPY_PP: ((P*)D)[di] = ((const P*)A)[ai]; break;
    case X265CU_COPY_SS: ((int16_t*)D)[di] = ((const int16_t*)A)[ai]; break;
    case X265CU_COPY_SP: ((P*)D)[di] = (P)((const int16_t*)A)[ai]; break;
    case X265CU_COPY_PS: ((int16_t*)D)[di] = (int16_t)((const P*)A)[ai]; break;
    case X265CU_SUB_PS:  ((int16_t*)D)[di] = (int16_t)((int)((const P*)A)[ai] - (int)((const P*)Bv)[bi]); break;
    case X265CU_ADD_PS:  ((P*)D)[di] = (P)clip3i(0, maxv, (int)((const P*)A)[ai] + (int)((const int16_t*)Bv)[bi]); break;
    case X265CU_PIXELAVG_PP: ((P*)D)[di] = (P)(((int)((const P*)A)[ai] + (int)((const P*)Bv)[bi] + 1) >> 1); break;
    case X265CU_ADDAVG:
    {
        constexpr int shift = 14 + 1 - depth;
        constexpr int offset = (1 << (shift - 1)) + 2 * 8192;
        ((P*)D)[di] = (P)clip3i(0, maxv, ((int)((const int16_t*)A)[ai] + (int)((const int16_t*)Bv)[bi] + offset) >> shift);
        break;
    }
    case X265CU_P2S: ((int16_t*)D)[di] = (int16_t)((int)(int16_t)(((const P*)A)[ai] << (14 - depth)) - 8192); break;
    case X265CU_TRANSPOSE: ((P*)D)[jb.d_off + (int64_t)y * jb.w + x] = ((const P*)A)[jb.a_off + (int64_t)x * jb.a_stride + y]; break;
    case X265CU_BLOCKFILL_S: ((int16_t*)D)[di] = (int16_t)jb.p0; break;
    case X265CU_CPY2DTO1D_SHL: case X265CU_CPY1DTO2D_SHL:
        ((int16_t*)D)[di] = (int16_t)(((const int16_t*)A)[ai] << jb.p0); break;
    case X265CU_CPY2DTO1D_SHR: case X265CU_CPY1DTO2D_SHR:
        ((int16_t*)D)[di] = (int16_t)((((const int16_t*)A)[ai] + (int16_t)(1 << (jb.p0 - 1))) >> jb.p0); break;
    case X265CU_WEIGHT_PP:
    {
        int16_t v = (int16_t)(((const P*)A)[ai] << (14 - depth));
        ((P*)D)[di] = (P)clip3i(0, maxv, ((jb.p0 * v + jb.p1) >> jb.p2) + jb.p3);
        break;
    }
    case X265CU_WEIGHT_SP:
        ((P*)D)[di] = (P)clip3i(0, maxv, ((jb.p0 * (((const int16_t*)A)[ai] + 8192) + jb.p1) >> jb.p2) + jb.p3); break;
    case X265CU_SCALE2D_64TO32:
    {
        const P* p = (const P*)A + jb.a_off + (int64_t)(2 * y) * jb.a_stride + 2 * x;
        ((P*)D)[jb.d_off + y * 32 + x] = (P)((p[0] + p[1] + p[jb.a_stride] + p[jb.a_stride + 1] + 2) >> 2);
        break;
    }
    case X265CU_DEQUANT_NORMAL:
        ((int16_t*)D)[di] = (int16_t)clip16((((const int16_t*)A)[ai] * jb.p0 + (1 << (jb.p1 - 1))) >> jb.p1); break;
    }
}

// ---- vector path for the element-wise ops: a thread handles 8 consecutive elements of a row ---------------
// operand element kinds per op: 0 = none, 1 = pixel, 2 = int16
__device__ __forceinline__ void blockop_kinds(int op, int& kd, int& ka, int& kb)
{
    kd = ka = kb = 0;
    switch (op)
    {
    case X265CU_COPY_PP: kd = 1; ka = 1; break;
    case X265CU_COPY_SS: kd = 2; ka = 2; break;
    case X265CU_COPY_SP: kd = 1; ka = 2; break;
    case X265CU_COPY_PS: kd = 2; ka = 1; break;
    case X265CU_SUB_PS:  kd = 2; ka = 1; kb = 1; break;
    case X265CU_ADD_PS:  kd = 1; ka = 1; kb = 2; break;
    case X265CU_PIXELAVG_PP: kd = 1; ka = 1; kb = 1; break;
    case X265CU_ADDAVG:  kd = 1; ka = 2; kb = 2; break;
    case X265CU_P2S:     kd = 2; ka = 1; break;
    case X265CU_BLOCKFILL_S: kd = 2; break;
    case X265CU_CPY2DTO1D_SHL: case X265CU_CPY1DTO2D_SHL: case X265CU_CPY2DTO1D_SHR: case X265CU_CPY1DTO2D_SHR:
    case X265CU_DEQUANT_NORMAL: kd = 2; ka = 2; break;
    case X265CU_WEIGHT_PP: kd = 1; ka = 1; break;
    case X265CU_WEIGHT_SP: kd = 1; ka = 2; break;
    default: break;                                   // transpose / scale2D: not element-wise, scalar path only
    }
}

// the value an element-wise op writes for inputs a, b (same arithmetic as blockop_elem)
template <typename P>
__device__ __forceinline__ int blockop_value(int op, const x265cu_blk_job& jb, int a, int b)
{
    constexpr int depth = PixTraits<P>::depth;
    constexpr int maxv = PixTraits<P>::maxv;
    switch (op)
    {
    case X265CU_SUB_PS:  return (int)(int16_t)(a - b);
    case X265CU_ADD_PS:  return clip3i(0, maxv, a + b);
    case X265CU_PIXELAVG_PP: return (a + b + 1) >> 1;
    case X265CU_ADDAVG:
    {
        constexpr int shift = 14 + 1 - depth;
        constexpr int offset = (1 << (shift - 1)) + 2 * 8192;
        return clip3i(0, maxv, (a + b + offset) >> shift);
    }
    case X265CU_P2S: return (int)(int16_t)((int)(int16_t)(a << (14 - depth)) - 8192);
    case X265CU_BLOCKFILL_S: return (int)(int16_t)jb.p0;
    case X265CU_CPY2DTO1D_SHL: case X265CU_CPY1DTO2D_SHL: return (int)(int16_t)(a << jb.p0);
    case X265CU_CPY2DTO1D_SHR: case X265CU_CPY1DTO2D_SHR: return (int)(int16_t)((a + (int16_t)(1 << (jb.p0 - 1))) >> jb.p0);
    case X265CU_WEIGHT_PP: { int16_t v = (int16_t)(a << (14 - depth)); return clip3i(0, maxv, ((jb.p0 * v + jb.p1) >> jb.p2) + jb.p3); }
    case X265CU_WEIGHT_SP: return clip3i(0, maxv, ((jb.p0 * (a + 8192) + jb.p1) >> jb.p2) + jb.p3);
    case X265CU_DEQUANT_NORMAL: return (int)(int16_t)clip16((a * jb.p0 + (1 << (jb.p1 - 1))) >> jb.p1);
    default: return a;                                // the copies
    }
}

// 8 consecutive elements of `bytes`-wide type (1: u8, 2: u16 / int16 with `sgn`) at p, 8 x bytes aligned
__device__ __forceinline__ void blk_load8(const void* __restrict__ p, int bytes, bool sgn, int (&v)[8])
{
    if (bytes == 1)
    {
        const uint2 w = __ldg((const uint2*)p);
#pragma unroll
        for (int k = 0; k < 4; k++) { v[k] = (int)((w.x >> (8 * k)) & 255u); v[4 + k] = (int)((w.y >> (8 * k)) & 255u); }
    }
    else
    {
        const uint4 w = __ldg((const uint4*)p);
        const uint32_t ww[4] = { w.x, w.y, w.z, w.w };
#pragma unroll
        for (int k = 0; k < 4; k++)
        {
            v[2 * k]     = sgn ? (int)(int16_t)(ww[k] & 0xffffu) : (int)(ww[k] & 0xffffu);
            v[2 * k + 1] = sgn ? (int)(int16_t)(ww[k] >> 16) : (int)(ww[k] >> 16);
        }
    }
}
__device__ __forceinline__ void blk_store8(void* __restrict__ p, int bytes, const int (&v)[8])
{
    if (bytes == 1)
        *(uint2*)p = make_uint2((uint32_t)(v[0] & 255) | ((uint32_t)(v[1] & 255) << 8) | ((uint32_t)(v[2] & 255) << 16) | ((uint32_t)v[3] << 24),
                                (uint32_t)(v[4] & 255) | ((uint32_t)(v[5] & 255) << 8) | ((uint32_t)(v[6] & 255) << 16) | ((uint32_t)v[7] << 24));
    else
        *(uint4*)p = make_uint4(((uint32_t)v[0] & 0xffffu) | ((uint32_t)v[1] << 16), ((uint32_t)v[2] & 0xffffu) | ((uint32_t)v[3] << 16),
                                ((uint32_t)v[4] & 0xffffu) | ((uint32_t)v[5] << 16), ((uint32_t)v[6] & 0xffffu) | ((uint32_t)v[7] << 16));
}

// one block per job (grid-stride over jobs), threads stride over the w*h elements.  OPT >= 0: the operation as a compile-time
// constant (the hot element-wise ops get their own instantiation: with a run-time `op` the per-element switch of
// blockop_value survives in the unrolled loop); OPT = -1: any op.
template <typename P, int OPT>
__global__ void __launch_bounds__(256) k_blockop(int op_rt, void* __restrict__ D, const void* __restrict__ A, const void* __restrict__ B,
                                                 const x265cu_blk_job* __restrict__ jobs, int n)
{
    const int op = OPT >= 0 ? OPT : op_rt;
    for (int j = blockIdx.x; j < n; j += gridDim.x)
    {
        const x265cu_blk_job jb = jobs[j];
        const int w = jb.w, cnt = jb.w * jb.h;
        int kd, ka, kb;
        blockop_kinds(op, kd, ka, kb);
        if (kd && (w & 7) == 0)
        {
            // element sizes and the 8-element alignment of every operand row
            const int sd = kd == 1 ? (int)sizeof(P) : 2, sa = ka == 1 ? (int)sizeof(P) : 2, sb = kb == 1 ? (int)sizeof(P) : 2;
            const uintptr_t pd = (uintptr_t)D + (size_t)jb.d_off * sd, pa = (uintptr_t)A + (size_t)jb.a_off * sa, pb = (uintptr_t)B + (size_t)jb.b_off * sb;
            bool ok = ((pd | (uintptr_t)((size_t)jb.d_stride * sd)) & (8 * sd - 1)) == 0;
            if (ka) ok = ok && ((pa | (uintptr_t)((size_t)jb.a_stride * sa)) & (8 * sa - 1)) == 0;
            if (kb) ok = ok && ((pb | (uintptr_t)((size_t)jb.b_stride * sb)) & (8 * sb - 1)) == 0;
            if (ok)
            {
                const int upr = w >> 3;
                for (int u = threadIdx.x; u < upr * jb.h; u += blockDim.x)
                {
                    const int y = u / upr, x = (u - y * upr) * 8;
                    int a[8], b[8], v[8];
                    if (ka) blk_load8((const void*)(pa + ((size_t)y * jb.a_stride + x) * sa), sa, ka == 2, a);
                    if (kb) blk_load8((const void*)(pb + ((size_t)y * jb.b_stride + x) * sb), sb, kb == 2, b);
#pragma unroll
                    for (int k = 0; k < 8; k++) v[k] = blockop_value<P>(op, jb, ka ? a[k] : 0, kb ? b[k] : 0);
                    blk_store8((void*)(pd + ((size_t)y * jb.d_stride + x) * sd), sd, v);
                }
                continue;
            }
        }
        for (int i = threadIdx.x; i < cnt; i += blockDim.x)
        {
            int y = i / w, x = i - y * w;
            blockop_elem<P>(op, jb, D, A, B, x, y);
        }
    }
}

static int launch_blockop(x265cu_ctx* ctx, int depth, int op, void* D, const void* A, const void* B, const x265cu_blk_job* jobs, int n)
{
    if (n <= 0) return 0;
    int blocks = n < ctx->sm_count * 16 ? n : ctx->sm_count * 16;
#define BLK_LAUNCH(OPT) do { if (depth == 8) k_blockop<uint8_t, OPT><<<blocks, 256, 0, ctx->stream>>>(op, D, A, B, jobs, n); \
                             else            k_blockop<uint16_t, OPT><<<blocks, 256, 0, ctx->stream>>>(op, D, A, B, jobs, n); } while (0)
    switch (op)
    {
    case X265CU_SUB_PS:      BLK_LAUNCH(X265CU_SUB_PS); break;
    case X265CU_ADD_PS:      BLK_LAUNCH(X265CU_ADD_PS); break;
    case X265CU_PIXELAVG_PP: BLK_LAUNCH(X265CU_PIXELAVG_PP); break;
    case X265CU_ADDAVG:      BLK_LAUNCH(X265CU_ADDAVG); break;
    case X265CU_COPY_PP:     BLK_LAUNCH(X265CU_COPY_PP); break;
    case X265CU_COPY_SS:     BLK_LAUNCH(X265CU_COPY_SS); break;
    case X265CU_COPY_PS:     BLK_LAUNCH(X265CU_COPY_PS); break;
    case X265CU_COPY_SP:     BLK_LAUNCH(X265CU_COPY_SP); break;
    case X265CU_P2S:         BLK_LAUNCH(X265CU_P2S); break;
    default:                 BLK_LAUNCH(-1); break;
    }
#undef BLK_LAUNCH
    CU_LAUNCH_CHECK(ctx);
    return 0;
}

// ---- frame_init_lowres (pixel.cpp:604-628) + border extension (pixel.cpp:1027-1041) ---------
// Each thread produces 4 adjacent lowres pixels of all 4 planes from a 3x9 full-res window.
template <typename P>
__global__ void __launch_bounds__(256) k_lowres_init(const P* __restrict__ src, int sstride, P* __restrict__ d0, P* __restrict__ dh,
                                                     P* __restrict__ dv, P* __restrict__ dc, int dstride, int width, int height)
{
    const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x0 >= width || y >= height) return;
    const P* r0 = src + (int64_t)(2 * y) * sstride + 2 * x0;
    const P* r1 = r0 + sstride;
    const P* r2 = r1 + sstride;
    int a[9], b[9], c[9];
    const int nload = min(9, 2 * (width - x0) + 1);
#pragma unroll
    for (int i = 0; i < 9; i++)
    {
        int k = i < nload ? i : nload - 1;
        a[i] = r0[k]; b[i] = r1[k]; c[i] = r2[k];
    }
    // vertical pair averages: v01[i] = avg(r0,r1), v12[i] = avg(r1,r2)
    int v01[9], v12[9];
#pragma unroll
    for (int i = 0; i < 9; i++) { v01[i] = (a[i] + b[i] + 1) >> 1; v12[i] = (b[i] + c[i] + 1) >> 1; }
    const int nout = min(4, width - x0);
    const int64_t o = (int64_t)y * dstride + x0;
#pragma unroll
    for (int k = 0; k < 4; k++)
    {
        if (k < nout)
        {
            d0[o + k] = (P)((v01[2 * k] + v01[2 * k + 1] + 1) >> 1);
            dh[o + k] = (P)((v01[2 * k + 1] + v01[2 * k + 2] + 1) >> 1);
            dv[o + k] = (P)((v12[2 * k] + v12[2 * k + 1] + 1) >> 1);
            dc[o + k] = (P)((v12[2 * k + 1] + v12[2 * k + 2] + 1) >> 1);
        }
    }
}

// 8-bit fast path: a thread produces 8 adjacent lowres pixels of all 4 planes with packed-byte arithmetic: three
// 16-byte row loads (+ the 17th pixel), VAVGU4 (the reference's (a + b + 1) >> 1 on four bytes at once) for the
// vertical pairs, PRMT to split even / odd columns, VAVGU4 again, four 8-byte stores.
__global__ void __launch_bounds__(256) k_lowres_init_u8x8(const uint8_t* __restrict__ src, int sstride, uint8_t* __restrict__ d0, uint8_t* __restrict__ dh,
                                                          uint8_t* __restrict__ dv, uint8_t* __restrict__ dc, int dstride, int width8, int height)
{
    const int xu = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (xu >= width8 || y >= height) return;
    const uint8_t* r0 = src + (int64_t)(2 * y) * sstride + 16 * xu;
    const uint8_t* r1 = r0 + sstride;
    const uint8_t* r2 = r1 + sstride;
    const uint4 a = __ldg((const uint4*)r0), b = __ldg((const uint4*)r1), c = __ldg((const uint4*)r2);
    const uint32_t a16 = __ldg(r0 + 16), b16 = __ldg(r1 + 16), c16 = __ldg(r2 + 16);
    const uint32_t A[4] = { a.x, a.y, a.z, a.w }, B[4] = { b.x, b.y, b.z, b.w }, C4[4] = { c.x, c.y, c.z, c.w };
    uint32_t out[4][2];
#pragma unroll
    for (int half = 0; half < 2; half++)
    {
        uint32_t V[4];
#pragma unroll
        for (int i = 0; i < 4; i++) V[i] = half ? __vavgu4(B[i], C4[i]) : __vavgu4(A[i], B[i]);
        const uint32_t t = half ? (b16 + c16 + 1) >> 1 : (a16 + b16 + 1) >> 1;
        const uint32_t E0 = __byte_perm(V[0], V[1], 0x6420), O0 = __byte_perm(V[0], V[1], 0x7531);
        const uint32_t E1 = __byte_perm(V[2], V[3], 0x6420), O1 = __byte_perm(V[2], V[3], 0x7531);
        const uint32_t ES0 = __byte_perm(E0, E1, 0x4321), ES1 = __byte_perm(E1, t, 0x4321);
        out[2 * half][0] = __vavgu4(E0, O0);      out[2 * half][1] = __vavgu4(E1, O1);         // even/odd pair: columns 2k, 2k+1
        out[2 * half + 1][0] = __vavgu4(O0, ES0); out[2 * half + 1][1] = __vavgu4(O1, ES1);    // columns 2k+1, 2k+2
    }
    const int64_t o = (int64_t)y * dstride + 8 * xu;
    *(uint2*)(d0 + o) = make_uint2(out[0][0], out[0][1]);
    *(uint2*)(dh + o) = make_uint2(out[1][0], out[1][1]);
    *(uint2*)(dv + o) = make_uint2(out[2][0], out[2][1]);
    *(uint2*)(dc + o) = make_uint2(out[3][0], out[3][1]);
}

// 16-bit fast path (10 / 12-bit pixels): a thread produces 4 adjacent lowres pixels of all 4 planes on packed halfword pairs:
// (a + b + 1) >> 1 of two pixels per 32-bit add (no carry between the halves: sums stay below 2^13), PRMT for the
// even / odd column split, three 16-byte row loads (+ the ninth pixel), four 8-byte stores.
__device__ __forceinline__ uint32_t avg2_u16(uint32_t a, uint32_t b) { return ((a + b + 0x00010001u) >> 1) & 0x7fff7fffu; }
__global__ void __launch_bounds__(256) k_lowres_init_u16x4(const uint16_t* __restrict__ src, int sstride, uint16_t* __restrict__ d0, uint16_t* __restrict__ dh,
                                                           uint16_t* __restrict__ dv, uint16_t* __restrict__ dc, int dstride, int width4, int height)
{
    const int xu = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (xu >= width4 || y >= height) return;
    const uint16_t* r0 = src + (int64_t)(2 * y) * sstride + 8 * xu;
    const uint16_t* r1 = r0 + sstride;
    const uint16_t* r2 = r1 + sstride;
    const uint4 a = __ldg((const uint4*)r0), b = __ldg((const uint4*)r1), c = __ldg((const uint4*)r2);
    const uint32_t a8 = __ldg(r0 + 8), b8 = __ldg(r1 + 8), c8 = __ldg(r2 + 8);
    const uint32_t A[4] = { a.x, a.y, a.z, a.w }, B[4] = { b.x, b.y, b.z, b.w }, C4[4] = { c.x, c.y, c.z, c.w };
    uint32_t out[4][2];
#pragma unroll
    for (int half = 0; half < 2; half++)
    {
        uint32_t V[4];
#pragma unroll
        for (int i = 0; i < 4; i++) V[i] = half ? avg2_u16(B[i], C4[i]) : avg2_u16(A[i], B[i]);
        const uint32_t t = half ? (b8 + c8 + 1) >> 1 : (a8 + b8 + 1) >> 1;
        const uint32_t E0 = __byte_perm(V[0], V[1], 0x5410), O0 = __byte_perm(V[0], V[1], 0x7632);       // (v0, v2), (v1, v3)
        const uint32_t E1 = __byte_perm(V[2], V[3], 0x5410), O1 = __byte_perm(V[2], V[3], 0x7632);       // (v4, v6), (v5, v7)
        const uint32_t ES0 = __byte_perm(E0, E1, 0x5432), ES1 = __byte_perm(E1, t, 0x5432);              // (v2, v4), (v6, v8)
        out[2 * half][0] = avg2_u16(E0, O0);      out[2 * half][1] = avg2_u16(E1, O1);
        out[2 * half + 1][0] = avg2_u16(O0, ES0); out[2 * half + 1][1] = avg2_u16(O1, ES1);
    }
    const int64_t o = (int64_t)y * dstride + 4 * xu;
    *(uint2*)(d0 + o) = make_uint2(out[0][0], out[0][1]);
    *(uint2*)(dh + o) = make_uint2(out[1][0], out[1][1]);
    *(uint2*)(dv + o) = make_uint2(out[2][0], out[2][1]);
    *(uint2*)(dc + o) = make_uint2(out[3][0], out[3][1]);
}

// extendPicBorder (pixel.cpp:1027-1041) in ONE launch for up to four planes of the same geometry (round 1: a left/right
// and a top/bottom launch per plane, nine launches for a lowres init).  The reference replicates the edge pixels of every
// row, then copies `stride` elements of the (extended) first / last row into the margin rows; every output here is a pure
// function of the un-extended picture (margin rows read the source row and its two edge pixels directly), so the two
// passes need no ordering.  Block = one output row of one plane.
template <typename P> struct ExtPlanes { P* p[4]; };
template <typename P>
__global__ void __launch_bounds__(256) k_extend_border(ExtPlanes<P> pl, int stride, int width, int height, int mx, int my)
{
    // a WARP per output row (8 rows per CTA): a CTA per row meant 100 K tiny CTAs for a stacked batch of lowres planes
    P* pic = pl.p[blockIdx.y];
    const int lane = threadIdx.x & 31;
    const int r = (int)(blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) - my;      // output row: -my .. height + my - 1
    if (r >= height + my) return;
    const int sr = min(max(r, 0), height - 1);
    const P* srow = pic + (int64_t)sr * stride;
    P* drow = pic + (int64_t)r * stride;
    const P l = srow[0], rt = srow[width - 1];
    if (r == sr)
    {
        for (int x = lane; x < mx; x += 32) { drow[-mx + x] = l; drow[width + x] = rt; }
    }
    else
    {   // `stride` elements from column -mx: margins replicated, the row itself, and whatever padding follows (as memcpy does)
        for (int x = lane; x < stride; x += 32)
        {
            const int sx = x - mx;
            drow[sx] = sx < 0 ? l : sx < width ? srow[sx] : sx < width + mx ? rt : srow[sx];
        }
    }
}

template <typename P>
static int extend_border_n(x265cu_ctx* ctx, P* const* pics, int nplanes, int stride, int width, int height, int mx, int my)
{
    ExtPlanes<P> pl;
    for (int i = 0; i < 4; i++) pl.p[i] = pics[i < nplanes ? i : 0];
    k_extend_border<P><<<dim3((height + 2 * my + 7) / 8, nplanes), 256, 0, ctx->stream>>>(pl, stride, width, height, mx, my);
    CU_LAUNCH_CHECK(ctx);
    return 0;
}
template <typename P>
static int extend_border_t(x265cu_ctx* ctx, P* pic, int stride, int width, int height, int mx, int my)
{
    return extend_border_n<P>(ctx, &pic, 1, stride, width, height, mx, my);
}
