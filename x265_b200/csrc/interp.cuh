// x265_b200/csrc/interp.cuh -- sub-pel interpolation class (8-tap luma / 4-tap chroma).
// Semantics: /root/reference/source/common/ipfilter.cpp:79-118 (hpp), :120-162 (hps, rowExt),
// :164-203 (vpp), :205-239 (vps), :241-282 (vsp), :284-317 (vss), :362-369 (hvpp = hps+vsp).
// IF_INTERNAL_PREC 14, IF_FILTER_PREC 6, IF_INTERNAL_OFFS 8192 (common/constants.h:66-70).
#pragma once
#include "common.cuh"

__device__ __forceinline__ const int16_t* interp_taps(int ntaps, int idx)
{
    return ntaps == 8 ? c_lumaFilter[idx] : c_chromaFilter[idx];
}

// rounding / output stage shared by all variants.  `kind`: 0 = pp (pixel in, pixel out),
// 1 = ps (pixel in, short out), 2 = sp (short in, pixel out), 3 = ss (short in, short out)
template <int DEPTH>
__device__ __forceinline__ int interp_finish(int sum, int kind)
{
    constexpr int headroom = 14 - DEPTH;
    constexpr int maxv = (1 << DEPTH) - 1;
    switch (kind)
    {
    case 0:  return clip3i(0, maxv, (int)(int16_t)((sum + 32) >> 6));
    case 1:  { constexpr int shift = 6 - headroom; return (int)(int16_t)((sum + (int)((unsigned)-8192 << shift)) >> shift); }
    case 2:  { constexpr int shift = 6 + headroom; return clip3i(0, maxv, (int)(int16_t)((sum + (1 << (shift - 1)) + (8192 << 6)) >> shift)); }
    default: return (int)(int16_t)(sum >> 6);
    }
}

// ---- row-segment helpers shared by the interpolation fast path and the motion-estimation sub-pel code ----
// A lane owns NPX (8 or 4) consecutive output pixels of one row.
// 8-tap horizontal luma sum of the 8 pixels starting at s (ipfilter.cpp:79-118 inner loop).  8-bit planes:
// three aligned words, two funnel shifts and two DP4A (u8 pixels x s8 taps, exact in int32) instead of
// eight byte loads and eight IMADs; the third word is within the plane margin even when unused.
__device__ __forceinline__ int dp4a_us(uint32_t a, uint32_t b, int acc)
{
    int d;
    asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(acc));
    return d;
}
// c_lumaFilter[xf] packed as 2 x 4 signed bytes (taps 0-3, taps 4-7), little-endian
__constant__ uint32_t c_luma4[4][2] = { { 0x40000000u, 0u }, { 0x3af604ffu, 0x0001fb11u }, { 0x28f504ffu, 0xff04f528u }, { 0x11fb0100u, 0xff04f63au } };
template <typename P>
__device__ __forceinline__ int me_hsum8(const P* __restrict__ s, const int16_t* __restrict__ cx, int xf)
{
    if (sizeof(P) == 1)
    {
        const uintptr_t a = (uintptr_t)s;
        const uint32_t* ap = (const uint32_t*)(a & ~(uintptr_t)3);
        const unsigned sh = ((unsigned)a & 3u) * 8u;
        const uint32_t w0 = __ldg(ap), w1 = __ldg(ap + 1), w2 = __ldg(ap + 2);
        const uint32_t lo = __funnelshift_r(w0, w1, sh), hi = __funnelshift_r(w1, w2, sh);
        return dp4a_us(hi, c_luma4[xf][1], dp4a_us(lo, c_luma4[xf][0], 0));
    }
    int sum = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) sum += (int)s[k] * cx[k];
    return sum;
}

__device__ __forceinline__ int dp2a_lo_ss(uint32_t a, uint32_t b, int acc)
{
    int d; asm("dp2a.lo.s32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(acc)); return d;
}
__device__ __forceinline__ int dp2a_hi_ss(uint32_t a, uint32_t b, int acc)
{
    int d; asm("dp2a.hi.s32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(acc)); return d;
}

// NPX horizontal 8-tap sums of the outputs starting at pixel s (reads s[-3 .. NPX+3]).  8-bit planes: NPX/4+3
// aligned words, one funnel shift per word to the row's byte phase, then every output is two DP4A on a
// byte-shifted window (shared between neighbouring outputs): 4.25 instructions per output.
template <typename P, int NPX>
__device__ __forceinline__ void me_hrow(const P* __restrict__ s, int xf, int (&sum)[NPX])
{
    if (sizeof(P) == 1)
    {
        constexpr int NA = NPX / 4 + 2;                          // window words
        const uintptr_t a = (uintptr_t)(s - 3);
        const uint32_t* ap = (const uint32_t*)(a & ~(uintptr_t)3);
        const unsigned sh = ((unsigned)a & 3u) * 8u;
        uint32_t W[NA + 1], A[NA];
#pragma unroll
        for (int i = 0; i <= NA; i++) W[i] = __ldg(ap + i);
#pragma unroll
        for (int i = 0; i < NA; i++) A[i] = __funnelshift_r(W[i], W[i + 1], sh);   // A[i] = window bytes 4i..4i+3, byte 0 = s[-3]
        const uint32_t t0 = c_luma4[xf][0], t1 = c_luma4[xf][1];
#pragma unroll
        for (int x = 0; x < NPX; x++)
        {
            const int jw = x >> 2, k = (x & 3) * 8;
            const uint32_t lo = k ? __funnelshift_r(A[jw], A[jw + 1], k) : A[jw];
            const uint32_t hi = k ? __funnelshift_r(A[jw + 1], A[jw + 2], k) : A[jw + 1];
            sum[x] = dp4a_us(hi, t1, dp4a_us(lo, t0, 0));
        }
    }
    else
    {
        const int16_t* cx = c_lumaFilter[xf];
#pragma unroll
        for (int x = 0; x < NPX; x++)
        {
            int v = 0;
#pragma unroll
            for (int k = 0; k < 8; k++) v += (int)s[x + k - 3] * cx[k];
            sum[x] = v;
        }
    }
}

// Stage 1 of hv (hps with rowExt, ipfilter.cpp:120-162) for the NPX outputs starting at pixel s: the horizontal sums
// rounded to the 14-bit intermediate, stored packed at d (one 16-byte store for 8 outputs, 8 bytes for 4).
template <typename P, int NPX>
__device__ __forceinline__ void me_hv_row(const P* __restrict__ s, int xf, int16_t* __restrict__ d)
{
    constexpr int DEPTH = PixTraits<P>::depth;
    int sum[NPX];
    me_hrow<P, NPX>(s, xf, sum);
    uint32_t pk[NPX / 2];
#pragma unroll
    for (int i = 0; i < NPX / 2; i++)
        pk[i] = ((uint32_t)interp_finish<DEPTH>(sum[2 * i], 1) & 0xffffu) | ((uint32_t)interp_finish<DEPTH>(sum[2 * i + 1], 1) << 16);
    if (NPX == 8) *(uint4*)d = make_uint4(pk[0], pk[1], pk[NPX / 2 - 2], pk[NPX / 2 - 1]);
    else          *(uint2*)d = make_uint2(pk[0], pk[NPX / 2 - 1]);
}

// NPX vertical 8-tap sums straight from pixel rows; s = (row y-3, first pixel of the segment).  8-bit: each
// 4x4 block of bytes is transposed in registers (8 PRMT) so that a pixel's four vertical taps are one DP4A.
template <typename P, int NPX>
__device__ __forceinline__ void me_vcol(const P* __restrict__ s, int rstride, int yf, int (&sum)[NPX])
{
    if (sizeof(P) == 1)
    {
        constexpr int NW = NPX / 4;
        uint32_t R[8][NW];
#pragma unroll
        for (int k = 0; k < 8; k++)
        {
            const uintptr_t a = (uintptr_t)(s + (ptrdiff_t)k * rstride);
            const uint32_t* ap = (const uint32_t*)(a & ~(uintptr_t)3);
            const unsigned sh = ((unsigned)a & 3u) * 8u;
            uint32_t w[NW + 1];
#pragma unroll
            for (int i = 0; i <= NW; i++) w[i] = __ldg(ap + i);
#pragma unroll
            for (int i = 0; i < NW; i++) R[k][i] = __funnelshift_r(w[i], w[i + 1], sh);
        }
        const uint32_t t0 = c_luma4[yf][0], t1 = c_luma4[yf][1];
#pragma unroll
        for (int i = 0; i < NW; i++)
        {
            uint32_t col[2][4];
#pragma unroll
            for (int g = 0; g < 2; g++)
            {
                const uint32_t r0 = R[4 * g][i], r1 = R[4 * g + 1][i], r2 = R[4 * g + 2][i], r3 = R[4 * g + 3][i];
                const uint32_t p0 = __byte_perm(r0, r1, 0x5140), p1 = __byte_perm(r2, r3, 0x5140);     // (r0b0 r1b0 r0b1 r1b1), (r2b0 r3b0 r2b1 r3b1)
                const uint32_t p2 = __byte_perm(r0, r1, 0x7362), p3 = __byte_perm(r2, r3, 0x7362);     // same for bytes 2, 3
                col[g][0] = __byte_perm(p0, p1, 0x5410); col[g][1] = __byte_perm(p0, p1, 0x7632);
                col[g][2] = __byte_perm(p2, p3, 0x5410); col[g][3] = __byte_perm(p2, p3, 0x7632);
            }
#pragma unroll
            for (int bb = 0; bb < 4; bb++) sum[4 * i + bb] = dp4a_us(col[1][bb], t1, dp4a_us(col[0][bb], t0, 0));
        }
    }
    else
    {
        const int16_t* cy = c_lumaFilter[yf];
#pragma unroll
        for (int x = 0; x < NPX; x++)
        {
            int v = 0;
#pragma unroll
            for (int k = 0; k < 8; k++) v += (int)s[(ptrdiff_t)k * rstride + x] * cy[k];
            sum[x] = v;
        }
    }
}

// NPX vertical 8-tap sums over int16 intermediate rows in shared memory (second stage of hv); m = (row y, first
// element of the segment), row pitch `pitch` elements.  Two vertically adjacent int16 of one column are packed
// with one PRMT and consumed by DP2A (2 x s16 . 2 x s8 taps): 4 DP2A per pixel.
template <int NPX>
__device__ __forceinline__ void me_vmid(const int16_t* __restrict__ m, int pitch, int yf, int (&sum)[NPX])
{
    constexpr int NW = NPX / 2;
    uint32_t M[8][NW];
#pragma unroll
    for (int k = 0; k < 8; k++)
    {
        if (NPX == 8) { const uint4 v = *(const uint4*)(m + k * pitch); M[k][0] = v.x; M[k][1] = v.y; M[k][NW - 2] = v.z; M[k][NW - 1] = v.w; }
        else          { const uint2 v = *(const uint2*)(m + k * pitch); M[k][0] = v.x; M[k][NW - 1] = v.y; }
    }
    const uint32_t t0 = c_luma4[yf][0], t1 = c_luma4[yf][1];
#pragma unroll
    for (int i = 0; i < NW; i++)
    {
        int s0 = 0, s1 = 0;
#pragma unroll
        for (int pr = 0; pr < 4; pr++)
        {
            const uint32_t lo = __byte_perm(M[2 * pr][i], M[2 * pr + 1][i], 0x5410);      // (m[2p][2i], m[2p+1][2i])
            const uint32_t hi = __byte_perm(M[2 * pr][i], M[2 * pr + 1][i], 0x7632);      // (m[2p][2i+1], m[2p+1][2i+1])
            const uint32_t t = pr < 2 ? t0 : t1;
            if (pr & 1) { s0 = dp2a_hi_ss(lo, t, s0); s1 = dp2a_hi_ss(hi, t, s1); }
            else        { s0 = dp2a_lo_ss(lo, t, s0); s1 = dp2a_lo_ss(hi, t, s1); }
        }
        sum[2 * i] = s0; sum[2 * i + 1] = s1;
    }
}


// ---- 4-row units: a lane owns 4 consecutive rows of an 8-pixel column strip ---------------------------------------
// Vertical filters re-use their source rows: 11 rows feed 4 output rows (2.75 row loads per output row instead of 8).

// 8 pixels of a row at any byte phase as two packed words (8-bit planes); the third aligned word is inside the plane
// margin even when it is not needed
__device__ __forceinline__ void ip_row8_packed(const uint8_t* __restrict__ p, uint32_t& x0, uint32_t& x1)
{
    const uintptr_t a = (uintptr_t)p;
    const uint32_t* ap = (const uint32_t*)(a & ~(uintptr_t)3);
    const unsigned sh = ((unsigned)a & 3u) * 8u;
    const uint32_t w0 = __ldg(ap), w1 = __ldg(ap + 1), w2 = __ldg(ap + 2);
    x0 = __funnelshift_r(w0, w1, sh); x1 = __funnelshift_r(w1, w2, sh);
}

// 4 x 8 vertical 8-tap sums straight from pixel rows; s = (row y-3 of the first output row, first pixel of the strip).
// 8-bit: the 11 source rows are transposed once in 4-row groups G0 = rows 0-3, G1 = 4-7, G2 = 8-10 (one byte per row in
// a word per column), then output row y is DP4A(G0, A[y]) + DP4A(G1, B[y]) + DP4A(G2, C[y]) with the 8 taps shifted by
// y bytes and zero padded (A[0], B[0] = the plain tap words, C[0] = 0): exact integer sums, same as ipfilter.cpp:164-203.
template <typename P>
__device__ __forceinline__ void me_vcol4(const P* __restrict__ s, int rstride, int yf, int (&sum)[4][8])
{
    if (sizeof(P) == 1)
    {
        const uint32_t TL = c_luma4[yf][0], TH = c_luma4[yf][1];
        uint32_t A[4], B[4], C[4];
        A[0] = TL; B[0] = TH; C[0] = 0u;
        A[1] = TL << 8;  B[1] = __funnelshift_r(TL, TH, 24); C[1] = TH >> 24;
        A[2] = TL << 16; B[2] = __funnelshift_r(TL, TH, 16); C[2] = TH >> 16;
        A[3] = TL << 24; B[3] = __funnelshift_r(TL, TH, 8);  C[3] = TH >> 8;
        uint32_t R[12][2];
#pragma unroll
        for (int k = 0; k < 11; k++) ip_row8_packed((const uint8_t*)(s + (ptrdiff_t)k * rstride), R[k][0], R[k][1]);
        R[11][0] = 0u; R[11][1] = 0u;
#pragma unroll
        for (int i = 0; i < 2; i++)
        {
            uint32_t col[3][4];
#pragma unroll
            for (int g = 0; g < 3; g++)
            {
                const uint32_t r0 = R[4 * g][i], r1 = R[4 * g + 1][i], r2 = R[4 * g + 2][i], r3 = R[4 * g + 3][i];
                const uint32_t p0 = __byte_perm(r0, r1, 0x5140), p1 = __byte_perm(r2, r3, 0x5140);
                const uint32_t p2 = __byte_perm(r0, r1, 0x7362), p3 = __byte_perm(r2, r3, 0x7362);
                col[g][0] = __byte_perm(p0, p1, 0x5410); col[g][1] = __byte_perm(p0, p1, 0x7632);
                col[g][2] = __byte_perm(p2, p3, 0x5410); col[g][3] = __byte_perm(p2, p3, 0x7632);
            }
#pragma unroll
            for (int bb = 0; bb < 4; bb++)
            {
                sum[0][4 * i + bb] = dp4a_us(col[1][bb], B[0], dp4a_us(col[0][bb], A[0], 0));
#pragma unroll
                for (int y = 1; y < 4; y++)
                    sum[y][4 * i + bb] = dp4a_us(col[2][bb], C[y], dp4a_us(col[1][bb], B[y], dp4a_us(col[0][bb], A[y], 0)));
            }
        }
    }
    else
    {
        const int16_t* cy = c_lumaFilter[yf];
#pragma unroll
        for (int x = 0; x < 8; x++)
        {
            int p[11];
#pragma unroll
            for (int k = 0; k < 11; k++) p[k] = (int)__ldg(s + (ptrdiff_t)k * rstride + x);
#pragma unroll
            for (int y = 0; y < 4; y++)
            {
                int v = 0;
#pragma unroll
                for (int k = 0; k < 8; k++) v += p[y + k] * cy[k];
                sum[y][x] = v;
            }
        }
    }
}

// 4 x 8 vertical 8-tap sums over int16 intermediate rows in shared memory (second stage of hv); m = (row y of the first
// output row, first element of the strip), 16-byte aligned, row pitch `pitch` elements.  The 10 vertically adjacent row
// pairs (q, q+1) of a column are packed once (PRMT); output row y consumes pairs y, y+2, y+4, y+6 with DP2A.
__device__ __forceinline__ void me_vmid4(const int16_t* __restrict__ m, int pitch, int yf, int (&sum)[4][8])
{
    const uint32_t t0 = c_luma4[yf][0], t1 = c_luma4[yf][1];
#pragma unroll
    for (int hf = 0; hf < 2; hf++)
    {
        uint32_t M[11][2];
#pragma unroll
        for (int k = 0; k < 11; k++) { const uint2 v = *(const uint2*)(m + k * pitch + 4 * hf); M[k][0] = v.x; M[k][1] = v.y; }
#pragma unroll
        for (int i = 0; i < 2; i++)
        {
            uint32_t lo[10], hi[10];
#pragma unroll
            for (int q = 0; q < 10; q++)
            {
                lo[q] = __byte_perm(M[q][i], M[q + 1][i], 0x5410);       // (m[q][c], m[q+1][c]), c = 4 hf + 2 i
                hi[q] = __byte_perm(M[q][i], M[q + 1][i], 0x7632);       // column c + 1
            }
#pragma unroll
            for (int y = 0; y < 4; y++)
            {
                int s0 = 0, s1 = 0;
                s0 = dp2a_lo_ss(lo[y], t0, s0);     s1 = dp2a_lo_ss(hi[y], t0, s1);
                s0 = dp2a_hi_ss(lo[y + 2], t0, s0); s1 = dp2a_hi_ss(hi[y + 2], t0, s1);
                s0 = dp2a_lo_ss(lo[y + 4], t1, s0); s1 = dp2a_lo_ss(hi[y + 4], t1, s1);
                s0 = dp2a_hi_ss(lo[y + 6], t1, s0); s1 = dp2a_hi_ss(hi[y + 6], t1, s1);
                sum[y][4 * hf + 2 * i] = s0; sum[y][4 * hf + 2 * i + 1] = s1;
            }
        }
    }
}

// jobs the row-segment kernel (k_interp_rows, below) takes; the generic kernel skips them
__device__ __forceinline__ bool interp_fast_eligible(int op, const x265cu_interp_job& jb)
{
    return jb.ntaps == 8 && (jb.w & 7) == 0 && jb.w <= 64 && jb.h > 0 &&
           (op == X265CU_HPP || op == X265CU_HPS || op == X265CU_VPP || op == X265CU_VPS || op == X265CU_HVPP);
}

// One CTA per job.  The source window (block + filter halo) is staged once in shared memory as int16,
// the horizontal pass writes a second shared tile, the vertical pass reads it: every source sample is
// fetched from HBM/L2 exactly once per job.
template <typename P>
__global__ void __launch_bounds__(256) k_interp(int op, const void* __restrict__ srcv, void* __restrict__ dstv,
                                                const x265cu_interp_job* __restrict__ jobs, int n)
{
    constexpr int DEPTH = PixTraits<P>::depth;
    __shared__ int16_t win[72 * 72];
    __shared__ int16_t mid[72 * 64];
    for (int j = blockIdx.x; j < n; j += gridDim.x)
    {
        const x265cu_interp_job jb = jobs[j];
        if (interp_fast_eligible(op, jb)) continue;                        // k_interp_rows owns this job
        const int w = jb.w, h = jb.h, nt = jb.ntaps;
        const bool srcShort = (op == X265CU_VSP || op == X265CU_VSS);
        const bool doH = (op == X265CU_HPP || op == X265CU_HPS || op == X265CU_HVPP);
        const bool doV = (op == X265CU_VPP || op == X265CU_VPS || op == X265CU_VSP || op == X265CU_VSS || op == X265CU_HVPP);
        const bool vHalo = doV || (op == X265CU_HPS && jb.rowExt);
        const int hl = doH ? nt / 2 - 1 : 0, hr = doH ? nt / 2 : 0;         // left / right halo
        const int vt = vHalo ? nt / 2 - 1 : 0, vb = vHalo ? nt / 2 : 0;      // top / bottom halo
        const int ww = w + hl + hr, wh = h + vt + vb;
        // stage window
        for (int i = threadIdx.x; i < ww * wh; i += blockDim.x)
        {
            int r = i / ww, c = i - r * ww;
            int64_t si = jb.s_off + (int64_t)(r - vt) * jb.s_stride + (c - hl);
            win[r * 72 + c] = srcShort ? ((const int16_t*)srcv)[si] : (int16_t)((const P*)srcv)[si];
        }
        __syncthreads();
        const int16_t* cx = interp_taps(nt, jb.idxX);
        const int16_t* cy = interp_taps(nt, jb.idxY);
        if (op == X265CU_HPP || op == X265CU_HPS)
        {
            const int16_t* c = cx;
            const int kind = (op == X265CU_HPP) ? 0 : 1;
            for (int i = threadIdx.x; i < w * wh; i += blockDim.x)
            {
                int r = i / w, x = i - r * w;
                int sum = 0;
                for (int k = 0; k < nt; k++) sum += (int)win[r * 72 + x + k] * c[k];
                int v = interp_finish<DEPTH>(sum, kind);
                int64_t di = jb.d_off + (int64_t)r * jb.d_stride + x;      // rowExt: dst row 0 = 3 rows above the block
                if (kind == 0) ((P*)dstv)[di] = (P)v; else ((int16_t*)dstv)[di] = (int16_t)v;
            }
        }
        else if (op == X265CU_HVPP)
        {
            for (int i = threadIdx.x; i < w * wh; i += blockDim.x)
            {
                int r = i / w, x = i - r * w;
                int sum = 0;
                for (int k = 0; k < nt; k++) sum += (int)win[r * 72 + x + k] * cx[k];
                mid[r * 64 + x] = (int16_t)interp_finish<DEPTH>(sum, 1);
            }
            __syncthreads();
            for (int i = threadIdx.x; i < w * h; i += blockDim.x)
            {
                int y = i / w, x = i - y * w;
                int sum = 0;
                for (int k = 0; k < nt; k++) sum += (int)mid[(y + k) * 64 + x] * cy[k];
                ((P*)dstv)[jb.d_off + (int64_t)y * jb.d_stride + x] = (P)interp_finish<DEPTH>(sum, 2);
            }
        }
        else
        {
            // vertical-only variants; coefficient index is idxX for the single-index signatures
            const int16_t* c = cx;
            const int kind = op == X265CU_VPP ? 0 : (op == X265CU_VPS ? 1 : (op == X265CU_VSP ? 2 : 3));
            for (int i = threadIdx.x; i < w * h; i += blockDim.x)
            {
                int y = i / w, x = i - y * w;
                int sum = 0;
                for (int k = 0; k < nt; k++) sum += (int)win[(y + k) * 72 + x] * c[k];
                int v = interp_finish<DEPTH>(sum, kind);
                int64_t di = jb.d_off + (int64_t)y * jb.d_stride + x;
                if (kind == 0 || kind == 2) ((P*)dstv)[di] = (P)v; else ((int16_t*)dstv)[di] = (int16_t)v;
            }
        }
        __syncthreads();
    }
}

// ---- fast path: one warp per job, one lane per 8-pixel row segment -----------------------------------------
// Eligible jobs: luma (8 taps), pixel source (hpp / hps / vpp / vps / hvpp), width a multiple of 8.  Everything
// stays in registers except hvpp's intermediate, which goes through shared memory in bands of 16 rows.
// Source rows are read as aligned 4-byte words funnel-shifted to the row's byte phase (any source alignment);
// a segment is stored with one 8 / 16-byte store when the destination allows it.
#define IP_BAND 16

template <typename P, typename D>
__device__ __forceinline__ void interp_store8(D* __restrict__ d, const int (&v)[8], bool vec)
{
    if (vec)
    {
        if (sizeof(D) == 1)
            *(uint2*)d = make_uint2((uint32_t)v[0] | ((uint32_t)v[1] << 8) | ((uint32_t)v[2] << 16) | ((uint32_t)v[3] << 24),
                                    (uint32_t)v[4] | ((uint32_t)v[5] << 8) | ((uint32_t)v[6] << 16) | ((uint32_t)v[7] << 24));
        else
            *(uint4*)d = make_uint4(((uint32_t)v[0] & 0xffffu) | ((uint32_t)v[1] << 16), ((uint32_t)v[2] & 0xffffu) | ((uint32_t)v[3] << 16),
                                    ((uint32_t)v[4] & 0xffffu) | ((uint32_t)v[5] << 16), ((uint32_t)v[6] & 0xffffu) | ((uint32_t)v[7] << 16));
    }
    else
    {
#pragma unroll
        for (int x = 0; x < 8; x++) d[x] = (D)v[x];
    }
}

// GROUP: 0 = horizontal (hpp, hps), 1 = vertical (vpp, vps), 2 = hvpp -- separate instantiations so that each pass
// keeps its own register budget (the 8x4-unit vertical path needs 80 registers, the horizontal one 48).
template <typename P, int GROUP>
__global__ void __launch_bounds__(256) k_interp_rows(int op, const P* __restrict__ src, void* __restrict__ dstv,
                                                     const x265cu_interp_job* __restrict__ jobs, int n)
{
    constexpr int DEPTH = PixTraits<P>::depth;
    __shared__ __align__(16) int16_t s_mid[GROUP == 2 ? 8 : 1][GROUP == 2 ? (IP_BAND + 7) * 64 : 8];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int16_t* mid = s_mid[GROUP == 2 ? warp : 0];
    for (int j = blockIdx.x * 8 + warp; j < n; j += gridDim.x * 8)
    {
        const x265cu_interp_job jb = jobs[j];
        if (!interp_fast_eligible(op, jb)) continue;
        const int w = jb.w, segs = w >> 3;
        const P* s0 = src + jb.s_off;
        if (GROUP == 2)
        {
            P* d0 = (P*)dstv + jb.d_off;
            const bool vec = (((uintptr_t)d0 | (uintptr_t)((size_t)jb.d_stride * sizeof(P))) & 7) == 0 && sizeof(P) == 1 ||
                             (((uintptr_t)d0 | (uintptr_t)((size_t)jb.d_stride * sizeof(P))) & 15) == 0 && sizeof(P) == 2;
            for (int y0 = 0; y0 < jb.h; y0 += IP_BAND)
            {
                const int rows = min(IP_BAND, jb.h - y0);
                __syncwarp();
                for (int t = lane; t < (rows + 7) * segs; t += 32)
                {
                    const int mrow = t / segs, seg = t - mrow * segs;
                    me_hv_row<P, 8>(s0 + (ptrdiff_t)(y0 - 3 + mrow) * jb.s_stride + seg * 8, jb.idxX, mid + mrow * w + seg * 8);
                }
                __syncwarp();
                for (int u = lane; u < rows * segs; u += 32)
                {
                    const int row = u / segs, seg = u - row * segs;
                    int v[8];
                    me_vmid<8>(mid + row * w + seg * 8, w, jb.idxY, v);
#pragma unroll
                    for (int x = 0; x < 8; x++) v[x] = interp_finish<DEPTH>(v[x], 2);
                    interp_store8<P, P>(d0 + (ptrdiff_t)(y0 + row) * jb.d_stride + seg * 8, v, vec);
                }
            }
        }
        else
        {
            const bool toShort = op == X265CU_HPS || op == X265CU_VPS;
            const int ext = (op == X265CU_HPS && jb.rowExt) ? 3 : 0;          // rowExt: 3 rows above .. 4 rows below, dst row 0 = first of them
            const int rows = jb.h + (ext ? 7 : 0);
            const size_t dsz = toShort ? 2 : sizeof(P);
            const uintptr_t dbase = (uintptr_t)dstv + (size_t)jb.d_off * dsz;
            const bool vec = ((dbase | (uintptr_t)((size_t)jb.d_stride * dsz)) & (dsz == 1 ? 7 : 15)) == 0;
            if (GROUP == 1 && (jb.h & 3) == 0 && (jb.h >> 2) * segs >= 32)
            {   // vertical, a warp's worth of 8x4 units: 11 source rows feed 4 output rows (me_vcol4)
                for (int u = lane; u < (jb.h >> 2) * segs; u += 32)
                {
                    const int grp = u / segs, seg = u - grp * segs, row = grp * 4;
                    int v[4][8];
                    me_vcol4<P>(s0 + (ptrdiff_t)(row - 3) * jb.s_stride + seg * 8, jb.s_stride, jb.idxX, v);
#pragma unroll
                    for (int y = 0; y < 4; y++)
                    {
#pragma unroll
                        for (int x = 0; x < 8; x++) v[y][x] = interp_finish<DEPTH>(v[y][x], toShort ? 1 : 0);
                        if (toShort) interp_store8<P, int16_t>((int16_t*)dbase + (ptrdiff_t)(row + y) * jb.d_stride + seg * 8, v[y], vec);
                        else         interp_store8<P, P>((P*)dbase + (ptrdiff_t)(row + y) * jb.d_stride + seg * 8, v[y], vec);
                    }
                }
                continue;
            }
            for (int u = lane; u < rows * segs; u += 32)
            {
                const int row = u / segs, seg = u - row * segs;
                const P* s = s0 + (ptrdiff_t)(row - ext) * jb.s_stride + seg * 8;
                int v[8];
                if (GROUP == 0) me_hrow<P, 8>(s, jb.idxX, v);
                else            me_vcol<P, 8>(s - 3 * (ptrdiff_t)jb.s_stride, jb.s_stride, jb.idxX, v);
#pragma unroll
                for (int x = 0; x < 8; x++) v[x] = interp_finish<DEPTH>(v[x], toShort ? 1 : 0);
                if (toShort) interp_store8<P, int16_t>((int16_t*)dbase + (ptrdiff_t)row * jb.d_stride + seg * 8, v, vec);
                else         interp_store8<P, P>((P*)dbase + (ptrdiff_t)row * jb.d_stride + seg * 8, v, vec);
            }
        }
    }
}

template <typename P>
static void launch_interp_rows(x265cu_ctx* ctx, int fb, int op, const void* src, void* dst, const x265cu_interp_job* jobs, int n)
{
    if (op == X265CU_HVPP)                          k_interp_rows<P, 2><<<fb, 256, 0, ctx->stream>>>(op, (const P*)src, dst, jobs, n);
    else if (op == X265CU_VPP || op == X265CU_VPS)  k_interp_rows<P, 1><<<fb, 256, 0, ctx->stream>>>(op, (const P*)src, dst, jobs, n);
    else                                            k_interp_rows<P, 0><<<fb, 256, 0, ctx->stream>>>(op, (const P*)src, dst, jobs, n);
}

static int launch_interp(x265cu_ctx* ctx, int depth, int op, const void* src, void* dst, const x265cu_interp_job* jobs, int n)
{
    if (n <= 0) return 0;
    int blocks = n < ctx->sm_count * 8 ? n : ctx->sm_count * 8;
    const bool pixelSrc = !(op == X265CU_VSP || op == X265CU_VSS);
    if (pixelSrc)
    {   // the row-segment kernel takes the eligible jobs (one warp each), the generic kernel the rest
        int fb = (n + 7) / 8;
        if (fb > ctx->sm_count * 8) fb = ctx->sm_count * 8;
        if (depth == 8) launch_interp_rows<uint8_t>(ctx, fb, op, src, dst, jobs, n);
        else            launch_interp_rows<uint16_t>(ctx, fb, op, src, dst, jobs, n);
        CU_LAUNCH_CHECK(ctx);
    }
    if (depth == 8) k_interp<uint8_t><<<blocks, 256, 0, ctx->stream>>>(op, src, dst, jobs, n);
    else            k_interp<uint16_t><<<blocks, 256, 0, ctx->stream>>>(op, src, dst, jobs, n);
    CU_LAUNCH_CHECK(ctx);
    return 0;
}
