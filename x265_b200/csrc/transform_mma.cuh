// x265_b200/csrc/transform_mma.cuh -- 16x16 / 32x32 integer DCT and IDCT on the int8 tensor-core pipe (IMMA),
// bit-exact to /root/reference/source/common/dct.cpp:83-203 (forward) and :302-416 (inverse).
//
// There is no int16 MMA.  The HEVC matrix fits s8 (|c| <= 90); every int16 operand x is split exactly as
// x = 256*hi + lo with hi = x >> 8 (s8) and lo = x & 255 (u8), two IMMAs (s8 x s8 and s8 x u8) accumulate in
// s32 and are recombined as (hi_acc << 8) + lo_acc  (|acc| <= 32*90*32768 < 2^31, SURVEY hard part 4).
// The reference's per-pass `(acc + add) >> shift` with int16 truncation (forward) or clip (inverse) is the
// epilogue between the two passes.
//
// One warp transforms one TU entirely in registers: pass 1's accumulator fragment IS pass 2's B operand.
// With D = A x B, A = the constant matrix (row-major, m16 tiles) and B = the data (col fragment), pass 1
// yields D1[k1][j1]; pass 2 needs B2[i2][j2] = D1[j2][i2], i.e. the accumulator ROW becomes the B COLUMN --
// which is exactly how the C and B fragments are distributed over lanes (row/col = lane >> 2) -- and the
// accumulator columns 8*nt + 2t + {0,1} become B's K slots 16r + 4t + e through a fixed permutation that is
// folded into the constant A operand of pass 2.  HBM traffic is the compulsory 4*N*N bytes per TU.
#pragma once
#include "common.cuh"

template <int K32>
__device__ __forceinline__ void imma(int (&d)[4], const uint32_t* a, const uint32_t* b, bool b_unsigned)
{
    if (K32)
    {
        if (b_unsigned)
            asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                         : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
        else
            asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                         : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
    }
    else
    {
        if (b_unsigned)
            asm volatile("mma.sync.aligned.m16n8k16.row.col.s32.s8.u8.s32 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                         : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(b[0]));
        else
            asm volatile("mma.sync.aligned.m16n8k16.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                         : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(b[0]));
    }
}
// the data as the A operand (u8 low bytes or s8 high bytes) against the s8 constant matrix as B
template <int K32>
__device__ __forceinline__ void imma_da(int (&d)[4], const uint32_t* a, const uint32_t* b, bool a_unsigned)
{
    if (K32)
    {
        if (a_unsigned)
            asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                         : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
        else
            asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                         : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
    }
    else
    {
        if (a_unsigned)
            asm volatile("mma.sync.aligned.m16n8k16.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                         : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(b[0]));
        else
            asm volatile("mma.sync.aligned.m16n8k16.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                         : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(b[0]));
    }
}

// four int16 values -> (4 high bytes, 4 low bytes)
__device__ __forceinline__ void split4(int v0, int v1, int v2, int v3, uint32_t& hi, uint32_t& lo)
{
    const uint32_t w0 = ((uint32_t)(uint16_t)v0) | ((uint32_t)(uint16_t)v1 << 16);
    const uint32_t w1 = ((uint32_t)(uint16_t)v2) | ((uint32_t)(uint16_t)v3 << 16);
    lo = __byte_perm(w0, w1, 0x6420);
    hi = __byte_perm(w0, w1, 0x7531);
}

// N = 16 or 32.  FWD: src strided (stride / tu_pitch in elements), dst contiguous N*N per TU; INV: the reverse.
template <int DEPTH, int N, bool FWD>
__global__ void __launch_bounds__(256) k_transform_mma(const int16_t* __restrict__ src, int16_t* __restrict__ dst, int stride, int64_t tu_pitch, int n, int swapStore)
{
    constexpr int IP = N + 2;                                        // inverse: input tile pitch (halfwords)
    __shared__ __align__(16) int16_t s_in[FWD ? 1 : 8][FWD ? 8 : N * IP];
    const bool in16 = (((uintptr_t)src) & 15) == 0;                 // contiguous TUs of N * N int16: 16-byte pieces when the base allows
    constexpr int LG = N == 32 ? 5 : 4;
    constexpr int MT = N / 16, NT = N / 8, KR = N / 16;          // m tiles, n tiles, B registers per n tile
    constexpr int K32 = N == 32;
    constexpr int shift1 = FWD ? LG - 1 + (DEPTH - 8) : 7;
    constexpr int shift2 = FWD ? LG + 6 : 12 - (DEPTH - 8);
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
    // the matrix through shared memory: the fragment set-up below indexes it per lane (see d_dct in common.cuh)
    __shared__ __align__(16) int8_t M[N * N];
    for (int i = threadIdx.x * 4; i < N * N; i += blockDim.x * 4) *(uint32_t*)(M + i) = *(const uint32_t*)(d_dct[LG - 2] + i);
    __syncthreads();

    // constant A fragments: pass 1 uses the natural K order, pass 2 the accumulator-induced permutation.
    // forward: A[row][k] = M[row][k];  inverse: A[row][k] = M[k][row]  (A = M^T)
    uint32_t a1[MT][2 * KR], a2[MT][2 * KR];
#pragma unroll
    for (int mt = 0; mt < MT; mt++)
#pragma unroll
        for (int r = 0; r < KR; r++)
#pragma unroll
            for (int h = 0; h < 2; h++)
            {
                const int row = g + 8 * h + 16 * mt;
                uint32_t w1 = 0, w2 = 0;
#pragma unroll
                for (int e = 0; e < 4; e++)
                {
                    const int k1 = 16 * r + 4 * t + e;
                    const int k2 = 8 * (2 * r + (e >> 1)) + 2 * t + (e & 1);
                    const int c1 = FWD ? M[row * N + k1] : M[k1 * N + row];
                    const int c2 = FWD ? M[row * N + k2] : M[k2 * N + row];
                    w1 |= (uint32_t)(uint8_t)(int8_t)c1 << (8 * e);
                    w2 |= (uint32_t)(uint8_t)(int8_t)c2 << (8 * e);
                }
                a1[mt][2 * r + h] = w1; a2[mt][2 * r + h] = w2;      // register order: (r0,h0) (r0,h1) (r1,h0) (r1,h1)
            }

    // inverse with 4-byte aligned destination rows (swapStore): pass 2 runs with the operand roles SWAPPED -- the pass-1 results are
    // the A operand (rows = residual rows) and the matrix the B operand (B[k][i] = M[k][i], K slots in the accumulator-induced
    // order), so the accumulators come out row-major (two adjacent residual columns per register pair) and leave as 4-byte stores
    // like the forward transform's coefficients; the un-swapped form leaves residual COLUMNS along the lanes (2-byte scattered
    // stores, half of every sector wasted)
    uint32_t b2c[NT][KR];
    if (!FWD)
    {
#pragma unroll
        for (int nt = 0; nt < NT; nt++)
#pragma unroll
            for (int r = 0; r < KR; r++)
            {
                uint32_t w = 0;
#pragma unroll
                for (int e = 0; e < 4; e++)
                {
                    const int k2 = 8 * (2 * r + (e >> 1)) + 2 * t + (e & 1);
                    w |= (uint32_t)(uint8_t)(int8_t)M[k2 * N + 8 * nt + g] << (8 * e);
                }
                b2c[nt][r] = w;
            }
    }

    constexpr bool PRE = !FWD && N == 16;                           // (32x32: the 16 prefetch registers would cost a resident CTA)
    uint4 pre[PRE ? N * N / 256 : 1];
    if (PRE && in16 && warp < n)
    {
        const int16_t* sn = src + (int64_t)warp * N * N;
#pragma unroll
        for (int q = 0; q < N * N / 256; q++) pre[PRE ? q : 0] = __ldg((const uint4*)(sn + (q * 32 + lane) * 8));
    }
    for (int tu = warp; tu < n; tu += nwarps)
    {
        // ---- pass-1 B fragments from memory ----
        uint32_t bh[NT][KR], bl[NT][KR];
        if (FWD)
        {
            const int16_t* s = src + (int64_t)tu * tu_pitch;
#pragma unroll
            for (int nt = 0; nt < NT; nt++)
#pragma unroll
                for (int r = 0; r < KR; r++)
                {   // B[k][j]: j = g + 8 nt (input row), k = 16 r + 4 t + e (input column): 4 consecutive int16
                    const uint2 w = *(const uint2*)(s + (int64_t)(g + 8 * nt) * stride + 16 * r + 4 * t);
                    bl[nt][r] = __byte_perm(w.x, w.y, 0x6420);
                    bh[nt][r] = __byte_perm(w.x, w.y, 0x7531);
                }
        }
        else
        {
            // The fragments need four coefficients of one COLUMN per lane (2-byte loads N elements apart from global memory:
            // half of every sector wasted).  The warp copies its TU with 16-byte row pieces into a padded shared tile (pitch N + 2
            // halfwords: the four rows a quad of lanes reads are 4 banks apart) and picks the columns out of that.
            const int16_t* s = src + (int64_t)tu * N * N;
            int16_t* tile = s_in[threadIdx.x >> 5];
            __syncwarp();
            uint4 wv[N * N / 256];                                   // all pieces requested before the first shared store
            if (in16)
            {
#pragma unroll
                for (int q = 0; q < N * N / 256; q++) wv[q] = PRE ? pre[PRE ? q : 0] : __ldg((const uint4*)(s + (q * 32 + lane) * 8));
            }
#pragma unroll
            for (int q = 0; q < N * N / 256; q++)
            {
                const int e0 = (q * 32 + lane) * 8, row = e0 >> LG, col = e0 & (N - 1);
                uint32_t* tp = (uint32_t*)(tile + row * IP + col);
                if (in16)
                {
                    const uint4 w = wv[q];
                    tp[0] = w.x; tp[1] = w.y; tp[2] = w.z; tp[3] = w.w;
                }
                else
                {
#pragma unroll
                    for (int k = 0; k < 8; k++) tile[row * IP + col + k] = s[e0 + k];
                }
            }
            __syncwarp();
            // the NEXT TU's coefficients are requested now and land while this TU is transformed (one warp per TU is a long
            // dependent chain: load -> tile -> fragments -> 2 x MMA passes -> stores, which the prefetch overlaps with the
            // loads)
            if (PRE && in16 && tu + nwarps < n)
            {
                const int16_t* sn = src + (int64_t)(tu + nwarps) * N * N;
#pragma unroll
                for (int q = 0; q < N * N / 256; q++) pre[PRE ? q : 0] = __ldg((const uint4*)(sn + (q * 32 + lane) * 8));
            }
#pragma unroll
            for (int nt = 0; nt < NT; nt++)
#pragma unroll
                for (int r = 0; r < KR; r++)
                {   // B[k][j] = In[k][j]: k = 16 r + 4 t + e (coefficient row), j = g + 8 nt
                    const int16_t* p = tile + (16 * r + 4 * t) * IP + g + 8 * nt;
                    split4(p[0], p[IP], p[2 * IP], p[3 * IP], bh[nt][r], bl[nt][r]);
                }
        }
        // ---- pass 1 ----
        int o1[MT][NT][4];
#pragma unroll
        for (int mt = 0; mt < MT; mt++)
#pragma unroll
            for (int nt = 0; nt < NT; nt++)
            {
                int ah[4] = { 0, 0, 0, 0 }, al[4] = { 0, 0, 0, 0 };
                imma<K32>(ah, a1[mt], bh[nt], false);
                imma<K32>(al, a1[mt], bl[nt], true);
#pragma unroll
                for (int q = 0; q < 4; q++)
                {
                    const int v = (((ah[q] << 8) + al[q]) + (1 << (shift1 - 1))) >> shift1;
                    o1[mt][nt][q] = FWD ? (int)(int16_t)v : clip16(v);
                }
            }
        // ---- pass-2 B fragments straight from the pass-1 accumulators ----
        // n tile 2*mt + half takes accumulator rows g + 8*half of m tile mt; K slots (r, e) <- (nt = 2r + (e>>1), col e&1)
        uint32_t ch[NT][KR], cl[NT][KR];
#pragma unroll
        for (int mt = 0; mt < MT; mt++)
#pragma unroll
            for (int half = 0; half < 2; half++)
#pragma unroll
                for (int r = 0; r < KR; r++)
                    split4(o1[mt][2 * r][2 * half], o1[mt][2 * r][2 * half + 1], o1[mt][2 * r + 1][2 * half], o1[mt][2 * r + 1][2 * half + 1],
                           ch[2 * mt + half][r], cl[2 * mt + half][r]);
        // ---- pass 2 + store ----
        int16_t* d = dst + (int64_t)tu * (FWD ? (int64_t)N * N : tu_pitch);
        if (!FWD && swapStore)
        {
#pragma unroll
            for (int mt = 0; mt < MT; mt++)
            {
                uint32_t aH[2 * KR], aL[2 * KR];
#pragma unroll
                for (int r = 0; r < KR; r++)
#pragma unroll
                    for (int h = 0; h < 2; h++) { aH[2 * r + h] = ch[2 * mt + h][r]; aL[2 * r + h] = cl[2 * mt + h][r]; }
#pragma unroll
                for (int nt = 0; nt < NT; nt++)
                {
                    int ah[4] = { 0, 0, 0, 0 }, al[4] = { 0, 0, 0, 0 };
                    imma_da<K32>(ah, aH, b2c[nt], false);
                    imma_da<K32>(al, aL, b2c[nt], true);
                    int v[4];
#pragma unroll
                    for (int q = 0; q < 4; q++) v[q] = clip16((((ah[q] << 8) + al[q]) + (1 << (shift2 - 1))) >> shift2);
                    // accumulator element q: residual row = g + 8*(q>>1) + 16 mt, column = 8 nt + 2 t + (q&1)
                    *(uint32_t*)(d + (int64_t)(g + 16 * mt) * stride + 8 * nt + 2 * t)     = ((uint32_t)(uint16_t)v[0]) | ((uint32_t)(uint16_t)v[1] << 16);
                    *(uint32_t*)(d + (int64_t)(g + 8 + 16 * mt) * stride + 8 * nt + 2 * t) = ((uint32_t)(uint16_t)v[2]) | ((uint32_t)(uint16_t)v[3] << 16);
                }
            }
            continue;
        }
#pragma unroll
        for (int mt = 0; mt < MT; mt++)
#pragma unroll
            for (int nt = 0; nt < NT; nt++)
            {
                int ah[4] = { 0, 0, 0, 0 }, al[4] = { 0, 0, 0, 0 };
                imma<K32>(ah, a2[mt], ch[nt], false);
                imma<K32>(al, a2[mt], cl[nt], true);
                int v[4];
#pragma unroll
                for (int q = 0; q < 4; q++)
                {
                    const int x = (((ah[q] << 8) + al[q]) + (1 << (shift2 - 1))) >> shift2;
                    v[q] = FWD ? (int)(int16_t)x : clip16(x);
                }
                // accumulator element q: row = g + 8*(q>>1) + 16 mt, col = 8 nt + 2 t + (q&1)
                if (FWD)
                {   // dst[k2 * N + j2]: rows are coefficient rows, two adjacent columns per 32-bit store
                    *(uint32_t*)(d + (g + 16 * mt) * N + 8 * nt + 2 * t)     = ((uint32_t)(uint16_t)v[0]) | ((uint32_t)(uint16_t)v[1] << 16);
                    *(uint32_t*)(d + (g + 8 + 16 * mt) * N + 8 * nt + 2 * t) = ((uint32_t)(uint16_t)v[2]) | ((uint32_t)(uint16_t)v[3] << 16);
                }
                else
                {   // D2[i2][j2] = Out[j2][i2]: dst[j2 * stride + i2]
                    const int j0 = 8 * nt + 2 * t, i0 = g + 16 * mt;
                    d[(int64_t)j0 * stride + i0] = (int16_t)v[0];
                    d[(int64_t)(j0 + 1) * stride + i0] = (int16_t)v[1];
                    d[(int64_t)j0 * stride + i0 + 8] = (int16_t)v[2];
                    d[(int64_t)(j0 + 1) * stride + i0 + 8] = (int16_t)v[3];
                }
            }
    }
}

// returns 1 if the tensor-core path took the launch, 0 if the caller must use the shared-memory kernel
template <int DEPTH>
static int launch_transform_mma(x265cu_ctx* ctx, int op, int N, const int16_t* src, int16_t* dst, int stride, int64_t tu_pitch, int n)
{
    if (N != 16 && N != 32) return 0;
    const bool fwd = (op == X265CU_DCT);
    if (!fwd && op != X265CU_IDCT) return 0;
    if (fwd)
    {   // 8-byte vector loads of the residual rows, 4-byte stores of the coefficients
        if ((((uintptr_t)src) & 7) || (stride & 3) || (tu_pitch & 3) || (((uintptr_t)dst) & 3)) return 0;
    }
    int blocks = (n + 7) / 8;
    if (blocks > ctx->sm_count * 8) blocks = ctx->sm_count * 8;
    // inverse: role-swapped pass 2 with 4-byte stores when every destination row is 4-byte aligned
    const int vec = !fwd && !(((uintptr_t)dst) & 3) && !(stride & 1) && !(tu_pitch & 1);
    if (N == 32)
    {
        if (fwd) k_transform_mma<DEPTH, 32, true><<<blocks, 256, 0, ctx->stream>>>(src, dst, stride, tu_pitch, n, 0);
        else     k_transform_mma<DEPTH, 32, false><<<blocks, 256, 0, ctx->stream>>>(src, dst, stride, tu_pitch, n, vec);
    }
    else
    {
        if (fwd) k_transform_mma<DEPTH, 16, true><<<blocks, 256, 0, ctx->stream>>>(src, dst, stride, tu_pitch, n, 0);
        else     k_transform_mma<DEPTH, 16, false><<<blocks, 256, 0, ctx->stream>>>(src, dst, stride, tu_pitch, n, vec);
    }
    return 1;
}
