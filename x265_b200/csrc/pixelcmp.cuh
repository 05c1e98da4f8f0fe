// x265_b200/csrc/pixelcmp.cuh -- pixel-compare class: SAD / SATD / SA8D / SSE / SSD_S / VAR / PSY.
// Semantics: /root/reference/source/common/pixel.cpp:40-377 (sad, satd_4x4/8x4, sa8d), :167-186 (sse),
// :379-391 (ssd_s), :703-720 (var), :726-757 (psyCost_pp).  Bit-exact integer arithmetic.
#pragma once
#include "common.cuh"

// ---- Hadamard cores (per thread, registers only) -------------------------------------------
__device__ __forceinline__ void had4(int& a, int& b, int& c, int& d)
{
    int s01 = a + b, d01 = a - b, s23 = c + d, d23 = c - d;
    a = s01 + s23; c = s01 - s23; b = d01 + d23; d = d01 - d23;
}

// sum |H4 D H4^T| of one 4x4 tile, un-normalised (pixel.cpp:210-236 before the >>1)
template <typename PA, typename PB>
__device__ __forceinline__ int had4x4_abs(const PA* __restrict__ a, int sa, const PB* __restrict__ b, int sb)
{
    int m[4][4];
#pragma unroll
    for (int y = 0; y < 4; y++)
    {
#pragma unroll
        for (int x = 0; x < 4; x++) m[y][x] = (int)a[y * sa + x] - (int)b[y * sb + x];
        had4(m[y][0], m[y][1], m[y][2], m[y][3]);
    }
    int acc = 0;
#pragma unroll
    for (int x = 0; x < 4; x++)
    {
        had4(m[0][x], m[1][x], m[2][x], m[3][x]);
        acc += abs(m[0][x]) + abs(m[1][x]) + abs(m[2][x]) + abs(m[3][x]);
    }
    return acc;
}

// same, but plane b is implicit zero (psy cost energy term)
template <typename PA>
__device__ __forceinline__ int had4x4_abs_zero(const PA* __restrict__ a, int sa)
{
    int m[4][4];
#pragma unroll
    for (int y = 0; y < 4; y++)
    {
#pragma unroll
        for (int x = 0; x < 4; x++) m[y][x] = (int)a[y * sa + x];
        had4(m[y][0], m[y][1], m[y][2], m[y][3]);
    }
    int acc = 0;
#pragma unroll
    for (int x = 0; x < 4; x++)
    {
        had4(m[0][x], m[1][x], m[2][x], m[3][x]);
        acc += abs(m[0][x]) + abs(m[1][x]) + abs(m[2][x]) + abs(m[3][x]);
    }
    return acc;
}

// un-normalised 8x8 Hadamard abs-sum (pixel.cpp:299-334); `zero_b` skips plane b
template <typename PA, typename PB, bool ZERO_B>
__device__ __forceinline__ int had8x8_abs(const PA* __restrict__ a, int sa, const PB* __restrict__ b, int sb)
{
    int m[8][8];
#pragma unroll
    for (int y = 0; y < 8; y++)
    {
#pragma unroll
        for (int x = 0; x < 8; x++) m[y][x] = ZERO_B ? (int)a[y * sa + x] : (int)a[y * sa + x] - (int)b[y * sb + x];
        had4(m[y][0], m[y][1], m[y][2], m[y][3]);
        had4(m[y][4], m[y][5], m[y][6], m[y][7]);
#pragma unroll
        for (int k = 0; k < 4; k++) { int p = m[y][k], q = m[y][k + 4]; m[y][k] = p + q; m[y][k + 4] = p - q; }
    }
    int acc = 0;
#pragma unroll
    for (int x = 0; x < 8; x++)
    {
        had4(m[0][x], m[1][x], m[2][x], m[3][x]);
        had4(m[4][x], m[5][x], m[6][x], m[7][x]);
#pragma unroll
        for (int k = 0; k < 4; k++) acc += abs(m[k][x] + m[k + 4][x]) + abs(m[k][x] - m[k + 4][x]);
    }
    return acc;
}

// ---- warp-cooperative block costs (all 32 lanes call; result valid in every lane) ----------

template <typename PA, typename PB>
__device__ __forceinline__ int warp_sad(const PA* __restrict__ a, int sa, const PB* __restrict__ b, int sb, int w, int h, int lane)
{
    int acc = 0;
    const int n = w * h;
    if ((w & (w - 1)) == 0)
    {
        const int lg = 31 - __clz(w);
        for (int i = lane; i < n; i += 32)
        {
            int y = i >> lg, x = i & (w - 1);
            acc += abs((int)a[y * sa + x] - (int)b[y * sb + x]);
        }
    }
    else
    {
        for (int i = lane; i < n; i += 32)
        {
            int y = i / w, x = i - y * w;
            acc += abs((int)a[y * sa + x] - (int)b[y * sb + x]);
        }
    }
    return warp_sum(acc);
}

// SATD with the reference's tiling (pixel.cpp:263-297, table :1134-1158): width % 8 == 0 -> 8x4
// tiles halved once per tile; otherwise 4x4 tiles halved per tile.
template <typename PA, typename PB>
__device__ __forceinline__ int warp_satd(const PA* __restrict__ a, int sa, const PB* __restrict__ b, int sb, int w, int h, int lane)
{
    int acc = 0;
    if ((w & 7) == 0)
    {
        const int tw = w >> 3, nt = tw * (h >> 2);
        for (int t = lane; t < nt; t += 32)
        {
            int ty = t / tw, tx = t - ty * tw;
            const PA* pa = a + (ty * 4) * sa + tx * 8; const PB* pb = b + (ty * 4) * sb + tx * 8;
            acc += (had4x4_abs(pa, sa, pb, sb) + had4x4_abs(pa + 4, sa, pb + 4, sb)) >> 1;
        }
    }
    else
    {
        const int tw = w >> 2, nt = tw * (h >> 2);
        for (int t = lane; t < nt; t += 32)
        {
            int ty = t / tw, tx = t - ty * tw;
            acc += had4x4_abs(a + (ty * 4) * sa + tx * 4, sa, b + (ty * 4) * sb + tx * 4, sb) >> 1;
        }
    }
    return warp_sum(acc);
}

// SA8D (pixel.cpp:336-377, table :1166-1170 and the chroma aliases): <8 -> satd; multiples of 16 ->
// 16x16 tiles rounded once; otherwise 8x8 tiles each rounded.
template <typename PA, typename PB>
__device__ __forceinline__ int warp_sa8d(const PA* __restrict__ a, int sa, const PB* __restrict__ b, int sb, int w, int h, int lane)
{
    if (w < 8 || h < 8) return warp_satd(a, sa, b, sb, w, h, lane);
    const int tw = w >> 3, nt = tw * (h >> 3);
    int acc = 0;
    if (((w | h) & 15) == 0)
    {
        // one lane per 8x8; the 4 lanes of a 16x16 tile are combined before rounding
        for (int t0 = 0; t0 < nt; t0 += 32)
        {
            int t = t0 + lane;
            int v = 0;
            // order 8x8 tiles so that 4 consecutive t form one 16x16: t = (tile16 * 4 + sub)
            if (t < nt)
            {
                int t16 = t >> 2, sub = t & 3;
                int tw16 = w >> 4;
                int y16 = t16 / tw16, x16 = t16 - y16 * tw16;
                int y = y16 * 16 + (sub >> 1) * 8, x = x16 * 16 + (sub & 1) * 8;
                v = had8x8_abs<PA, PB, false>(a + y * sa + x, sa, b + y * sb + x, sb);
            }
            v += __shfl_xor_sync(0xffffffffu, v, 1);
            v += __shfl_xor_sync(0xffffffffu, v, 2);
            if ((lane & 3) == 0 && t < nt) acc += (v + 2) >> 2;
        }
    }
    else
    {
        for (int t = lane; t < nt; t += 32)
        {
            int ty = t / tw, tx = t - ty * tw;
            acc += (had8x8_abs<PA, PB, false>(a + ty * 8 * sa + tx * 8, sa, b + ty * 8 * sb + tx * 8, sb) + 2) >> 2;
        }
    }
    return warp_sum(acc);
}

template <typename PA, typename PB>
__device__ __forceinline__ unsigned long long warp_sse(const PA* __restrict__ a, int sa, const PB* __restrict__ b, int sb, int w, int h, int lane)
{
    unsigned long long acc = 0;
    const int n = w * h;
    for (int i = lane; i < n; i += 32)
    {
        int y = i / w, x = i - y * w;
        int d = (int)a[y * sa + x] - (int)b[y * sb + x];
        acc += (unsigned)(d * d);
    }
    return warp_sum64(acc);
}

// psyCost_pp (pixel.cpp:726-757)
template <typename P>
__device__ __forceinline__ int warp_psy(const P* __restrict__ s, int ss, const P* __restrict__ r, int rs, int n, int lane)
{
    if (n == 4)
    {
        int v = 0;
        if (lane == 0)
        {
            int sadS = 0, sadR = 0;
            for (int y = 0; y < 4; y++) for (int x = 0; x < 4; x++) { sadS += s[y * ss + x]; sadR += r[y * rs + x]; }
            int es = (had4x4_abs_zero(s, ss) >> 1) - (sadS >> 2);
            int er = (had4x4_abs_zero(r, rs) >> 1) - (sadR >> 2);
            v = abs(es - er);
        }
        return __shfl_sync(0xffffffffu, v, 0);
    }
    const int tw = n >> 3, nt = tw * tw;
    int acc = 0;
    for (int t = lane; t < nt; t += 32)
    {
        int ty = t / tw, tx = t - ty * tw;
        const P* ps = s + ty * 8 * ss + tx * 8; const P* pr = r + ty * 8 * rs + tx * 8;
        int sadS = 0, sadR = 0;
        for (int y = 0; y < 8; y++) for (int x = 0; x < 8; x++) { sadS += ps[y * ss + x]; sadR += pr[y * rs + x]; }
        int es = ((had8x8_abs<P, P, true>(ps, ss, ps, ss) + 2) >> 2) - (sadS >> 2);
        int er = ((had8x8_abs<P, P, true>(pr, rs, pr, rs) + 2) >> 2) - (sadR >> 2);
        acc += abs(es - er);
    }
    return warp_sum(acc);
}

// ---- batched job-list kernel ---------------------------------------------------------------------------------
// One warp per job would keep 2 of 32 lanes busy on an 8x8 SATD and pay a 5-step reduction for 64 pixels of an 8x8 SAD.
// Instead a warp takes 32 consecutive jobs (one coalesced
// 1 KB read of the records), picks the SUB-GROUP width the largest of them needs -- lanes per job = pow2ceil(work units),
// units = 8x4 tiles for SATD, 8x8 tiles for SA8D / PSY, 16-pixel groups for the element-wise costs -- and runs
// 32 / width jobs side by side per pass; results go back to the lane that read the job, so the 32 outputs are one
// coalesced store.  width = 32 is exactly the old behaviour (64x64 blocks).  The arithmetic per job is unchanged.
__device__ __forceinline__ int grp_sum(int v, int lpj)
{
    for (int o = 1; o < lpj; o <<= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ unsigned long long grp_sum64(unsigned long long v, int lpj)
{
    for (int o = 1; o < lpj; o <<= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ uint32_t pc_ld32(uintptr_t a)          // 4 bytes at any alignment (planes have margins)
{
    const uint32_t* ap = (const uint32_t*)(a & ~(uintptr_t)3);
    const uint32_t sh = (uint32_t)(a & 3) * 8;
    const uint32_t lo = __ldg(ap);
    return sh ? __funnelshift_r(lo, __ldg(ap + 1), sh) : lo;
}

// SAD on packed words: 4 (8-bit) / 2 (16-bit) pixels per VABSDIFF4 / max-min pair
template <typename P>
__device__ __forceinline__ int grp_sad(const P* __restrict__ a, int sa, const P* __restrict__ b, int sb, int w, int h, int sub, int lpj)
{
    constexpr int PPW = 4 / (int)sizeof(P);                       // pixels per word
    const int wq = w / PPW, nq = wq * h;
    const bool p2 = (wq & (wq - 1)) == 0;                         // no integer division per word for the power-of-two widths
    const int lgq = 31 - __clz(wq);
    uint32_t acc = 0;
#pragma unroll 4
    for (int i = sub; i < nq; i += lpj)
    {
        const int y = p2 ? i >> lgq : i / wq, x = (i - y * wq) * PPW;
        const uint32_t wa = pc_ld32((uintptr_t)(a + y * sa + x)), wb = pc_ld32((uintptr_t)(b + y * sb + x));
        if (sizeof(P) == 1) acc = __vsadu4(wa, wb) + acc;
        else { const uint32_t t = __vmaxu2(wa, wb) - __vminu2(wa, wb); acc += (t & 0xffffu) + (t >> 16); }
    }
    return grp_sum((int)acc, lpj);
}

template <typename PA, typename PB>
__device__ __forceinline__ int grp_satd(const PA* __restrict__ a, int sa, const PB* __restrict__ b, int sb, int w, int h, int sub, int lpj)
{
    int acc = 0;
    if ((w & 7) == 0)
    {
        const int tw = w >> 3, nt = tw * (h >> 2);
        for (int t = sub; t < nt; t += lpj)
        {
            const int ty = t / tw, tx = t - ty * tw;
            const PA* pa = a + (ty * 4) * sa + tx * 8; const PB* pb = b + (ty * 4) * sb + tx * 8;
            acc += (had4x4_abs(pa, sa, pb, sb) + had4x4_abs(pa + 4, sa, pb + 4, sb)) >> 1;
        }
    }
    else
    {
        const int tw = w >> 2, nt = tw * (h >> 2);
        for (int t = sub; t < nt; t += lpj)
        {
            const int ty = t / tw, tx = t - ty * tw;
            acc += had4x4_abs(a + (ty * 4) * sa + tx * 4, sa, b + (ty * 4) * sb + tx * 4, sb) >> 1;
        }
    }
    return grp_sum(acc, lpj);
}

// `ntmax` = the largest 8x8-tile count among the jobs of this pass (warp-uniform): the 16x16 rounding combines four
// lanes by shuffles inside the loop, so every lane runs the same number of trips
template <typename PA, typename PB>
__device__ __forceinline__ int grp_sa8d(const PA* __restrict__ a, int sa, const PB* __restrict__ b, int sb, int w, int h, int sub, int lpj, int ntmax)
{
    const int tw = w >> 3, nt = tw * (h >> 3);
    const bool r16 = ((w | h) & 15) == 0;
    int acc = 0;
    for (int t0 = 0; t0 < ntmax; t0 += lpj)
    {
        const int t = t0 + sub;
        int v = 0;
        if (t < nt)
        {
            int y, x;
            if (r16)
            {   // four consecutive t form one 16x16
                const int t16 = t >> 2, q = t & 3, tw16 = w >> 4;
                const int y16 = t16 / tw16, x16 = t16 - y16 * tw16;
                y = y16 * 16 + (q >> 1) * 8; x = x16 * 16 + (q & 1) * 8;
            }
            else { const int ty = t / tw; y = ty * 8; x = (t - ty * tw) * 8; }
            v = had8x8_abs<PA, PB, false>(a + y * sa + x, sa, b + y * sb + x, sb);
        }
        const int v4 = v + __shfl_xor_sync(0xffffffffu, v, 1);
        const int v16 = v4 + __shfl_xor_sync(0xffffffffu, v4, 2);
        if (t < nt) acc += r16 ? ((sub & 3) == 0 ? (v16 + 2) >> 2 : 0) : (v + 2) >> 2;
    }
    return grp_sum(acc, lpj);
}

// sse_pp on packed words.  8-bit: |a - b| of four pixels (VABSDIFF4), squared and summed by ONE DP4A(d, d) into a 32-bit partial
// (a lane adds at most 4 * 255^2 per word and sees at most 1024 words of a 64x64 block: no overflow).  16-bit pixels: the two
// halves' differences (max - min, no borrow) squared and added in 64 bits.
template <typename P>
__device__ __forceinline__ unsigned long long grp_sse_pp(const P* __restrict__ a, int sa, const P* __restrict__ b, int sb, int w, int h, int sub, int lpj)
{
    constexpr int PPW = 4 / (int)sizeof(P);
    const int wq = w / PPW, nq = wq * h;
    const bool p2 = (wq & (wq - 1)) == 0;
    const int lgq = 31 - __clz(wq);
    unsigned long long acc = 0;
    uint32_t part = 0;
#pragma unroll 4
    for (int i = sub; i < nq; i += lpj)
    {
        const int y = p2 ? i >> lgq : i / wq, x = (i - y * wq) * PPW;
        const uint32_t wa = pc_ld32((uintptr_t)(a + y * sa + x)), wb = pc_ld32((uintptr_t)(b + y * sb + x));
        if (sizeof(P) == 1)
        {
            const uint32_t d = __vabsdiffu4(wa, wb);
            part = __dp4a(d, d, part);
        }
        else
        {
            const uint32_t t = __vmaxu2(wa, wb) - __vminu2(wa, wb);
            const uint32_t d0 = t & 0xffffu, d1 = t >> 16;
            acc += (unsigned long long)(d0 * d0) + (unsigned long long)(d1 * d1);
        }
    }
    acc += part;
    return grp_sum64(acc, lpj);
}

template <typename PA, typename PB>
__device__ __forceinline__ unsigned long long grp_sse(const PA* __restrict__ a, int sa, const PB* __restrict__ b, int sb, int w, int h, int sub, int lpj)
{
    unsigned long long acc = 0;
    const int n = w * h;
    const bool p2 = (w & (w - 1)) == 0;
    const int lgw = 31 - __clz(w);
#pragma unroll 4
    for (int i = sub; i < n; i += lpj)
    {
        const int y = p2 ? i >> lgw : i / w, x = i - y * w;
        const int d = (int)a[y * sa + x] - (int)b[y * sb + x];
        acc += (unsigned)(d * d);
    }
    return grp_sum64(acc, lpj);
}

template <typename P>
__device__ __forceinline__ int grp_psy(const P* __restrict__ s, int ss, const P* __restrict__ r, int rs, int n, int sub, int lpj)
{
    int acc = 0;
    if (n == 4)
    {
        if (sub == 0)
        {
            int sadS = 0, sadR = 0;
            for (int y = 0; y < 4; y++) for (int x = 0; x < 4; x++) { sadS += s[y * ss + x]; sadR += r[y * rs + x]; }
            const int es = (had4x4_abs_zero(s, ss) >> 1) - (sadS >> 2);
            const int er = (had4x4_abs_zero(r, rs) >> 1) - (sadR >> 2);
            acc = abs(es - er);
        }
        return grp_sum(acc, lpj);
    }
    const int tw = n >> 3, nt = tw * tw;
    for (int t = sub; t < nt; t += lpj)
    {
        const int ty = t / tw, tx = t - ty * tw;
        const P* ps = s + ty * 8 * ss + tx * 8; const P* pr = r + ty * 8 * rs + tx * 8;
        int sadS = 0, sadR = 0;
        for (int y = 0; y < 8; y++) for (int x = 0; x < 8; x++) { sadS += ps[y * ss + x]; sadR += pr[y * rs + x]; }
        const int es = ((had8x8_abs<P, P, true>(ps, ss, ps, ss) + 2) >> 2) - (sadS >> 2);
        const int er = ((had8x8_abs<P, P, true>(pr, rs, pr, rs) + 2) >> 2) - (sadR >> 2);
        acc += abs(es - er);
    }
    return grp_sum(acc, lpj);
}

// work units of a job for the sub-group width (see above)
__device__ __forceinline__ int pixelcmp_units(int op, int w, int h)
{
    switch (op)
    {
    case X265CU_SATD: return (w & 7) ? (w >> 2) * (h >> 2) : (w >> 3) * (h >> 2);
    case X265CU_SA8D: return (w < 8 || h < 8) ? ((w & 7) ? (w >> 2) * (h >> 2) : (w >> 3) * (h >> 2)) : max(4, (w >> 3) * (h >> 3));
    case X265CU_PSY:  return max(1, (w >> 3) * (w >> 3));
    default:          return max(1, (w * h) >> 4);
    }
}

// HAD = false: the element-wise costs (SAD, SSE, SSD_S, VAR); HAD = true: the Hadamard costs (SATD, SA8D, PSY).  Two
// instantiations because the 8x8 Hadamard needs 128 registers (16 resident warps per SM), which starved the latency-bound
// element-wise loops: on their own they need ~40 registers and run with 64 warps per SM.
template <typename P, bool HAD>
__global__ void __launch_bounds__(256) k_pixelcmp(int op, const P* __restrict__ A, const P* __restrict__ B,
                                                  const x265cu_cmp_job* __restrict__ jobs, int n, uint64_t* __restrict__ out, int lgChunk)
{
    // a warp takes 2^lgChunk consecutive jobs (32 for long lists; fewer when the list is too short to give every SM its warps)
    const int lane = threadIdx.x & 31;
    const int wpb = blockDim.x >> 5;
    const int nchunks = (n + (1 << lgChunk) - 1) >> lgChunk;
    for (int ch = blockIdx.x * wpb + (threadIdx.x >> 5); ch < nchunks; ch += gridDim.x * wpb)
    {
        const int j0 = ch << lgChunk, cnt = min(1 << lgChunk, n - j0);
        x265cu_cmp_job mine;
        mine.a_off = 0; mine.b_off = 0; mine.a_stride = 0; mine.b_stride = 0; mine.w = 4; mine.h = 4;
        if (lane < cnt) mine = jobs[j0 + lane];
        const int units = lane < cnt ? pixelcmp_units(op, mine.w, mine.h) : 1;
        const int umax = __reduce_max_sync(0xffffffffu, units);
        int lpj = 1;
        while (lpj < umax && lpj < 32) lpj <<= 1;
        const int lglpj = 31 - __clz(lpj), jpp = 32 >> lglpj;                  // jobs per pass
        const int sub = lane & (lpj - 1);
        uint64_t myres = 0;
        for (int pass = 0; pass < lpj && pass * jpp < cnt; pass++)
        {
            const int k = pass * jpp + (lane >> lglpj);                       // the job (lane of this chunk) my sub-group works on
            const int ks = min(k, cnt - 1);
            const long long a_off = __shfl_sync(0xffffffffu, (long long)mine.a_off, ks), b_off = __shfl_sync(0xffffffffu, (long long)mine.b_off, ks);
            const int sa = __shfl_sync(0xffffffffu, (int)mine.a_stride, ks), sb = __shfl_sync(0xffffffffu, (int)mine.b_stride, ks);
            const int wh = __shfl_sync(0xffffffffu, ((int)mine.w << 16) | (int)(uint16_t)mine.h, ks);
            const int w = wh >> 16, h = wh & 0xffff;
            uint64_t res = 0;
            switch (HAD ? op : (op == X265CU_SATD || op == X265CU_SA8D || op == X265CU_PSY ? -1 : op))
            {
            case X265CU_SAD:  res = (uint32_t)grp_sad<P>(A + a_off, sa, B + b_off, sb, w, h, sub, lpj); break;
            case X265CU_SATD: if (HAD) res = (uint32_t)grp_satd(A + a_off, sa, B + b_off, sb, w, h, sub, lpj); break;
            case X265CU_SA8D:
            if (HAD)
            {
                // blocks below 8x8 take the SATD path; a pass mixing both kinds would diverge around the in-loop shuffles
                const bool small = w < 8 || h < 8;
                const unsigned anySmall = __ballot_sync(0xffffffffu, small), anyBig = __ballot_sync(0xffffffffu, !small);
                const int nt = small ? 0 : (w >> 3) * (h >> 3);
                const int ntmax = __reduce_max_sync(0xffffffffu, nt);
                int v = 0;
                if (anyBig)  v = grp_sa8d(A + a_off, sa, B + b_off, sb, small ? 8 : w, small ? 8 : h, sub, lpj, ntmax);
                if (anySmall) { const int v2 = grp_satd(A + a_off, sa, B + b_off, sb, small ? w : 4, small ? h : 4, sub, lpj); if (small) v = v2; }
                res = (uint32_t)v;
            }
            break;
            case X265CU_SSE_PP:
            {
                const unsigned long long v = grp_sse_pp<P>(A + a_off, sa, B + b_off, sb, w, h, sub, lpj);
                res = PixTraits<P>::depth == 8 ? (uint64_t)(uint32_t)v : v;     // sse_t width (common.h:144-148)
                break;
            }
            case X265CU_SSE_SS:
            {
                const int16_t* a = (const int16_t*)A + a_off; const int16_t* b = (const int16_t*)B + b_off;
                const unsigned long long v = grp_sse(a, sa, b, sb, w, h, sub, lpj);
                res = PixTraits<P>::depth == 8 ? (uint64_t)(uint32_t)v : v;
                break;
            }
            case X265CU_SSD_S:
            {
                const int16_t* a = (const int16_t*)A + a_off;
                unsigned long long acc = 0;
                for (int i = sub; i < w * h; i += lpj) { const int y = i / w, x = i - y * w; const int v = a[y * sa + x]; acc += (unsigned)(v * v); }
                acc = grp_sum64(acc, lpj);
                res = PixTraits<P>::depth == 8 ? (uint64_t)(uint32_t)acc : acc;
                break;
            }
            case X265CU_VAR:
            {
                const P* a = A + a_off;
                unsigned s = 0, q = 0;
                for (int i = sub; i < w * h; i += lpj) { const int y = i / w, x = i - y * w; const unsigned v = a[y * sa + x]; s += v; q += v * v; }
                s = (unsigned)grp_sum((int)s, lpj); q = (unsigned)grp_sum((int)q, lpj);
                res = (uint64_t)s + ((uint64_t)q << 32);
                break;
            }
            case X265CU_PSY: if (HAD) res = (uint32_t)grp_psy(A + a_off, sa, B + b_off, sb, w, sub, lpj); break;
            }
            // hand the result to the lane that owns job k: lane L's job was worked on in pass L / jpp by sub-group L % jpp
            const unsigned long long got = __shfl_sync(0xffffffffu, (unsigned long long)res, (lane & (jpp - 1)) << lglpj);
            if ((lane >> (5 - lglpj)) == pass) myres = got;
        }
        if (lane < cnt) out[j0 + lane] = myres;
    }
}

static int launch_pixelcmp(x265cu_ctx* ctx, int depth, int op, const void* A, const void* B,
                           const x265cu_cmp_job* jobs, int n, uint64_t* out)
{
    if (n <= 0) return 0;
    const int threads = 256, wpb = threads / 32;
    // jobs per warp chunk: 32 when that still leaves every SM ~32 warps of work, else the largest power of two that does
    int lgChunk = 5;
    while (lgChunk > 0 && (n >> lgChunk) < ctx->sm_count * 32) lgChunk--;
    const int nchunks = (n + (1 << lgChunk) - 1) >> lgChunk;
    int blocks = (nchunks + wpb - 1) / wpb;
    int maxb = ctx->sm_count * 8;
    if (blocks > maxb) blocks = maxb;
    const bool had = op == X265CU_SATD || op == X265CU_SA8D || op == X265CU_PSY;
    if (depth == 8)
    {
        if (had) k_pixelcmp<uint8_t, true><<<blocks, threads, 0, ctx->stream>>>(op, (const uint8_t*)A, (const uint8_t*)B, jobs, n, out, lgChunk);
        else     k_pixelcmp<uint8_t, false><<<blocks, threads, 0, ctx->stream>>>(op, (const uint8_t*)A, (const uint8_t*)B, jobs, n, out, lgChunk);
    }
    else
    {
        if (had) k_pixelcmp<uint16_t, true><<<blocks, threads, 0, ctx->stream>>>(op, (const uint16_t*)A, (const uint16_t*)B, jobs, n, out, lgChunk);
        else     k_pixelcmp<uint16_t, false><<<blocks, threads, 0, ctx->stream>>>(op, (const uint16_t*)A, (const uint16_t*)B, jobs, n, out, lgChunk);
    }
    CU_LAUNCH_CHECK(ctx);
    return 0;
}
