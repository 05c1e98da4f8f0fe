// x265_b200/csrc/frame.cuh -- frame-level fused kernels of the CTU-analysis pipeline (DESIGN.md):
//   k_build_me_jobs : PU geometry table + predictor field -> motionEstimate jobs
//                     (Search::setSearchRange search.cpp:2724-2768, CUData::clipMv cudata.cpp:1915-1928)
//   k_intra_cu      : per CU (8/16/32): neighbours from the source plane, 1:2:1 filter, 35 predictions
//                     evaluated in registers, SA8D by an 8-lane shuffle Hadamard (search.cpp:1358-1444)
// The residual chain of the luma and chroma planes (k_cu_residual) is in resid.cuh.
#pragma once
#include "common.cuh"
#include "interp.cuh"
#include "intra.cuh"

#include "geometry.h"        // PuDesc / CuDesc / TuDesc and the host-side table builder

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return min(max(v, lo), hi); }

__global__ void __launch_bounds__(256) k_build_me_jobs(const PuDesc* __restrict__ pus, int n, const int16_t* __restrict__ field,
                                                       int fw, int fh, int width, int height, int stride,
                                                       int method, int subme, int merange, x265cu_me_job* __restrict__ jobs)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const PuDesc d = pus[i];
    const int y = d.offset / stride, x = d.offset - y * stride;
    const int bx = x >> 4, by = y >> 4, r = d.ref;
    const int16_t* f  = field + ((size_t)(r * fh + by) * fw + bx) * 2;
    const int16_t* fr = field + ((size_t)(r * fh + by) * fw + clampi(bx + 1, 0, fw - 1)) * 2;
    const int16_t* fb = field + ((size_t)(r * fh + clampi(by + 1, 0, fh - 1)) * fw + bx) * 2;
    x265cu_me_job j;
    j.offset = d.offset; j.ref = d.ref; j.pw = d.pw; j.ph = d.ph;
    j.qmvp[0] = f[0]; j.qmvp[1] = f[1];
    j.mvc[0] = fr[0]; j.mvc[1] = fr[1]; j.mvc[2] = fb[0]; j.mvc[3] = fb[1];
    j.mvc[4] = j.mvc[5] = j.mvc[6] = j.mvc[7] = 0;
    j.numCand = 2; j.method = (int8_t)method; j.subme = (int8_t)subme; j.merange = (int8_t)merange;
    const int dist = merange << 2;
    const int xmax = (width + 8 - d.cuX - 1) << 2, xmin = -((64 + 8 + d.cuX - 1) << 2);
    const int ymax = (height + 8 - d.cuY - 1) << 2, ymin = -((64 + 8 + d.cuY - 1) << 2);
    int mnx = clampi(f[0] - dist, xmin, xmax) >> 2, mxx = clampi(f[0] + dist, xmin, xmax) >> 2;
    int mny = clampi(f[1] - dist, ymin, ymax) >> 2, mxy = clampi(f[1] + dist, ymin, ymax) >> 2;
    if (mxy < mny) mxy = mny;
    j.mvmin[0] = (int16_t)mnx; j.mvmin[1] = (int16_t)mny; j.mvmax[0] = (int16_t)mxx; j.mvmax[1] = (int16_t)mxy;
    jobs[i] = j;
}

// {cost, mvx, mvy, 0} int32 x4 -> {cost int32, mvx int16, mvy int16}: what the host mode decision reads back
__global__ void k_pack_me(const int32_t* __restrict__ me_out, int n, int2* __restrict__ packed)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int4 v = ((const int4*)me_out)[i];
    packed[i] = make_int2(v.x, (int)(((uint32_t)(uint16_t)(int16_t)v.y) | ((uint32_t)(uint16_t)(int16_t)v.z << 16)));
}

// ---------------------------------------------------------------------------------------------
// closed-form intra prediction of one pixel (intrapred.cpp:53-204); nb/filt in shared memory
__device__ __forceinline__ int intra_pixel(const int16_t* __restrict__ nbs, int N, int lg, int mode, int bFilter, int dc, int y, int x, int maxv)
{
    const int N2 = 2 * N;
    if (mode == 0)
        return ((N - 1 - x) * nbs[N2 + 1 + y] + (N - 1 - y) * nbs[1 + x] + (x + 1) * nbs[1 + N] + (y + 1) * nbs[N2 + 1 + N] + N) >> (lg + 1);
    if (mode == 1)
    {
        if (bFilter)
        {
            if (x == 0 && y == 0) return (nbs[1] + nbs[N2 + 1] + 2 * dc + 2) >> 2;
            if (y == 0) return (nbs[1 + x] + 3 * dc + 2) >> 2;
            if (x == 0) return (nbs[N2 + 1 + y] + 3 * dc + 2) >> 2;
        }
        return dc;
    }
    const bool hor = mode < 18;
    const int angOff = hor ? 10 - mode : mode - 26;
    const int angle = c_angle[8 + angOff];
    const int mainBase = hor ? N2 + 1 : 1, sideBase = hor ? 1 : N2 + 1;
    const int r = hor ? x : y, c = hor ? y : x;           // vertical-family frame coordinates
    if (angle == 0)
    {
        int v = nbs[mainBase + c];
        if (bFilter && c == 0) v = clip3i(0, maxv, (int)(int16_t)(nbs[mainBase] + ((nbs[sideBase + r] - nbs[0]) >> 1)));
        return v;
    }
    const int pos = (r + 1) * angle, o = pos >> 5, f = pos & 31;
    const int inv = angle < 0 ? c_invAngle[-angOff - 1] : 0;
    auto ref_at = [&](int idx) -> int {
        if (idx >= 0) return nbs[mainBase + idx];
        if (idx == -1) return nbs[0];
        const int i = -idx - 2;                                    // projected side neighbours (intrapred.cpp:150-160)
        return nbs[sideBase - 1 + ((128 + (i + 1) * inv) >> 8)];
    };
    const int a = ref_at(o + c);
    if (!f) return a;
    return ((32 - f) * a + f * ref_at(o + c + 1) + 16) >> 5;
}

// 8x8 Hadamard abs-sum over an 8-lane group: each lane holds one row of differences
__device__ __forceinline__ int had8_group(int d[8], int lane)
{
    had4(d[0], d[1], d[2], d[3]); had4(d[4], d[5], d[6], d[7]);
#pragma unroll
    for (int k = 0; k < 4; k++) { int p = d[k], q = d[k + 4]; d[k] = p + q; d[k + 4] = p - q; }
#pragma unroll
    for (int s = 1; s < 8; s <<= 1)
    {
#pragma unroll
        for (int k = 0; k < 8; k++)
        {
            int v = __shfl_xor_sync(0xffffffffu, d[k], s);
            d[k] = (lane & s) ? (v - d[k]) : (d[k] + v);
        }
    }
    int acc = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) acc += abs(d[k]);
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    acc += __shfl_xor_sync(0xffffffffu, acc, 2);
    acc += __shfl_xor_sync(0xffffffffu, acc, 4);
    return acc;          // raw 8x8 sum, identical in the 8 lanes of the group
}

// ---- intra mode search of the frame analyser (search.cpp:1358-1444): per CU of 8, 16 or 32 the 35 modes' SA8D costs and the
// best mode, ties to the lowest.  Neighbours come from the source plane (like slicetype.cpp:729-733) and are 1:2:1 filtered
// for the modes intra_use_filtered picks (no strong smoothing at 32x32); DC and angle-0 edge filters only for S <= 16.
// A WARP per 8x8 CU or per 16x16 quadrant of a CU: S = 8 and 16 take one warp per CU and several CUs per CTA, with warp
// barriers only; S = 32 takes a 4-warp CTA.  Lanes hold 8 pixels of one row of an 8x8 tile (had8_group's layout), and both
// that source row and the matching row of the transposed source block, loaded once.  Angular modes are predicted by
// intra_ang_item in the vertical-family frame, so a horizontal mode's block comes out transposed and is compared with the
// transposed source: the sum of absolute 8x8 Hadamard coefficients does not change under transposition, and the
// transpose maps 8x8 tiles onto 8x8 tiles and 16x16 rounding groups onto 16x16 groups (the reference's m_fencTransposed,
// search.cpp:1379).  Planar and DC are evaluated per pixel.
// Predicted pixels x0 .. x0 + 7 of row r of mode `mode` of an S x S block: planar and DC in the picture frame, angular
// modes in the vertical-family frame (refbuf built by intra_ang_ref)
template <typename P, int S>
__device__ __forceinline__ void intra_row8(const P* nbs, const P* refbuf, int mode, int dc, int r, int x0, int pred[8])
{
    constexpr int N2 = 2 * S, lg = S == 8 ? 3 : (S == 16 ? 4 : 5), bFilter = S <= 16;
    constexpr int UW = 2 * (int)sizeof(P);                        // 8 pixels per item
    if (mode >= 2)
    {
        uint32_t o32[UW];
        intra_ang_item<P, UW>(refbuf, nbs, S, mode, bFilter, r, x0, o32);
#pragma unroll
        for (int k = 0; k < 8; k++)
            pred[k] = sizeof(P) == 1 ? (int)((o32[k >> 2] >> (8 * (k & 3))) & 0xffu) : (int)((o32[k >> 1] >> (16 * (k & 1))) & 0xffffu);
    }
    else if (mode == 1)
    {
#pragma unroll
        for (int k = 0; k < 8; k++)
        {
            const int x = x0 + k;
            int v = dc;
            if (bFilter)
            {
                if (x == 0 && r == 0) v = ((int)nbs[1] + (int)nbs[N2 + 1] + 2 * dc + 2) >> 2;
                else if (r == 0)      v = ((int)nbs[1 + x] + 3 * dc + 2) >> 2;
                else if (x == 0)      v = ((int)nbs[N2 + 1 + r] + 3 * dc + 2) >> 2;
            }
            pred[k] = v;
        }
    }
    else
    {
        const int left = nbs[N2 + 1 + r], tr = nbs[1 + S], bl = nbs[N2 + 1 + S];
#pragma unroll
        for (int k = 0; k < 8; k++)
        {
            const int x = x0 + k;
            pred[k] = ((S - 1 - x) * left + (S - 1 - r) * (int)nbs[1 + x] + (x + 1) * tr + (r + 1) * bl + S) >> (lg + 1);
        }
    }
}

template <typename P, int S>
__global__ void __launch_bounds__(128) k_intra_cu(const P* __restrict__ fenc, int stride, const CuDesc* __restrict__ cus,
                                                  const int32_t* __restrict__ list, int n, uint32_t* __restrict__ intra_cost)
{
    constexpr int QW = S == 32 ? 4 : 1;                           // warps per CU
    constexpr int CPB = 4 / QW;                                   // CUs per 128-thread CTA
    constexpr int NB = (4 * S + 1 + 7) & ~7;                      // neighbour array, padded
    constexpr int SLOTS = S == 8 ? 4 : 1;                         // modes a warp evaluates side by side
    constexpr int RB = (3 * S + 12 + 7) & ~7;                     // projected reference row (intra_ang_item)
    constexpr int N2 = 2 * S;
    __shared__ __align__(16) P s_nb[CPB][2][NB];                  // [CU][unfiltered, filtered]
    __shared__ __align__(16) P s_ref[4][SLOTS][RB];               // per warp
    __shared__ uint32_t s_part[S == 32 ? 4 : 1][36];              // S = 32: per-quadrant costs
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int cslot = warp / QW, q = warp % QW, gt = threadIdx.x % (32 * QW);
    const int grp = lane >> 3, row = lane & 7;
    for (int i = blockIdx.x * CPB + cslot; i < n; i += gridDim.x * CPB)
    {
        const int c = list[i];
        const CuDesc cu = cus[c];
        const P* o = fenc + (ptrdiff_t)cu.y * stride + cu.x;
        P* nb = s_nb[cslot][0]; P* nf = s_nb[cslot][1];
        if (QW == 1) __syncwarp(); else __syncthreads();          // the previous CU's neighbours have been read
        for (int k = gt; k < 4 * S + 1; k += 32 * QW)
            nb[k] = k == 0 ? o[-stride - 1] : (k <= N2 ? o[-stride + (k - 1)] : o[(ptrdiff_t)(k - N2 - 1) * stride - 1]);
        if (QW == 1) __syncwarp(); else __syncthreads();
        for (int k = gt; k < 4 * S + 1; k += 32 * QW) nf[k] = (P)intra_filter_elem(nb, k, S);
        int dsum = 0;
        for (int k = lane; k < N2; k += 32) dsum += k < S ? nb[1 + k] : nb[N2 + 1 + k - S];
        const int dc = (warp_sum(dsum) + S) / N2;
        if (QW == 1) __syncwarp(); else __syncthreads();
        // this lane's 8x8 tile: S = 8 the CU; else tile grp of the warp's 16x16 quadrant q
        const int ty = S == 8 ? 0 : (q >> 1) * 16 + (grp >> 1) * 8, tx = S == 8 ? 0 : (q & 1) * 16 + (grp & 1) * 8;
        const int r = ty + row;
        int src[8], srcT[8];
#pragma unroll
        for (int k = 0; k < 8; k++) { src[k] = o[(ptrdiff_t)r * stride + tx + k]; srcT[k] = o[(ptrdiff_t)(tx + k) * stride + r]; }
        uint32_t* out = intra_cost + (size_t)c * 36;
        uint32_t best = 0xffffffffu;
        P* refbuf = s_ref[warp][S == 8 ? grp : 0];
        for (int m0 = 0; m0 < 35; m0 += SLOTS)
        {
            const int m = m0 + (S == 8 ? grp : 0), mode = min(m, 34);
            const P* nbs = intra_use_filtered(mode, S) ? nf : nb;
            __syncwarp();                                         // the previous mode's reference row has been read
            if (mode >= 2) intra_ang_ref<P>(refbuf, nbs, S, mode, S == 8 ? row : lane, S == 8 ? 8 : 32);
            __syncwarp();
            int pred[8], d[8];
            intra_row8<P, S>(nbs, refbuf, mode, dc, r, tx, pred);
            const bool tr = mode >= 2 && mode < 18;               // horizontal: transposed block against the transposed source
#pragma unroll
            for (int k = 0; k < 8; k++) d[k] = (tr ? srcT[k] : src[k]) - pred[k];
            int raw = had8_group(d, lane);
            uint32_t cost;
            if (S == 8) cost = (uint32_t)((raw + 2) >> 2);        // sa8d_8x8 rounds per 8x8 (pixel.cpp:341-351)
            else
            {
                raw += __shfl_xor_sync(0xffffffffu, raw, 8);
                raw += __shfl_xor_sync(0xffffffffu, raw, 16);
                cost = (uint32_t)((raw + 2) >> 2);                // sa8d_16x16 rounds once per 16x16
            }
            if (S == 32) { if (lane == 0) s_part[q][m] = cost; }
            else if (m < 35)
            {
                if (row == 0) out[m] = cost;
                best = min(best, (cost << 6) | (uint32_t)m);
            }
        }
        if (S == 32)
        {
            __syncthreads();
            if (warp == 0)
            {
                for (int m = lane; m < 35; m += 32)
                {
                    const uint32_t cost = s_part[0][m] + s_part[1][m] + s_part[2][m] + s_part[3][m];
                    out[m] = cost;
                    best = min(best, (cost << 6) | (uint32_t)m);
                }
            }
        }
        // costs stay below 2^26 (a 32x32 10-bit block: 16 groups of at most 2^19 after rounding), so (cost << 6) | mode is
        // an exact arg-min key with ties to the lowest mode
        if (warp == cslot * QW)
        {
            best = __reduce_min_sync(0xffffffffu, best);
            if (lane == 0) out[35] = best & 63u;
        }
    }
}

// CU 64 rows of the intra table: zeros (no intra search at 64x64)
__global__ void k_intra_zero(const int32_t* __restrict__ list, int n, uint32_t* __restrict__ intra_cost)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n * 36) intra_cost[(size_t)list[i / 36] * 36 + i % 36] = 0;
}

template <typename P, int S>
static int intra_launch(x265cu_ctx* c, const void* fenc, int stride, const CuDesc* cus, const int32_t* list, int n, uint32_t* intra_cost)
{
    if (n == 0) return 0;
    constexpr int CPB = S == 32 ? 1 : 4;
    k_intra_cu<P, S><<<min((n + CPB - 1) / CPB, c->sm_count * 16), 128, 0, c->stream>>>((const P*)fenc, stride, cus, list, n, intra_cost);
    CU_LAUNCH_CHECK(c);
    return 0;
}

// one launch per CU size over its own list (lists[k] = CUs of size 8 << k, n[k] entries); CU and intra table indices are absolute
template <typename P>
static int launch_intra(x265cu_ctx* c, const void* fenc, int stride, const CuDesc* cus, const int32_t* const lists[4], const int n[4],
                        uint32_t* intra_cost)
{
    if (intra_launch<P, 8>(c, fenc, stride, cus, lists[0], n[0], intra_cost) ||
        intra_launch<P, 16>(c, fenc, stride, cus, lists[1], n[1], intra_cost) ||
        intra_launch<P, 32>(c, fenc, stride, cus, lists[2], n[2], intra_cost)) return -1;
    if (n[3])
    {
        k_intra_zero<<<(n[3] * 36 + 255) / 256, 256, 0, c->stream>>>(lists[3], n[3], intra_cost);
        CU_LAUNCH_CHECK(c);
    }
    return 0;
}
