// x265_b200/csrc/frame.cuh -- frame-level fused kernels of the CTU-analysis pipeline (DESIGN.md):
//   k_build_me_jobs : PU geometry table + predictor field -> motionEstimate jobs
//                     (Search::setSearchRange search.cpp:2724-2768, CUData::clipMv cudata.cpp:1915-1928)
//   k_intra_search  : per CU (8/16/32): neighbours from the source plane, 1:2:1 filter, 35 predictions
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

template <typename P>
__global__ void __launch_bounds__(256) k_intra_search(const P* __restrict__ fenc, int stride, const CuDesc* __restrict__ cus, int ncu,
                                                      uint32_t* __restrict__ intra_cost)
{
    constexpr int maxv = PixTraits<P>::maxv;
    __shared__ int16_t s_nb[129], s_filt[129];
    __shared__ uint32_t s_cost[36];
    __shared__ int s_dc;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
    const int grp = lane >> 3, row = lane & 7;
    for (int c = blockIdx.x; c < ncu; c += gridDim.x)
    {
        const CuDesc cu = cus[c];
        const int S = cu.size;
        uint32_t* out = intra_cost + (size_t)c * 36;
        if (S == 64) { if (tid < 36) out[tid] = 0; continue; }
        const int lg = 31 - __clz(S), N2 = 2 * S;
        const P* o = fenc + (size_t)cu.y * stride + cu.x;
        __syncthreads();
        for (int i = tid; i < 4 * S + 1; i += blockDim.x)
        {
            int v;
            if (i == 0) v = o[-stride - 1];
            else if (i <= N2) v = o[-stride + (i - 1)];
            else v = o[(ptrdiff_t)(i - N2 - 1) * stride - 1];
            s_nb[i] = (int16_t)v;
        }
        __syncthreads();
        for (int i = tid; i < 4 * S + 1; i += blockDim.x) s_filt[i] = (int16_t)intra_filter_elem(s_nb, i, S);
        if (tid == 0)
        {
            int sum = S;
            for (int i = 0; i < S; i++) sum += s_nb[1 + i] + s_nb[N2 + 1 + i];
            s_dc = sum / N2;
        }
        __syncthreads();
        const int dc = s_dc;
        const int bFilter = S <= 16;
        if (S == 8)
        {   // 4 modes per warp pass: lane group g -> mode, lane row -> block row
            for (int m0 = warp * 4; m0 < 35; m0 += nwarps * 4)
            {
                const int mode = min(m0 + grp, 34);
                const int16_t* nbs = intra_use_filtered(mode, S) ? s_filt : s_nb;
                int d[8];
#pragma unroll
                for (int x = 0; x < 8; x++)
                    d[x] = (int)o[(size_t)row * stride + x] - intra_pixel(nbs, S, lg, mode, bFilter, dc, row, x, maxv);
                int raw = had8_group(d, lane);
                if (row == 0 && m0 + grp < 35) s_cost[m0 + grp] = (uint32_t)((raw + 2) >> 2);
            }
        }
        else
        {   // one mode per warp pass; 4 tiles (one 16x16) per pass: group g -> 8x8 tile of the 16x16
            for (int mode = warp; mode < 35; mode += nwarps)
            {
                const int16_t* nbs = intra_use_filtered(mode, S) ? s_filt : s_nb;
                int total = 0;
                for (int by = 0; by < S; by += 16)
                    for (int bx = 0; bx < S; bx += 16)
                    {
                        const int y = by + (grp >> 1) * 8 + row, x0 = bx + (grp & 1) * 8;
                        int d[8];
#pragma unroll
                        for (int x = 0; x < 8; x++)
                            d[x] = (int)o[(size_t)y * stride + x0 + x] - intra_pixel(nbs, S, lg, mode, bFilter, dc, y, x0 + x, maxv);
                        int raw = had8_group(d, lane);
                        raw += __shfl_xor_sync(0xffffffffu, raw, 8);
                        raw += __shfl_xor_sync(0xffffffffu, raw, 16);
                        total += (raw + 2) >> 2;                       // sa8d_16x16 rounds once per 16x16 (pixel.cpp:341-351)
                    }
                if (lane == 0) s_cost[mode] = (uint32_t)total;
            }
        }
        __syncthreads();
        if (tid < 35) out[tid] = s_cost[tid];
        if (tid == 0)
        {
            uint32_t bc = 0xffffffffu; int bm = 0;
            for (int m = 0; m < 35; m++) if (s_cost[m] < bc) { bc = s_cost[m]; bm = m; }
            out[35] = (uint32_t)bm;
        }
    }
}
