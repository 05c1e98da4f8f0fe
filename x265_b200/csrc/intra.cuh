// x265_b200/csrc/intra.cuh -- intra prediction class (DC, planar, angular 2..34, all-angs, 1:2:1 filter).
// Semantics: /root/reference/source/common/intrapred.cpp:31-51 (filter), :53-85 (DC), :87-100 (planar),
// :102-204 (angular), :206-234 (all-angs).  Neighbour layout: [0]=top-left, [1..2N]=top(+right),
// [2N+1..4N]=left(+bottom).
#pragma once
#include "common.cuh"
#include "interp.cuh"

__constant__ int8_t  c_angle[17]   = { -32, -26, -21, -17, -13, -9, -5, -2, 0, 2, 5, 9, 13, 17, 21, 26, 32 };
__constant__ int16_t c_invAngle[8] = { 4096, 1638, 910, 630, 482, 390, 315, 256 };

// which TU sizes use the filtered neighbours for an angular / planar mode (constants.cpp:561,
// HEVC 8.4.4.2.3): min(|m-26|,|m-10|) > thr(N), thr = 7 (N=8), 1 (N=16), 0 (N=32); never N=4 / DC.
__device__ __forceinline__ bool intra_use_filtered(int mode, int N)
{
    if (mode == 1 || N == 4) return false;
    if (mode == 0) return N >= 8;
    int d = min(abs(mode - 26), abs(mode - 10));
    int thr = N == 8 ? 7 : (N == 16 ? 1 : 0);
    return d > thr;
}

// Cooperative predictor.  nbs: neighbours in shared memory (4N+1), ref: shared scratch >= 3N+2.
// Writes an N x N block; `vframe` = leave horizontal modes untransposed (all-angs storage).
// Must be called by all threads of the CTA (contains __syncthreads()).
template <typename P>
__device__ void intra_predict_block(const int16_t* nbs, int16_t* refbuf, P* __restrict__ dst, int64_t dstStride,
                                    int N, int mode, int bFilter, bool vframe)
{
    constexpr int maxv = PixTraits<P>::maxv;
    const int lg = 31 - __clz(N), N2 = 2 * N;
    if (mode == 0)
    {
        const int tr = nbs[1 + N], bl = nbs[N2 + 1 + N];
        for (int i = threadIdx.x; i < N * N; i += blockDim.x)
        {
            int y = i >> lg, x = i & (N - 1);
            dst[y * dstStride + x] = (P)(((N - 1 - x) * nbs[N2 + 1 + y] + (N - 1 - y) * nbs[1 + x] + (x + 1) * tr + (y + 1) * bl + N) >> (lg + 1));
        }
        return;
    }
    if (mode == 1)
    {
        int sum = N;
        for (int i = 0; i < N; i++) sum += nbs[1 + i] + nbs[N2 + 1 + i];
        const int dc = sum / N2;
        for (int i = threadIdx.x; i < N * N; i += blockDim.x)
        {
            int y = i >> lg, x = i & (N - 1);
            int v = dc;
            if (bFilter)
            {
                if (x == 0 && y == 0) v = (nbs[1] + nbs[N2 + 1] + 2 * dc + 2) >> 2;
                else if (y == 0)      v = (nbs[1 + x] + 3 * dc + 2) >> 2;
                else if (x == 0)      v = (nbs[N2 + 1 + y] + 3 * dc + 2) >> 2;
            }
            dst[y * dstStride + x] = (P)v;
        }
        return;
    }
    const bool hor = mode < 18;
    const int angOff = hor ? 10 - mode : mode - 26;
    const int angle = c_angle[8 + angOff];
    // main/side edges in the vertical-family frame
    const int mainBase = hor ? N2 + 1 : 1;     // nbs[mainBase + i], i = 0..2N-1
    const int sideBase = hor ? 1 : N2 + 1;
    if (angle == 0)
    {
        for (int i = threadIdx.x; i < N * N; i += blockDim.x)
        {
            int r = i >> lg, c = i & (N - 1);
            int v = nbs[mainBase + c];
            if (bFilter && c == 0) v = clip3i(0, maxv, (int)(int16_t)(nbs[mainBase] + ((nbs[sideBase + r] - nbs[0]) >> 1)));
            int y = (hor && !vframe) ? c : r, x = (hor && !vframe) ? r : c;
            dst[y * dstStride + x] = (P)v;
        }
        return;
    }
    // reference line: refbuf[off + 1 + idx] holds ref[idx], idx in [-N-1 .. 2N]
    const int off = N + 1;
    __syncthreads();
    if (angle < 0)
    {
        const int nproj = -((N * angle) >> 5) - 1;
        const int inv = c_invAngle[-angOff - 1];
        for (int i = threadIdx.x; i < nproj; i += blockDim.x)
            refbuf[off + 1 + (-2 - i)] = nbs[sideBase - 1 + ((128 + (i + 1) * inv) >> 8)];     // side[k-1], k = acc>>8
        for (int i = threadIdx.x; i < N + 1; i += blockDim.x)
            refbuf[off + 1 + (-1 + i)] = (i == 0) ? nbs[0] : nbs[mainBase + i - 1];
    }
    else
    {
        for (int i = threadIdx.x; i < N2; i += blockDim.x) refbuf[off + 1 + i] = nbs[mainBase + i];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < N * N; i += blockDim.x)
    {
        int r = i >> lg, c = i & (N - 1);
        int pos = (r + 1) * angle;
        int o = pos >> 5, f = pos & 31;
        int a = refbuf[off + 1 + o + c];
        int v = f ? (((32 - f) * a + f * refbuf[off + 1 + o + c + 1] + 16) >> 5) : a;
        int y = (hor && !vframe) ? c : r, x = (hor && !vframe) ? r : c;
        dst[y * dstStride + x] = (P)v;
    }
}

// 1:2:1 neighbour smoothing (intrapred.cpp:31-51), element i of 4N+1
template <typename T>
__device__ __forceinline__ int intra_filter_elem(const T* s, int i, int N)
{
    const int N2 = 2 * N, N4 = 4 * N;
    if (i == 0) return (2 * (int)s[0] + (int)s[1] + (int)s[N2 + 1] + 2) >> 2;
    if (i == N2 || i == N4) return s[i];
    if (i == N2 + 1) return (2 * (int)s[N2 + 1] + (int)s[0] + (int)s[N2 + 2] + 2) >> 2;
    return (2 * (int)s[i] + (int)s[i - 1] + (int)s[i + 1] + 2) >> 2;
}

template <typename P>
__global__ void __launch_bounds__(256) k_intra_pred(int N, const P* __restrict__ nb, int64_t nb_pitch, P* __restrict__ dst, int64_t dst_pitch,
                                                    int dst_stride, const x265cu_intra_job* __restrict__ jobs, int n)
{
    __shared__ int16_t s_nb[129];
    __shared__ int16_t s_ref[128];
    for (int j = blockIdx.x; j < n; j += gridDim.x)
    {
        __syncthreads();
        for (int i = threadIdx.x; i < 4 * N + 1; i += blockDim.x) s_nb[i] = nb[j * nb_pitch + i];
        __syncthreads();
        intra_predict_block<P>(s_nb, s_ref, dst + j * dst_pitch, dst_stride, N, jobs[j].mode, jobs[j].bFilter, false);
    }
}

// one WARP per neighbour array (4N+1 <= 129 elements): no shared staging, no CTA barriers (a CTA per job would pay two
// __syncthreads for 65 elements)
template <typename P>
__global__ void __launch_bounds__(256) k_intra_filter(int N, const P* __restrict__ nb, P* __restrict__ filt, int64_t pitch, int n)
{
    const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
    const int N2 = 2 * N, N4 = 4 * N;
    for (int j = blockIdx.x * wpb + (threadIdx.x >> 5); j < n; j += gridDim.x * wpb)
    {
        const P* s = nb + j * pitch;
        P* d = filt + j * pitch;
        for (int i = lane; i <= N4; i += 32)
        {
            int v;
            if (i == 0) v = (2 * (int)s[0] + (int)s[1] + (int)s[N2 + 1] + 2) >> 2;
            else if (i == N2 || i == N4) v = s[i];
            else if (i == N2 + 1) v = (2 * (int)s[N2 + 1] + (int)s[0] + (int)s[N2 + 2] + 2) >> 2;
            else v = (2 * (int)s[i] + (int)s[i - 1] + (int)s[i + 1] + 2) >> 2;
            d[i] = (P)v;
        }
    }
}

// all-angs, one CTA per block: the neighbours (unfiltered and filtered) are staged once, each of the 8 warps takes
// every 8th mode, a lane produces 4 consecutive pixels of a row and stores them with one 4 / 8-byte store
// (33*N*N contiguous per job, 128 contiguous bytes per warp store).  Same per-pixel arithmetic as
// intra_predict_block (intrapred.cpp:102-234).
template <typename P>
__global__ void __launch_bounds__(256) k_intra_allangs_cta(int N, const P* __restrict__ refp, const P* __restrict__ filtp, int64_t nb_pitch,
                                                           P* __restrict__ dst, int bLuma, int n)
{
    constexpr int maxv = PixTraits<P>::maxv;
    __shared__ int16_t s_nb[2][132];
    __shared__ int16_t s_ref[8][132];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int lg = 31 - __clz(N), N2 = 2 * N, upr = N >> 2, nunits = (N * N) >> 2;      // units of 4 pixels
    for (int j = blockIdx.x; j < n; j += gridDim.x)
    {
        __syncthreads();
        for (int i = threadIdx.x; i < 2 * (4 * N + 1); i += blockDim.x)
        {
            const int which = i >= 4 * N + 1, e = which ? i - (4 * N + 1) : i;
            s_nb[which][e] = (int16_t)(which ? filtp : refp)[j * nb_pitch + e];
        }
        __syncthreads();
        int16_t* refbuf = s_ref[warp];
        for (int mode = 2 + warp; mode < 35; mode += 8)
        {
            const int16_t* nbs = s_nb[intra_use_filtered(mode, N) ? 1 : 0];
            P* out = dst + ((int64_t)j * 33 + (mode - 2)) * N * N;
            const bool hor = mode < 18;
            const int angOff = hor ? 10 - mode : mode - 26;
            const int angle = c_angle[8 + angOff];
            const int mainBase = hor ? N2 + 1 : 1, sideBase = hor ? 1 : N2 + 1;
            const int off = N + 1;
            __syncwarp();
            if (angle < 0)
            {
                const int nproj = -((N * angle) >> 5) - 1;
                const int inv = c_invAngle[-angOff - 1];
                for (int i = lane; i < nproj; i += 32) refbuf[off + 1 + (-2 - i)] = nbs[sideBase - 1 + ((128 + (i + 1) * inv) >> 8)];
                for (int i = lane; i < N + 1; i += 32) refbuf[off + 1 + (-1 + i)] = (i == 0) ? nbs[0] : nbs[mainBase + i - 1];
            }
            else if (angle > 0)
            {
                for (int i = lane; i < N2; i += 32) refbuf[off + 1 + i] = nbs[mainBase + i];
            }
            __syncwarp();
            for (int u = lane; u < nunits; u += 32)
            {
                const int r = u / upr, c0 = (u - r * upr) * 4;
                int v[4];
                if (angle == 0)
                {
#pragma unroll
                    for (int k = 0; k < 4; k++) v[k] = nbs[mainBase + c0 + k];
                    if (bLuma && c0 == 0) v[0] = clip3i(0, maxv, (int)(int16_t)(nbs[mainBase] + ((nbs[sideBase + r] - nbs[0]) >> 1)));
                }
                else
                {
                    const int pos = (r + 1) * angle, o = pos >> 5, f = pos & 31;
                    const int16_t* rp = refbuf + off + 1 + o + c0;
                    int a = rp[0];
#pragma unroll
                    for (int k = 0; k < 4; k++)
                    {
                        const int b = rp[k + 1];
                        v[k] = f ? (((32 - f) * a + f * b + 16) >> 5) : a;
                        a = b;
                    }
                }
                P* d = out + (r << lg) + c0;
                if (sizeof(P) == 1) *(uint32_t*)d = (uint32_t)v[0] | ((uint32_t)v[1] << 8) | ((uint32_t)v[2] << 16) | ((uint32_t)v[3] << 24);
                else                *(uint2*)d = make_uint2((uint32_t)v[0] | ((uint32_t)v[1] << 16), (uint32_t)v[2] | ((uint32_t)v[3] << 16));
            }
        }
    }
}

// ---- packed angular prediction, shared by k_intra_allangs_packed and the frame analyser's intra search (frame.cuh) ----
// Projected reference row of angular mode `mode` (2..34) of an N x N block in the vertical-family frame, kept as PIXELS:
// refbuf[N + 2 + idx] = ref[idx], idx in [-N, 2N) (intrapred.cpp:120-160).  Built by the nl lanes li = 0..nl-1 of a group;
// modes 10 / 26 (angle 0) need none.  The caller syncs the group before and after.
template <typename P>
__device__ __forceinline__ void intra_ang_ref(P* refbuf, const P* nbs, int N, int mode, int li, int nl)
{
    const bool hor = mode < 18;
    const int angOff = hor ? 10 - mode : mode - 26, angle = c_angle[8 + angOff];
    const int N2 = 2 * N, mainBase = hor ? N2 + 1 : 1, sideBase = hor ? 1 : N2 + 1, off = N + 1;
    if (angle < 0)
    {
        const int nproj = -((N * angle) >> 5) - 1;
        const int inv = c_invAngle[-angOff - 1];
        for (int i = li; i < nproj; i += nl) refbuf[off + 1 + (-2 - i)] = nbs[sideBase - 1 + ((128 + (i + 1) * inv) >> 8)];
        for (int i = li; i < N + 1; i += nl) refbuf[off + 1 + (-1 + i)] = (i == 0) ? nbs[0] : nbs[mainBase + i - 1];
    }
    else if (angle > 0)
    {
        for (int i = li; i < N2; i += nl) refbuf[off + 1 + i] = nbs[mainBase + i];
    }
}

// Pixels c0 .. c0 + UW * 4 / sizeof(P) - 1 of row r of angular mode `mode` in the vertical-family frame (a horizontal mode's
// block transposed), packed 4 (8-bit) / 2 (16-bit) per word.  From the projected row of intra_ang_ref: UW + 2 aligned words,
// funnel shifts to the item's byte phase, then one DP4A (bytes p[k], p[k+1] against the weights (32 - f, f), + 16 in the
// accumulator) or DP2A per pixel and one shift; f == 0 needs no special case: (32 p + 16) >> 5 == p.  Modes 10 / 26 (angle 0)
// copy the main reference, with the edge filter on column 0 when bFilter.  refbuf must be 4-byte aligned and hold
// 3N + 12 pixels (the words past the last used pixel are read and weighted by 0).
template <typename P, int UW>
__device__ __forceinline__ void intra_ang_item(const P* refbuf, const P* nbs, int N, int mode, int bFilter, int r, int c0, uint32_t o32[UW])
{
    constexpr int maxv = PixTraits<P>::maxv;
    constexpr int ES = (int)sizeof(P), UPX = UW * 4 / ES;
    const bool hor = mode < 18;
    const int angOff = hor ? 10 - mode : mode - 26, angle = c_angle[8 + angOff];
    const int N2 = 2 * N, mainBase = hor ? N2 + 1 : 1, sideBase = hor ? 1 : N2 + 1, off = N + 1;
    if (angle == 0)
    {
        int v[UPX];
#pragma unroll
        for (int q = 0; q < UPX; q++) v[q] = nbs[mainBase + c0 + q];
        if (bFilter && c0 == 0) v[0] = clip3i(0, maxv, (int)(int16_t)((int)nbs[mainBase] + (((int)nbs[sideBase + r] - (int)nbs[0]) >> 1)));
#pragma unroll
        for (int w = 0; w < UW; w++)
            o32[w] = ES == 1 ? ((uint32_t)v[4 * w] | ((uint32_t)v[4 * w + 1] << 8) | ((uint32_t)v[4 * w + 2] << 16) | ((uint32_t)v[4 * w + 3] << 24))
                             : ((uint32_t)v[(2 * w) % UPX] | ((uint32_t)v[(2 * w + 1) % UPX] << 16));
        return;
    }
    const int pos = (r + 1) * angle, o = pos >> 5, f = pos & 31;
    const uint32_t W = (uint32_t)(32 - f) | ((uint32_t)f << 8);
    const unsigned bo = (unsigned)(off + 1 + o + c0) * ES;
    const uint32_t* wp = (const uint32_t*)refbuf + (bo >> 2);
    const unsigned sh = (bo & 3u) * 8u;
    uint32_t wd[UW + 2], x[UW + 1];
#pragma unroll
    for (int w = 0; w < UW + 2; w++) wd[w] = wp[w];
#pragma unroll
    for (int w = 0; w < UW + 1; w++) x[w] = __funnelshift_r(wd[w], wd[w + 1], sh);
#pragma unroll
    for (int w = 0; w < UW; w++)
    {
        if (ES == 1)
        {
            const uint32_t p0 = (uint32_t)dp4a_us(x[w], W, 16) >> 5, p1 = (uint32_t)dp4a_us(x[w], W << 8, 16) >> 5;
            const uint32_t p2 = (uint32_t)dp4a_us(x[w], W << 16, 16) >> 5;
            const uint32_t p3 = (uint32_t)dp4a_us(__funnelshift_r(x[w], x[w + 1], 24), W, 16) >> 5;
            o32[w] = p0 | (p1 << 8) | (p2 << 16) | (p3 << 24);
        }
        else
        {
            const uint32_t p0 = (uint32_t)dp2a_lo_ss(x[w], W, 16) >> 5;
            const uint32_t p1 = (uint32_t)dp2a_lo_ss(__funnelshift_r(x[w], x[w + 1], 16), W, 16) >> 5;
            o32[w] = p0 | (p1 << 16);
        }
    }
}

// all-angs on packed pixels: same per-pixel arithmetic as k_intra_allangs_cta, issued 4 (8-bit) / 2 (16-bit) pixels per word.
// The CTA kernel above spends ~45 instructions per 4 pixels (two shared loads, two IMADs, shift and select per pixel, the
// packing) and keeps half a warp idle on a 16x16 block (a mode has 16 row units there): issue bound.  Here
//   * neighbours and the projected reference row are kept as PIXELS in shared memory, a work item is a 16-byte piece of an
//     output row (a whole row up to 16 / 8 pixels), computed by intra_ang_item;
//   * a warp runs 32 / items-per-mode modes side by side (two for a 16x16 8-bit block, four for 8x8), each with its own
//     reference row, so all lanes are busy for every block size.
// Modes 10 / 26 (angle 0: a copy of the main reference plus the edge filter) stay scalar.
template <typename P, int UW>
__global__ void __launch_bounds__(256) k_intra_allangs_packed(int N, const P* __restrict__ refp, const P* __restrict__ filtp, int64_t nb_pitch,
                                                              P* __restrict__ dst, int bLuma, int n)
{
    constexpr int ES = (int)sizeof(P), UPX = UW * 4 / ES;          // pixels per work item
    __shared__ __align__(16) P s_nb[2][136];
    __shared__ __align__(16) P s_ref[8][8][136];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int lg = 31 - __clz(N);
    const int cpr = N / UPX, ipm = N * cpr;                        // items per row / per mode (both powers of two, ipm <= 64)
    const int G = ipm >= 32 ? 1 : 32 / ipm;                        // modes a warp runs side by side
    const int g = ipm >= 32 ? 0 : lane / ipm, li = ipm >= 32 ? lane : lane - g * ipm, lstep = ipm >= 32 ? 32 : ipm;
    const int slot = warp * G + g, nslots = 8 * G, rounds = (33 + nslots - 1) / nslots;
    P* refbuf = s_ref[warp][g];
    for (int j = blockIdx.x; j < n; j += gridDim.x)
    {
        __syncthreads();
        for (int i = threadIdx.x; i < 2 * (4 * N + 1); i += blockDim.x)
        {
            const int which = i >= 4 * N + 1, e = which ? i - (4 * N + 1) : i;
            s_nb[which][e] = (which ? filtp : refp)[j * nb_pitch + e];
        }
        __syncthreads();
        for (int k = 0; k < rounds; k++)
        {
            const int mode = 2 + slot + k * nslots;
            const bool active = mode < 35;
            const P* nbs = s_nb[active && intra_use_filtered(mode, N) ? 1 : 0];
            __syncwarp();
            if (active) intra_ang_ref<P>(refbuf, nbs, N, mode, li, lstep);
            __syncwarp();
            if (active)
            {
                P* out = dst + ((int64_t)j * 33 + (mode - 2)) * N * N;
                for (int it = li; it < ipm; it += lstep)
                {
                    const int r = it / cpr, c0 = (it - r * cpr) * UPX;
                    uint32_t o32[UW];
                    intra_ang_item<P, UW>(refbuf, nbs, N, mode, bLuma, r, c0, o32);
                    P* d = out + (r << lg) + c0;
                    if (UW == 4)      *(uint4*)d = make_uint4(o32[0], o32[1], o32[2], o32[3]);
                    else if (UW == 2) *(uint2*)d = make_uint2(o32[0], o32[1]);
                    else              *(uint32_t*)d = o32[0];
                }
            }
        }
    }
}

// all-angs (intrapred.cpp:206-234): grid = (33 modes, jobs); 33*N*N contiguous per job
template <typename P>
__global__ void __launch_bounds__(256) k_intra_allangs(int N, const P* __restrict__ refp, const P* __restrict__ filtp, int64_t nb_pitch,
                                                       P* __restrict__ dst, int bLuma, int n)
{
    __shared__ int16_t s_nb[129];
    __shared__ int16_t s_ref[128];
    const int mode = 2 + blockIdx.x;
    for (int j = blockIdx.y; j < n; j += gridDim.y)
    {
        const P* src = intra_use_filtered(mode, N) ? filtp : refp;
        __syncthreads();
        for (int i = threadIdx.x; i < 4 * N + 1; i += blockDim.x) s_nb[i] = src[j * nb_pitch + i];
        __syncthreads();
        intra_predict_block<P>(s_nb, s_ref, dst + ((int64_t)j * 33 + (mode - 2)) * N * N, N, N, mode, bLuma, true);
    }
}
