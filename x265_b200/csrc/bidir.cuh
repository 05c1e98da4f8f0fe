// x265_b200/csrc/bidir.cuh -- BIDIR stage of the frame analyser (stage bit 4, a B slice): per CU (8 to 64) the uni-directional
// 2Nx2N estimate of checkInter_rd0_4 and the bidirectional one of Analysis::checkBidir2Nx2N (analysis.cpp:3062-3071,
// 3145-3265) on the analyser's cost model (include/x265_b200.h, x265cu_analyser_set_lists): the best 2Nx2N job of each list,
// sa8d of the uni prediction, of the addAvg bi-prediction and of the zero pair (+ the chroma twins) plus the ME's mvcost, and
// the decision.  Predictions are predcost.cuh's pc_plane (the uni pixel path, or the two 14-bit predictions and addAvg), the
// costs grp_sa8d / had4x4_abs against the prediction in shared memory.  One launch per CU size over the per-size CU lists
// (geometry.h cuBy): CU 8 a warp each (four per CTA), CU 16 a 128-thread CTA, CU 32 and 64 a 256-thread CTA.
#pragma once
#include "common.cuh"
#include "predcost.cuh"
#include "resid.cuh"
#include "geometry.h"

// fenc / refs [plane] = luma, Cb, Cr (origin pointers, refs device tables indexed by slot); jobs / me_out / cu_jobs are the
// whole tables (absolute indices), list / n the launch's slice of one per-size CU list; mvc the centred mvcost table
struct BidirArgs
{
    const void* fenc[3]; const void* const* refs[3]; int stride, cstride, chroma;
    const CuDesc* cus; const int32_t* list; int n;
    const int32_t* cu_jobs; int numRefs, numRefL0; const int32_t* me_out; const x265cu_me_job* jobs;
    const uint16_t* mvc; int width, height;
    x265cu_bidir_cu* out;
};

// sa8d of the w x w block, source in global memory, prediction in shared memory (pitch DP), summed over the job group: the
// cu[].sa8d of the block (8x8 transforms, rounded per 16x16 when w is a multiple of 16), satd 4x4 when w == 4 (the 4:2:0
// chroma of a CU 8, primitives.cpp:185-188).  A warp per 16-row band; every thread of the group calls.
template <typename P, int TPJ, int DP>
__device__ __forceinline__ int bd_sa8d(const P* __restrict__ fe, int fs, const int16_t* __restrict__ pr, int w, int* s_red, int t)
{
    const int lane = t & 31, warp = t >> 5;
    int v = 0;
    if (w == 4) { if (t == 0) v = had4x4_abs(fe, fs, pr, DP) >> 1; }
    else if (warp < (w == 8 ? 1 : w >> 4))
    {
        const int h = w == 8 ? 8 : 16;
        const int s = grp_sa8d(fe + (ptrdiff_t)(warp * h) * fs, fs, pr + warp * h * DP, DP, w, h, lane, 32, (w >> 3) * (h >> 3));
        v = lane == 0 ? s : 0;
    }
    return resid_group_sum<TPJ>(v, s_red);
}

// luma + (chroma) sa8d of the CU's prediction: uni (r1 < 0: list slot r0 at mv0, pixel path) or bi (slots r0, r1 at mv0, mv1:
// addAvg of the 14-bit predictions)
template <typename P, int TPJ, int S>
__device__ __forceinline__ int bd_cost(const BidirArgs& a, const CuDesc& cu, int r0, int r1, int mx0, int my0, int mx1, int my1,
                                       int16_t* s_p0, int16_t* s_p1, int16_t* s_win, int16_t* s_mid, int* s_red, int t)
{
    x265cu_pred_job jb;
    jb.mv0[0] = (int16_t)mx0; jb.mv0[1] = (int16_t)my0; jb.mv1[0] = (int16_t)mx1; jb.mv1[1] = (int16_t)my1; jb.flags = 0;
    int cost = 0;
    for (int pl = 0; pl < (a.chroma ? 3 : 1); pl++)
    {
        const int st = pl ? a.cstride : a.stride, w = pl ? S / 2 : S;
        const ptrdiff_t off = pl ? (ptrdiff_t)(cu.y >> 1) * st + (cu.x >> 1) : (ptrdiff_t)cu.y * st + cu.x;
        const P* const* tab = (const P* const*)a.refs[pl];
        const P* p0 = tab[r0] + off;
        const P* p1 = r1 >= 0 ? tab[r1] + off : nullptr;
        if (pl) pc_plane<P, TPJ, S, 4>(p0, p1, st, jb, w, w, s_p0, s_p1, s_win, s_mid, t);
        else    pc_plane<P, TPJ, S, 8>(p0, p1, st, jb, w, w, s_p0, s_p1, s_win, s_mid, t);
        cost += bd_sa8d<P, TPJ, S>((const P*)a.fenc[pl] + off, st, s_p0, w, s_red, t);
    }
    return cost;
}

template <typename P, int TPJ, int S>
__global__ void __launch_bounds__(TPJ > 128 ? TPJ : 128) k_cu_bidir(const BidirArgs a)
{
    constexpr int JPB = (TPJ > 128 ? TPJ : 128) / TPJ;
    constexpr int WIN = (S + 7) * (S + 8), MID = (S + 7) * S, PRD = S * S;
    __shared__ int16_t s_all[JPB][WIN + MID + 2 * PRD];
    __shared__ int s_red[TPJ / 32];
    const int grp = JPB == 1 ? 0 : threadIdx.x / TPJ, t = JPB == 1 ? threadIdx.x : threadIdx.x % TPJ;
    int16_t* s_win = s_all[grp]; int16_t* s_mid = s_win + WIN; int16_t* s_p0 = s_mid + MID; int16_t* s_p1 = s_p0 + PRD;
    for (int j = blockIdx.x * JPB + grp; j < a.n; j += gridDim.x * JPB)
    {
        const int c = a.list[j];
        const CuDesc cu = a.cus[c];
        // 1. the best 2Nx2N job of each list (ties to the lowest slot); scalars, so that nothing is indexed at run time
        int b0 = 0, b1 = a.numRefL0, c0 = 0x7fffffff, c1 = 0x7fffffff;
        for (int r = 0; r < a.numRefs; r++)
        {
            const int cost = a.me_out[(size_t)a.cu_jobs[c * a.numRefs + r] * 4];
            if (r < a.numRefL0) { if (cost < c0) { c0 = cost; b0 = r; } }
            else if (cost < c1) { c1 = cost; b1 = r; }
        }
        const int j0 = a.cu_jobs[c * a.numRefs + b0], j1 = a.cu_jobs[c * a.numRefs + b1];
        const int m0x = a.me_out[(size_t)j0 * 4 + 1], m0y = a.me_out[(size_t)j0 * 4 + 2];
        const int m1x = a.me_out[(size_t)j1 * 4 + 1], m1y = a.me_out[(size_t)j1 * 4 + 2];
        const int p0x = a.jobs[j0].qmvp[0], p0y = a.jobs[j0].qmvp[1], p1x = a.jobs[j1].qmvp[0], p1y = a.jobs[j1].qmvp[1];
        const bool u1 = c0 > c1;
        // 2. uni, 3. bi
        const uint32_t uniCost = bd_cost<P, TPJ, S>(a, cu, u1 ? b1 : b0, -1, u1 ? m1x : m0x, u1 ? m1y : m0y, 0, 0, s_p0, s_p1, s_win, s_mid, s_red, t) +
                                 (u1 ? me_mvcost(a.mvc, p1x, p1y, m1x, m1y) : me_mvcost(a.mvc, p0x, p0y, m0x, m0y));
        uint32_t biCost = bd_cost<P, TPJ, S>(a, cu, b0, b1, m0x, m0y, m1x, m1y, s_p0, s_p1, s_win, s_mid, s_red, t) +
                          me_mvcost(a.mvc, p0x, p0y, m0x, m0y) + me_mvcost(a.mvc, p1x, p1y, m1x, m1y);
        // 4. the zero pair, when both MVPs lie in setSearchRange(cu, 0, max(width, height)) widened by 2 rows
        bool tryZero = (m0x | m0y | m1x | m1y) != 0;
        if (tryZero)
        {
            const int dist = max(a.width, a.height) << 2;
            const int xmax = (a.width + 8 - cu.x - 1) << 2, xmin = -((64 + 8 + cu.x - 1) << 2);
            const int ymax = (a.height + 8 - cu.y - 1) << 2, ymin = -((64 + 8 + cu.y - 1) << 2);
            const int mnx = max(min(max(-dist, xmin), xmax), -32767) >> 2, mxx = min(min(max(dist, xmin), xmax), 32767) >> 2;
            const int mny = max(min(max(-dist, ymin), ymax), -32767) >> 2;
            const int mxy = max(min(min(max(dist, ymin), ymax), 32767) >> 2, mny) + 2;
            tryZero = p0x >= mnx * 4 && p0x <= mxx * 4 && p0y >= mny * 4 && p0y <= mxy * 4 &&
                      p1x >= mnx * 4 && p1x <= mxx * 4 && p1y >= mny * 4 && p1y <= mxy * 4;
        }
        bool zero = false;
        if (tryZero)
        {
            const uint32_t zCost = bd_cost<P, TPJ, S>(a, cu, b0, b1, 0, 0, 0, 0, s_p0, s_p1, s_win, s_mid, s_red, t) +
                                   me_mvcost(a.mvc, p0x, p0y, 0, 0) + me_mvcost(a.mvc, p1x, p1y, 0, 0);
            if (zCost < biCost) { biCost = zCost; zero = true; }
        }
        // 5. the decision
        if (t == 0)
        {
            x265cu_bidir_cu o;
            o.uniCost = uniCost; o.biCost = biCost;
            o.interDir = (int8_t)(biCost < uniCost ? 3 : u1 ? 2 : 1);
            o.ref[0] = (int8_t)b0; o.ref[1] = (int8_t)b1; o.zero = zero;
            o.mv[0][0] = (int16_t)(zero ? 0 : m0x); o.mv[0][1] = (int16_t)(zero ? 0 : m0y);
            o.mv[1][0] = (int16_t)(zero ? 0 : m1x); o.mv[1][1] = (int16_t)(zero ? 0 : m1y);
            a.out[c] = o;
        }
    }
}

template <typename P, int TPJ, int S>
static int bidir_launch(x265cu_ctx* c, int maxPerSm, BidirArgs a, const int32_t* list, int n)
{
    constexpr int JPB = (TPJ > 128 ? TPJ : 128) / TPJ;
    if (n == 0) return 0;
    a.list = list; a.n = n;
    k_cu_bidir<P, TPJ, S><<<min((n + JPB - 1) / JPB, c->sm_count * maxPerSm), TPJ > 128 ? TPJ : 128, 0, c->stream>>>(a);
    CU_LAUNCH_CHECK(c);
    return 0;
}

// one launch per CU size, lists[k] = the CUs of size 8 << k (n[k] entries)
template <typename P>
static int launch_bidir(x265cu_ctx* c, const BidirArgs& a, const int32_t* const lists[4], const int n[4])
{
    if (bidir_launch<P, 32, 8>(c, 16, a, lists[0], n[0]) || bidir_launch<P, 128, 16>(c, 16, a, lists[1], n[1]) ||
        bidir_launch<P, 256, 32>(c, 8, a, lists[2], n[2]) || bidir_launch<P, 256, 64>(c, 4, a, lists[3], n[3])) return -1;
    return 0;
}
