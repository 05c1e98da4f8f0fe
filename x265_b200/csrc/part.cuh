// x265_b200/csrc/part.cuh -- PART stage of the frame analyser (stage bit 5, a P slice): per CU (8 to 64) and per partition the
// geometry emits, the sa8dCost of checkInter_rd0_4 (analysis.cpp:3023-3071) on the analyser's cost model (include/x265_b200.h,
// x265cu_part_cu): each PU's slot of lowest ME cost, its prediction at its ME vector into the CU's S x S prediction in shared
// memory (pc_predict: the pixel path, or for a weighted slot the 14-bit prediction and resid_weight_sp, as the residual stage
// predicts), bd_sa8d of the CU (+ the chroma twins) plus the PUs' ME mvcost.  One launch per CU size over the per-size CU lists
// (geometry.h cuBy), with k_cu_bidir's shapes: CU 8 a warp each (four per CTA), CU 16 a 128-thread CTA, CU 32 and 64 a
// 256-thread CTA.
#pragma once
#include "common.cuh"
#include "predcost.cuh"
#include "resid.cuh"
#include "bidir.cuh"
#include "geometry.h"

// fenc / refs [plane] = luma, Cb, Cr (origin pointers; refs device tables of the unweighted planes, indexed by slot); pus, jobs,
// me_out and cu_jobs are the whole tables (absolute indices), list / n the launch's slice of one per-size CU list; mvc the
// centred mvcost table; wt the residual stage's weight table ([16][3], resid.cuh), null while no slot is weighted
struct PartArgs
{
    const void* fenc[3]; const void* const* refs[3]; int stride, cstride, chroma;
    const CuDesc* cus; const PuDesc* pus; const int32_t* list; int n;
    const int32_t* cu_jobs; int numRefs, rect, amp; const int32_t* me_out; const x265cu_me_job* jobs;
    const uint16_t* mvc; const int4* wt;
    x265cu_part_cu* out;
};

// PU k's slot of lowest ME cost over its jobs (ties to the lowest slot) and that job
__device__ __forceinline__ int part_best_job(const PartArgs& a, int c, int k, int& slot)
{
    int best = 0, bcost = 0x7fffffff;
    for (int r = 0; r < a.numRefs; r++)
    {
        const int cost = a.me_out[(size_t)(a.cu_jobs[c * a.numRefs + r] + k) * 4];
        if (cost < bcost) { bcost = cost; best = r; }
    }
    slot = best;
    return a.cu_jobs[c * a.numRefs + best] + k;
}

// the prediction of one PU of one plane into its place in the CU's prediction (pitch S): the PU is pw x ph (luma) at (rx, ry)
// in the CU; sub = 0 luma, 1 the 4:2:0 chroma planes
template <typename P, int TPJ, int S, int NT>
__device__ __forceinline__ void part_pu_pred(const PartArgs& a, const CuDesc& cu, int pl, int slot, int mvx, int mvy, int rx, int ry,
                                             int pw, int ph, int16_t* s_pred, int16_t* s_win, int16_t* s_mid, int t)
{
    constexpr int maxv = PixTraits<P>::maxv, sub = NT == 8 ? 0 : 1;
    const int st = pl ? a.cstride : a.stride, w = pw >> sub, h = ph >> sub;
    const P* ref = ((const P* const*)a.refs[pl])[slot] + (ptrdiff_t)((cu.y + ry) >> sub) * st + ((cu.x + rx) >> sub);
    int16_t* dst = s_pred + (ry >> sub) * S + (rx >> sub);
    pc_sync<TPJ>();                                               // the previous PU's window / the previous plane's cost is read
    if (a.wt && a.wt[3 * slot].x)
    {
        pc_predict<P, TPJ, S, NT, true>(ref, st, mvx, mvy, w, h, dst, s_win, s_mid, t);
        pc_sync<TPJ>();
        const int4 wv = a.wt[3 * slot + pl];                      // luma entry 0, Cb / Cr entries 1 / 2
        const PcDiv dw = pc_div(w);
        for (int i = t; i < w * h; i += TPJ)
        {
            int y, x; pc_split(dw, i, y, x);
            dst[y * S + x] = (int16_t)resid_weight_sp<maxv>((int)dst[y * S + x], wv);
        }
    }
    else
        pc_predict<P, TPJ, S, NT, false>(ref, st, mvx, mvy, w, h, dst, s_win, s_mid, t);
    pc_sync<TPJ>();
}

template <typename P, int TPJ, int S>
__global__ void __launch_bounds__(TPJ > 128 ? TPJ : 128) k_cu_part(const PartArgs a)
{
    constexpr int JPB = (TPJ > 128 ? TPJ : 128) / TPJ;
    constexpr int WIN = (S + 7) * (S + 8), MID = (S + 7) * S, PRD = S * S;
    __shared__ int16_t s_all[JPB][WIN + MID + PRD];
    __shared__ int s_red[TPJ / 32];
    const int grp = JPB == 1 ? 0 : threadIdx.x / TPJ, t = JPB == 1 ? threadIdx.x : threadIdx.x % TPJ;
    int16_t* s_win = s_all[grp]; int16_t* s_mid = s_win + WIN; int16_t* s_pred = s_mid + MID;
    // the partitions geometry_cu_parts emits at this size, in its order: 2Nx2N; 2NxN, Nx2N (rect); 2NxnU, 2NxnD, nLx2N, nRx2N
    // (amp, CU >= 16)
    const bool amp = a.amp && S >= 16;
    const int nparts = 1 + (a.rect ? 2 : 0) + (amp ? 4 : 0);
    for (int j = blockIdx.x * JPB + grp; j < a.n; j += gridDim.x * JPB)
    {
        const int c = a.list[j];
        const CuDesc cu = a.cus[c];
        x265cu_part_cu* o = a.out + c;
        for (int pi = 0; pi < nparts; pi++)
        {
            const int ps = pi == 0 ? 0 : (a.rect ? (pi < 3 ? pi : pi + 1) : pi + 3);    // PartSize
            const int k0 = pi == 0 ? 0 : 2 * pi - 1, npu = pi == 0 ? 1 : 2;           // its first PU job, its PUs
            // 1. per PU the slot and the vector; PU 0 lies at the CU origin, PU 1 fills the rest of the CU (its bottom-right)
            int s0, s1 = -1;
            const int j0 = part_best_job(a, c, k0, s0);
            const int j1 = npu > 1 ? part_best_job(a, c, k0 + 1, s1) : j0;
            const int m0x = a.me_out[(size_t)j0 * 4 + 1], m0y = a.me_out[(size_t)j0 * 4 + 2];
            const int m1x = a.me_out[(size_t)j1 * 4 + 1], m1y = a.me_out[(size_t)j1 * 4 + 2];
            const int pw0 = a.pus[j0].pw, ph0 = a.pus[j0].ph, pw1 = a.pus[j1].pw, ph1 = a.pus[j1].ph;
            uint32_t mvcost = me_mvcost(a.mvc, a.jobs[j0].qmvp[0], a.jobs[j0].qmvp[1], m0x, m0y);
            if (npu > 1) mvcost += me_mvcost(a.mvc, a.jobs[j1].qmvp[0], a.jobs[j1].qmvp[1], m1x, m1y);
            // 2. the CU's prediction, 3. its sa8d per plane
            uint32_t sa8d = 0;
            for (int pl = 0; pl < (a.chroma ? 3 : 1); pl++)
            {
#pragma unroll 1
                for (int u = 0; u < npu; u++)
                {
                    const int slot = u ? s1 : s0, mx = u ? m1x : m0x, my = u ? m1y : m0y, pw = u ? pw1 : pw0, ph = u ? ph1 : ph0;
                    const int rx = u ? S - pw : 0, ry = u ? S - ph : 0;
                    if (pl) part_pu_pred<P, TPJ, S, 4>(a, cu, pl, slot, mx, my, rx, ry, pw, ph, s_pred, s_win, s_mid, t);
                    else    part_pu_pred<P, TPJ, S, 8>(a, cu, pl, slot, mx, my, rx, ry, pw, ph, s_pred, s_win, s_mid, t);
                }
                const int st = pl ? a.cstride : a.stride;
                const ptrdiff_t off = pl ? (ptrdiff_t)(cu.y >> 1) * st + (cu.x >> 1) : (ptrdiff_t)cu.y * st + cu.x;
                sa8d += bd_sa8d<P, TPJ, S>((const P*)a.fenc[pl] + off, st, s_pred, pl ? S / 2 : S, s_red, t);
            }
            // the record, field by field
            if (t == 0)
            {
                o->cost[ps] = sa8d + mvcost; o->sa8d[ps] = sa8d;
                o->ref[ps][0] = (int8_t)s0; o->ref[ps][1] = (int8_t)s1;
                o->mv[ps][0][0] = (int16_t)m0x; o->mv[ps][0][1] = (int16_t)m0y;
                o->mv[ps][1][0] = (int16_t)(npu > 1 ? m1x : 0); o->mv[ps][1][1] = (int16_t)(npu > 1 ? m1y : 0);
            }
        }
        // the partitions not evaluated: NxN always, the rect / AMP ones the geometry does not emit
        if (t == 0)
            for (int ps = 1; ps < 8; ps++)
                if (ps == 3 || (ps < 3 && !a.rect) || (ps > 3 && !amp))
                {
                    o->cost[ps] = 0xffffffffu; o->sa8d[ps] = 0xffffffffu;
                    o->ref[ps][0] = o->ref[ps][1] = -1;
                    o->mv[ps][0][0] = o->mv[ps][0][1] = o->mv[ps][1][0] = o->mv[ps][1][1] = 0;
                }
    }
}

template <typename P, int TPJ, int S>
static int part_launch(x265cu_ctx* c, int maxPerSm, PartArgs a, const int32_t* list, int n)
{
    constexpr int JPB = (TPJ > 128 ? TPJ : 128) / TPJ;
    if (n == 0) return 0;
    a.list = list; a.n = n;
    k_cu_part<P, TPJ, S><<<min((n + JPB - 1) / JPB, c->sm_count * maxPerSm), TPJ > 128 ? TPJ : 128, 0, c->stream>>>(a);
    CU_LAUNCH_CHECK(c);
    return 0;
}

// one launch per CU size, lists[k] = the CUs of size 8 << k (n[k] entries)
template <typename P>
static int launch_part(x265cu_ctx* c, const PartArgs& a, const int32_t* const lists[4], const int n[4])
{
    if (part_launch<P, 32, 8>(c, 16, a, lists[0], n[0]) || part_launch<P, 128, 16>(c, 16, a, lists[1], n[1]) ||
        part_launch<P, 256, 32>(c, 8, a, lists[2], n[2]) || part_launch<P, 256, 64>(c, 4, a, lists[3], n[3])) return -1;
    return 0;
}
