// x265_b200/csrc/part.cuh -- PART stage of the frame analyser (stage bit 5, a P slice): per CU (8 to 64) and per partition the
// geometry emits, the sa8dCost of checkInter_rd0_4 (analysis.cpp:3023-3071) on the analyser's cost model (include/x265_b200.h,
// x265cu_part_cu): each PU's slot of lowest ME cost, its prediction at its ME vector into the CU's S x S prediction in shared
// memory (pc_predict: the pixel path, or for a weighted slot the 14-bit prediction and resid_weight_sp, as the residual stage
// predicts), bd_sa8d of the CU (+ the chroma twins) plus the PUs' ME mvcost.  One launch per CU size over the per-size CU lists
// (geometry.h cuBy), with k_cu_bidir's shapes: CU 8 a warp each (four per CTA), CU 16 a 128-thread CTA, CU 32 and 64 a
// 256-thread CTA.  k_cu_part_b (stage bit 6, a B slice) is the same over the same shapes, with predInterSearch's per-PU list
// choice and bi-prediction (below).
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

// ---- stage bit 6 (PART_B, a B slice): per PU the best job of each list, the bi try with its zero pair, the direction
// (predInterSearch's B-slice path, search.cpp:2473-2644), then the CU's prediction and costs as above (include/x265_b200.h,
// x265cu_part_b_cu).  A bi PU's predictions are pc_plane's: the two pixel predictions and pixelavg_pp, or the two 14-bit ones
// and addAvg.  Slots are unweighted (a B slice is refused while weighted), so `p.wt` is null.
struct PartBArgs
{
    PartArgs p; int numRefL0, width, height, chromaSatd;   // chromaSatd: chroma enabled and subme > 2
    x265cu_part_b_cu* out;
};

// The zero try's range of the CU at (cx, cy), quarter-pel: setSearchRange(cu, 0, max(width, height)) with k_build_me_jobs'
// clip and the maxMvLen clamp, then mvmax.y += 2 and both bounds << 2 (search.cpp:2515-2529), k_cu_bidir's range; and
// MV::checkRange of an MVP against it
struct BdRange { int mnx, mxx, mny, mxy; };
__device__ __forceinline__ BdRange bd_zero_range(int width, int height, int cx, int cy)
{
    const int dist = max(width, height) << 2;
    const int xmax = (width + 8 - cx - 1) << 2, xmin = -((64 + 8 + cx - 1) << 2);
    const int ymax = (height + 8 - cy - 1) << 2, ymin = -((64 + 8 + cy - 1) << 2);
    const int mnx = max(min(max(-dist, xmin), xmax), -32767) >> 2, mxx = min(min(max(dist, xmin), xmax), 32767) >> 2;
    const int mny = max(min(max(-dist, ymin), ymax), -32767) >> 2;
    const int mxy = max(min(min(max(dist, ymin), ymax), 32767) >> 2, mny) + 2;
    BdRange r; r.mnx = mnx * 4; r.mxx = mxx * 4; r.mny = mny * 4; r.mxy = mxy * 4;
    return r;
}
__device__ __forceinline__ bool bd_in_range(const BdRange& r, int px, int py)
{
    return px >= r.mnx && px <= r.mxx && py >= r.mny && py <= r.mxy;
}

// one PU of a partition: each list's best slot, ME cost, searched vector and MVP; its place and size in the CU; the bi try's
// result and the direction
struct PartBPu
{
    int slot0, slot1, cost0, cost1, m0x, m0y, m1x, m1y, p0x, p0y, p1x, p1y, rx, ry, pw, ph, dir, zero;
    uint32_t biCost;
};

// the bi-prediction of plane pl of the PU at the pair (mx0, my0) / (mx1, my1) into dst (pitch S); flags X265CU_PRED_AVG_PP:
// pixelavg_pp of the pixel predictions, else addAvg of the 14-bit ones
template <typename P, int TPJ, int S>
__device__ __forceinline__ void part_b_bipred(const PartArgs& a, const CuDesc& cu, int pl, const PartBPu& q, int mx0, int my0, int mx1,
                                              int my1, int flags, int16_t* dst, int16_t* s_p1, int16_t* s_win, int16_t* s_mid, int t)
{
    x265cu_pred_job jb;
    jb.mv0[0] = (int16_t)mx0; jb.mv0[1] = (int16_t)my0; jb.mv1[0] = (int16_t)mx1; jb.mv1[1] = (int16_t)my1; jb.flags = (uint8_t)flags;
    const int sub = pl ? 1 : 0, st = pl ? a.cstride : a.stride;
    const ptrdiff_t off = (ptrdiff_t)((cu.y + q.ry) >> sub) * st + ((cu.x + q.rx) >> sub);
    const P* const* tab = (const P* const*)a.refs[pl];
    if (pl) pc_plane<P, TPJ, S, 4>(tab[q.slot0] + off, tab[q.slot1] + off, st, jb, q.pw >> 1, q.ph >> 1, dst, s_p1, s_win, s_mid, t);
    else    pc_plane<P, TPJ, S, 8>(tab[q.slot0] + off, tab[q.slot1] + off, st, jb, q.pw, q.ph, dst, s_p1, s_win, s_mid, t);
}

// bufSATD (+ bufChromaSATD with chromaSatd) of the PU's bi-prediction at the pair, summed over the job group; the prediction
// is staged in s_p0 (pitch S)
template <typename P, int TPJ, int S>
__device__ __forceinline__ int part_b_satd(const PartArgs& a, const CuDesc& cu, const PartBPu& q, int mx0, int my0, int mx1, int my1,
                                           bool chromaSatd, int16_t* s_p0, int16_t* s_p1, int16_t* s_win, int16_t* s_mid, int* s_red, int t)
{
    int acc = 0;
    for (int pl = 0; pl < (chromaSatd ? 3 : 1); pl++)
    {
        part_b_bipred<P, TPJ, S>(a, cu, pl, q, mx0, my0, mx1, my1, chromaSatd ? 0 : X265CU_PRED_AVG_PP, s_p0, s_p1, s_win, s_mid, t);
        const int sub = pl ? 1 : 0, st = pl ? a.cstride : a.stride;
        const ptrdiff_t off = (ptrdiff_t)((cu.y + q.ry) >> sub) * st + ((cu.x + q.rx) >> sub);
        acc += pc_cost<P, TPJ, S>((const P*)a.fenc[pl] + off, st, s_p0, q.pw >> sub, q.ph >> sub, true, t);
    }
    return resid_group_sum<TPJ>(acc, s_red);
}

// steps 1-3 for PU u (job k of the CU's jobs) of CU c; BI: the bi try runs (not 2Nx2N, not a CU 8)
template <typename P, int TPJ, int S>
__device__ __forceinline__ PartBPu part_b_pu(const PartBArgs& b, const CuDesc& cu, int c, int k, int u, bool bi, const BdRange& zr,
                                             int16_t* s_p0, int16_t* s_p1, int16_t* s_win, int16_t* s_mid, int* s_red, int t)
{
    const PartArgs& a = b.p;
    PartBPu q;
    q.slot0 = 0; q.slot1 = b.numRefL0; q.cost0 = q.cost1 = 0x7fffffff;
    for (int r = 0; r < a.numRefs; r++)
    {
        const int cost = a.me_out[(size_t)(a.cu_jobs[c * a.numRefs + r] + k) * 4];
        if (r < b.numRefL0) { if (cost < q.cost0) { q.cost0 = cost; q.slot0 = r; } }
        else if (cost < q.cost1) { q.cost1 = cost; q.slot1 = r; }
    }
    const int j0 = a.cu_jobs[c * a.numRefs + q.slot0] + k, j1 = a.cu_jobs[c * a.numRefs + q.slot1] + k;
    q.m0x = a.me_out[(size_t)j0 * 4 + 1]; q.m0y = a.me_out[(size_t)j0 * 4 + 2];
    q.m1x = a.me_out[(size_t)j1 * 4 + 1]; q.m1y = a.me_out[(size_t)j1 * 4 + 2];
    q.p0x = a.jobs[j0].qmvp[0]; q.p0y = a.jobs[j0].qmvp[1]; q.p1x = a.jobs[j1].qmvp[0]; q.p1y = a.jobs[j1].qmvp[1];
    q.pw = a.pus[j0].pw; q.ph = a.pus[j0].ph;
    q.rx = u ? S - q.pw : 0; q.ry = u ? S - q.ph : 0;          // PU 0 at the CU origin, PU 1 fills the rest of the CU
    q.biCost = 0xffffffffu; q.zero = 0;
    if (bi)
    {
        const bool chromaSatd = b.chromaSatd && !(((q.pw >> 1) | (q.ph >> 1)) & 3);
        q.biCost = part_b_satd<P, TPJ, S>(a, cu, q, q.m0x, q.m0y, q.m1x, q.m1y, chromaSatd, s_p0, s_p1, s_win, s_mid, s_red, t) +
                   me_mvcost(a.mvc, q.p0x, q.p0y, q.m0x, q.m0y) + me_mvcost(a.mvc, q.p1x, q.p1y, q.m1x, q.m1y);
        if ((q.m0x | q.m0y | q.m1x | q.m1y) && bd_in_range(zr, q.p0x, q.p0y) && bd_in_range(zr, q.p1x, q.p1y))
        {
            const uint32_t zCost = part_b_satd<P, TPJ, S>(a, cu, q, 0, 0, 0, 0, chromaSatd, s_p0, s_p1, s_win, s_mid, s_red, t) +
                                   me_mvcost(a.mvc, q.p0x, q.p0y, 0, 0) + me_mvcost(a.mvc, q.p1x, q.p1y, 0, 0);
            if (zCost < q.biCost) { q.biCost = zCost; q.zero = 1; }
        }
    }
    q.dir = q.biCost < (uint32_t)q.cost0 && q.biCost < (uint32_t)q.cost1 ? 3 : q.cost0 <= q.cost1 ? 1 : 2;
    return q;
}

// the mvcost of the PU's final vectors: the used list's vector of a uni PU, both of a bi PU (the pair after the zero try)
__device__ __forceinline__ uint32_t part_b_mvcost(const uint16_t* mvc, const PartBPu& q)
{
    const int z = q.zero ? 0 : 1;
    if (q.dir == 3) return me_mvcost(mvc, q.p0x, q.p0y, q.m0x * z, q.m0y * z) + me_mvcost(mvc, q.p1x, q.p1y, q.m1x * z, q.m1y * z);
    return q.dir == 1 ? me_mvcost(mvc, q.p0x, q.p0y, q.m0x, q.m0y) : me_mvcost(mvc, q.p1x, q.p1y, q.m1x, q.m1y);
}

// PU u's fields of entry ps of the record (has: the partition has that PU)
__device__ __forceinline__ void part_b_store(x265cu_part_b_cu* o, int ps, int u, const PartBPu& q, bool has)
{
    const int z = q.zero ? 0 : 1;
    o->biCost[ps][u] = has ? q.biCost : 0xffffffffu;
    o->interDir[ps][u] = (int8_t)(has ? q.dir : 0);
    o->ref[ps][u][0] = (int8_t)(has ? q.slot0 : -1); o->ref[ps][u][1] = (int8_t)(has ? q.slot1 : -1);
    o->zero[ps][u] = (uint8_t)(has ? q.zero : 0);
    o->mv[ps][u][0][0] = (int16_t)(has ? q.m0x * z : 0); o->mv[ps][u][0][1] = (int16_t)(has ? q.m0y * z : 0);
    o->mv[ps][u][1][0] = (int16_t)(has ? q.m1x * z : 0); o->mv[ps][u][1][1] = (int16_t)(has ? q.m1y * z : 0);
}

template <typename P, int TPJ, int S>
__global__ void __launch_bounds__(TPJ > 128 ? TPJ : 128) k_cu_part_b(const PartBArgs b)
{
    const PartArgs& a = b.p;
    constexpr bool BI = S > 8;                                    // isBipredRestriction: a CU 8's PUs are never bi
    constexpr int JPB = (TPJ > 128 ? TPJ : 128) / TPJ;
    // window, intermediate, the CU's prediction (also where a bi try stages its prediction), and the second list's prediction
    // of a bi PU at the same pitch S: a PU as tall as the CU (Nx2N, nLx2N, nRx2N) needs all S rows of it
    constexpr int WIN = (S + 7) * (S + 8), MID = (S + 7) * S, PRD = S * S, BUF = BI ? PRD : 0;
    __shared__ int16_t s_all[JPB][WIN + MID + PRD + BUF];
    __shared__ int s_red[TPJ / 32];
    const int grp = JPB == 1 ? 0 : threadIdx.x / TPJ, t = JPB == 1 ? threadIdx.x : threadIdx.x % TPJ;
    int16_t* s_win = s_all[grp]; int16_t* s_mid = s_win + WIN; int16_t* s_pred = s_mid + MID; int16_t* s_p1 = s_pred + PRD;
    // the partitions in k_cu_part's order
    const bool amp = a.amp && S >= 16;
    const int nparts = 1 + (a.rect ? 2 : 0) + (amp ? 4 : 0);
    for (int j = blockIdx.x * JPB + grp; j < a.n; j += gridDim.x * JPB)
    {
        const int c = a.list[j];
        const CuDesc cu = a.cus[c];
        x265cu_part_b_cu* o = b.out + c;
        const BdRange zr = bd_zero_range(b.width, b.height, cu.x, cu.y);    // per CU, not per PU (search.cpp:2515-2529)
        for (int pi = 0; pi < nparts; pi++)
        {
            const int ps = pi == 0 ? 0 : (a.rect ? (pi < 3 ? pi : pi + 1) : pi + 3);    // PartSize
            const int k0 = pi == 0 ? 0 : 2 * pi - 1, npu = pi == 0 ? 1 : 2;           // its first PU job, its PUs
            const bool bi = BI && pi > 0;
            const PartBPu q0 = part_b_pu<P, TPJ, S>(b, cu, c, k0, 0, bi, zr, s_pred, s_p1, s_win, s_mid, s_red, t);
            const PartBPu q1 = npu > 1 ? part_b_pu<P, TPJ, S>(b, cu, c, k0 + 1, 1, bi, zr, s_pred, s_p1, s_win, s_mid, s_red, t) : q0;
            uint32_t mvcost = part_b_mvcost(a.mvc, q0);
            if (npu > 1) mvcost += part_b_mvcost(a.mvc, q1);
            // the CU's prediction, its sa8d per plane
            uint32_t sa8d = 0;
            for (int pl = 0; pl < (a.chroma ? 3 : 1); pl++)
            {
#pragma unroll 1
                for (int u = 0; u < npu; u++)
                {
                    const PartBPu q = u ? q1 : q0;
                    if (BI && q.dir == 3)
                    {
                        const int z = q.zero ? 0 : 1;
                        int16_t* dst = s_pred + (q.ry >> (pl ? 1 : 0)) * S + (q.rx >> (pl ? 1 : 0));
                        part_b_bipred<P, TPJ, S>(a, cu, pl, q, q.m0x * z, q.m0y * z, q.m1x * z, q.m1y * z, 0, dst, s_p1, s_win, s_mid, t);
                    }
                    else
                    {
                        const int slot = q.dir == 1 ? q.slot0 : q.slot1, mx = q.dir == 1 ? q.m0x : q.m1x, my = q.dir == 1 ? q.m0y : q.m1y;
                        if (pl) part_pu_pred<P, TPJ, S, 4>(a, cu, pl, slot, mx, my, q.rx, q.ry, q.pw, q.ph, s_pred, s_win, s_mid, t);
                        else    part_pu_pred<P, TPJ, S, 8>(a, cu, pl, slot, mx, my, q.rx, q.ry, q.pw, q.ph, s_pred, s_win, s_mid, t);
                    }
                }
                const int st = pl ? a.cstride : a.stride;
                const ptrdiff_t off = pl ? (ptrdiff_t)(cu.y >> 1) * st + (cu.x >> 1) : (ptrdiff_t)cu.y * st + cu.x;
                sa8d += bd_sa8d<P, TPJ, S>((const P*)a.fenc[pl] + off, st, s_pred, pl ? S / 2 : S, s_red, t);
            }
            if (t == 0)
            {
                o->cost[ps] = sa8d + mvcost; o->sa8d[ps] = sa8d;
                part_b_store(o, ps, 0, q0, true);
                part_b_store(o, ps, 1, q1, npu > 1);
            }
        }
        // the partitions not evaluated: NxN always, the rect / AMP ones the geometry does not emit
        if (t == 0)
            for (int ps = 1; ps < 8; ps++)
                if (ps == 3 || (ps < 3 && !a.rect) || (ps > 3 && !amp))
                {
                    const PartBPu none = {};
                    o->cost[ps] = 0xffffffffu; o->sa8d[ps] = 0xffffffffu;
                    part_b_store(o, ps, 0, none, false);
                    part_b_store(o, ps, 1, none, false);
                }
    }
}

template <typename P, int TPJ, int S>
static int part_b_launch(x265cu_ctx* c, int maxPerSm, PartBArgs b, const int32_t* list, int n)
{
    constexpr int JPB = (TPJ > 128 ? TPJ : 128) / TPJ;
    if (n == 0) return 0;
    b.p.list = list; b.p.n = n;
    k_cu_part_b<P, TPJ, S><<<min((n + JPB - 1) / JPB, c->sm_count * maxPerSm), TPJ > 128 ? TPJ : 128, 0, c->stream>>>(b);
    CU_LAUNCH_CHECK(c);
    return 0;
}

// one launch per CU size, lists[k] = the CUs of size 8 << k (n[k] entries)
template <typename P>
static int launch_part_b(x265cu_ctx* c, const PartBArgs& b, const int32_t* const lists[4], const int n[4])
{
    if (part_b_launch<P, 32, 8>(c, 16, b, lists[0], n[0]) || part_b_launch<P, 128, 16>(c, 16, b, lists[1], n[1]) ||
        part_b_launch<P, 256, 32>(c, 8, b, lists[2], n[2]) || part_b_launch<P, 256, 64>(c, 4, b, lists[3], n[3])) return -1;
    return 0;
}
