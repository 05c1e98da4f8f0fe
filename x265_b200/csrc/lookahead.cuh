// x265_b200/csrc/lookahead.cuh -- lookahead frame-cost estimation on device (BASELINE configs[1]):
//   k_lowres_intra   : LookaheadTLD::lowresIntraEstimate  (encoder/slicetype.cpp:696-805): per 8x8 lowres CU,
//                      neighbours from the source plane, DC / planar / coarse-to-fine angular scan, SATD 8x8
//   k_lookahead_cost : CostEstimateGroup::estimateFrameCost + estimateCUCost (slicetype.cpp:3115-3388, serial
//                      path, no HME / weightp): reverse-raster CU order with MV predictors from the right /
//                      below / below-left / below-right neighbours => anti-diagonal wavefront; one CTA per
//                      (p0, p1, b) triple, one warp per CU of the current diagonal, the motion search itself is
//                      me_run_job() (HEX, subme 1, merange 16 on the 4 hpel planes).
#pragma once
#include "common.cuh"
#include "me.cuh"
#include "frame.cuh"

#define LA_COST_MAX (1 << 28)
#define LA_COST_MASK ((1 << 14) - 1)
#define LA_COST_SHIFT 14

// SATD 8x8 (= two 8x4 tiles, pixel.cpp:239-297) over an 8-lane group: lane `row` holds one row of 8 differences
__device__ __forceinline__ int satd8x8_group(int d[8], int lane)
{
    had4(d[0], d[1], d[2], d[3]); had4(d[4], d[5], d[6], d[7]);          // horizontal 4-point on both halves
#pragma unroll
    for (int s = 1; s < 4; s <<= 1)                                        // vertical 4-point inside each 4-row tile
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
    acc += __shfl_xor_sync(0xffffffffu, acc, 2);                            // sum of one 8x4 tile (4 lanes)
    int tile = acc >> 1;                                                    // halved per 8x4 tile
    return tile + __shfl_xor_sync(0xffffffffu, tile, 4);                    // + the other tile of the CU
}

template <typename P>
__global__ void __launch_bounds__(256) k_lowres_intra(const x265cu_la_intra_job* __restrict__ jobs, int stride, int w8, int h8, int lambda)
{
    constexpr int maxv = PixTraits<P>::maxv;
    __shared__ int16_t s_nb[32][33], s_filt[32][33];
    const x265cu_la_intra_job jb = jobs[blockIdx.y];
    const P* plane0 = (const P*)jb.plane0;
    const int tid = threadIdx.x, lane = tid & 31, grp = tid >> 3, row = tid & 7;      // 32 CUs per CTA, 8 lanes each
    const int ncu = w8 * h8;
    const int intraPenalty = 5 * lambda, lowresPenalty = 4;
    for (int base = blockIdx.x * 32; base < ncu; base += gridDim.x * 32)
    {
        const int cu = base + grp;
        const bool act = cu < ncu;
        const int cuXY = act ? cu : ncu - 1;
        const int cuY = cuXY / w8, cuX = cuXY - cuY * w8;
        const P* cur = plane0 + 8 * cuX + (size_t)8 * cuY * stride;
        __syncthreads();
        // neighbours: [0] top-left, [1..16] top, [17..32] left (slicetype.cpp:729-733)
        for (int i = row; i < 33; i += 8)
        {
            const P* tl = cur - stride - 1;
            s_nb[grp][i] = (int16_t)(i <= 16 ? tl[i] : tl[(ptrdiff_t)(i - 16) * stride]);
        }
        __syncthreads();
        for (int i = row; i < 33; i += 8) s_filt[grp][i] = (int16_t)intra_filter_elem(s_nb[grp], i, 8);
        __syncthreads();
        int dcsum = 8;
        for (int i = 0; i < 8; i++) dcsum += s_nb[grp][1 + i] + s_nb[grp][17 + i];
        const int dc = dcsum / 16;
        int f[8];
#pragma unroll
        for (int x = 0; x < 8; x++) f[x] = cur[(size_t)row * stride + x];
        auto cost_of = [&](int mode, const int16_t* nbs) -> int {
            int d[8];
#pragma unroll
            for (int x = 0; x < 8; x++) d[x] = f[x] - intra_pixel(nbs, 8, 3, mode, 1, dc, row, x, maxv);
            return satd8x8_group(d, lane);
        };
        int icost = LA_COST_MAX, ilow = 0, cost;
        cost = cost_of(1, s_nb[grp]);   if (cost < icost) { icost = cost; ilow = 1; }
        cost = cost_of(0, s_filt[grp]); if (cost < icost) { icost = cost; ilow = 0; }
        int acost = LA_COST_MAX, alow = 4;
        for (int mode = 5; mode < 35; mode += 5)
        {
            cost = cost_of(mode, intra_use_filtered(mode, 8) ? s_filt[grp] : s_nb[grp]);
            if (cost < acost) { acost = cost; alow = mode; }
        }
        for (int dist = 2; dist >= 1; dist--)
        {
            const int minus = alow - dist, plus = alow + dist;
            cost = cost_of(minus, intra_use_filtered(minus, 8) ? s_filt[grp] : s_nb[grp]);
            if (cost < acost) { acost = cost; alow = minus; }
            cost = cost_of(plus, intra_use_filtered(plus, 8) ? s_filt[grp] : s_nb[grp]);
            if (cost < acost) { acost = cost; alow = plus; }
        }
        if (acost < icost) { icost = acost; ilow = alow; }
        icost += intraPenalty + lowresPenalty;
        if (act && row == 0)
        {
            jb.lowresCosts[cuXY] = (uint16_t)min(icost, LA_COST_MASK);
            jb.intraCost[cuXY] = icost;
            jb.intraMode[cuXY] = (uint8_t)ilow;
            const bool score = (cuX > 0 && cuX < w8 - 1 && cuY > 0 && cuY < h8 - 1) || w8 <= 2 || h8 <= 2;
            const int icostAq = (score && jb.invQscale) ? ((icost * jb.invQscale[cuXY] + 128) >> 8) : icost;
            if (score) { atomicAdd((unsigned long long*)&jb.out[0], (unsigned long long)icost); atomicAdd((unsigned long long*)&jb.out[1], (unsigned long long)icostAq); }
            atomicAdd(&jb.rowSatds[cuY], icostAq);
        }
    }
}

__global__ void k_la_zero(int32_t* a, int n, int64_t* out, int nout)
{
    for (int i = threadIdx.x; i < n; i += blockDim.x) a[i] = 0;
    for (int i = threadIdx.x; i < nout; i += blockDim.x) out[i] = 0;
}

// ---------------------------------------------------------------------------------------------
#define LA_WARPS 16
template <typename P>
__global__ void __launch_bounds__(LA_WARPS * 32, 1) k_lookahead_cost(const x265cu_la_job* __restrict__ jobs, int stride, int w8, int h8,
                                                                      const uint16_t* __restrict__ mvcost)
{
    extern __shared__ unsigned char la_smem[];
    __shared__ int32_t s_out[LA_WARPS][4];
    // One thread-block CLUSTER per triple: the CTAs of the cluster (1..4, chosen at launch from the diagonal length)
    // split the CUs of every anti-diagonal, so a diagonal of up to 64 CUs is one round of warps instead of four; the
    // per-diagonal barrier is the cluster barrier, whose release / acquire pair also publishes the MVs and costs the
    // other CTAs wrote to global memory.
    unsigned crank, csize;
    asm("mov.u32 %0, %%cluster_ctarank;" : "=r"(crank));
    asm("mov.u32 %0, %%cluster_nctarank;" : "=r"(csize));
    const x265cu_la_job jb = jobs[blockIdx.x / csize];
    const int lane = threadIdx.x & 31, warp = (int)crank * LA_WARPS + (threadIdx.x >> 5);      // warp index inside the cluster
    const int nwarps = (int)csize * LA_WARPS;
    MeShared* sm = (MeShared*)la_smem + (threadIdx.x >> 5);
    // Cooperative slices (CostEstimateGroup::processTasks, slicetype.cpp:3075-3112; estimateFrameCost :3143-3173): a job may
    // cover only the CU rows [y0, y1) of the frame; its bottom row is the slice's `lastRow` (no MV predictors from below),
    // the rows' costs accumulate into the SAME frame totals (jb.out, zeroed by x265cu_lookahead_cost_batch before the launch).
    // rows == 0: the whole frame (the serial path, :3178-3196).  Slices of one triple are independent wavefronts.
    const int y0 = jb.rows ? (jb.rows & 0xffff) : 0, y1 = jb.rows ? ((jb.rows >> 16) & 0xffff) : h8;
    const int hs = y1 - y0;
    if (crank == 0)
        for (int i = y0 + threadIdx.x; i < y1; i += blockDim.x) jb.rowSatds[i] = 0;
    const int ndiag = (w8 - 1) + 2 * (hs - 1) + 1;
    for (int t = 0; t < ndiag; t++)
    {
        // MVs / costs of the previous diagonals are visible to every CTA of the cluster
        asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
        // CUs on this diagonal: k = 0.. with cuY = y1-1-k, cuX = w8-1-(t-2k)
        const int kmin = max(0, (t - (w8 - 1) + 1) >> 1), kmax = min(hs - 1, t >> 1);
        for (int k = kmin + warp; k <= kmax; k += nwarps)
        {
            const int cuY = y1 - 1 - k, cuX = w8 - 1 - (t - 2 * k);
            if (cuX < 0 || cuX >= w8) continue;
            const int cuXY = cuX + cuY * w8;
            const bool lastRow = (cuY == y1 - 1);
            const int off = 8 * cuX + 8 * cuY * stride;
            x265cu_me_job mj;
            mj.offset = off; mj.ref = 0; mj.pw = 8; mj.ph = 8;
            mj.mvmin[0] = (int16_t)(-cuX * 8 - 8); mj.mvmin[1] = (int16_t)(-cuY * 8 - 8);
            mj.mvmax[0] = (int16_t)((w8 - cuX - 1) * 8 + 8); mj.mvmax[1] = (int16_t)((h8 - cuY - 1) * 8 + 8);
            mj.numCand = 0; mj.method = 1; mj.subme = 1; mj.merange = 16;
            MeCtx<P> c;
            c.fenc = (const P*)jb.fenc[0] + off; c.fstride = stride; c.rstride = stride; c.mvc = mvcost;
            c.minx = mj.mvmin[0]; c.miny = mj.mvmin[1]; c.maxx = mj.mvmax[0]; c.maxy = mj.mvmax[1];
            c.w = 8; c.h = 8; c.lgw = 3; c.lane = lane; c.lowres = 1; c.sm = sm;
            me_set_shape<P>(c);                 // source and reference share the stride
            int bcost = LA_COST_MAX, listused = 0;
            int lmx[2] = { 0, 0 }, lmy[2] = { 0, 0 };            // final MV of each list for the bidir candidates
            for (int i = 0; i < 1 + jb.bidir; i++)
            {
                int32_t* fencCost = jb.mvcosts[i] + cuXY;
                const bool doSearch = i ? jb.doSearch1 : jb.doSearch0;
                if (!doSearch)
                {
                    const int fc = *fencCost;
                    lmx[i] = jb.mvs[i][2 * cuXY]; lmy[i] = jb.mvs[i][2 * cuXY + 1];       // written by an earlier launch
                    if (fc < bcost) { bcost = fc; listused = i + 1; }
                    continue;
                }
                int32_t* fmv = jb.mvs[i] + 2 * cuXY;
                const void* const* fref = i ? jb.ref1 : jb.ref0;
                for (int q = 0; q < 4; q++) c.ref[q] = (const P*)fref[q] + off;
                // reverse-order MV prediction (slicetype.cpp:3271-3280): right, below, below-left, below-right
                int numc = 0, mvcx[4], mvcy[4];
                if (cuX < w8 - 1) { mvcx[numc] = fmv[2]; mvcy[numc] = fmv[3]; numc++; }
                if (!lastRow)
                {
                    mvcx[numc] = fmv[2 * w8]; mvcy[numc] = fmv[2 * w8 + 1]; numc++;
                    if (cuX > 0) { mvcx[numc] = fmv[2 * (w8 - 1)]; mvcy[numc] = fmv[2 * (w8 - 1) + 1]; numc++; }
                    if (cuX < w8 - 1) { mvcx[numc] = fmv[2 * (w8 + 1)]; mvcy[numc] = fmv[2 * (w8 + 1) + 1]; numc++; }
                }
                int mvpx = 0, mvpy = 0, skipCost = 0x7fffffff;
                if (numc)
                {
                    int mvpcost = LA_COST_MAX;
                    // bufSATD(lowresMC(mvc)) of all candidates in one burst, then the reference's sequential fold
                    const int lq = min(lane, numc - 1);
                    const int cqx = lq == 0 ? mvcx[0] : lq == 1 ? mvcx[1] : lq == 2 ? mvcx[2] : mvcx[3];
                    const int cqy = lq == 0 ? mvcy[0] : lq == 1 ? mvcy[1] : lq == 2 ? mvcy[2] : mvcy[3];
                    const int ccost = me_lowres_multi(c, numc, cqx, cqy, true);
#pragma unroll
                    for (int idx = 0; idx < 4; idx++)
                    {
                        if (idx >= numc) break;
                        const int cost = __shfl_sync(0xffffffffu, ccost, idx);
                        if (cost < mvpcost) { mvpcost = cost; mvpx = mvcx[idx]; mvpy = mvcy[idx]; }
                        if (!(mvpx | mvpy) && jb.bidir) skipCost = cost;
                    }
                }
                c.mvpx = mvpx; c.mvpy = mvpy;
                mj.qmvp[0] = (int16_t)mvpx; mj.qmvp[1] = (int16_t)mvpy;
                __syncwarp();
                me_run_job<P>(c, mj, s_out[threadIdx.x >> 5]);
                __syncwarp();
                int fc = s_out[threadIdx.x >> 5][0], mx = s_out[threadIdx.x >> 5][1], my = s_out[threadIdx.x >> 5][2];
                __syncwarp();
                if (skipCost < 64 && skipCost < fc && jb.bidir) { fc = skipCost; mx = 0; my = 0; }
                if (lane == 0) { *fencCost = fc; fmv[0] = mx; fmv[1] = my; }
                lmx[i] = mx; lmy[i] = my;
                if (fc < bcost) { bcost = fc; listused = i + 1; }
            }
            if (jb.bidir)
            {
                // avg(L0 MC, L1 MC) then the co-located average (slicetype.cpp:3326-3346); both through SATD
                const int m0x = lmx[0], m0y = lmy[0], m1x = lmx[1], m1y = lmy[1];
                for (int pass = 0; pass < 2; pass++)
                {
                    __syncwarp();
                    for (int i = lane; i < 64; i += 32)
                    {
                        const int y = i >> 3, x = i & 7;
                        int s0, s1;
                        if (pass == 0)
                        {
                            int mv[2][2] = { { m0x, m0y }, { m1x, m1y } };
                            int v[2];
                            for (int l = 0; l < 2; l++)
                            {
                                const void* const* fr = l ? jb.ref1 : jb.ref0;
                                const int qx = mv[l][0], qy = mv[l][1];
                                const int ha = (qy & 2) | ((qx & 2) >> 1);
                                const P* a = (const P*)fr[ha] + off + (qx >> 2) + (ptrdiff_t)(qy >> 2) * stride;
                                int va = a[(ptrdiff_t)y * stride + x];
                                if ((qx | qy) & 1)
                                {
                                    const int rx = qx + (qx & 1), ry = qy + (qy & 1);
                                    const int hb = (ry & 2) | ((rx & 2) >> 1);
                                    const P* b = (const P*)fr[hb] + off + (rx >> 2) + (ptrdiff_t)(ry >> 2) * stride;
                                    va = (va + (int)b[(ptrdiff_t)y * stride + x] + 1) >> 1;
                                }
                                v[l] = va;
                            }
                            s0 = v[0]; s1 = v[1];
                        }
                        else
                        {
                            s0 = ((const P*)jb.ref0[0])[off + (ptrdiff_t)y * stride + x];
                            s1 = ((const P*)jb.ref1[0])[off + (ptrdiff_t)y * stride + x];
                        }
                        sm->pred[y * 64 + x] = (uint16_t)((s0 + s1 + 1) >> 1);
                    }
                    __syncwarp();
                    const int bicost = warp_sum(me_band_cost(c, 0, 8, true));
                    if (bicost < bcost) { bcost = bicost; listused = 3; }
                }
                bcost += 4;
            }
            else
            {
                bcost += 4;
                const int ic = jb.intraCost[cuXY];
                if (ic < bcost) { bcost = ic; listused = 0; }
            }
            if (lane == 0)
            {
                const bool score = (cuX > 0 && cuX < w8 - 1 && cuY > 0 && cuY < h8 - 1) || w8 <= 2 || h8 <= 2;
                const int bcostAq = (score && jb.invQscale) ? ((bcost * jb.invQscale[cuXY] + 128) >> 8) : bcost;
                if (score)
                {
                    atomicAdd((unsigned long long*)&jb.out[0], (unsigned long long)bcost);
                    atomicAdd((unsigned long long*)&jb.out[1], (unsigned long long)bcostAq);
                    if (!listused && !jb.bidir) atomicAdd((unsigned long long*)&jb.out[2], 1ull);
                }
                atomicAdd(&jb.rowSatds[cuY], bcostAq);
                jb.lowresCosts[cuXY] = (uint16_t)(min(bcost, LA_COST_MASK) | (listused << LA_COST_SHIFT));
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// cuTree: estimateCUPropagateCost (common/pixel.cpp:914-940), the per-CU amount of "influence on future quality" that
// Lookahead::estimateCUPropagate (slicetype.cpp:2641-2670) scatters over the reference frames.  Double precision, each
// operation rounded on its own as the host's scalar code does (no FMA contraction: __dmul_rn / __dadd_rn / __ddiv_rn), and
// the final double -> int conversion with x86 cvttsd2si semantics (NaN / out of range -> INT_MIN) so that degenerate
// inputs (intraCost 0) match the C primitive bit for bit too.  One thread per CU.
__device__ __forceinline__ int la_cvttsd2si(double v)
{
    return (v >= -2147483648.0 && v < 2147483648.0) ? (int)v : (int)0x80000000;
}
// The amount of one CU: shared by k_propagate_cost and cuTree's step kernels (k_cutree_amount).
__device__ __forceinline__ int la_propagate_amount(int propagateIn, int intraCost, int interCostWord, int invQscale, double fps)
{
    const int interCost = min(intraCost, interCostWord & LA_COST_MASK);
    // Q16 x Q8.8 = Q24.8, an int32 product converted to double: it wraps past 2^31 as the reference's does
    const double propagateIntra = (double)(int)((unsigned)intraCost * (unsigned)invQscale);
    const double propagateAmount = __dadd_rn((double)propagateIn, __dmul_rn(propagateIntra, fps));
    const double propagateNum = (double)(intraCost - interCost);
    const double propagateDenom = (double)intraCost;
    return la_cvttsd2si(__dadd_rn(__ddiv_rn(__dmul_rn(propagateAmount, propagateNum), propagateDenom), 0.5));
}
__global__ void __launch_bounds__(256) k_propagate_cost(int* __restrict__ dst, const uint16_t* __restrict__ propagateIn, const int32_t* __restrict__ intraCosts,
                                                        const uint16_t* __restrict__ interCosts, const int32_t* __restrict__ invQscales, double fpsFactor, int64_t len)
{
    const double fps = fpsFactor / 256;                             // range [0.01, 1.00]
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < len; i += (int64_t)gridDim.x * blockDim.x)
        dst[i] = la_propagate_amount(propagateIn[i], intraCosts[i], interCosts[i], invQscales[i], fps);
}

// ---------------------------------------------------------------------------------------------
// cuTree's propagation chain (Lookahead::cuTree / estimateCUPropagate, slicetype.cpp:2538-2747).  x265cu_cutree groups the
// window's steps into levels: steps of which none reads an array that another one writes (the non-referenced B steps of a
// mini-GOP; then the middle B of a b-pyramid; then the anchor).  A level is two launches in stream order:
//   k_cutree_amount  : every CU's propagate_amount into scratch, and the level's overflow flag;
//   k_cutree_scatter : the bipred weighting, the MV-0 shortcut, the bilinear split and the edge tests of :2690-2738.
// Why the parallel scatter is exact: every add is CLIP_ADD(s, x) = (uint16)min(s + x, 65535).  For x >= 0 the result of
// any sequence of such adds on one word is min(s0 + sum(x), 65535) whatever their order (each add is monotone and the clamp
// absorbs), so the adds of a whole level may land in any order -- as a compare-and-swap loop on the 16-bit word that
// applies min(s + x, 65535) atomically.  x >= 0 holds when every propagating amount is below 2^21: then
// amount * bipredWeight + 32 (weights <= 64) and listamount * idxNweight + 512 (weights <= 1024) stay inside int32.  The
// reference computes those products in int32 and wraps (x86 imul): a wrapped add can be negative, CLIP_ADD then wraps
// modulo 2^16 and the result depends on the order.  k_cutree_amount raises the flag for any amount >= 2^21; the scatter
// then replays the whole level on one thread, in the reference's step and raster order, with its int32 wrap-around.
#define CUTREE_MAX_STEPS 16
#define CUTREE_SAFE_AMOUNT (1 << 21)
struct CuTreeStep
{
    const int32_t* intraCost; const int32_t* invQscale;
    const uint16_t* propagateIn;        // frame b's own propagateCost when referenced, NULL: zeros (:2656-2658)
    const uint16_t* lowresCosts;        // lowresCosts[b - p0][p1 - b]
    const int32_t* mvs[2];              // lowresMvs[list][listDist[list]] as int32 pairs
    uint16_t* ref[2];                   // propagateCost of p0 and p1
    int32_t bipredWeight[2];
};
struct CuTreeLevel
{
    CuTreeStep s[CUTREE_MAX_STEPS];
    int n;
};

__global__ void __launch_bounds__(256) k_cutree_amount(const CuTreeLevel L, int ncu, double fpsFactor, int* __restrict__ amounts, int* __restrict__ flag)
{
    const CuTreeStep& s = L.s[blockIdx.y];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ncu) return;
    const int amount = la_propagate_amount(s.propagateIn ? s.propagateIn[i] : 0, s.intraCost[i], s.lowresCosts[i], s.invQscale[i], fpsFactor / 256);
    amounts[blockIdx.y * ncu + i] = amount;
    if (amount >= CUTREE_SAFE_AMOUNT) *flag = 1;
}

// CLIP_ADD(s, x) exactly as the compiled reference computes it: int32 sum (wrapping), min with 65535, truncation to 16 bits
__device__ __forceinline__ void cutree_clip_add_serial(uint16_t* p, int x)
{
    *p = (uint16_t)min((int)((unsigned)*p + (unsigned)x), 65535);
}
// the same for 0 <= x < 2^31 - 65535, atomically: min(s + x, 65535) on the 16-bit word
__device__ __forceinline__ void cutree_clip_add_atomic(uint16_t* p, int x)
{
    if (x <= 0) return;
    unsigned short old = *(volatile unsigned short*)p, assumed;
    do
    {
        assumed = old;
        if (assumed == 0xffff) return;
        old = atomicCAS((unsigned short*)p, assumed, (unsigned short)min((int)assumed + x, 65535));
    } while (old != assumed);
}

// One CU of one step (:2676-2741); products in unsigned arithmetic so that they wrap as the reference's int32 ones do
template <bool Serial>
__device__ __forceinline__ void cutree_scatter_cu(const CuTreeStep& s, int cu, int amount, int w8, int h8)
{
    if (amount <= 0) return;                                          // intra blocks do not propagate
    const int listsUsed = s.lowresCosts[cu] >> LA_COST_SHIFT;
    const int blocky = cu / w8, blockx = cu - blocky * w8;
    auto add = [&](uint16_t* p, int x) { if (Serial) cutree_clip_add_serial(p, x); else cutree_clip_add_atomic(p, x); };
    auto part = [](int a, int w) { return (int)((unsigned)a * (unsigned)w + 512u) >> 10; };
    for (int list = 0; list < 2; list++)
    {
        if (!((listsUsed >> list) & 1)) continue;
        int listamount = amount;
        if (listsUsed == 3) listamount = (int)((unsigned)listamount * (unsigned)s.bipredWeight[list] + 32u) >> 6;
        uint16_t* ref = s.ref[list];
        const int mx = s.mvs[list][2 * cu], my = s.mvs[list][2 * cu + 1];
        if (!(mx | my)) { add(ref + cu, listamount); continue; }     // the MV-0 shortcut
        const int cux = (mx >> 5) + blockx, cuy = (my >> 5) + blocky;
        const int idx0 = cux + cuy * w8, x = mx & 31, y = my & 31;
        const int w0 = (32 - y) * (32 - x), w1 = (32 - y) * x, w2 = y * (32 - x), w3 = y * x;
        const bool x0 = cux >= 0 && cux < w8, x1 = cux + 1 >= 0 && cux + 1 < w8;
        const bool y0 = cuy >= 0 && cuy < h8, y1 = cuy + 1 >= 0 && cuy + 1 < h8;
        if (x0 && y0) add(ref + idx0, part(listamount, w0));
        if (x1 && y0) add(ref + idx0 + 1, part(listamount, w1));
        if (x0 && y1) add(ref + idx0 + w8, part(listamount, w2));
        if (x1 && y1) add(ref + idx0 + w8 + 1, part(listamount, w3));
    }
}

__global__ void __launch_bounds__(256) k_cutree_scatter(const CuTreeLevel L, int w8, int h8, const int* __restrict__ amounts, const int* __restrict__ flag)
{
    const int ncu = w8 * h8;
    if (*flag)
    {
        // an amount of the level may overflow: the whole level on one thread, in the reference's order
        if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0)
            for (int k = 0; k < L.n; k++)
                for (int cu = 0; cu < ncu; cu++)
                    cutree_scatter_cu<true>(L.s[k], cu, amounts[k * ncu + cu], w8, h8);
        return;
    }
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < ncu) cutree_scatter_cu<false>(L.s[blockIdx.y], i, amounts[blockIdx.y * ncu + i], w8, h8);
}
