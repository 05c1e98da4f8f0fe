// x265_b200/csrc/resid.cuh -- residual chain of every CU's best inter prediction, for luma (analyser stage bit 1) and for
// both 4:2:0 chroma planes (stage bit 3).  Per luma TU of the CU (T = min(S, 32)) and per plane, one TU of T >> sub
// (geometry_plane_tu), fully on-chip:
//   best-ref select -> MC (luma predict.cpp:245-266; chroma predInterChromaPixel, predict.cpp:306-353: the luma quarter-pel
//   vector read as eighth-pel) -> sub_ps -> dct -> quant -> dequant_normal -> idct / DC shortcut -> add_ps -> sse_pp
//   (search.cpp:3178 estimateResidualQT, search.cpp:2990-3080; quant.cpp:397-470, :543-605, non-RDOQ path).
// The reference and vector are the lowest ME cost of the CU's 2Nx2N jobs, ties to the lowest index.  The MC is pc_predict
// (predcost.cuh).  A job group of TPJ threads takes one (TU, plane) item at a time, and every launch reads the list of one
// luma TU size (geometry.h tuBy): TUs of 4 and 8 take a WARP each (four per CTA, private shared tiles, warp barriers only),
// TUs of 16 a 128-thread CTA each, luma TUs of 32 a 256-thread CTA each.
#pragma once
#include "common.cuh"
#include "predcost.cuh"
#include "geometry.h"

// quantiser scalars of a TU: flat scaling lists, non-I slice rounding offset (scalinglist.cpp:129-130; quant.cpp:411, 465-466,
// 556, 567)
struct ResidQuant { int scale, invScale, qbits, add, dqshift; };
template <int DEPTH>
__device__ __forceinline__ ResidQuant resid_quant(int qp, int lg)
{
    const int per = qp / 6, rem = qp - per * 6;
    ResidQuant q;
    q.scale = rem == 0 ? 26214 : rem == 1 ? 23302 : rem == 2 ? 20560 : rem == 3 ? 18396 : rem == 4 ? 16384 : 14564;
    q.invScale = (rem == 0 ? 40 : rem == 1 ? 45 : rem == 2 ? 51 : rem == 3 ? 57 : rem == 4 ? 64 : 72) << per;
    const int transformShift = 15 - DEPTH - lg;
    q.qbits = 14 + per + transformShift;
    q.add = 85 << (q.qbits - 9);
    q.dqshift = 20 - 14 - transformShift;
    return q;
}
// the residual value of every sample of a TU whose only nonzero level is the DC one (quant.cpp:588-598)
template <int DEPTH>
__device__ __forceinline__ int resid_dc_only(int dequantDc)
{
    constexpr int shift = 12 - (DEPTH - 8) - 3;
    return (((dequantDc + 1) >> 1) * 8 + (1 << (shift - 1))) >> shift;
}

// weight_sp of one 14-bit prediction sample with addWeightUni's round 1 << (shift - 1) (predict.cpp:525-578, pixel.cpp:493-516);
// w = {weighted, w0, offset, shift} as in the residual stage's weight table (cu_residual below)
template <int MAXV>
__device__ __forceinline__ int resid_weight_sp(int v, const int4& w)
{
    return clip3i(0, MAXV, ((w.y * (v + 8192) + (1 << (w.w - 1))) >> w.w) + w.z);
}

// sum over the TPJ threads of a job group, in every thread of the group.  TPJ is a multiple of 32; a group of more than one
// warp is the whole CTA.
template <int TPJ, typename T>
__device__ __forceinline__ T resid_group_sum(T v, T* s_red)
{
    if constexpr (sizeof(T) == 8) v = warp_sum64(v);
    else v = warp_sum(v);
    if (TPJ == 32) return v;
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
    __syncthreads();
    T s = 0;
#pragma unroll
    for (int w = 0; w < TPJ / 32; w++) s += s_red[w];
    return s;
}

// Per-plane inputs and outputs of the stage.  NPL planes (1 luma, 2 Cb / Cr) share the stride and the TU list; levels and
// recon of a plane share its geometry.  tus is the whole TU table, tul the launch's slice of one per-size list (ntu
// entries).  recon = origin pointers [NPL * depthIdx + plane]; cu_sse / cu_numsig are [NPL * cu + plane] and accumulate;
// cu_ref (luma) receives the chosen reference, or is null.
struct ResidArgs
{
    const void* fenc[2]; const void* const* refs[2]; int16_t* coef[2]; int qp[2];
    int stride; void* const* recon;
    const CuDesc* cus; const TuDesc* tus; const int32_t* tul; int ntu; const int32_t* cu_jobs; int numRefs; const int32_t* me_out;
    unsigned long long* cu_sse; uint32_t* cu_numsig; int32_t* cu_ref;
};

// Item j of [0, NPL * ntu) = plane j % NPL of TU tul[j / NPL].  NT = 8 is the luma plane, NT = 4 the two chroma planes at half
// resolution.  Every TU of the list is at most MAXS wide in the launch's planes.
// WT: the P-slice weighted uni-prediction (Predict::motionCompensation with wp0->wtPresent, predict.cpp:82-112).  wt[3 * ref +
// plane] = {weighted, w0, offset, shift}: weighted = the reference's luma wtPresent (the same in its three entries), w0 =
// inputWeight, offset = inputOffset << (depth - 8), shift = log2WeightDenom + 14 - depth.  A CU whose reference is weighted
// takes the 14-bit prediction of the unweighted plane (predInterLumaShort / predInterChromaShort) and weight_sp with
// addWeightUni's round 1 << (shift - 1) (predict.cpp:525-578, pixel.cpp:493-516); chroma uses entries 1 and 2 whatever
// their wtPresent.  WT = false compiles to the unweighted stage alone.
// BI: a B slice (the BIDIR stage's record bd[cu], bidir.cuh).  A CU with interDir 3 predicts each TU through the two 14-bit
// predictions of its list-0 / list-1 slots at its pair of vectors and addAvg (predict.cpp:168-189, pixel.cpp:842-862); its
// cu_ref is its list-0 slot.  Any other CU takes the path above: its uni-directional winner is the lowest ME cost over all
// slots, ties to the lowest, because the list-0 slots come first.
template <typename P, int TPJ, int MAXS, int NT, bool WT, bool BI = false>
__device__ __forceinline__ void cu_residual(const ResidArgs& a, const int4* __restrict__ wt, const x265cu_bidir_cu* __restrict__ bd = nullptr)
{
    constexpr int DEPTH = PixTraits<P>::depth, maxv = PixTraits<P>::maxv;
    constexpr int JPB = (TPJ > 128 ? TPJ : 128) / TPJ, NPL = NT == 8 ? 1 : 2, SUB = NPL - 1;
    constexpr int WR = MAXS + NT - 1;                            // rows of the MC source window and intermediate
    // The transform tiles reuse the MC's window / intermediate storage once the prediction is made.  Their rows are padded
    // to MAXS + 2 so that the column reads of the forward passes fall in distinct banks.
    constexpr int TP = MAXS + 2, MC = WR * (MAXS + 8) + WR * MAXS, TILES = 2 * MAXS * TP;
    constexpr int SCR = MC > TILES ? MC : TILES, DP = MAXS;
    __shared__ int16_t s_all[JPB][SCR + (BI ? 2 : 1) * MAXS * MAXS];   // BI: the list-1 prediction after s_pred
    __shared__ int8_t s_mat[JPB][MAXS * MAXS];                    // the TU size's DCT matrix
    __shared__ int s_red[TPJ / 32];
    __shared__ unsigned long long s_red64[TPJ / 32];
    __shared__ int s_lvl0[JPB];                                   // quantised DC level of the group's TU
    // With one group per CTA the group is 0 and the tile bases are constants: the luma launch needs 32 registers instead of the
    // 48 it takes when the group is derived from threadIdx.x
    const int grp = JPB == 1 ? 0 : threadIdx.x / TPJ, t = JPB == 1 ? threadIdx.x : threadIdx.x % TPJ;
    int16_t* s_win = s_all[grp]; int16_t* s_mid = s_win + WR * (MAXS + 8); int16_t* s_pred = s_win + SCR;
    int16_t* s_a = s_win; int16_t* s_b = s_a + MAXS * TP;
    int8_t* M = s_mat[grp];
    for (int j = blockIdx.x * JPB + grp; j < NPL * a.ntu; j += gridDim.x * JPB)
    {
        const TuDesc tu = a.tus[a.tul[j / NPL]];
        const int plane = j % NPL;
        const CuDesc cu = a.cus[tu.cu];
        const PlaneTu pt = geometry_plane_tu(cu, tu, SUB);
        const int T = pt.size;
        const int lg = 31 - __clz(T), N = T * T;
        int best = 0, bcost = 0x7fffffff;
        for (int r = 0; r < a.numRefs; r++)
        {
            const int cost = a.me_out[(size_t)a.cu_jobs[tu.cu * a.numRefs + r] * 4];
            if (cost < bcost) { bcost = cost; best = r; }
        }
        const bool bi = BI && bd[tu.cu].interDir == 3;
        if (bi) best = bd[tu.cu].ref[0];
        const int32_t* mo = a.me_out + (size_t)a.cu_jobs[tu.cu * a.numRefs + best] * 4;
        const ptrdiff_t off = (ptrdiff_t)pt.y * a.stride + pt.x;
        const P* ref = ((const P* const*)(plane ? a.refs[1] : a.refs[0]))[best] + off;
        const P* fe = (const P*)(plane ? a.fenc[1] : a.fenc[0]) + off;
        pc_sync<TPJ>();                                           // the previous item's tiles have been read
        for (int i = t; i < N; i += TPJ) M[i] = d_dct[lg - 2][i];
        if (bi)
        {
            // the record's words 2..4: {interDir, ref[0], ref[1], zero}, mv[0] (x | y << 16), mv[1]
            const int* w = reinterpret_cast<const int*>(bd + tu.cu);
            const int rw = w[2], v0 = w[3], v1 = w[4];
            const P* const* tab = (const P* const*)(plane ? a.refs[1] : a.refs[0]);
            int16_t* s_p1 = s_pred + MAXS * MAXS;
            pc_predict<P, TPJ, MAXS, NT, true>(tab[(int8_t)(rw >> 8)] + off, a.stride, (v0 << 16) >> 16, v0 >> 16, T, T, s_pred, s_win, s_mid, t);
            pc_sync<TPJ>();
            pc_predict<P, TPJ, MAXS, NT, true>(tab[(int8_t)(rw >> 16)] + off, a.stride, (v1 << 16) >> 16, v1 >> 16, T, T, s_p1, s_win, s_mid, t);
            pc_sync<TPJ>();
            constexpr int shift = 15 - DEPTH, offset = (1 << (shift - 1)) + 2 * 8192;
            for (int i = t; i < N; i += TPJ)
            {
                const int y = i >> lg, x = i & (T - 1);
                s_pred[y * DP + x] = (int16_t)clip3i(0, maxv, ((int)s_pred[y * DP + x] + (int)s_p1[y * DP + x] + offset) >> shift);
            }
        }
        else if (WT && wt[3 * best].x)
        {
            pc_predict<P, TPJ, MAXS, NT, true>(ref, a.stride, mo[1], mo[2], T, T, s_pred, s_win, s_mid, t);
            pc_sync<TPJ>();
            const int4 w = wt[3 * best + SUB + plane];             // luma entry 0, Cb / Cr entries 1 / 2
            for (int i = t; i < N; i += TPJ)
            {
                const int y = i >> lg, x = i & (T - 1);
                s_pred[y * DP + x] = (int16_t)resid_weight_sp<maxv>((int)s_pred[y * DP + x], w);
            }
        }
        else
            pc_predict<P, TPJ, MAXS, NT, false>(ref, a.stride, mo[1], mo[2], T, T, s_pred, s_win, s_mid, t);
        pc_sync<TPJ>();
        // ---- residual ----
        for (int i = t; i < N; i += TPJ)
        {
            const int y = i >> lg, x = i & (T - 1);
            s_a[y * TP + x] = (int16_t)((int)fe[(ptrdiff_t)y * a.stride + x] - (int)s_pred[y * DP + x]);
        }
        pc_sync<TPJ>();
        // ---- forward DCT, rows then columns (dct.cpp:83-240, 442-525) ----
        {
            const int sh1 = lg - 1 + (DEPTH - 8), sh2 = lg + 6;
            for (int i = t; i < N; i += TPJ)
            {
                const int k = i >> lg, jj = i & (T - 1);
                int acc = 0;
                for (int q = 0; q < T; q++) acc += (int)M[k * T + q] * s_a[jj * TP + q];
                s_b[k * TP + jj] = (int16_t)((acc + (1 << (sh1 - 1))) >> sh1);
            }
            pc_sync<TPJ>();
            for (int i = t; i < N; i += TPJ)
            {
                const int k = i >> lg, jj = i & (T - 1);
                int acc = 0;
                for (int q = 0; q < T; q++) acc += (int)M[k * T + q] * s_b[jj * TP + q];
                s_a[i] = (int16_t)((acc + (1 << (sh2 - 1))) >> sh2);      // coefficients in linear k * T + j order
            }
            pc_sync<TPJ>();
        }
        // ---- quant (dct.cpp:664-686) + dequant_normal (dct.cpp:612-634) ----
        const ResidQuant rq = resid_quant<DEPTH>(plane ? a.qp[1] : a.qp[0], lg);
        int16_t* qout = (plane ? a.coef[1] : a.coef[0]) + pt.off;
        int cnt = 0;
        for (int i = t; i < N; i += TPJ)
        {
            const int v = s_a[i];
            int lvl = (abs(v) * rq.scale + rq.add) >> rq.qbits;
            cnt += lvl != 0;
            if (v < 0) lvl = -lvl;
            const int q = clip16(lvl);
            qout[i] = (int16_t)q;
            if (i == 0) s_lvl0[grp] = q;
            s_b[i] = (int16_t)clip16((q * rq.invScale + (1 << (rq.dqshift - 1))) >> rq.dqshift);
        }
        const int numSig = resid_group_sum<TPJ>(cnt, s_red);
        pc_sync<TPJ>();
        // the reference tests coeff[0] != 0 on the QUANTISED level (quant.cpp:588)
        const bool dcOnly = numSig == 1 && s_lvl0[grp] != 0;
        // ---- inverse transform: residual in `res` ----
        const int16_t* res = s_a;
        if (dcOnly)
        {
            const int dc = resid_dc_only<DEPTH>(s_b[0]);
            for (int i = t; i < N; i += TPJ) s_a[i] = (int16_t)dc;
        }
        else if (numSig)
        {
            const int sh2 = 12 - (DEPTH - 8);
            for (int i = t; i < N; i += TPJ)
            {
                const int jj = i >> lg, i2 = i & (T - 1);
                int acc = 0;
                for (int q = 0; q < T; q++) acc += (int)M[q * T + i2] * s_b[q * T + jj];
                s_a[i] = (int16_t)clip16((acc + 64) >> 7);
            }
            pc_sync<TPJ>();
            for (int i = t; i < N; i += TPJ)
            {
                const int jj = i >> lg, i2 = i & (T - 1);
                int acc = 0;
                for (int q = 0; q < T; q++) acc += (int)M[q * T + i2] * s_a[q * T + jj];
                s_b[i] = (int16_t)clip16((acc + (1 << (sh2 - 1))) >> sh2);
            }
            res = s_b;
        }
        pc_sync<TPJ>();
        // ---- reconstruction (add_ps with the clip, or the prediction) + distortion ----
        const int dIdx = cu.size == 64 ? 0 : (cu.size == 32 ? 1 : (cu.size == 16 ? 2 : 3));
        P* rc = (P*)a.recon[NPL * dIdx + plane] + off;
        unsigned long long sse = 0;
        for (int i = t; i < N; i += TPJ)
        {
            const int y = i >> lg, x = i & (T - 1);
            const int p = s_pred[y * DP + x];
            const int v = numSig ? clip3i(0, maxv, p + (int)res[i]) : p;
            rc[(ptrdiff_t)y * a.stride + x] = (P)v;
            const int d = (int)fe[(ptrdiff_t)y * a.stride + x] - v;
            sse += (unsigned)(d * d);
        }
        sse = resid_group_sum<TPJ>(sse, s_red64);
        if (t == 0)
        {
            if (sse) atomicAdd(&a.cu_sse[NPL * tu.cu + plane], sse);
            if (numSig) atomicAdd(&a.cu_numsig[NPL * tu.cu + plane], (uint32_t)numSig);
            if (a.cu_ref) a.cu_ref[tu.cu] = best;
        }
    }
}

template <typename P, int TPJ, int MAXS, int NT>
__global__ void __launch_bounds__(TPJ > 128 ? TPJ : 128) k_cu_residual(const ResidArgs a)
{
    cu_residual<P, TPJ, MAXS, NT, false>(a, nullptr);
}

// the stage of a frame with at least one weighted reference (the unweighted ones take the same path as in k_cu_residual)
template <typename P, int TPJ, int MAXS, int NT>
__global__ void __launch_bounds__(TPJ > 128 ? TPJ : 128) k_cu_residual_wp(const ResidArgs a, const int4* __restrict__ wt)
{
    cu_residual<P, TPJ, MAXS, NT, true>(a, wt);
}

// the stage of a B slice (bd = the BIDIR records; the uni-predicted CUs take the same path as in k_cu_residual)
template <typename P, int TPJ, int MAXS, int NT>
__global__ void __launch_bounds__(TPJ > 128 ? TPJ : 128) k_cu_residual_bi(const ResidArgs a, const x265cu_bidir_cu* __restrict__ bd)
{
    cu_residual<P, TPJ, MAXS, NT, false, true>(a, nullptr, bd);
}

template <typename P, int TPJ, int MAXS, int NT>
static int resid_launch(x265cu_ctx* c, int maxPerSm, const ResidArgs& a, const int4* wt, const x265cu_bidir_cu* bd)
{
    constexpr int JPB = (TPJ > 128 ? TPJ : 128) / TPJ;
    const int items = (NT == 8 ? 1 : 2) * a.ntu;
    if (items == 0) return 0;
    const int grid = min((items + JPB - 1) / JPB, c->sm_count * maxPerSm), block = TPJ > 128 ? TPJ : 128;
    if (bd) k_cu_residual_bi<P, TPJ, MAXS, NT><<<grid, block, 0, c->stream>>>(a, bd);
    else if (wt) k_cu_residual_wp<P, TPJ, MAXS, NT><<<grid, block, 0, c->stream>>>(a, wt);
    else    k_cu_residual<P, TPJ, MAXS, NT><<<grid, block, 0, c->stream>>>(a);
    CU_LAUNCH_CHECK(c);
    return 0;
}

// One launch per luma TU size, each over its own list (lists[k] = TUs of luma size 8 << k, n[k] entries): luma TUs of 8 a
// warp each, of 16 a 128-thread CTA, of 32 a 256-thread CTA (at most 8 per SM); chroma TUs of 4 and 8 a warp each, of 16 a
// 128-thread CTA; at most 16 CTAs per SM otherwise.  wt (device, [16][3]) non-null: the weighted stage (k_cu_residual_wp);
// bd (device, [ncu]) non-null: the stage of a B slice (k_cu_residual_bi).
template <typename P>
static int launch_resid(x265cu_ctx* c, bool chroma, ResidArgs a, const int32_t* const lists[3], const int n[3], const int4* wt = nullptr,
                        const x265cu_bidir_cu* bd = nullptr)
{
    for (int k = 0; k < 3; k++)
    {
        a.tul = lists[k]; a.ntu = n[k];
        const int e = chroma ? (k < 2 ? resid_launch<P, 32, 8, 4>(c, 16, a, wt, bd) : resid_launch<P, 128, 16, 4>(c, 16, a, wt, bd))
                             : (k == 0 ? resid_launch<P, 32, 8, 8>(c, 16, a, wt, bd) : k == 1 ? resid_launch<P, 128, 16, 8>(c, 16, a, wt, bd)
                                                                                             : resid_launch<P, 256, 32, 8>(c, 8, a, wt, bd));
        if (e) return -1;
    }
    return 0;
}
