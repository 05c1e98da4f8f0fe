// x265_b200/csrc/chroma_resid.cuh -- 4:2:0 chroma residual chain of every CU's best inter prediction (analyser stage bit 3):
// per luma TU of the CU (T = min(S, 32)) and per chroma plane, one (T/2) x (T/2) chroma TU (geometry_chroma_tu):
//   chroma MC (predInterChromaPixel, predict.cpp:306-353: the luma quarter-pel vector read as eighth-pel) -> sub_ps -> dct
//   -> quant -> dequant_normal -> idct / DC shortcut -> add_ps -> sse_pp  (search.cpp:2990-3080, quant.cpp:397-470, :543-605,
//   non-RDOQ path; the same chain as k_cu_residual with the chroma TU size and the plane's chroma QP).
// The reference and vector are the luma stage's choice: lowest ME cost of the CU's 2Nx2N jobs, ties to the lowest index.
// Chroma TUs are 4, 8 and 16 wide.  Two launches over the same (TU, plane) list: TUs of 4 and 8 take one WARP each (four per
// CTA, private shared tiles, warp barriers only), TUs of 16 one 128-thread CTA each.  The MC is pc_predict (predcost.cuh).
#pragma once
#include "common.cuh"
#include "predcost.cuh"
#include "frame.cuh"

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

// sum over the TPJ threads of a job group, in every thread of the group
template <int TPJ>
__device__ __forceinline__ int cr_group_sum(int v, int* s_red)
{
    v = warp_sum(v);
    if (TPJ == 32) return v;
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
    __syncthreads();
    return s_red[0] + s_red[1] + s_red[2] + s_red[3];
}

// Item j of [0, 2 * ntu) = plane j & 1 (0 Cb, 1 Cr) of TU j >> 1.  recon = 8 origin pointers [depthIdx][plane]; levels and
// recon of a plane share its chroma geometry (cstride); cu_sse / cu_numsig are [cu][plane] and accumulate.
template <typename P, int TPJ, int MAXS>
__global__ void __launch_bounds__(128) k_cu_chroma_residual(const P* __restrict__ fcb, const P* __restrict__ fcr,
                                                            const P* const* __restrict__ rcb, const P* const* __restrict__ rcr, int cstride,
                                                            const CuDesc* __restrict__ cus, const TuDesc* __restrict__ tus, int ntu,
                                                            const int32_t* __restrict__ cu_jobs, int numRefs, const int32_t* __restrict__ me_out,
                                                            int qpCb, int qpCr, int16_t* __restrict__ coefCb, int16_t* __restrict__ coefCr,
                                                            P* const* __restrict__ recon, unsigned long long* __restrict__ cu_sse,
                                                            uint32_t* __restrict__ cu_numsig)
{
    constexpr int DEPTH = PixTraits<P>::depth, maxv = PixTraits<P>::maxv;
    constexpr int JPB = 128 / TPJ, DP = MAXS;
    constexpr int WIN = (MAXS + 3) * (MAXS + 8), MID = (MAXS + 3) * MAXS, NN = MAXS * MAXS;
    __shared__ int16_t s_all[JPB][WIN + MID + 3 * NN];
    __shared__ int s_red[4];
    __shared__ int s_lvl0[JPB];                                   // quantised DC level of the group's TU
    const int grp = threadIdx.x / TPJ, t = threadIdx.x % TPJ;
    int16_t* s_win = s_all[grp]; int16_t* s_mid = s_win + WIN; int16_t* s_pred = s_mid + MID;
    int16_t* s_a = s_pred + NN; int16_t* s_b = s_a + NN;
    for (int j = blockIdx.x * JPB + grp; j < 2 * ntu; j += gridDim.x * JPB)
    {
        const TuDesc tu = tus[j >> 1];
        const int plane = j & 1;
        const CuDesc cu = cus[tu.cu];
        const ChromaTu c = geometry_chroma_tu(cu, tu);
        const int Tc = c.size;
        if ((Tc > 8) != (MAXS == 16)) continue;                  // the sibling launch owns this TU
        const int lg = 31 - __clz(Tc), N = Tc * Tc;
        int best = 0, bcost = 0x7fffffff;
        for (int r = 0; r < numRefs; r++)
        {
            const int cost = me_out[(size_t)cu_jobs[tu.cu * numRefs + r] * 4];
            if (cost < bcost) { bcost = cost; best = r; }
        }
        const int32_t* mo = me_out + (size_t)cu_jobs[tu.cu * numRefs + best] * 4;
        const int qx = mo[1], qy = mo[2];
        const ptrdiff_t off = (ptrdiff_t)c.y * cstride + c.x;
        const P* ref = (plane ? rcr : rcb)[best] + off;
        const P* fe = (plane ? fcr : fcb) + off;
        pc_sync<TPJ>();                                           // the previous item's tiles have been read
        pc_predict<P, TPJ, MAXS, 4, false>(ref, cstride, qx, qy, Tc, Tc, s_pred, s_win, s_mid, t);
        pc_sync<TPJ>();
        // ---- residual ----
        for (int i = t; i < N; i += TPJ)
        {
            const int y = i >> lg, x = i & (Tc - 1);
            s_a[i] = (int16_t)((int)fe[(ptrdiff_t)y * cstride + x] - (int)s_pred[y * DP + x]);
        }
        pc_sync<TPJ>();
        // ---- forward DCT, rows then columns (dct.cpp:83-240, 442-525) ----
        const int8_t* M = d_dct[lg - 2];
        {
            const int sh1 = lg - 1 + (DEPTH - 8), sh2 = lg + 6;
            for (int i = t; i < N; i += TPJ)
            {
                const int k = i >> lg, jj = i & (Tc - 1);
                int acc = 0;
                for (int q = 0; q < Tc; q++) acc += (int)M[k * Tc + q] * s_a[jj * Tc + q];
                s_b[k * Tc + jj] = (int16_t)((acc + (1 << (sh1 - 1))) >> sh1);
            }
            pc_sync<TPJ>();
            for (int i = t; i < N; i += TPJ)
            {
                const int k = i >> lg, jj = i & (Tc - 1);
                int acc = 0;
                for (int q = 0; q < Tc; q++) acc += (int)M[k * Tc + q] * s_b[jj * Tc + q];
                s_a[i] = (int16_t)((acc + (1 << (sh2 - 1))) >> sh2);
            }
            pc_sync<TPJ>();
        }
        // ---- quant (dct.cpp:664-686) + dequant_normal (dct.cpp:612-634) ----
        const ResidQuant rq = resid_quant<DEPTH>(plane ? qpCr : qpCb, lg);
        int16_t* qout = (plane ? coefCr : coefCb) + c.off;
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
        const int numSig = cr_group_sum<TPJ>(cnt, s_red);
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
                const int jj = i >> lg, i2 = i & (Tc - 1);
                int acc = 0;
                for (int q = 0; q < Tc; q++) acc += (int)M[q * Tc + i2] * s_b[q * Tc + jj];
                s_a[i] = (int16_t)clip16((acc + 64) >> 7);
            }
            pc_sync<TPJ>();
            for (int i = t; i < N; i += TPJ)
            {
                const int jj = i >> lg, i2 = i & (Tc - 1);
                int acc = 0;
                for (int q = 0; q < Tc; q++) acc += (int)M[q * Tc + i2] * s_a[q * Tc + jj];
                s_b[i] = (int16_t)clip16((acc + (1 << (sh2 - 1))) >> sh2);
            }
            res = s_b;
        }
        pc_sync<TPJ>();
        // ---- reconstruction (add_ps with the clip, or the prediction) + distortion ----
        const int dIdx = cu.size == 64 ? 0 : (cu.size == 32 ? 1 : (cu.size == 16 ? 2 : 3));
        P* rc = recon[2 * dIdx + plane] + off;
        unsigned long long sse = 0;
        for (int i = t; i < N; i += TPJ)
        {
            const int y = i >> lg, x = i & (Tc - 1);
            const int p = s_pred[y * DP + x];
            const int v = numSig ? clip3i(0, maxv, p + (int)res[i]) : p;
            rc[(ptrdiff_t)y * cstride + x] = (P)v;
            const int d = (int)fe[(ptrdiff_t)y * cstride + x] - v;
            sse += (unsigned)(d * d);
        }
        sse = warp_sum64(sse);
        if ((t & 31) == 0 && sse) atomicAdd(&cu_sse[2 * tu.cu + plane], sse);
        if (t == 0 && numSig) atomicAdd(&cu_numsig[2 * tu.cu + plane], (uint32_t)numSig);
    }
}

template <typename P>
static int launch_cu_chroma_residual(x265cu_ctx* c, const void* fcb, const void* fcr, const void* const* rcb, const void* const* rcr, int cstride,
                                     const CuDesc* cus, const TuDesc* tus, int ntu, const int32_t* cu_jobs, int numRefs, const int32_t* me_out,
                                     int qpCb, int qpCr, int16_t* coefCb, int16_t* coefCr, void* const* recon,
                                     unsigned long long* cu_sse, uint32_t* cu_numsig)
{
    const int n = 2 * ntu, maxb = c->sm_count * 16;
    int b1 = (n + 3) / 4; if (b1 > maxb) b1 = maxb;
    const int b2 = n < maxb ? n : maxb;
    k_cu_chroma_residual<P, 32, 8><<<b1, 128, 0, c->stream>>>((const P*)fcb, (const P*)fcr, (const P* const*)rcb, (const P* const*)rcr, cstride,
        cus, tus, ntu, cu_jobs, numRefs, me_out, qpCb, qpCr, coefCb, coefCr, (P* const*)recon, cu_sse, cu_numsig);
    CU_LAUNCH_CHECK(c);
    k_cu_chroma_residual<P, 128, 16><<<b2, 128, 0, c->stream>>>((const P*)fcb, (const P*)fcr, (const P* const*)rcb, (const P* const*)rcr, cstride,
        cus, tus, ntu, cu_jobs, numRefs, me_out, qpCb, qpCr, coefCb, coefCr, (P* const*)recon, cu_sse, cu_numsig);
    CU_LAUNCH_CHECK(c);
    return 0;
}
