// x265_b200/csrc/predcost.cuh -- prediction costs of predInterSearch around the motion search, batched:
//   Search::selectMVP        (/root/reference/source/encoder/search.cpp:1992-2023)  SAD of the luma prediction at an AMVP candidate
//   Search::mergeEstimation  (search.cpp:1901-1960)  SATD (+ Cb/Cr SATD) of a merge candidate's motion-compensated prediction
//   bidir of predInterSearch (search.cpp:2474-2607)  SATD of the bi-prediction: addAvg of the two 14-bit intermediates
//                                                    (+ chroma) when bChromaSATD, else pixelavg_pp of two pixel predictions
// The prediction is Predict::motionCompensation's unweighted path (common/predict.cpp:76-240): predInterLumaPixel /
// predInterLumaShort / predInterChromaPixel / predInterChromaShort (predict.cpp:242-407), Yuv::addAvg (yuv.cpp:189-211);
// the costs are MotionEstimate::bufSAD / bufSATD / bufChromaSATD (encoder/motion.h:87-95).  4:2:0, vectors clipped by the
// caller (CUData::clipMv).  One job = one (PU, candidate); nothing is written but the cost.
//
// Four launches over the same list: one-list jobs on the motion search's sub-pel code (k_pred_uni, small / large PUs), two-list
// jobs staged through shared memory (k_pred_cost): PUs up to 16x16 take one WARP each (four per CTA, private tiles, warp
// barriers only), larger PUs one 128-thread CTA each; the prediction lives in shared memory from the source window to the cost.
#pragma once
#include "common.cuh"
#include "interp.cuh"
#include "pixelcmp.cuh"

template <int TPJ> __device__ __forceinline__ void pc_sync() { if (TPJ == 32) __syncwarp(); else __syncthreads(); }

// i -> (row, column) of a block `w` wide: a shift for the power-of-two widths (every symmetric PU), a division for 12 / 24 / 48
struct PcDiv { int w, lg; };
__device__ __forceinline__ PcDiv pc_div(int width) { PcDiv d; d.w = width; d.lg = (width & (width - 1)) ? -1 : 31 - __clz(width); return d; }
__device__ __forceinline__ void pc_split(const PcDiv& d, int i, int& y, int& x) { y = d.lg >= 0 ? i >> d.lg : i / d.w; x = i - y * d.w; }

// One plane's prediction of a w x h block into dst (int16, pitch DP): pixel domain (SHORT = false: copy / hpp / vpp / hvpp)
// or the 14-bit intermediate (SHORT = true: p2s / hps / vps / hps + vss).  NT = 8 (luma, quarter-pel) or 4 (chroma, eighth).
template <typename P, int TPJ, int MAXS, int NT, bool SHORT>
__device__ __forceinline__ void pc_predict(const P* __restrict__ ref, int stride, int mvx, int mvy, int w, int h,
                                           int16_t* __restrict__ dst, int16_t* __restrict__ s_win, int16_t* __restrict__ s_mid, int t)
{
    constexpr int DEPTH = PixTraits<P>::depth;
    constexpr int FB = NT == 8 ? 2 : 3, HL = NT / 2 - 1;          // fraction bits; taps left of / above the sample
    constexpr int WP = MAXS + 8, DP = MAXS;                       // window / destination pitch
    const int xf = mvx & ((1 << FB) - 1), yf = mvy & ((1 << FB) - 1);
    const P* src = ref + (mvx >> FB) + (ptrdiff_t)(mvy >> FB) * stride;
    if (!(xf | yf))
    {
        const PcDiv dw = pc_div(w);
        for (int i = t; i < w * h; i += TPJ)
        {
            int y, x; pc_split(dw, i, y, x);
            const int p = src[(ptrdiff_t)y * stride + x];
            dst[y * DP + x] = (int16_t)(SHORT ? (p << (14 - DEPTH)) - 8192 : p);
        }
        return;
    }
    const int hl = xf ? HL : 0, vt = yf ? HL : 0;
    const int ww = w + (xf ? NT - 1 : 0), wh = h + (yf ? NT - 1 : 0);
    const PcDiv dw = pc_div(w);
    for (int i = t; i < ww * wh; i += TPJ)
    {
        const int r = i / ww, c = i - r * ww;
        s_win[r * WP + c] = (int16_t)src[(ptrdiff_t)(r - vt) * stride + (c - hl)];
    }
    pc_sync<TPJ>();
    const int16_t* cx = NT == 8 ? c_lumaFilter[xf] : c_chromaFilter[xf];
    const int16_t* cy = NT == 8 ? c_lumaFilter[yf] : c_chromaFilter[yf];
    if (!yf || !xf)
    {
        const int step = !yf ? 1 : WP;
        const int16_t* cf = !yf ? cx : cy;
        for (int i = t; i < w * h; i += TPJ)
        {
            int y, x; pc_split(dw, i, y, x);
            int sum = 0;
#pragma unroll
            for (int k = 0; k < NT; k++) sum += (int)s_win[y * WP + x + k * step] * cf[k];
            dst[y * DP + x] = (int16_t)interp_finish<DEPTH>(sum, SHORT ? 1 : 0);
        }
    }
    else
    {
        for (int i = t; i < w * wh; i += TPJ)
        {
            int r, x; pc_split(dw, i, r, x);
            int sum = 0;
#pragma unroll
            for (int k = 0; k < NT; k++) sum += (int)s_win[r * WP + x + k] * cx[k];
            s_mid[r * DP + x] = (int16_t)interp_finish<DEPTH>(sum, 1);
        }
        pc_sync<TPJ>();
        for (int i = t; i < w * h; i += TPJ)
        {
            int y, x; pc_split(dw, i, y, x);
            int sum = 0;
#pragma unroll
            for (int k = 0; k < NT; k++) sum += (int)s_mid[(y + k) * DP + x] * cy[k];
            dst[y * DP + x] = (int16_t)interp_finish<DEPTH>(sum, SHORT ? 3 : 2);
        }
    }
}

// prediction of one plane for the job's lists into s_p0 (pixel values), per motionCompensation / the bidir estimate
template <typename P, int TPJ, int MAXS, int NT>
__device__ __forceinline__ void pc_plane(const P* r0, const P* r1, int stride, const x265cu_pred_job& jb, int w, int h,
                                         int16_t* s_p0, int16_t* s_p1, int16_t* s_win, int16_t* s_mid, int t)
{
    constexpr int DEPTH = PixTraits<P>::depth, maxv = PixTraits<P>::maxv, DP = MAXS;
    const bool bi = r0 && r1;
    pc_sync<TPJ>();                                               // the previous plane's cost has been read
    if (!bi)
    {
        pc_predict<P, TPJ, MAXS, NT, false>(r0 ? r0 : r1, stride, r0 ? jb.mv0[0] : jb.mv1[0], r0 ? jb.mv0[1] : jb.mv1[1], w, h, s_p0, s_win, s_mid, t);
        pc_sync<TPJ>();
        return;
    }
    if (jb.flags & X265CU_PRED_AVG_PP)
    {
        pc_predict<P, TPJ, MAXS, NT, false>(r0, stride, jb.mv0[0], jb.mv0[1], w, h, s_p0, s_win, s_mid, t);
        pc_sync<TPJ>();
        pc_predict<P, TPJ, MAXS, NT, false>(r1, stride, jb.mv1[0], jb.mv1[1], w, h, s_p1, s_win, s_mid, t);
        pc_sync<TPJ>();
        const PcDiv dw = pc_div(w);
        for (int i = t; i < w * h; i += TPJ)
        {
            int y, x; pc_split(dw, i, y, x);
            s_p0[y * DP + x] = (int16_t)(((int)s_p0[y * DP + x] + (int)s_p1[y * DP + x] + 1) >> 1);       // pixelavg_pp (pixel.cpp:545-557)
        }
    }
    else
    {
        pc_predict<P, TPJ, MAXS, NT, true>(r0, stride, jb.mv0[0], jb.mv0[1], w, h, s_p0, s_win, s_mid, t);
        pc_sync<TPJ>();
        pc_predict<P, TPJ, MAXS, NT, true>(r1, stride, jb.mv1[0], jb.mv1[1], w, h, s_p1, s_win, s_mid, t);
        pc_sync<TPJ>();
        constexpr int shift = 15 - DEPTH, offset = (1 << (shift - 1)) + 2 * 8192;                       // addAvg (pixel.cpp:842-862)
        const PcDiv dw = pc_div(w);
        for (int i = t; i < w * h; i += TPJ)
        {
            int y, x; pc_split(dw, i, y, x);
            s_p0[y * DP + x] = (int16_t)clip3i(0, maxv, ((int)s_p0[y * DP + x] + (int)s_p1[y * DP + x] + offset) >> shift);
        }
    }
    pc_sync<TPJ>();
}

// SAD / SATD of (source block in global memory, prediction in shared memory); the SATD tiling is the reference's per size
// (8x4 tiles halved once when the width is a multiple of 8, else 4x4 tiles: pixel.cpp:263-297, 1131-1155)
template <typename P, int TPJ, int MAXS>
__device__ __forceinline__ int pc_cost(const P* __restrict__ f, int fs, const int16_t* __restrict__ pr, int w, int h, bool satd, int t)
{
    constexpr int DP = MAXS;
    int acc = 0;
    if (!satd)
    {
        const PcDiv dw = pc_div(w);
        for (int i = t; i < w * h; i += TPJ) { int y, x; pc_split(dw, i, y, x); acc += abs((int)f[(ptrdiff_t)y * fs + x] - (int)pr[y * DP + x]); }
    }
    else if (!(w & 7))
    {
        const int tw = w >> 3, nt = tw * (h >> 2);
        for (int q = t; q < nt; q += TPJ)
        {
            const int ty = q / tw, tx = q - ty * tw;
            const P* pf = f + (ptrdiff_t)(ty * 4) * fs + tx * 8; const int16_t* pp = pr + (ty * 4) * DP + tx * 8;
            acc += (had4x4_abs(pf, fs, pp, DP) + had4x4_abs(pf + 4, fs, pp + 4, DP)) >> 1;
        }
    }
    else
    {
        const int tw = w >> 2, nt = tw * (h >> 2);
        for (int q = t; q < nt; q += TPJ)
        {
            const int ty = q / tw, tx = q - ty * tw;
            acc += had4x4_abs(f + (ptrdiff_t)(ty * 4) * fs + tx * 4, fs, pr + (ty * 4) * DP + tx * 4, DP) >> 1;
        }
    }
    return acc;
}

struct PredChroma { const void* fcb; const void* fcr; const void* const* rcb; const void* const* rcr; int cstride; };

// TPJ = 32: a warp per job (PUs up to MAXS = 16); TPJ = 128: a CTA per job (MAXS = 64)
template <typename P, int TPJ, int MAXS>
__global__ void __launch_bounds__(128, TPJ == 32 ? 8 : 4) k_pred_cost(const P* __restrict__ fenc, int fstride, const P* const* __restrict__ refs, int rstride,
                                                   PredChroma ch, const x265cu_pred_job* __restrict__ jobs, int n, int32_t* __restrict__ out, int uniElsewhere)
{
    constexpr int JPB = 128 / TPJ;
    constexpr int WIN = (MAXS + 7) * (MAXS + 8), MID = (MAXS + 7) * MAXS, PRD = MAXS * MAXS;
    __shared__ int16_t s_all[JPB][WIN + MID + 2 * PRD];
    __shared__ int s_red[4];
    const int grp = threadIdx.x / TPJ, t = threadIdx.x % TPJ;
    int16_t* s_win = s_all[grp]; int16_t* s_mid = s_win + WIN; int16_t* s_p0 = s_mid + MID; int16_t* s_p1 = s_p0 + PRD;
    for (int j = blockIdx.x * JPB + grp; j < n; j += gridDim.x * JPB)
    {
        const x265cu_pred_job jb = jobs[j];
        const int w = jb.pw, h = jb.ph;
        const bool small = w <= 16 && h <= 16;
        if (small != (MAXS == 16)) continue;                     // the sibling launch owns this job
        if (uniElsewhere && (jb.ref0 < 0 || jb.ref1 < 0)) continue;   // one-list jobs: k_pred_uni (the motion search's sub-pel code)
        if (uniElsewhere && small && !((w & (w - 1)) | (h & (h - 1)))) continue;   // ... and so are the two-list jobs of small pow2 PUs
        const P* r0 = jb.ref0 >= 0 ? refs[jb.ref0] + jb.offset : nullptr;
        const P* r1 = jb.ref1 >= 0 ? refs[jb.ref1] + jb.offset : nullptr;
        pc_plane<P, TPJ, MAXS, 8>(r0, r1, rstride, jb, w, h, s_p0, s_p1, s_win, s_mid, t);
        int acc = pc_cost<P, TPJ, MAXS>(fenc + jb.offset, fstride, s_p0, w, h, jb.cost == X265CU_PRED_SATD, t);
        const int cw = w >> 1, chh = h >> 1;
        const bool bi = r0 && r1;
        if (jb.cost == X265CU_PRED_SATD && (jb.flags & X265CU_PRED_CHROMA) && !(bi && (jb.flags & X265CU_PRED_AVG_PP)) && ch.fcb && !((cw | chh) & 3))
        {
            const int py = jb.offset / fstride, px = jb.offset - py * fstride;
            const ptrdiff_t coff = (ptrdiff_t)(py >> 1) * ch.cstride + (px >> 1);
            for (int p = 0; p < 2; p++)
            {
                const P* const* tab = (const P* const*)(p ? ch.rcr : ch.rcb);
                const P* c0 = jb.ref0 >= 0 ? tab[jb.ref0] + coff : nullptr;
                const P* c1 = jb.ref1 >= 0 ? tab[jb.ref1] + coff : nullptr;
                pc_plane<P, TPJ, MAXS, 4>(c0, c1, ch.cstride, jb, cw, chh, s_p0, s_p1, s_win, s_mid, t);
                acc += pc_cost<P, TPJ, MAXS>((const P*)(p ? ch.fcr : ch.fcb) + coff, ch.cstride, s_p0, cw, chh, true, t);
            }
        }
        acc = warp_sum(acc);
        if (TPJ == 32) { if (t == 0) out[j] = acc; }
        else
        {
            __syncthreads();
            if ((t & 31) == 0) s_red[t >> 5] = acc;
            __syncthreads();
            if (t == 0) out[j] = s_red[0] + s_red[1] + s_red[2] + s_red[3];
        }
    }
}

// ---- two-list jobs of small PUs (pow2, up to 16x16: 94 % of a frame's PUs) on the search's lane-per-row-segment code ------------
// The lane's row segment (NPX pixels of one row) of a prediction of the PU at the quarter-pel vector (qx, qy) on plane `ref`:
// SHORT = the 14-bit intermediate of predInterLumaShort (p2s / hps / vps / hps + vss), else the pixel prediction of
// predInterLumaPixel.  Same helpers and lane mapping as me_subpel_small_t (lane = row + h * segment; lanes >= h * segments idle);
// the hv case stages its h + 7 horizontally filtered rows in the warp's scratch.  All 32 lanes call.
template <typename P, int NPX, bool SHORT>
__device__ __forceinline__ void pb_seg(const MeCtx<P>& c, const P* __restrict__ ref, int qx, int qy, int (&pr)[NPX])
{
    const int lane = c.lane;
    const int lgsegs = NPX == 8 ? c.lgw - 3 : 0, lgh = 31 - __clz(c.h);
    const int lpc = 1 << (lgh + lgsegs);
    const int tasksPer = (c.h + 7) << lgsegs;
    int16_t* mid = c.sm->mid;
    const int xf = qx & 3, yf = qy & 3;
    __syncwarp();
    if (xf && yf)
        for (int t = lane; t < tasksPer; t += 32)
        {
            const int mrow = t >> lgsegs, seg = t & ((1 << lgsegs) - 1);
            me_hv_row<P, NPX>(ref + (qx >> 2) + (ptrdiff_t)((qy >> 2) - 3 + mrow) * c.rstride + seg * 8, xf, mid + mrow * c.w + seg * 8);
        }
    __syncwarp();
    const int sub = lane & (lpc - 1), row = sub & (c.h - 1), seg = sub >> lgh;
    if (lane < lpc)
        me_pred_seg<P, NPX, SHORT>(ref + (qx >> 2) + (ptrdiff_t)((qy >> 2) + row) * c.rstride + seg * 8, c.rstride, xf, yf,
                                   mid + row * c.w + seg * 8, c.w, pr);
    else
    {
#pragma unroll
        for (int x = 0; x < NPX; x++) pr[x] = 0;
    }
}

// luma cost of a bi-prediction: addAvg of the two 14-bit predictions (Yuv::addAvg) or, with avgpp, pixelavg_pp of the two
// pixel predictions; SAD or SATD against the source rows as in me_subpel_small_t's stage 3.  Result in lane 0.
template <typename P, int NPX>
__device__ __forceinline__ int pb_bi_luma(const MeCtx<P>& c, const P* __restrict__ ref0, const P* __restrict__ ref1, int qx0, int qy0, int qx1, int qy1,
                                          bool avgpp, bool satd)
{
    constexpr int DEPTH = PixTraits<P>::depth, maxv = PixTraits<P>::maxv;
    const int lane = c.lane;
    const int lgsegs = NPX == 8 ? c.lgw - 3 : 0, lgh = 31 - __clz(c.h);
    const int lpc = 1 << (lgh + lgsegs);
    int a[NPX], b[NPX], d[NPX];
    if (avgpp) { pb_seg<P, NPX, false>(c, ref0, qx0, qy0, a); pb_seg<P, NPX, false>(c, ref1, qx1, qy1, b); }
    else       { pb_seg<P, NPX, true>(c, ref0, qx0, qy0, a);  pb_seg<P, NPX, true>(c, ref1, qx1, qy1, b); }
    const int sub = lane & (lpc - 1), row = sub & (c.h - 1), seg = sub >> lgh;
    if (lane < lpc)
    {
        constexpr int shift = 15 - DEPTH, offset = (1 << (shift - 1)) + 2 * 8192;
        int fv[NPX];
        me_load_fenc<P, NPX>(c, c.fenc + (ptrdiff_t)row * c.fstride + seg * 8, fv);
#pragma unroll
        for (int x = 0; x < NPX; x++)
        {
            const int pr = avgpp ? (a[x] + b[x] + 1) >> 1 : clip3i(0, maxv, (a[x] + b[x] + offset) >> shift);
            d[x] = fv[x] - pr;
        }
    }
    else
    {
#pragma unroll
        for (int x = 0; x < NPX; x++) d[x] = 0;
    }
    return __shfl_sync(0xffffffffu, me_seg_cost<NPX>(d, satd, lane, lpc), 0);
}

// Cb + Cr SATD of a bi-prediction's chroma (predInterChromaShort x 2 + addAvg), small PUs: me_chroma_batch_cols' lane mapping
// (four lanes per 4x4 tile, one column each) for ONE candidate with two lists.  The single separable path (hps with rowExt, then
// vss) reproduces p2s / hps / vps exactly for zero phases through the identity taps {0, 64, 0, 0}: mid = 64 p - 8192 (8-bit) or
// 16 p - 8192 (10-bit) is exact and sum(c) = 64, so (sum(c mid)) >> 6 equals the direct forms (see DESIGN.md section 4).
template <typename P>
__device__ __forceinline__ int pb_bi_chroma(const MeCtx<P>& c, const MeChromaCtx<P>& c0, const MeChromaCtx<P>& c1, int qx0, int qy0, int qx1, int qy1)
{
    constexpr int DEPTH = PixTraits<P>::depth, maxv = PixTraits<P>::maxv;
    const int lgtpr = c.lgw - 3;
    const int lgnt = lgtpr + (31 - __clz(c.h)) - 3;
    const int lgipc = lgnt + 3, total = 1 << lgipc;                // lane-items of the candidate: 8 / 16 / 32
    const int lggs = 2 + lgtpr;
    const int it = min(c.lane, total - 1);
    const int col = it & 3, t = it >> 2;
    const bool cr = (t >> lgnt) != 0;
    const int tt = t & ((1 << lgnt) - 1);
    const int ty = tt >> lgtpr, tx = tt & ((1 << lgtpr) - 1);
    const ptrdiff_t o = (ptrdiff_t)(ty * 4) * c0.cstride + tx * 4 + col;
    const P* f = (cr ? c0.fcr : c0.fcb) + o;
    int sh[2][4];
#pragma unroll
    for (int l = 0; l < 2; l++)
    {
        const MeChromaCtx<P>& cc = l ? c1 : c0;
        const int qx = l ? qx1 : qx0, qy = l ? qy1 : qy0;
        const P* r = (cr ? cc.rcr : cc.rcb) + o + (qx >> 3) + (ptrdiff_t)(qy >> 3) * cc.cstride - 1 - cc.cstride;
        const uint32_t th = __ldg(&d_chromaTaps4[qx & 7]), tv = __ldg(&d_chromaTaps4[qy & 7]);
        const int v0 = (int)(int8_t)tv, v1 = (int)(int8_t)(tv >> 8), v2 = (int)(int8_t)(tv >> 16), v3 = (int)tv >> 24;
        int mid[7];
#pragma unroll
        for (int q = 0; q < 7; q++) mid[q] = interp_finish<DEPTH>(me_chroma_hsum<P>(r + q * cc.cstride, th), 1);
#pragma unroll
        for (int y = 0; y < 4; y++) sh[l][y] = interp_finish<DEPTH>(v0 * mid[y] + v1 * mid[y + 1] + v2 * mid[y + 2] + v3 * mid[y + 3], 3);
    }
    constexpr int shift = 15 - DEPTH, offset = (1 << (shift - 1)) + 2 * 8192;
    int d[4];
#pragma unroll
    for (int y = 0; y < 4; y++) d[y] = (int)__ldg(f + y * c0.cstride) - clip3i(0, maxv, (sh[0][y] + sh[1][y] + offset) >> shift);
    had4(d[0], d[1], d[2], d[3]);
    const int s1 = (c.lane & 1) ? -1 : 1, s2 = (c.lane & 2) ? -1 : 1;
#pragma unroll
    for (int y = 0; y < 4; y++)
    {
        d[y] = __shfl_xor_sync(0xffffffffu, d[y], 1) + s1 * d[y];
        d[y] = __shfl_xor_sync(0xffffffffu, d[y], 2) + s2 * d[y];
    }
    int v = abs(d[0]) + abs(d[1]) + abs(d[2]) + abs(d[3]);
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    if (lggs == 3) v += __shfl_xor_sync(0xffffffffu, v, 4);
    v >>= 1;
    for (int s = lggs; s < lgipc; s++) v += __shfl_xor_sync(0xffffffffu, v, 1 << s);
    return __shfl_sync(0xffffffffu, v, 0);
}

// One-list jobs (AMVP candidates, uni-directional merge candidates) are exactly what MotionEstimate::subpelCompare computes for
// one candidate (motion.cpp:1571-1664: the same copy / hpp / vpp / hvpp prediction, SAD or SATD, + the chroma-SATD term), so
// they run on the motion search's own sub-pel code (me.cuh: me_subpel_batch, me_chroma_batch -- lane-per-row-segment DP4A
// interpolation straight from the planes) instead of the staged generic path above: a warp per job, small-PU and large-PU
// instantiations as in the search.  Same arithmetic, ~5x fewer instructions per job.
template <typename P, int CLS>
__global__ void __launch_bounds__(256, CLS == 1 ? ME_BIG_BLOCKS : ME_MIN_BLOCKS) k_pred_uni(const P* __restrict__ fenc, int fstride, const P* const* __restrict__ refs, int rstride,
                                                                                        MeChromaArgs ch, int haveChroma, const x265cu_pred_job* __restrict__ jobs, int n,
                                                                                        int32_t* __restrict__ out, int* __restrict__ counter)
{
    extern __shared__ unsigned char me_smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    MeShared* sm = (MeShared*)me_smem + warp;
    for (;;)
    {
        int jid = 0;
        if (lane == 0) jid = atomicAdd(counter, 1);
        jid = __shfl_sync(0xffffffffu, jid, 0);
        if (jid >= n) break;
        const x265cu_pred_job pj = jobs[jid];
        const bool bi = pj.ref0 >= 0 && pj.ref1 >= 0;
        if (bi && CLS != 0) continue;                              // two lists, large PUs: k_pred_cost
        const bool l0 = pj.ref0 >= 0;
        x265cu_me_job j;
        j.offset = pj.offset; j.ref = (int16_t)(l0 ? pj.ref0 : pj.ref1); j.pw = (int8_t)pj.pw; j.ph = (int8_t)pj.ph;
        j.mvmin[0] = j.mvmin[1] = j.mvmax[0] = j.mvmax[1] = 0; j.qmvp[0] = j.qmvp[1] = 0;
#pragma unroll
        for (int k = 0; k < 8; k++) j.mvc[k] = 0;
        j.numCand = 0; j.method = 3; j.merange = 0;
        j.subme = (int8_t)((pj.flags & X265CU_PRED_CHROMA) ? 3 : 2);
        MeCtx<P> c;
        me_make_ctx<P>(c, j, fenc, fstride, refs, rstride, 0, nullptr, lane, sm);
        if (me_subpel_class(c) != CLS) continue;                   // the sibling launch owns this job (two lists: k_pred_cost)
        const bool satd = pj.cost == X265CU_PRED_SATD;
        if (bi)
        {   // CLS 0 only: both lists on the lane-per-row-segment code
            const P* ref1 = refs[pj.ref1] + pj.offset;
            const bool avgpp = (pj.flags & X265CU_PRED_AVG_PP) != 0;
            int cost = c.w >= 8 ? pb_bi_luma<P, 8>(c, c.ref[0], ref1, pj.mv0[0], pj.mv0[1], pj.mv1[0], pj.mv1[1], avgpp, satd)
                                : pb_bi_luma<P, 4>(c, c.ref[0], ref1, pj.mv0[0], pj.mv0[1], pj.mv1[0], pj.mv1[1], avgpp, satd);
            if (satd && !avgpp && haveChroma && (pj.flags & X265CU_PRED_CHROMA))
            {
                MeChromaCtx<P> c0, c1;
                me_set_chroma<P>(c0, c, j, ch, fstride);
                j.ref = (int16_t)pj.ref1;
                me_set_chroma<P>(c1, c, j, ch, fstride);
                if (c0.on) cost += pb_bi_chroma<P>(c, c0, c1, pj.mv0[0], pj.mv0[1], pj.mv1[0], pj.mv1[1]);
            }
            if (lane == 0) out[jid] = cost;
            __syncwarp();
            continue;
        }
        const int qx = l0 ? pj.mv0[0] : pj.mv1[0], qy = l0 ? pj.mv0[1] : pj.mv1[1];
        int cost = me_subpel_batch<P, CLS>(c, 1, qx, qy, satd);
        if (satd && haveChroma && (pj.flags & X265CU_PRED_CHROMA))
        {
            MeChromaCtx<P> cc;
            me_set_chroma<P>(cc, c, j, ch, fstride);
            if (cc.on) cost += me_chroma_batch<P, CLS>(c, cc, 1, qx, qy, 1u);
        }
        if (lane == 0) out[jid] = cost;
        __syncwarp();
    }
}

template <typename P>
static int launch_pred_cost_t(x265cu_ctx* ctx, const void* fenc, int fstride, const void* const* refs, int rstride, const PredChroma& ch,
                              const x265cu_pred_job* jobs, int n, int32_t* out)
{
    // one-list jobs
    {
        CU_CHECK(cudaMemsetAsync(ctx->d_counter + 12, 0, 2 * sizeof(int), ctx->stream));
        MeChromaArgs a; a.fencCb = ch.fcb; a.fencCr = ch.fcr; a.refCb = ch.rcb; a.refCr = ch.rcr; a.cstride = ch.cstride;
        const int threads = 256, warps = threads / 32;
        const size_t smem = sizeof(MeShared) * warps;
        const int need = (n + warps - 1) / warps;
        int b0 = ctx->sm_count * ME_MIN_BLOCKS, b1 = ctx->sm_count * ME_BIG_BLOCKS;
        if (b0 > need) b0 = need;
        if (b1 > need) b1 = need;
        k_pred_uni<P, 0><<<b0, threads, smem, ctx->stream>>>((const P*)fenc, fstride, (const P* const*)refs, rstride, a, ch.fcb != NULL, jobs, n, out, ctx->d_counter + 12);
        CU_LAUNCH_CHECK(ctx);
        k_pred_uni<P, 1><<<b1, threads, smem, ctx->stream>>>((const P*)fenc, fstride, (const P* const*)refs, rstride, a, ch.fcb != NULL, jobs, n, out, ctx->d_counter + 13);
        CU_LAUNCH_CHECK(ctx);
    }
    // two-list jobs
    const int maxb = ctx->sm_count * 16;
    int b1 = (n + 3) / 4; if (b1 > maxb) b1 = maxb;
    int b2 = n < maxb ? n : maxb;
    k_pred_cost<P, 32, 16><<<b1, 128, 0, ctx->stream>>>((const P*)fenc, fstride, (const P* const*)refs, rstride, ch, jobs, n, out, 1);
    CU_LAUNCH_CHECK(ctx);
    k_pred_cost<P, 128, 64><<<b2, 128, 0, ctx->stream>>>((const P*)fenc, fstride, (const P* const*)refs, rstride, ch, jobs, n, out, 1);
    CU_LAUNCH_CHECK(ctx);
    return 0;
}
