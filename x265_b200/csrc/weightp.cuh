// x265_b200/csrc/weightp.cuh -- the frame encoder's weighted-prediction analysis, weightAnalyse
// (encoder/weightPrediction.cpp:222-539), on the lookahead's device-resident planes and motion fields.
//   k_weightp_costs : weightCost (:169-218) of a list of candidates for one plane.  One warp per 8x8 block: the block of
//                     the (motion-compensated) reference -- mcLuma / Lowres::lowresMC (:60-89) or mcChroma (:93-163) with
//                     its four filter paths -- and of the source go to shared memory, then 8-lane groups score four
//                     candidates at a time (weight_pp, satd8x8_group, the luma min with intraCost).  The per-candidate
//                     sums wrap in uint32 as the reference's do; the order of additions does not matter.
//   host            : the search (:260-501) restated literally; its candidates depend on the picture statistics only, so
//                     each (list, plane) takes one launch and one download.
#pragma once
#include "common.cuh"
#include "interp.cuh"
#include "lookahead.cuh"
#include <limits.h>
#include <math.h>

#define WP_MAX_CANDS 48

struct WpCostArgs
{
    const void* fenc;            // luma: lowres plane 0 of fenc; chroma: the fenc chroma plane (both at picture origin)
    const void* ref[4];          // luma: the 4 hpel planes of ref; chroma: ref[0] = the ref chroma plane
    int fs, rs;                  // strides (pixels) of fenc / ref
    const int32_t* mvs;          // int32 pairs per lowres CU, or NULL
    const int32_t* intraCost;    // luma only
    int chroma;                  // 0 luma, 1 chroma
    int width, height;           // analysed area: w8 * 8 x h8 * 8 (luma), cw x ch (chroma)
    int w8, h8;                  // lowresWidthInCU / lowresHeightInCU
    int ncand;
    x265cu_wp_cand cand[WP_MAX_CANDS];
};

// one pixel (r, k) of the 8x8 reference block at (x, y), as mcLuma / mcChroma / the plain plane give it
template <typename P, int DEPTH>
__device__ __forceinline__ int wp_ref_pixel(const WpCostArgs& a, int x, int y, int r, int k)
{
    constexpr int maxv = (1 << DEPTH) - 1;
    const int rs = a.rs;
    if (!a.chroma)
    {
        const P* const* pl = (const P* const*)a.ref;
        if (!a.mvs) return pl[0][(ptrdiff_t)(y + r) * rs + x + k];
        const int cu = (y >> 3) * a.w8 + (x >> 3);
        const int qx = clip3i((-x - 8) * 4, (a.width - x - 1 + 8) * 4, a.mvs[2 * cu]);
        const int qy = clip3i((-y - 8) * 4, (a.height - y - 1 + 8) * 4, a.mvs[2 * cu + 1]);
        const int ha = (qy & 2) | ((qx & 2) >> 1);
        const int va = pl[ha][(ptrdiff_t)(y + r + (qy >> 2)) * rs + x + k + (qx >> 2)];
        if (!((qx | qy) & 1)) return va;
        const int rx = qx + (qx & 1), ry = qy + (qy & 1);          // lowresMC's second plane, pixelavg_pp
        const int hb = (ry & 2) | ((rx & 2) >> 1);
        return (va + pl[hb][(ptrdiff_t)(y + r + (ry >> 2)) * rs + x + k + (rx >> 2)] + 1) >> 1;
    }
    const P* src = (const P*)a.ref[0];
    if (!a.mvs || !(x < a.w8 && y < a.h8))                          // mcChroma compares pixel x / y with CU counts
        return src[(ptrdiff_t)(y + r) * rs + x + k];
    const int cu = y * a.w8 + (x >> 3);                             // y is a pixel row (:114)
    // mv <<= 1, then >>= 1 (4:2:0), clipped in units of 4
    const int mx = clip3i((-x - 8) * 4, (a.width - x - 1 + 8) * 4, (int)((unsigned)a.mvs[2 * cu] << 1) >> 1);
    const int my = clip3i((-y - 8) * 4, (a.height - y - 1 + 8) * 4, (int)((unsigned)a.mvs[2 * cu + 1] << 1) >> 1);
    const P* t = src + (ptrdiff_t)(y + (my >> 2)) * rs + x + (mx >> 2);
    const int xf = mx & 7, yf = my & 7;
    if (!(xf | yf)) return t[(ptrdiff_t)r * rs + k];
    const int16_t* cx = c_chromaFilter[xf];
    const int16_t* cy = c_chromaFilter[yf];
    if (!yf)                                                        // filter_hpp
    {
        const P* s = t + (ptrdiff_t)r * rs + k - 1;
        return interp_finish<DEPTH>(s[0] * cx[0] + s[1] * cx[1] + s[2] * cx[2] + s[3] * cx[3], 0);
    }
    if (!xf)                                                        // filter_vpp
    {
        const P* s = t + (ptrdiff_t)(r - 1) * rs + k;
        return interp_finish<DEPTH>(s[0] * cy[0] + s[rs] * cy[1] + s[2 * rs] * cy[2] + s[3 * rs] * cy[3], 0);
    }
    int sum = 0;                                                    // filter_hps (row extension) + filter_vsp
#pragma unroll
    for (int i = 0; i < 4; i++)
    {
        const P* s = t + (ptrdiff_t)(r - 1 + i) * rs + k - 1;
        sum += interp_finish<DEPTH>(s[0] * cx[0] + s[1] * cx[1] + s[2] * cx[2] + s[3] * cx[3], 1) * cy[i];
    }
    (void)maxv;
    return interp_finish<DEPTH>(sum, 2);
}

template <typename P>
__global__ void __launch_bounds__(256) k_weightp_costs(const __grid_constant__ WpCostArgs a, uint32_t* __restrict__ costs)
{
    constexpr int DEPTH = PixTraits<P>::depth, maxv = PixTraits<P>::maxv, corr = 14 - DEPTH;
    __shared__ int16_t s_ref[8][64], s_fenc[8][64];
    __shared__ uint32_t s_sum[WP_MAX_CANDS];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, grp = lane >> 3, row = lane & 7;
    for (int i = threadIdx.x; i < WP_MAX_CANDS; i += blockDim.x) s_sum[i] = 0;
    __syncthreads();
    const int bw = a.width >> 3, nblk = bw * (a.height >> 3);
    const P* fenc = (const P*)a.fenc;
    uint32_t acc[WP_MAX_CANDS / 4];
#pragma unroll
    for (int i = 0; i < WP_MAX_CANDS / 4; i++) acc[i] = 0;
    for (int b = blockIdx.x * 8 + warp; b < nblk; b += gridDim.x * 8)
    {
        const int by = b / bw, x = (b - by * bw) * 8, y = by * 8;
#pragma unroll
        for (int h = 0; h < 2; h++)
        {
            const int j = lane + 32 * h, r = j >> 3, k = j & 7;
            s_ref[warp][j] = (int16_t)wp_ref_pixel<P, DEPTH>(a, x, y, r, k);
            s_fenc[warp][j] = (int16_t)fenc[(ptrdiff_t)(y + r) * a.fs + x + k];
        }
        __syncwarp();
        const int icost = a.chroma ? INT_MAX : a.intraCost[b];
#pragma unroll
        for (int it = 0; it < WP_MAX_CANDS / 4; it++)
        {
            if (it * 4 >= a.ncand) break;                           // warp-uniform
            const x265cu_wp_cand c = a.cand[min(it * 4 + grp, a.ncand - 1)];
            const int round = (c.denom ? 1 << (c.denom - 1) : 0) << corr, shift = c.denom + corr;
            const int off = c.offset * (1 << (DEPTH - 8));
            int d[8];
#pragma unroll
            for (int k = 0; k < 8; k++)
            {
                int rv = s_ref[warp][row * 8 + k];
                if (c.weighted) rv = clip3i(0, maxv, ((c.w0 * (int)(int16_t)(rv << corr) + round) >> shift) + off);
                d[k] = rv - s_fenc[warp][row * 8 + k];
            }
            const int satd = satd8x8_group(d, lane);
            acc[it] += (uint32_t)min(satd, icost);
        }
        __syncwarp();
    }
#pragma unroll
    for (int it = 0; it < WP_MAX_CANDS / 4; it++)
        if (row == 0 && it * 4 + grp < a.ncand) atomicAdd(&s_sum[it * 4 + grp], acc[it]);
    __syncthreads();
    for (int i = threadIdx.x; i < a.ncand; i += blockDim.x) atomicAdd(&costs[i], s_sum[i]);
}

namespace wpa {

// (int) of a float as x86's cvttss2si computes it (law::la_cvttss2si): refMean == 0 in the offset rescale divides by zero
static inline int cvt(float v) { return (v >= -2147483648.f && v < 2147483648.f) ? (int)v : INT_MIN; }
static inline int clip3(int lo, int hi, int v) { return v < lo ? lo : (v > hi ? hi : v); }
// bitSize (common/bitstream.h:94-112)
static int bitsize(unsigned v) { int n = 0; while (v >> (n + 1)) n++; return v ? 2 * n + 1 : 1; }
static int bs_size_se(int val)
{
    int tmp = 1 - val * 2;
    if (tmp < 0) tmp = val * 2;
    return tmp < 256 ? bitsize((unsigned)tmp) : bitsize((unsigned)tmp >> 8) + 16;
}
// sliceHeaderCost (:49-56)
static int slice_header_cost(int weight, int denom, int offset, int lambda, int bChroma)
{
    if (bChroma) lambda *= 4;
    const int denomCost = bitsize((unsigned)denom + 1) * (2 - bChroma);
    return lambda * (10 + denomCost + 2 * (bs_size_se(weight) + bs_size_se(offset)));
}
static void set_w(x265cu_wp_entry& w, int present, int scale, int denom, int off)
{
    w.wtPresent = present; w.inputWeight = scale; w.log2WeightDenom = denom; w.inputOffset = off;
}

static const char* check_params(int depth, const x265cu_wp_params* p)
{
    if (depth != 8 && depth != 10) return "depth must be 8 or 10";
    if (!p) return "params is NULL";
    if (p->sliceType != 0 && p->sliceType != 1) return "sliceType must be 0 (B) or 1 (P)";
    if (p->csp != 0 && p->csp != 1) return "csp must be 0 (4:0:0) or 1 (4:2:0)";
    if (p->width < 16 || p->height < 16 || (p->width & 7) || (p->height & 7)) return "width / height must be multiples of 8, at least 16";
    if (p->bframes < 0 || p->bframes > 16) return "bframes must be 0..16";
    for (int l = 0; l < (p->sliceType == 1 ? 1 : 2); l++)
        if (p->numRefIdx[l] < 1 || p->numRefIdx[l] > 16) return "numRefIdx must be 1..16";
    return NULL;
}

static int refuse(const char* fn, const char* why)
{
    char msg[200];
    snprintf(msg, sizeof(msg), "%s: %s", fn, why);
    x265cu_set_error(msg, cudaErrorInvalidValue, __FILE__, __LINE__);
    return -1;
}

} // namespace wpa

static const char* weightp_costs_check(int depth, const x265cu_wp_params* p, const x265cu_wp_frame* fenc,
                                       const x265cu_wp_frame* ref, const int32_t* intraCost, int plane,
                                       const x265cu_wp_cand* cands, int ncand, const uint32_t* costs)
{
    const char* bad = wpa::check_params(depth, p);
    if (bad) return bad;
    if (!fenc || !ref || !cands || !costs) return "NULL record, candidate or cost pointer";
    if (plane < 0 || plane > 2 || (plane && !p->csp)) return "plane must be 0, or 1 / 2 in 4:2:0";
    if (ncand < 1 || ncand > WP_MAX_CANDS) return "ncand must be 1..48";
    for (int i = 0; i < ncand; i++)
    {
        const x265cu_wp_cand& c = cands[i];
        if (c.weighted && (c.w0 < 0 || c.w0 > 127 || c.denom < 0 || c.denom > 7 || c.offset < -128 || c.offset > 127))
            return "candidate out of range (w0 0..127, denom 0..7, offset -128..127)";
    }
    if (plane == 0)
    {
        if (!intraCost) return "intraCost is NULL";
        for (int k = 0; k < 4; k++)
            if (!fenc->lowres[k] || !ref->lowres[k]) return "NULL lowres plane";
        if (fenc->lowresStride < p->width / 2 || ref->lowresStride < p->width / 2) return "lowres stride smaller than the row";
    }
    else
    {
        const void* f = plane == 1 ? fenc->cb : fenc->cr;
        const void* r = plane == 1 ? ref->cb : ref->cr;
        if (!f || !r) return "NULL chroma plane";
        if (fenc->chromaStride < p->width / 2 || ref->chromaStride < p->width / 2) return "chroma stride smaller than the row";
    }
    return NULL;
}

// one launch of k_weightp_costs and one download of the sums (the scratch sums live in the context's staging arena)
static int weightp_costs_run(x265cu_ctx* c, int depth, const x265cu_wp_params* p, const x265cu_wp_frame* fenc,
                             const x265cu_wp_frame* ref, const int32_t* intraCost, const int32_t* mvs, int plane,
                             const x265cu_wp_cand* cands, int ncand, uint32_t* costs)
{
    WpCostArgs a;
    memset(&a, 0, sizeof(a));
    a.chroma = plane != 0;
    a.w8 = ((p->width / 2) + 7) >> 3; a.h8 = ((p->height / 2) + 7) >> 3;
    a.mvs = mvs; a.intraCost = intraCost;
    if (!plane)
    {
        a.fenc = fenc->lowres[0];
        for (int k = 0; k < 4; k++) a.ref[k] = ref->lowres[k];
        a.fs = fenc->lowresStride; a.rs = ref->lowresStride;
        a.width = a.w8 * 8; a.height = a.h8 * 8;
    }
    else
    {
        a.fenc = plane == 1 ? fenc->cb : fenc->cr;
        a.ref[0] = plane == 1 ? ref->cb : ref->cr;
        a.fs = fenc->chromaStride; a.rs = ref->chromaStride;
        a.width = ((p->width >> 4) << 4) >> 1; a.height = ((p->height >> 4) << 4) >> 1;   // :377-378
    }
    a.ncand = ncand;
    memcpy(a.cand, cands, sizeof(x265cu_wp_cand) * ncand);
    cudaSetDevice(c->device);
    uint32_t* d_sum = (uint32_t*)c->d_stage;
    uint32_t* h_sum = (uint32_t*)c->h_stage;
    CU_CHECK(cudaStreamSynchronize(c->stream));                     // the staging arena is free
    CU_CHECK(cudaMemsetAsync(d_sum, 0, sizeof(uint32_t) * ncand, c->stream));
    const int nblk = (a.width >> 3) * (a.height >> 3);
    int grid = (nblk + 7) / 8;
    if (grid > c->sm_count * 8) grid = c->sm_count * 8;
    if (grid < 1) grid = 1;
    if (depth == 8) k_weightp_costs<uint8_t><<<grid, 256, 0, c->stream>>>(a, d_sum);
    else            k_weightp_costs<uint16_t><<<grid, 256, 0, c->stream>>>(a, d_sum);
    CU_LAUNCH_CHECK(c);
    CU_CHECK(cudaMemcpyAsync(h_sum, d_sum, sizeof(uint32_t) * ncand, cudaMemcpyDeviceToHost, c->stream));
    CU_CHECK(cudaStreamSynchronize(c->stream));
    memcpy(costs, h_sum, sizeof(uint32_t) * ncand);
    return 0;
}

extern "C" int x265cu_weightp_costs(x265cu_ctx* c, int depth, const x265cu_wp_params* p, const x265cu_wp_frame* fenc,
                                    const x265cu_wp_frame* ref, const int32_t* intraCost_dev, const int32_t* mvs_dev, int plane,
                                    const x265cu_wp_cand* cands, int ncand, uint32_t* costs)
{
    const char* bad = c ? weightp_costs_check(depth, p, fenc, ref, intraCost_dev, plane, cands, ncand, costs) : "NULL context";
    if (bad) return wpa::refuse("x265cu_weightp_costs", bad);
    return weightp_costs_run(c, depth, p, fenc, ref, intraCost_dev, mvs_dev, plane, cands, ncand, costs);
}

extern "C" int x265cu_weightp_decide(int depth, const x265cu_wp_params* p, const x265cu_wp_frame* fenc,
                                     const x265cu_wp_frame* const* refs, const int32_t* has_mvs, x265cu_wp_cost_fn cost,
                                     void* user, x265cu_wp_entry* out)
{
    using namespace wpa;
    const char* bad = check_params(depth, p);
    if (!bad && (!fenc || !refs || !has_mvs || !cost || !out)) bad = "NULL argument";
    const int numPredDir = !bad && p->sliceType == 1 ? 1 : 2;
    for (int l = 0; !bad && l < numPredDir; l++)
        if (!refs[l]) bad = "NULL reference record";
    if (bad) return refuse("x265cu_weightp_decide", bad);
    x265cu_wp_entry (*wp)[16][3] = (x265cu_wp_entry (*)[16][3])out;
    const int nplanes = p->csp ? 3 : 1;
    const int lambda = depth == 8 ? 1 : 16;                  // (int)x265_lambda_tab[X265_LOOKAHEAD_QP]
    const float epsilon = 1.f / 128.f;
    int chromaDenom = 7, lumaDenom = 7, denom;
    int numpixels[3];
    const int w16 = ((p->width + 15) >> 4) << 4, h16 = ((p->height + 15) >> 4) << 4;
    numpixels[0] = w16 * h16;
    numpixels[1] = numpixels[2] = numpixels[0] >> 2;
    for (int list = 0; list < numPredDir; list++)
    {
        x265cu_wp_entry* weights = wp[list][0];
        const x265cu_wp_frame* ref = refs[list];
        const int diffPoc = abs(fenc->poc - ref->poc);
        float guessScale[3] = { 0, 0, 0 }, fencMean[3] = { 0, 0, 0 }, refMean[3] = { 0, 0, 0 };
        for (int plane = 0; plane < nplanes; plane++)
        {
            set_w(weights[plane], 0, 1, 0, 0);
            const uint64_t fencVar = fenc->wp_ssd[plane] + !ref->wp_ssd[plane];
            const uint64_t refVar = ref->wp_ssd[plane] + !ref->wp_ssd[plane];
            guessScale[plane] = sqrtf((float)fencVar / refVar);
            fencMean[plane] = (float)fenc->wp_sum[plane] / (numpixels[plane]) / (1 << (depth - 8));
            refMean[plane] = (float)ref->wp_sum[plane] / (numpixels[plane]) / (1 << (depth - 8));
        }
        while (!list && chromaDenom > 0)
        {
            const float thresh = 127.f / (1 << chromaDenom);
            if (guessScale[1] < thresh && guessScale[2] < thresh)
                break;
            chromaDenom--;
        }
        set_w(weights[1], 0, 1 << chromaDenom, chromaDenom, 0);
        set_w(weights[2], 0, 1 << chromaDenom, chromaDenom, 0);
        int useMvs = 0;
        for (int plane = 0; plane < nplanes; plane++)
        {
            denom = plane ? chromaDenom : lumaDenom;
            if (plane && !weights[0].wtPresent)
                break;
            if (fabsf(refMean[plane] - fencMean[plane]) < 0.5f && fabsf(1.f - guessScale[plane]) < epsilon)
            {
                set_w(weights[plane], 0, 1 << denom, denom, 0);
                continue;
            }
            if (plane)
            {
                const int scale = clip3(0, 255, cvt(guessScale[plane] * (1 << denom) + 0.5f));
                if (scale > 127)
                    continue;
                weights[plane].inputWeight = scale;
            }
            else
            {
                // setFromWeightAndOffset(w, 0, denom, bNormalize = !list) (slice.h:304-316)
                x265cu_wp_entry& w = weights[plane];
                w.inputOffset = 0; w.log2WeightDenom = denom; w.inputWeight = cvt(guessScale[plane] * (1 << denom) + 0.5f);
                while (!list && w.log2WeightDenom > 0 && w.inputWeight > 127) { w.log2WeightDenom--; w.inputWeight >>= 1; }
                if (w.inputWeight > 127) w.inputWeight = 127;
            }
            int mindenom = weights[plane].log2WeightDenom;
            int minscale = weights[plane].inputWeight;
            int minoff = 0;
            if (!plane && diffPoc <= p->bframes + 1)
                useMvs = has_mvs[list] != 0;
            // every candidate of the search in the reference's order, with the (scale, offset) range of each scale
            x265cu_wp_cand cand[1 + 9 * 5];
            int nc = 0, nsc = 0, scaleOf[9], offOf[9], firstOf[9];
            cand[nc++] = x265cu_wp_cand{ 0, 0, 0, 0 };
            const int startScale = clip3(0, 127, minscale - 4), endScale = clip3(0, 127, minscale + 4);
            for (int scale = startScale; scale <= endScale; scale++)
            {
                const int deltaWeight = scale - (1 << mindenom);
                if (deltaWeight > 127 || deltaWeight <= -128)
                    continue;
                int curScale = scale;
                int curOffset = cvt(fencMean[plane] - refMean[plane] * curScale / (1 << mindenom) + 0.5f);
                if (curOffset < -128 || curOffset > 127)
                {
                    curOffset = clip3(-128, 127, curOffset);
                    curScale = cvt((1 << mindenom) * (fencMean[plane] - curOffset) / refMean[plane] + 0.5f);
                    curScale = clip3(0, 127, curScale);
                }
                scaleOf[nsc] = curScale; offOf[nsc] = curOffset; firstOf[nsc] = nc; nsc++;
                const int so = clip3(-128, 127, curOffset - 2), eo = clip3(-128, 127, curOffset + 2);
                for (int off = so; off <= eo; off++) cand[nc++] = x265cu_wp_cand{ 1, curScale, mindenom, off };
            }
            uint32_t costs[1 + 9 * 5];
            if (cost(user, list, plane, useMvs, cand, nc, costs)) return -1;
            const uint32_t origscore = costs[0];
            if (!origscore)
            {
                set_w(weights[plane], 0, 1 << denom, denom, 0);
                continue;
            }
            uint32_t minscore = origscore;
            bool bFound = false;
            for (int k = 0; k < nsc; k++)
            {
                const int so = clip3(-128, 127, offOf[k] - 2), eo = clip3(-128, 127, offOf[k] + 2);
                for (int off = so, i = firstOf[k]; off <= eo; off++, i++)
                {
                    const uint32_t s = costs[i] + (uint32_t)slice_header_cost(scaleOf[k], mindenom, off, lambda, !!plane);
                    if (s < minscore) { minscore = s; minscale = scaleOf[k]; minoff = off; bFound = true; }
                    if (minoff == so && off != so)
                        break;
                }
            }
            if (!(plane || list) && mindenom > 0 && !(minscale & 1))
            {
                const int idx = minscale ? __builtin_ctz((unsigned)minscale) : 32;     // CTZ as tzcnt computes it
                const int shift = idx < mindenom ? idx : mindenom;
                mindenom -= shift;
                minscale >>= shift;
            }
            if (!bFound || (minscale == (1 << mindenom) && minoff == 0) || (float)minscore / origscore > 0.998f)
                set_w(weights[plane], 0, 1 << denom, denom, 0);
            else
                set_w(weights[plane], 1, minscale, mindenom, minoff);
        }
        if (weights[0].wtPresent && weights[1].wtPresent != weights[2].wtPresent)
        {
            if (weights[1].wtPresent) weights[2] = weights[1];
            else weights[1] = weights[2];
        }
        lumaDenom = weights[0].log2WeightDenom;
        chromaDenom = weights[1].log2WeightDenom;
        for (int r = 1; r < p->numRefIdx[list]; r++)
        {
            set_w(wp[list][r][0], 0, 1 << lumaDenom, lumaDenom, 0);
            set_w(wp[list][r][1], 0, 1 << chromaDenom, chromaDenom, 0);
            set_w(wp[list][r][2], 0, 1 << chromaDenom, chromaDenom, 0);
        }
    }
    return 0;
}

namespace wpa {
struct DeviceCosts
{
    x265cu_ctx* c; int depth; const x265cu_wp_params* p; const x265cu_wp_frame* fenc; const x265cu_wp_frame* const* refs;
    const int32_t* intraCost; const int32_t* const* mvs;
};
static int device_costs(void* user, int list, int plane, int use_mvs, const x265cu_wp_cand* cands, int n, uint32_t* costs)
{
    const DeviceCosts& d = *(const DeviceCosts*)user;
    const char* bad = weightp_costs_check(d.depth, d.p, d.fenc, d.refs[list], d.intraCost, plane, cands, n, costs);
    if (bad) return refuse("x265cu_weightp_analyse", bad);
    return weightp_costs_run(d.c, d.depth, d.p, d.fenc, d.refs[list], d.intraCost, use_mvs ? d.mvs[list] : NULL, plane,
                             cands, n, costs);
}
} // namespace wpa

extern "C" int x265cu_weightp_analyse(x265cu_ctx* c, int depth, const x265cu_wp_params* p, const x265cu_wp_frame* fenc,
                                      const int32_t* intraCost_dev, const x265cu_wp_frame* const* refs,
                                      const int32_t* const* mvs_dev, x265cu_wp_entry* out)
{
    const char* bad = !c ? "NULL context" : wpa::check_params(depth, p);
    if (!bad && (!fenc || !refs || !mvs_dev || !intraCost_dev || !out)) bad = "NULL argument";
    const int numPredDir = !bad && p->sliceType == 1 ? 1 : 2;
    // every plane the search could cost is checked before the first launch
    static const x265cu_wp_cand unweighted = { 0, 0, 0, 0 };
    uint32_t dummy;
    for (int l = 0; !bad && l < numPredDir; l++)
    {
        if (!refs[l]) { bad = "NULL reference record"; break; }
        for (int pl = 0; !bad && pl < (p->csp ? 3 : 1); pl++)
            bad = weightp_costs_check(depth, p, fenc, refs[l], intraCost_dev, pl, &unweighted, 1, &dummy);
    }
    if (bad) return wpa::refuse("x265cu_weightp_analyse", bad);
    int32_t has[2] = { 0, 0 };
    for (int l = 0; l < numPredDir; l++) has[l] = mvs_dev[l] != NULL;
    wpa::DeviceCosts d = { c, depth, p, fenc, refs, intraCost_dev, mvs_dev };
    return x265cu_weightp_decide(depth, p, fenc, refs, has, wpa::device_costs, &d, out);
}
