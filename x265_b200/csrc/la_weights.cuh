// x265_b200/csrc/la_weights.cuh -- the lookahead's weighted-prediction analysis on device-resident lowres planes:
// LookaheadTLD::weightsAnalyse + weightCostLuma (/root/reference/source/encoder/slicetype.cpp:807-840, 860-961).
// Host side = the reference's decision logic (float heuristics on the picture statistics, two trial weightings, the
// 0.998 acceptance test); device side = launches of kernels that already exist: `weight_pp` over the whole padded plane
// (k_blockop, pixel.cpp:518-543) and the 8x8 SATD map of the weighted reference against the source (k_pixelcmp_grid);
// the per-CU min(satd, intraCost) fold runs on the host over the downloaded map (4 B x CUs of traffic saved by doing it
// on the device would not matter: the call is dominated by the plane passes).
#pragma once
#include "common.cuh"
#include "blockops.cuh"
#include "pixelcmp_grid.cuh"
#include <limits.h>
#include <math.h>

namespace law {

struct Wp { int wtPresent, inputWeight, log2WeightDenom, inputOffset; };

// (int) of a float as x86's cvttss2si computes it: NaN and values outside the int range give INT_MIN.  C leaves those
// conversions undefined, and the analysis makes one on a fade from black: refMean == 0 with the offset clamped divides
// by zero (slicetype.cpp:921), and curScale then clamps +inf's INT_MIN to 0.
static inline int la_cvttss2si(float v)
{
    return (v >= -2147483648.f && v < 2147483648.f) ? (int)v : INT_MIN;
}

struct Run
{
    x265cu_ctx* c; int depth; size_t es;
    const uint8_t* fencBuf; const uint8_t* refBuf[4]; uint8_t* wbuf;
    int64_t planesize, padoffset; int stride, width, lines, paddedLines;
    const int32_t* intraCost;                // host
    int njobs; x265cu_blk_job* d_jobs; uint64_t* d_map; uint64_t* h_map; int nbx, nby;
};

// weight_pp of a whole padded plane: one job per 16-row band (the job list is shared by every plane: offsets are relative)
static int weight_plane(Run& r, const uint8_t* src, uint8_t* dst, const Wp& wp)
{
    const int offset = wp.inputOffset << (r.depth - 8);
    const int scale = wp.inputWeight, denom = wp.log2WeightDenom;
    const int round = denom ? 1 << (denom - 1) : 0;
    const int correction = 14 - r.depth;                        // IF_INTERNAL_PREC - X265_DEPTH
    // parameters travel in the job records: rewrite p0..p3 of the staged list, then upload it again
    x265cu_blk_job* hj = (x265cu_blk_job*)r.c->h_stage;
    CU_CHECK(cudaStreamSynchronize(r.c->stream));                  // the previous upload of this arena must be done
    for (int j = 0; j < r.njobs; j++) { hj[j].p0 = scale; hj[j].p1 = round << correction; hj[j].p2 = denom + correction; hj[j].p3 = offset; }
    CU_CHECK(cudaMemcpyAsync(r.d_jobs, hj, sizeof(x265cu_blk_job) * r.njobs, cudaMemcpyHostToDevice, r.c->stream));
    return launch_blockop(r.c, r.depth, X265CU_WEIGHT_PP, dst, src, NULL, r.d_jobs, r.njobs);
}

// weightCostLuma (slicetype.cpp:807-840)
static int cost_luma(Run& r, const Wp& wp, uint32_t* cost)
{
    const uint8_t* src = r.refBuf[0] + r.padoffset * r.es;
    if (wp.wtPresent)
    {
        if (weight_plane(r, r.refBuf[0], r.wbuf, wp)) return -1;
        src = r.wbuf + r.padoffset * r.es;
    }
    if (launch_pixelcmp_grid(r.c, r.depth, X265CU_SATD, src, r.stride, r.fencBuf + r.padoffset * r.es, r.stride, 8, 8, r.nbx, r.nby, r.d_map)) return -1;
    CU_CHECK(cudaMemcpyAsync(r.h_map, r.d_map, sizeof(uint64_t) * r.nbx * r.nby, cudaMemcpyDeviceToHost, r.c->stream));
    CU_CHECK(cudaStreamSynchronize(r.c->stream));
    uint32_t s = 0;
    for (int mb = 0; mb < r.nbx * r.nby; mb++)
    {
        const int satd = (int)r.h_map[mb];
        s += satd < r.intraCost[mb] ? (uint32_t)satd : (uint32_t)r.intraCost[mb];
    }
    *cost = s;
    return 0;
}

} // namespace law

// Planes are whole padded lowres buffers (Lowres::buffer[i], common/lowres.cpp:132-139: `planesize` pixels each, picture
// origin at `padoffset`), device resident; wbuf_dev = 4 * planesize pixels (LookaheadTLD::wbuffer).  intraCost_host[CUs]
// and stats = {fenc wp_sum, fenc wp_ssd, ref wp_sum, ref wp_ssd} (Lowres::wp_sum[0] / wp_ssd[0], accumulated by the caller
// as calcAdaptiveQuantFrame does, slicetype.cpp:49-57, 462-480, 665-676) are host inputs.  wp_out = {isWeighted, scale,
// log2 denominator, offset}; when isWeighted, wbuf_dev holds the 4 re-weighted planes the L0 search then uses
// (slicetype.cpp:3222).  Returns 0 / -1.
extern "C" int x265cu_lookahead_weights_analyse(x265cu_ctx* c, int depth, const void* fencBuf_dev, const void* const* refBuf_dev4 /* host array */,
                                                void* wbuf_dev, int64_t planesize, int stride, int width, int lines, int64_t padoffset,
                                                const int32_t* intraCost_host, const uint64_t* stats, int* wp_out)
{
    using namespace law;
    wp_out[0] = wp_out[1] = wp_out[2] = wp_out[3] = 0;
    if (!c || (depth != 8 && depth != 10) || stride <= 0 || width <= 0 || lines <= 0 || planesize < (int64_t)stride)
    {
        x265cu_set_error("x265cu_lookahead_weights_analyse: bad arguments", cudaErrorInvalidValue, __FILE__, __LINE__);
        return -1;
    }
    cudaSetDevice(c->device);
    static const float epsilon = 1.f / 128.f;
    Run r;
    r.c = c; r.depth = depth; r.es = depth == 8 ? 1 : 2;
    r.fencBuf = (const uint8_t*)fencBuf_dev; r.wbuf = (uint8_t*)wbuf_dev;
    for (int i = 0; i < 4; i++) r.refBuf[i] = (const uint8_t*)refBuf_dev4[i];
    r.planesize = planesize; r.padoffset = padoffset; r.stride = stride; r.width = width; r.lines = lines;
    r.paddedLines = (int)(planesize / stride);
    r.intraCost = intraCost_host;
    r.nbx = (width + 7) >> 3; r.nby = (lines + 7) >> 3;

    /* picture statistics -> guess, early termination (slicetype.cpp:885-897) */
    const uint64_t fencSum = stats[0], fencSsd = stats[1], refSum = stats[2], refSsd = stats[3];
    float guessScale, fencMean, refMean;
    if (fencSsd && refSsd) guessScale = sqrtf((float)fencSsd / refSsd);
    else                   guessScale = 1.0f;
    fencMean = (float)fencSum / (lines * width) / (1 << (depth - 8));
    refMean  = (float)refSum / (lines * width) / (1 << (depth - 8));
    if (fabsf(refMean - fencMean) < 0.5f && fabsf(1.f - guessScale) < epsilon)
        return 0;

    /* staging arena of the context: [0, 64 KB) the band job list, then the SATD map */
    const int band = 16;
    r.njobs = (r.paddedLines + band - 1) / band;
    const size_t mapOff = 64 << 10, mapBytes = sizeof(uint64_t) * (size_t)r.nbx * r.nby;
    if (sizeof(x265cu_blk_job) * (size_t)r.njobs > mapOff || mapOff + mapBytes > c->stage_bytes)
    {
        x265cu_set_error("x265cu_lookahead_weights_analyse: picture too large for the staging arena", cudaErrorInvalidValue, __FILE__, __LINE__);
        return -1;
    }
    CU_CHECK(cudaStreamSynchronize(c->stream));
    x265cu_blk_job* hj = (x265cu_blk_job*)c->h_stage;
    for (int j = 0; j < r.njobs; j++)
    {
        memset(&hj[j], 0, sizeof(hj[j]));
        hj[j].d_off = hj[j].a_off = (int64_t)j * band * stride;
        hj[j].d_stride = hj[j].a_stride = stride; hj[j].b_stride = stride;
        hj[j].w = (int16_t)stride;
        hj[j].h = (int16_t)((j + 1) * band <= r.paddedLines ? band : r.paddedLines - j * band);
    }
    r.d_jobs = (x265cu_blk_job*)c->d_stage;
    r.d_map = (uint64_t*)(c->d_stage + mapOff); r.h_map = (uint64_t*)(c->h_stage + mapOff);

    int minoff = 0, minscale, mindenom;
    unsigned int minscore = 0, origscore = 1;
    int found = 0;
    Wp wp = { 0, 0, 0, 0 };
    /* wp.setFromWeightAndOffset((int)(guessScale * 128 + 0.5f), 0, 7, true) (slice.h:304-316); wtPresent stays 0 */
    wp.inputOffset = 0; wp.log2WeightDenom = 7; wp.inputWeight = la_cvttss2si(guessScale * 128 + 0.5f);
    while (wp.log2WeightDenom > 0 && wp.inputWeight > 127) { wp.log2WeightDenom--; wp.inputWeight >>= 1; }
    if (wp.inputWeight > 127) wp.inputWeight = 127;
    mindenom = wp.log2WeightDenom;
    minscale = wp.inputWeight;

    uint32_t sc = 0;
    if (cost_luma(r, wp, &sc)) return -1;
    origscore = minscore = sc;
    if (!minscore)
        return 0;

    int curScale = minscale;
    int curOffset = la_cvttss2si(fencMean - refMean * curScale / (1 << mindenom) + 0.5f);
    if (curOffset < -128 || curOffset > 127)
    {
        curOffset = curOffset < -128 ? -128 : (curOffset > 127 ? 127 : curOffset);
        curScale = la_cvttss2si((1 << mindenom) * (fencMean - curOffset) / refMean + 0.5f);
        curScale = curScale < 0 ? 0 : (curScale > 127 ? 127 : curScale);
    }
    wp.inputWeight = curScale; wp.log2WeightDenom = mindenom; wp.inputOffset = curOffset; wp.wtPresent = 1;
    if (cost_luma(r, wp, &sc)) return -1;
    if (sc < minscore) { minscore = sc; minscale = curScale; minoff = curOffset; found = 1; }

    /* use a smaller denominator if possible (slicetype.cpp:925-932) */
    if (mindenom > 0 && minscale && !(minscale & 1))
    {
        int idx = 0;
        while (!((minscale >> idx) & 1)) idx++;
        const int shift = idx < mindenom ? idx : mindenom;
        mindenom -= shift;
        minscale >>= shift;
    }

    if (!found || (minscale == 1 << mindenom && minoff == 0) || (float)minscore / origscore > 0.998f)
        return 0;

    wp.inputWeight = minscale; wp.log2WeightDenom = mindenom; wp.inputOffset = minoff; wp.wtPresent = 1;
    for (int i = 0; i < 4; i++)
        if (weight_plane(r, r.refBuf[i], r.wbuf + (size_t)i * planesize * r.es, wp)) return -1;
    CU_CHECK(cudaStreamSynchronize(c->stream));
    wp_out[0] = 1; wp_out[1] = minscale; wp_out[2] = mindenom; wp_out[3] = minoff;
    return 0;
}
