/* oracle/oracle_lookahead.c -- TEST INFRASTRUCTURE ONLY (see oracle.h).
 * Restates the lookahead's per-frame cost estimation (BASELINE configs[1]):
 *   LookaheadTLD::lowresIntraEstimate        encoder/slicetype.cpp:696-805
 *   CostEstimateGroup::estimateFrameCost     encoder/slicetype.cpp:3115-3214 (serial path)
 *   CostEstimateGroup::estimateCUCost        encoder/slicetype.cpp:3216-3388 (no HME / weightp / AQ)
 *   ReferencePlanes::lowresMC                common/lowres.h:67-92
 *   LookaheadTLD::weightsAnalyse / weightCostLuma  encoder/slicetype.cpp:807-840, 860-961 (end of this file)
 * Pinned against the real classes through oracle/_ref (x265ref_la_*), tests/test_lookahead_oracle_vs_ref.py.
 */
#include "oracle.h"
#include <string.h>
#include <math.h>
#include <limits.h>

#define COST_MAX (1 << 28)               /* motion.h:65 */
#define LOWRES_COST_MASK ((1 << 14) - 1) /* slicetype.h:41-42 */
#define LOWRES_COST_SHIFT 14

int orc_intra_use_filtered(int mode, int n);

/* slicetype.cpp:696-805.  plane0: origin pixel of the lowres full-pel plane (margins extended). */
void orc_lowres_intra(const pixel* plane0, intptr_t stride, int w8, int h8, int lambda, const int32_t* invQscale,
                      int32_t* intraCost, uint8_t* intraMode, uint16_t* lowresCosts, int32_t* rowSatds, int64_t* costEst2)
{
    const int intraPenalty = 5 * lambda, lowresPenalty = 4;
    int64_t costEst = 0, costEstAq = 0;
    for (int cuY = 0; cuY < h8; cuY++)
    {
        rowSatds[cuY] = 0;
        for (int cuX = 0; cuX < w8; cuX++)
        {
            const int cuXY = cuX + cuY * w8;
            const pixel* cur = plane0 + 8 * cuX + (intptr_t)8 * cuY * stride;
            pixel fenc[64], pred[64], nb[2][33];
            orc_copy_pp(fenc, 8, cur, stride, 8, 8);
            const pixel* tl = cur - stride - 1;
            memcpy(nb[0], tl, 17 * sizeof(pixel));
            for (int i = 1; i <= 16; i++) nb[0][16 + i] = tl[(intptr_t)i * stride];
            orc_intra_filter(nb[0], nb[1], 8);
            int cost, icost = COST_MAX, ilow = 0;
            orc_intra_pred(pred, 8, nb[0], 1, 1, 8);            /* DC, bFilter = cuSize <= 16 */
            cost = orc_satd(fenc, 8, pred, 8, 8, 8);
            if (cost < icost) { icost = cost; ilow = 1; }
            orc_intra_pred(pred, 8, nb[1], 0, 0, 8);            /* planar on the filtered neighbours (cuSize >= 8) */
            cost = orc_satd(fenc, 8, pred, 8, 8, 8);
            if (cost < icost) { icost = cost; ilow = 0; }
            int acost = COST_MAX, alow = 4;
            for (int mode = 5; mode < 35; mode += 5)
            {
                orc_intra_pred(pred, 8, nb[orc_intra_use_filtered(mode, 8)], mode, 1, 8);
                cost = orc_satd(fenc, 8, pred, 8, 8, 8);
                if (cost < acost) { acost = cost; alow = mode; }
            }
            for (int dist = 2; dist >= 1; dist--)
            {
                int minus = alow - dist, plus = alow + dist;
                orc_intra_pred(pred, 8, nb[orc_intra_use_filtered(minus, 8)], minus, 1, 8);
                cost = orc_satd(fenc, 8, pred, 8, 8, 8);
                if (cost < acost) { acost = cost; alow = minus; }
                orc_intra_pred(pred, 8, nb[orc_intra_use_filtered(plus, 8)], plus, 1, 8);
                cost = orc_satd(fenc, 8, pred, 8, 8, 8);
                if (cost < acost) { acost = cost; alow = plus; }
            }
            if (acost < icost) { icost = acost; ilow = alow; }
            icost += intraPenalty + lowresPenalty;
            lowresCosts[cuXY] = (uint16_t)(icost < LOWRES_COST_MASK ? icost : LOWRES_COST_MASK);
            intraCost[cuXY] = icost;
            intraMode[cuXY] = (uint8_t)ilow;
            const int score = (cuX > 0 && cuX < w8 - 1 && cuY > 0 && cuY < h8 - 1) || w8 <= 2 || h8 <= 2;
            int icostAq = (score && invQscale) ? ((icost * invQscale[cuXY] + 128) >> 8) : icost;
            if (score) { costEst += icost; costEstAq += icostAq; }
            rowSatds[cuY] += icostAq;
        }
    }
    costEst2[0] = costEst; costEst2[1] = costEstAq;
}

/* lowres.h:67-92: pointer into a hpel plane, or the rounded average of two of them in buf */
static const pixel* lowres_mc(const pixel* const planes[4], intptr_t stride, intptr_t off, int qx, int qy, pixel* buf, intptr_t* outStride)
{
    if ((qx | qy) & 1)
    {
        int ha = (qy & 2) | ((qx & 2) >> 1);
        const pixel* a = planes[ha] + off + (qx >> 2) + (intptr_t)(qy >> 2) * stride;
        int rx = qx + (qx & 1), ry = qy + (qy & 1);
        int hb = (ry & 2) | ((rx & 2) >> 1);
        const pixel* b = planes[hb] + off + (rx >> 2) + (intptr_t)(ry >> 2) * stride;
        orc_pixelavg_pp(buf, *outStride, a, stride, b, stride, 8, 8);
        return buf;
    }
    *outStride = stride;
    int hp = (qy & 2) | ((qx & 2) >> 1);
    return planes[hp] + off + (qx >> 2) + (intptr_t)(qy >> 2) * stride;
}

typedef struct {
    const pixel* fenc[4];           /* origin pixels of the 4 hpel planes of frame b (only [0] is read) */
    const pixel* ref0[4];           /* frame p0 */
    const pixel* ref1[4];           /* frame p1 (bidir only) */
    intptr_t stride;
    int w8, h8;
    int bidir;                      /* b < p1 */
    int doSearch[2];
    int32_t* mvs[2];                /* [cu][2] qpel, in/out */
    int32_t* mvcosts[2];            /* [cu] in/out */
    const int32_t* intraCost;       /* frame b */
    const int32_t* invQscale;       /* NULL when AQ is off */
    const uint16_t* mvcost_tab;     /* centred, lambda of X265_LOOKAHEAD_QP */
    uint16_t* lowresCosts; int32_t* rowSatds;
    int64_t out[3];                 /* costEst, costEstAq, intraMbs */
    /* cooperative slices (slicetype.cpp:3075-3112, 3143-3173): numSlices > 1 splits the CU rows into numSlices ranges of
     * rowsPerSlice rows (the last one takes the remainder); every range starts with lastRow = true at its bottom row */
    int numSlices, rowsPerSlice;
} orc_la_job;

void orc_lookahead_frame_cost(orc_la_job* j)
{
    const int w8 = j->w8, h8 = j->h8;
    const intptr_t stride = j->stride;
    int64_t costEst = 0, costEstAq = 0, intraMbs = 0;
    const int nsl = j->numSlices > 1 ? j->numSlices : 1;
    for (int sl = 0; sl < nsl; sl++)
    {
    const int firstY = nsl > 1 ? j->rowsPerSlice * sl : 0;
    const int lastY = (nsl == 1 || sl == nsl - 1) ? h8 - 1 : j->rowsPerSlice * (sl + 1) - 1;
    for (int cuY = lastY; cuY >= firstY; cuY--)
    {
        const int lastRow = (cuY == lastY);
        j->rowSatds[cuY] = 0;
        for (int cuX = w8 - 1; cuX >= 0; cuX--)
        {
            const int cuXY = cuX + cuY * w8;
            const intptr_t off = 8 * cuX + (intptr_t)8 * cuY * stride;
            pixel fenc8[64 * 8];                                /* FENC_STRIDE cache */
            orc_copy_pp(fenc8, 64, j->fenc[0] + off, stride, 8, 8);
            int bcost = COST_MAX, listused = 0;
            const int mvmin[2] = { -cuX * 8 - 8, -cuY * 8 - 8 };
            const int mvmax[2] = { (w8 - cuX - 1) * 8 + 8, (h8 - cuY - 1) * 8 + 8 };
            for (int i = 0; i < 1 + j->bidir; i++)
            {
                int32_t* fencCost = &j->mvcosts[i][cuXY];
                int skipCost = 0x7fffffff;
                if (!j->doSearch[i])
                {
                    if (*fencCost < bcost) { bcost = *fencCost; listused = i + 1; }
                    continue;
                }
                int numc = 0, mvc[5][2], mvp[2] = { 0, 0 };
                int32_t* fmv = j->mvs[i] + 2 * cuXY;
                const pixel* const* fref = i ? j->ref1 : j->ref0;
#define MVC(k) do { mvc[numc][0] = fmv[2 * (k)]; mvc[numc][1] = fmv[2 * (k) + 1]; numc++; } while (0)
                if (cuX < w8 - 1) MVC(1);
                if (!lastRow)
                {
                    MVC(w8);
                    if (cuX > 0) MVC(w8 - 1);
                    if (cuX < w8 - 1) MVC(w8 + 1);
                }
#undef MVC
                if (numc)
                {
                    pixel buf[64];
                    int mvpcost = COST_MAX;
                    for (int idx = 0; idx < numc; idx++)
                    {
                        intptr_t st = 8;
                        const pixel* src = lowres_mc(fref, stride, off, mvc[idx][0], mvc[idx][1], buf, &st);
                        int cost = orc_satd(fenc8, 64, src, st, 8, 8);
                        if (cost < mvpcost) { mvpcost = cost; mvp[0] = mvc[idx][0]; mvp[1] = mvc[idx][1]; }
                        if (!(mvp[0] | mvp[1]) && j->bidir) skipCost = cost;
                    }
                }
                orc_me_job job;
                job.chroma = 0;
                job.fenc = j->fenc[0]; job.fencStride = stride; job.offset = off;
                for (int k = 0; k < 4; k++) job.ref[k] = fref[k];
                job.refStride = stride; job.lowres = 1; job.pw = 8; job.ph = 8; job.method = 1; job.subme = 1;
                job.mvmin[0] = mvmin[0]; job.mvmin[1] = mvmin[1]; job.mvmax[0] = mvmax[0]; job.mvmax[1] = mvmax[1];
                job.qmvp[0] = mvp[0]; job.qmvp[1] = mvp[1]; job.numCand = 0; job.mvc = NULL; job.merange = 16; job.mvcost = j->mvcost_tab;
                int out[2];
                *fencCost = orc_motion_estimate(&job, out);
                fmv[0] = out[0]; fmv[1] = out[1];
                if (skipCost < 64 && skipCost < *fencCost && j->bidir) { *fencCost = skipCost; fmv[0] = fmv[1] = 0; }
                if (*fencCost < bcost) { bcost = *fencCost; listused = i + 1; }
            }
            if (j->bidir)
            {
                pixel b0[64], b1[64], avg[64];
                intptr_t s0 = 8, s1 = 8;
                const pixel* src0 = lowres_mc(j->ref0, stride, off, j->mvs[0][2 * cuXY], j->mvs[0][2 * cuXY + 1], b0, &s0);
                const pixel* src1 = lowres_mc(j->ref1, stride, off, j->mvs[1][2 * cuXY], j->mvs[1][2 * cuXY + 1], b1, &s1);
                orc_pixelavg_pp(avg, 8, src0, s0, src1, s1, 8, 8);
                int bicost = orc_satd(fenc8, 64, avg, 8, 8, 8);
                if (bicost < bcost) { bcost = bicost; listused = 3; }
                orc_pixelavg_pp(avg, 8, j->ref0[0] + off, stride, j->ref1[0] + off, stride, 8, 8);
                bicost = orc_satd(fenc8, 64, avg, 8, 8, 8);
                if (bicost < bcost) { bcost = bicost; listused = 3; }
                bcost += 4;
            }
            else
            {
                bcost += 4;
                if (j->intraCost[cuXY] < bcost) { bcost = j->intraCost[cuXY]; listused = 0; }
            }
            const int score = (cuX > 0 && cuX < w8 - 1 && cuY > 0 && cuY < h8 - 1) || w8 <= 2 || h8 <= 2;
            int bcostAq = (score && j->invQscale) ? ((bcost * j->invQscale[cuXY] + 128) >> 8) : bcost;
            if (score)
            {
                costEst += bcost; costEstAq += bcostAq;
                if (!listused && !j->bidir) intraMbs++;
            }
            j->rowSatds[cuY] += bcostAq;
            j->lowresCosts[cuXY] = (uint16_t)((bcost < LOWRES_COST_MASK ? bcost : LOWRES_COST_MASK) | (listused << LOWRES_COST_SHIFT));
        }
    }
    }
    j->out[0] = costEst; j->out[1] = costEstAq; j->out[2] = intraMbs;
}

/* ------------------------------------------------------------------------------------------------------------
 * Lookahead weighted-prediction analysis: LookaheadTLD::weightCostLuma + weightsAnalyse
 * (encoder/slicetype.cpp:807-840, 860-961; WeightParam::setFromWeightAndOffset common/slice.h:304-316).
 * Planes are the whole padded lowres buffers (Lowres::buffer[i], common/lowres.cpp:132-139): `planesize` pixels each,
 * picture origin at `padoffset`.  The picture statistics wp_sum / wp_ssd of luma (accumulated by the reference in
 * calcAdaptiveQuantFrame, slicetype.cpp:49-57, 462-480, 665-676) are inputs.
 * Returns Lowres::weightedRef[].isWeighted; when 1, wbuf holds the 4 re-weighted planes and wp = {scale, denom, offset}.
 * wbuf (4 * planesize pixels) is also the scratch of the trial weightings, exactly like LookaheadTLD::wbuffer.
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct { int wtPresent, inputWeight, log2WeightDenom, inputOffset; } orc_wp;

/* (int) of a float with x86 cvttss2si semantics (NaN and out-of-range values -> INT_MIN), which the reference's casts get
 * from the compiler: on a fade from black refMean == 0 and the clamped offset's rescale divides by zero (slicetype.cpp:921). */
static int la_cvttss2si(float v)
{
    return (v >= -2147483648.f && v < 2147483648.f) ? (int)v : INT_MIN;
}

static uint32_t la_weight_cost_luma(const pixel* fencBuf, const pixel* const* refBuf, pixel* wbuf, intptr_t stride, int width, int lines,
                                    int paddedLines, intptr_t padoffset, const int32_t* intraCost, const orc_wp* wp)
{
    const pixel* src = refBuf[0] + padoffset;
    if (wp->wtPresent)
    {
        const int offset = wp->inputOffset << (ORC_DEPTH - 8);
        const int scale = wp->inputWeight, denom = wp->log2WeightDenom;
        const int round = denom ? 1 << (denom - 1) : 0;
        const int correction = 14 - ORC_DEPTH;
        orc_weight_pp(refBuf[0], wbuf, stride, (int)stride, paddedLines, scale, round << correction, denom + correction, offset);
        src = wbuf + padoffset;
    }
    const pixel* fenc = fencBuf + padoffset;
    uint32_t cost = 0;
    int mb = 0;
    for (int y = 0; y < lines; y += 8)
        for (int x = 0; x < width; x += 8, mb++)
        {
            const intptr_t pixoff = (intptr_t)y * stride + x;
            const int satd = orc_satd(src + pixoff, stride, fenc + pixoff, stride, 8, 8);
            cost += satd < intraCost[mb] ? (uint32_t)satd : (uint32_t)intraCost[mb];
        }
    return cost;
}

int orc_la_weights_analyse(const pixel* fencBuf, const pixel* const* refBuf, pixel* wbuf, intptr_t planesize, intptr_t stride,
                           int width, int lines, intptr_t padoffset, const int32_t* intraCost,
                           uint64_t fencSum, uint64_t fencSsd, uint64_t refSum, uint64_t refSsd, int* wpOut)
{
    static const float epsilon = 1.f / 128.f;
    const int paddedLines = (int)(planesize / stride);
    orc_wp wp = { 0, 0, 0, 0 };
    float guessScale, fencMean, refMean;
    if (fencSsd && refSsd) guessScale = sqrtf((float)fencSsd / refSsd);
    else                   guessScale = 1.0f;
    fencMean = (float)fencSum / (lines * width) / (1 << (ORC_DEPTH - 8));
    refMean  = (float)refSum / (lines * width) / (1 << (ORC_DEPTH - 8));
    if (fabsf(refMean - fencMean) < 0.5f && fabsf(1.f - guessScale) < epsilon)
        return 0;

    int minoff = 0, minscale, mindenom;
    unsigned int minscore = 0, origscore = 1;
    int found = 0;
    /* wp.setFromWeightAndOffset((int)(guessScale * 128 + 0.5f), 0, 7, true): note wtPresent stays 0 for the first cost */
    wp.inputOffset = 0; wp.log2WeightDenom = 7; wp.inputWeight = la_cvttss2si(guessScale * 128 + 0.5f);
    while (wp.log2WeightDenom > 0 && wp.inputWeight > 127) { wp.log2WeightDenom--; wp.inputWeight >>= 1; }
    if (wp.inputWeight > 127) wp.inputWeight = 127;
    mindenom = wp.log2WeightDenom;
    minscale = wp.inputWeight;

    origscore = minscore = la_weight_cost_luma(fencBuf, refBuf, wbuf, stride, width, lines, paddedLines, padoffset, intraCost, &wp);
    if (!minscore)
        return 0;

    unsigned int s = 0;
    int curScale = minscale;
    int curOffset = la_cvttss2si(fencMean - refMean * curScale / (1 << mindenom) + 0.5f);
    if (curOffset < -128 || curOffset > 127)
    {
        curOffset = curOffset < -128 ? -128 : (curOffset > 127 ? 127 : curOffset);
        curScale = la_cvttss2si((1 << mindenom) * (fencMean - curOffset) / refMean + 0.5f);
        curScale = curScale < 0 ? 0 : (curScale > 127 ? 127 : curScale);
    }
    wp.inputWeight = curScale; wp.log2WeightDenom = mindenom; wp.inputOffset = curOffset; wp.wtPresent = 1;
    s = la_weight_cost_luma(fencBuf, refBuf, wbuf, stride, width, lines, paddedLines, padoffset, intraCost, &wp);
    if (s < minscore) { minscore = s; minscale = curScale; minoff = curOffset; found = 1; }

    /* use a smaller denominator if possible */
    if (mindenom > 0 && !(minscale & 1))
    {
        int idx = 0;
        while (!((minscale >> idx) & 1) && idx < 31) idx++;         /* CTZ; minscale = 0 cannot get here with found = 1 mattering */
        if (minscale == 0) idx = 0;
        int shift = idx < mindenom ? idx : mindenom;
        mindenom -= shift;
        minscale >>= shift;
    }

    if (!found || (minscale == 1 << mindenom && minoff == 0) || (float)minscore / origscore > 0.998f)
        return 0;

    wp.inputWeight = minscale; wp.log2WeightDenom = mindenom; wp.inputOffset = minoff; wp.wtPresent = 1;
    {
        const int offset = wp.inputOffset << (ORC_DEPTH - 8);
        const int scale = wp.inputWeight, denom = wp.log2WeightDenom;
        const int round = denom ? 1 << (denom - 1) : 0;
        const int correction = 14 - ORC_DEPTH;
        for (int i = 0; i < 4; i++)
            orc_weight_pp(refBuf[i], wbuf + i * planesize, stride, (int)stride, paddedLines, scale, round << correction, denom + correction, offset);
    }
    wpOut[0] = minscale; wpOut[1] = mindenom; wpOut[2] = minoff;
    return 1;
}

/* cuTree: estimateCUPropagateCost (common/pixel.cpp:914-940): plain double arithmetic, `(int)` conversion of the host. */
void orc_propagate_cost(int* dst, const uint16_t* propagateIn, const int32_t* intraCosts, const uint16_t* interCosts,
                        const int32_t* invQscales, const double* fpsFactor, int len)
{
    const double fps = *fpsFactor / 256;
    for (int i = 0; i < len; i++)
    {
        const int intraCost = intraCosts[i];
        const int inter = interCosts[i] & LOWRES_COST_MASK;
        const int interCost = intraCost < inter ? intraCost : inter;
        const double propagateIntra = (double)intraCost * invQscales[i];
        const double propagateAmount = (double)propagateIn[i] + propagateIntra * fps;
        const double propagateNum = (double)(intraCost - interCost);
        const double propagateDenom = (double)intraCost;
        dst[i] = (int)(propagateAmount * propagateNum / propagateDenom + 0.5);
    }
}
