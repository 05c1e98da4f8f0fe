/* oracle/oracle_cutree.c -- TEST INFRASTRUCTURE ONLY: cuTree's propagation chain and its finish, restated in plain C.
 *
 * Lookahead::cuTree (encoder/slicetype.cpp:2538-2639), estimateCUPropagate (:2641-2747, with the propagateCost primitive of
 * common/pixel.cpp:914-940 inline) and the non-hevcAq cuTreeFinish (:2889-2937), over caller arrays.  The int32 products of
 * the scatter wrap as the compiled reference's do (x86 imul): they are computed in unsigned arithmetic here, so that this
 * file pins the wrapped order-dependent case too.  log2 is the host libm's, as the reference calls it (common.h:249).
 *
 * orc_cutree runs the chain in the reference's order, one CU at a time, and every cuTreeFinish call where the reference
 * makes it (when the frame has a qpCuTreeOffset); `finish` receives the calls as x265cu_cutree reports them. */
#include <math.h>
#include <stdint.h>
#include <string.h>

#define ORC_DIST 18                        /* X265_BFRAME_MAX + 2 */
#define TYPE_B 5
#define COST_MASK ((1 << 14) - 1)
#define COST_SHIFT 14

typedef struct {
    const int32_t* intraCost; const int32_t* invQscale; uint16_t* propagateCost;
    const uint16_t* lowresCosts[ORC_DIST][ORC_DIST];
    const int32_t* mvs[2][ORC_DIST];
    int32_t sliceType, reserved;
    /* cuTreeFinish: NULL qpCuTreeOffset = not finished here */
    const double* qpAqOffset; double* qpCuTreeOffset;
    double weightedCostDelta[ORC_DIST];
} orc_cutree_frame;

typedef struct {
    int32_t bIntra, lookaheadDepth, bBPyramid, bEnableWeightedBiPred, vbv, fpsNum, fpsDenom, qgSize;
    double qCompress;
} orc_cutree_params;

typedef struct {
    orc_cutree_frame* fr;
    const orc_cutree_params* p;
    int w8, h8, ncu, nfinish, maxFinish, missing;
    int32_t* finish;
    double averageDuration;
    int scratch[4096];
} Chain;

static double clip_duration(double f) { double v = 0.01 > f ? 0.01 : f; return v < 1.00 ? v : 1.00; }

/* CLIP_ADD(s, x) with the int32 sum wrapping */
static void clip_add(uint16_t* s, int32_t x)
{
    int32_t v = (int32_t)((uint32_t)*s + (uint32_t)x);
    *s = (uint16_t)(v < 65535 ? v : 65535);
}
static int32_t wmul_shift(int32_t a, int32_t w, uint32_t round, int shift) { return (int32_t)((uint32_t)a * (uint32_t)w + round) >> shift; }

/* estimateCUPropagateCost (pixel.cpp:914-940); out-of-range conversions as x86 cvttsd2si gives them */
static int32_t propagate_amount(int propagateIn, int intraCost, int interWord, int invQscale, double fps)
{
    int interCost = interWord & COST_MASK;
    if (interCost > intraCost) interCost = intraCost;
    double propagateIntra = (int32_t)((uint32_t)intraCost * (uint32_t)invQscale);     /* int32 product, wrapping */
    double propagateAmount = (double)propagateIn + propagateIntra * fps;
    double v = propagateAmount * (double)(intraCost - interCost) / (double)intraCost + 0.5;
    return (v >= -2147483648.0 && v < 2147483648.0) ? (int32_t)v : INT32_MIN;
}

static void finish_frame(Chain* c, int f, int ref0Distance);

static void step(Chain* c, int p0, int p1, int b, int referenced)
{
    orc_cutree_frame* fb = &c->fr[b];
    uint16_t* refCosts[2] = { c->fr[p0].propagateCost, c->fr[p1].propagateCost };
    int32_t distScaleFactor = (((b - p0) << 8) + ((p1 - p0) >> 1)) / (p1 - p0);
    int32_t bipredWeight = c->p->bEnableWeightedBiPred ? 64 - (distScaleFactor >> 2) : 32;
    int32_t bipredWeights[2] = { bipredWeight, 64 - bipredWeight };
    int listDist[2] = { b - p0, p1 - b };
    const uint16_t* costs = fb->lowresCosts[b - p0][p1 - b];
    double fpsFactor = clip_duration((double)c->p->fpsDenom / c->p->fpsNum) / clip_duration(c->averageDuration);
    const int w8 = c->w8, h8 = c->h8;
    const uint16_t* in = fb->propagateCost;
    if (!costs || !fb->mvs[0][b - p0] || (p1 > b && !fb->mvs[1][p1 - b]))
    {
        c->missing = 1;                                               /* an estimate the chain reads was not supplied */
        return;
    }
    if (!referenced)
        memset(fb->propagateCost, 0, w8 * sizeof(uint16_t));
    for (int blocky = 0; blocky < h8; blocky++)
    {
        int cuIndex = blocky * w8;
        for (int x = 0; x < w8; x++)
            c->scratch[x] = propagate_amount(in[x], fb->intraCost[cuIndex + x], costs[cuIndex + x], fb->invQscale[cuIndex + x], fpsFactor / 256);
        if (referenced)
            in += w8;
        for (int blockx = 0; blockx < w8; blockx++, cuIndex++)
        {
            int32_t amount = c->scratch[blockx];
            if (amount <= 0)
                continue;
            int lists = costs[cuIndex] >> COST_SHIFT;
            for (int list = 0; list < 2; list++)
            {
                if (!((lists >> list) & 1))
                    continue;
                int32_t listamount = amount;
                if (lists == 3)
                    listamount = wmul_shift(listamount, bipredWeights[list], 32, 6);
                const int32_t* mv = fb->mvs[list][listDist[list]] + 2 * cuIndex;
                uint16_t* ref = refCosts[list];
                if (!mv[0] && !mv[1])
                {
                    clip_add(&ref[cuIndex], listamount);
                    continue;
                }
                int32_t x = mv[0], y = mv[1];
                int32_t cux = (x >> 5) + blockx, cuy = (y >> 5) + blocky;
                int32_t idx0 = cux + cuy * w8;
                x &= 31; y &= 31;
                int32_t wt[4] = { (32 - y) * (32 - x), (32 - y) * x, y * (32 - x), y * x };
                int32_t idx[4] = { idx0, idx0 + 1, idx0 + w8, idx0 + w8 + 1 };
                for (int k = 0; k < 4; k++)
                {
                    int32_t cx = cux + (k & 1), cy = cuy + (k >> 1);
                    if (cx >= 0 && cx < w8 && cy >= 0 && cy < h8)
                        clip_add(&ref[idx[k]], wmul_shift(listamount, wt[k], 512, 10));
                }
            }
        }
    }
    if (c->p->vbv && c->p->lookaheadDepth && referenced)
        finish_frame(c, b, b == p1 ? b - p0 : 0);
}

/* cuTreeFinish, non-hevcAq (:2889-2937) */
static void finish_frame(Chain* c, int f, int ref0Distance)
{
    if (c->nfinish < c->maxFinish)
    {
        c->finish[2 * c->nfinish] = f;
        c->finish[2 * c->nfinish + 1] = ref0Distance;
    }
    c->nfinish++;
    orc_cutree_frame* fr = &c->fr[f];
    if (!fr->qpCuTreeOffset || ref0Distance < 0)
        return;
    const orc_cutree_params* p = c->p;
    const double strength = 5.0 * (1.0 - p->qCompress);
    int fpsFactor = (int)(clip_duration(c->averageDuration) / clip_duration((double)p->fpsDenom / p->fpsNum) * 256);
    double weightdelta = 0.0;
    if (ref0Distance && fr->weightedCostDelta[ref0Distance - 1] > 0)
        weightdelta = (1.0 - fr->weightedCostDelta[ref0Distance - 1]);
    if (p->qgSize == 8)
    {
        const int full = c->w8 * 2;                                   /* maxBlocksInRowFullRes */
        for (int cuY = 0; cuY < c->h8; cuY++)
            for (int cuX = 0; cuX < c->w8; cuX++)
            {
                const int cuXY = cuX + cuY * c->w8;
                int intracost = ((fr->intraCost[cuXY]) / 4 * fr->invQscale[cuXY] + 128) >> 8;
                if (!intracost)
                    continue;
                int propagateCost = ((fr->propagateCost[cuXY]) / 4 * fpsFactor + 128) >> 8;
                double log2_ratio = log2(intracost + propagateCost) - log2(intracost) + weightdelta;
                const int o = cuX * 2 + cuY * c->w8 * 4;
                const int at[4] = { o, o + 1, o + full, o + full + 1 };
                for (int k = 0; k < 4; k++)
                    fr->qpCuTreeOffset[at[k]] = fr->qpAqOffset[at[k]] - strength * (log2_ratio);
            }
    }
    else
    {
        for (int cuIndex = 0; cuIndex < c->ncu; cuIndex++)
        {
            int intracost = (fr->intraCost[cuIndex] * fr->invQscale[cuIndex] + 128) >> 8;
            if (!intracost)
                continue;
            int propagateCost = (fr->propagateCost[cuIndex] * fpsFactor + 128) >> 8;
            double log2_ratio = log2(intracost + propagateCost) - log2(intracost) + weightdelta;
            fr->qpCuTreeOffset[cuIndex] = fr->qpAqOffset[cuIndex] - strength * log2_ratio;
        }
    }
}

static void swap_costs(orc_cutree_frame* a, orc_cutree_frame* b)
{
    uint16_t* t = a->propagateCost; a->propagateCost = b->propagateCost; b->propagateCost = t;
}

/* Returns the number of cuTreeFinish calls (finish: (frame, ref0Distance) pairs, -1 = qpAqOffset copied), -1 for the
 * window the reference divides by zero on (estimateCUPropagate(0, 0, 0)), -2 when an estimate it read was not supplied. */
int orc_cutree(orc_cutree_frame* frames, int numframes, const orc_cutree_params* p, int w8, int h8, int32_t* finish, int maxFinish)
{
    static Chain cs;
    Chain* c = &cs;
    memset(c, 0, sizeof(*c));
    c->fr = frames; c->p = p; c->w8 = w8; c->h8 = h8; c->ncu = w8 * h8; c->finish = finish; c->maxFinish = maxFinish;
    const int ncu = w8 * h8;
    int idx = !p->bIntra;
    int lastnonb, curnonb = 1;
    int bframes = 0;
    double totalDuration = 0.0;
    for (int j = 0; j <= numframes; j++)
        totalDuration += (double)p->fpsDenom / p->fpsNum;
    c->averageDuration = totalDuration / (numframes + 1);
    int i = numframes;
    while (i > 0 && frames[i].sliceType == TYPE_B)
        i--;
    lastnonb = i;
    if (!p->lookaheadDepth)
    {
        if (p->bIntra)
        {
            memset(frames[0].propagateCost, 0, ncu * sizeof(uint16_t));
            if (frames[0].qpCuTreeOffset)
                memcpy(frames[0].qpCuTreeOffset, frames[0].qpAqOffset, (p->qgSize == 8 ? 4 : 1) * ncu * sizeof(double));
            finish_frame(c, 0, -1);
            return c->nfinish;
        }
        swap_costs(&frames[lastnonb], &frames[0]);
        memset(frames[0].propagateCost, 0, ncu * sizeof(uint16_t));
    }
    else
    {
        if (lastnonb < idx)
            return 0;
        memset(frames[lastnonb].propagateCost, 0, ncu * sizeof(uint16_t));
    }
    while (i-- > idx)
    {
        curnonb = i;
        while (frames[curnonb].sliceType == TYPE_B && curnonb > 0)
            curnonb--;
        if (curnonb < idx)
            break;
        memset(frames[curnonb].propagateCost, 0, ncu * sizeof(uint16_t));
        bframes = lastnonb - curnonb - 1;
        if (p->bBPyramid && bframes > 1)
        {
            int middle = (bframes + 1) / 2 + curnonb;
            memset(frames[middle].propagateCost, 0, ncu * sizeof(uint16_t));
            while (i > curnonb)
            {
                int p0 = i > middle ? middle : curnonb;
                int p1 = i < middle ? middle : lastnonb;
                if (i != middle)
                    step(c, p0, p1, i, 0);
                i--;
            }
            step(c, curnonb, lastnonb, middle, 1);
        }
        else
        {
            while (i > curnonb)
            {
                step(c, curnonb, lastnonb, i, 0);
                i--;
            }
        }
        step(c, curnonb, lastnonb, lastnonb, 1);
        lastnonb = curnonb;
    }
    if (!p->lookaheadDepth)
    {
        if (lastnonb == 0)
            return -1;
        step(c, 0, lastnonb, lastnonb, 1);
        swap_costs(&frames[lastnonb], &frames[0]);
    }
    finish_frame(c, lastnonb, lastnonb);
    if (p->bBPyramid && bframes > 1 && !p->vbv)
        finish_frame(c, lastnonb + (bframes + 1) / 2, 0);
    return c->missing ? -2 : c->nfinish;
}

/* cuTreeFinish of one frame on its current propagateCost (the host's half of the device chain) */
void orc_cutree_finish(orc_cutree_frame* frames, int numframes, const orc_cutree_params* p, int w8, int h8, int f, int ref0Distance)
{
    static Chain cs;
    Chain* c = &cs;
    memset(c, 0, sizeof(*c));
    c->fr = frames; c->p = p; c->w8 = w8; c->h8 = h8; c->ncu = w8 * h8;
    double totalDuration = 0.0;
    for (int j = 0; j <= numframes; j++)
        totalDuration += (double)p->fpsDenom / p->fpsNum;
    c->averageDuration = totalDuration / (numframes + 1);
    finish_frame(c, f, ref0Distance);
}
