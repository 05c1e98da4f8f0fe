/* oracle/oracle_pred.c -- TEST INFRASTRUCTURE ONLY (see oracle.h).
 *
 * Prediction costs of predInterSearch around the motion search, restated from the reference:
 *   - Search::selectMVP          encoder/search.cpp:1992-2023   SAD of the luma prediction at an AMVP candidate
 *   - Search::mergeEstimation    encoder/search.cpp:1901-1960   SATD (+ chroma SATD) of the merge candidate's prediction
 *   - bidir in predInterSearch   encoder/search.cpp:2474-2607   SATD of the bi-prediction (addAvg of the 14-bit
 *                                                                intermediates with bChromaSATD, pixelavg_pp of the two
 *                                                                pixel predictions without)
 * on Predict::motionCompensation's unweighted paths (common/predict.cpp:76-240), predInterLumaPixel / LumaShort /
 * ChromaPixel / ChromaShort (predict.cpp:242-420) and Yuv::addAvg (yuv.cpp -> primitives addAvg).  4:2:0 only.
 * Pinned to the real classes by tests/test_oracle_vs_ref.py::test_pred_cost (oracle/ref_shim.cpp: x265ref_pred_cost).
 */
#include <string.h>
#include "oracle.h"

typedef struct orc_pred_job_s
{
    const pixel* fenc[3];       /* source planes at the PU origin (chroma: at (x >> 1, y >> 1)) */
    const pixel* ref0[3];       /* list-0 reference planes at the PU origin; ref0[0] == NULL: list unused */
    const pixel* ref1[3];
    intptr_t stride, cstride;
    int w, h;
    int mv0[2], mv1[2];         /* quarter-pel, already clipped (CUData::clipMv is the caller's) */
    int cost;                   /* 0 = SAD (bufSAD), 1 = SATD (bufSATD) */
    int chroma;                 /* + bufChromaSATD (motion.h:91-95) */
    int biAvgPP;                /* two references: pixelavg_pp of the pixel predictions (search.cpp:2499-2510) instead of addAvg */
} orc_pred_job;

/* predict.cpp:242-265 */
static void luma_pixel(const pixel* ref, intptr_t stride, const int* mv, pixel* dst, intptr_t ds, int w, int h)
{
    const pixel* src = ref + (mv[0] >> 2) + (mv[1] >> 2) * stride;
    const int xf = mv[0] & 3, yf = mv[1] & 3;
    if (!(xf | yf)) orc_copy_pp(dst, ds, src, stride, w, h);
    else if (!yf)   orc_interp_hpp(src, stride, dst, ds, xf, 8, w, h);
    else if (!xf)   orc_interp_vpp(src, stride, dst, ds, yf, 8, w, h);
    else            orc_interp_hvpp(src, stride, dst, ds, xf, yf, 8, w, h);
}

/* predict.cpp:267-303 */
static void luma_short(const pixel* ref, intptr_t stride, const int* mv, int16_t* dst, intptr_t ds, int w, int h)
{
    const pixel* src = ref + (mv[0] >> 2) + (mv[1] >> 2) * stride;
    const int xf = mv[0] & 3, yf = mv[1] & 3;
    if (!(xf | yf)) orc_p2s(src, stride, dst, ds, w, h);
    else if (!yf)   orc_interp_hps(src, stride, dst, ds, xf, 0, 8, w, h);
    else if (!xf)   orc_interp_vps(src, stride, dst, ds, yf, 8, w, h);
    else
    {
        int16_t immed[64 * (64 + 7)];
        orc_interp_hps(src, stride, immed, w, xf, 1, 8, w, h);
        orc_interp_vss(immed + 3 * w, w, dst, ds, yf, 8, w, h);
    }
}

/* predict.cpp:305-351, one plane; 4:2:0: mvx = mv.x, eighth-pel */
static void chroma_pixel(const pixel* ref, intptr_t stride, const int* mv, pixel* dst, intptr_t ds, int cw, int ch)
{
    const pixel* src = ref + (mv[0] >> 3) + (mv[1] >> 3) * stride;
    const int xf = mv[0] & 7, yf = mv[1] & 7;
    if (!(xf | yf)) orc_copy_pp(dst, ds, src, stride, cw, ch);
    else if (!yf)   orc_interp_hpp(src, stride, dst, ds, xf, 4, cw, ch);
    else if (!xf)   orc_interp_vpp(src, stride, dst, ds, yf, 4, cw, ch);
    else
    {
        int16_t immed[64 * (64 + 3)];
        orc_interp_hps(src, stride, immed, cw, xf, 1, 4, cw, ch);
        orc_interp_vsp(immed + 1 * cw, cw, dst, ds, yf, 4, cw, ch);
    }
}

/* predict.cpp:353-407, one plane */
static void chroma_short(const pixel* ref, intptr_t stride, const int* mv, int16_t* dst, intptr_t ds, int cw, int ch)
{
    const pixel* src = ref + (mv[0] >> 3) + (mv[1] >> 3) * stride;
    const int xf = mv[0] & 7, yf = mv[1] & 7;
    if (!(xf | yf)) orc_p2s(src, stride, dst, ds, cw, ch);
    else if (!yf)   orc_interp_hps(src, stride, dst, ds, xf, 0, 4, cw, ch);
    else if (!xf)   orc_interp_vps(src, stride, dst, ds, yf, 4, cw, ch);
    else
    {
        int16_t immed[64 * (64 + 3)];
        orc_interp_hps(src, stride, immed, cw, xf, 1, 4, cw, ch);
        orc_interp_vss(immed + 1 * cw, cw, dst, ds, yf, 4, cw, ch);
    }
}

int orc_pred_cost(const orc_pred_job* j)
{
    pixel predY[64 * 64], predC[2][32 * 32];
    const int w = j->w, h = j->h, cw = w >> 1, ch = h >> 1;
    const int bi = j->ref0[0] && j->ref1[0];
    const int chroma = j->chroma && !(cw & 3) && !(ch & 3);     /* a chroma SATD exists for multiples of 4 only (motion.cpp:204-212) */
    if (bi && j->biAvgPP)
    {   /* search.cpp:2499-2510: two pixel predictions, pixelavg_pp; luma only */
        pixel p0[64 * 64], p1[64 * 64];
        luma_pixel(j->ref0[0], j->stride, j->mv0, p0, 64, w, h);
        luma_pixel(j->ref1[0], j->stride, j->mv1, p1, 64, w, h);
        orc_pixelavg_pp(predY, 64, p0, 64, p1, 64, w, h);
    }
    else if (bi)
    {   /* predict.cpp:167-186: both lists through the 14-bit intermediates, Yuv::addAvg */
        int16_t s0[64 * 64], s1[64 * 64];
        luma_short(j->ref0[0], j->stride, j->mv0, s0, 64, w, h);
        luma_short(j->ref1[0], j->stride, j->mv1, s1, 64, w, h);
        orc_addAvg(s0, s1, predY, 64, 64, 64, w, h);
        if (chroma)
            for (int p = 0; p < 2; p++)
            {
                chroma_short(j->ref0[1 + p], j->cstride, j->mv0, s0, 32, cw, ch);
                chroma_short(j->ref1[1 + p], j->cstride, j->mv1, s1, 32, cw, ch);
                orc_addAvg(s0, s1, predC[p], 32, 32, 32, cw, ch);
            }
    }
    else
    {   /* predict.cpp:188-239: one list, pixel prediction */
        const pixel* const* ref = j->ref0[0] ? j->ref0 : j->ref1;
        const int* mv = j->ref0[0] ? j->mv0 : j->mv1;
        luma_pixel(ref[0], j->stride, mv, predY, 64, w, h);
        if (chroma)
            for (int p = 0; p < 2; p++) chroma_pixel(ref[1 + p], j->cstride, mv, predC[p], 32, cw, ch);
    }
    if (!j->cost) return orc_sad(j->fenc[0], j->stride, predY, 64, w, h);
    int cost = orc_satd(j->fenc[0], j->stride, predY, 64, w, h);
    if (chroma && !(bi && j->biAvgPP))
        for (int p = 0; p < 2; p++) cost += orc_satd(predC[p], 32, j->fenc[1 + p], j->cstride, cw, ch);
    return cost;
}

/* orc_pred_cost over a job list in the batched entry point's layout (include/x265_b200.h: x265cu_pred_job), with the planes
 * and tables of x265ref_pred_cost_batch (oracle/ref_shim.cpp): planes at the picture origin, refs / refCb / refCr indexed by
 * ref0 / ref1, the chroma origin of the luma offset at ((offset / stride) >> 1) * cstride + ((offset % stride) >> 1).
 * fencCb == NULL: no chroma planes, so no job gets the chroma term (as x265cu_pred_cost_batch with chroma == NULL). */
typedef struct { int32_t offset; int16_t pw, ph; int8_t ref0, ref1; uint8_t cost, flags; int16_t mv0[2], mv1[2]; } orc_pred_batch_job;

int orc_pred_cost_batch(const pixel* fenc, const pixel* fencCb, const pixel* fencCr, const pixel* const* refs, const pixel* const* refCb,
                        const pixel* const* refCr, intptr_t stride, intptr_t cstride, const void* jobsv, int n, int32_t* out)
{
    const orc_pred_batch_job* jobs = (const orc_pred_batch_job*)jobsv;
    for (int i = 0; i < n; i++)
    {
        const orc_pred_batch_job* b = &jobs[i];
        const intptr_t coff = ((b->offset / stride) >> 1) * cstride + ((b->offset % stride) >> 1);
        const int chroma = (b->flags & 1) && fencCb;
        orc_pred_job j;
        memset(&j, 0, sizeof(j));
        j.fenc[0] = fenc + b->offset;
        if (chroma) { j.fenc[1] = fencCb + coff; j.fenc[2] = fencCr + coff; }
        if (b->ref0 >= 0)
        {
            j.ref0[0] = refs[b->ref0] + b->offset;
            if (chroma) { j.ref0[1] = refCb[b->ref0] + coff; j.ref0[2] = refCr[b->ref0] + coff; }
        }
        if (b->ref1 >= 0)
        {
            j.ref1[0] = refs[b->ref1] + b->offset;
            if (chroma) { j.ref1[1] = refCb[b->ref1] + coff; j.ref1[2] = refCr[b->ref1] + coff; }
        }
        j.stride = stride; j.cstride = cstride; j.w = b->pw; j.h = b->ph;
        j.mv0[0] = b->mv0[0]; j.mv0[1] = b->mv0[1]; j.mv1[0] = b->mv1[0]; j.mv1[1] = b->mv1[1];
        j.cost = b->cost; j.chroma = chroma; j.biAvgPP = (b->flags >> 1) & 1;
        out[i] = orc_pred_cost(&j);
    }
    return 0;
}
