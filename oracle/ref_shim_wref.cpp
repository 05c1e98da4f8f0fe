/* oracle/ref_shim_wref.cpp -- TEST INFRASTRUCTURE ONLY (never linked into the product).
 * ref_shim_chroma.cpp (included whole) plus weighted P-slice references (frame_wref.h) on the REAL reference code: the search
 * planes come from a real MotionReference (init + applyWeight as FrameEncoder calls them), the weighted prediction from a real
 * Predict (predInterLumaShort / predInterChromaShort + addWeightUni).  Built by Makefile.wref with the reference objects into
 * oracle/_ref/libx265ref_wref{8,10}.so. */
#include "ref_shim_chroma.cpp"
#include "reference.h"
#include "shortyuv.h"
#include <algorithm>

/* PredictionUnit's fields (predict.h:40-49) without its CUData constructor: a CU's 2Nx2N PU, z-order offsets 0 (the planes
 * handed to Predict start at the CU) */
struct RefPu { uint32_t ctuAddr, cuAbsPartIdx, puAbsPartIdx; int width, height; };
static_assert(sizeof(RefPu) == sizeof(PredictionUnit), "PredictionUnit layout");

struct drv_wref_s;
static void ref_wpred(const struct drv_wref_s* w, int r, int x, int y, int S, int qx, int qy, intptr_t stride, intptr_t cs, pixel* predY,
                      pixel (*predC)[32 * 32], int luma, int chroma);
#define DRV_WPRED(w, r, x, y, S, qx, qy, st, cs, pY, pC, l, c) ref_wpred(w, r, x, y, S, qx, qy, st, cs, pY, pC, l, c)
#include "frame_wref.h"

/* Predict::motionCompensation's P-slice path with wp0->wtPresent (predict.cpp:82-112) for the CU at (x, y): the real
 * predInterLumaShort / predInterChromaShort of the unweighted planes and the real addWeightUni with the WeightValues filled as
 * predict.cpp:96-102 fills them */
static void ref_wpred(const struct drv_wref_s* w, int r, int x, int y, int S, int qx, int qy, intptr_t stride, intptr_t cs, pixel* predY,
                      pixel (*predC)[32 * 32], int luma, int chroma)
{
    static thread_local Predict* pr = NULL;
    static thread_local ShortYuv* sy = NULL;
    static thread_local Yuv* py = NULL;
    if (!pr)
    {
        pr = new Predict(); pr->allocBuffers(X265_CSP_I420);
        sy = new ShortYuv(); sy->create(MAX_CU_SIZE, X265_CSP_I420);
        py = new Yuv(); py->create(MAX_CU_SIZE, X265_CSP_I420);
    }
    PicYuv pic;
    intptr_t zero = 0;
    pic.m_cuOffsetY = &zero; pic.m_cuOffsetC = &zero; pic.m_buOffsetY = &zero; pic.m_buOffsetC = &zero;
    pic.m_stride = stride; pic.m_strideC = cs;
    pic.m_picOrg[0] = (pixel*)w->refs[r] + (intptr_t)y * stride + x;
    pic.m_picOrg[1] = (pixel*)w->refC[r][0] + (intptr_t)(y / 2) * cs + x / 2;
    pic.m_picOrg[2] = (pixel*)w->refC[r][1] + (intptr_t)(y / 2) * cs + x / 2;
    const RefPu rpu = { 0, 0, 0, S, S };
    const PredictionUnit& pu = reinterpret_cast<const PredictionUnit&>(rpu);
    const MV mv(qx, qy);
    Predict::WeightValues wv[3];
    for (int plane = 0; plane < (chroma ? 3 : 1); plane++)
    {
        const int32_t* e = w->wp[r][plane];
        wv[plane].w      = e[1];
        wv[plane].offset = e[3] * (1 << (X265_DEPTH - 8));
        wv[plane].shift  = e[2];
        wv[plane].round  = e[2] >= 1 ? 1 << (e[2] - 1) : 0;
    }
    if (luma) pr->predInterLumaShort(pu, *sy, pic, mv);
    if (chroma) pr->predInterChromaShort(pu, *sy, pic, mv);
    pr->addWeightUni(pu, *py, *sy, wv, luma != 0, chroma != 0);
    for (int i = 0; i < S && luma; i++) memcpy(predY + i * S, py->m_buf[0] + i * py->m_size, sizeof(pixel) * S);
    for (int pl = 0; pl < 2 && chroma; pl++)
        for (int i = 0; i < S / 2; i++) memcpy(predC[pl] + i * (S / 2), py->m_buf[1 + pl] + i * py->m_csize, sizeof(pixel) * (S / 2));
    pic.m_cuOffsetY = pic.m_cuOffsetC = pic.m_buOffsetY = pic.m_buOffsetC = NULL;
    pic.m_picOrg[0] = pic.m_picOrg[1] = pic.m_picOrg[2] = NULL;
}

/* The search planes of one reference: a real PicYuv holding the picture (borders extended as the frame filter leaves a
 * reconstruction), a real MotionReference::init with the table row as FrameEncoder passes it (frameencoder.cpp:544-554: the row
 * when luma has wtPresent, else NULL), then applyWeight for every CTU row as compressFrame calls it once each row's
 * reference rows are reconstructed (frameencoder.cpp:895-905, m_refLagRows from :157-162), up to the last row.  fpelPlane[c]
 * is copied out with the analyser's margins (96 x 80, 48 x 40): the weighted plane, or the picture for an unweighted plane.
 * Returns MotionReference::isWeighted. */
extern "C" int x265ref_wref_planes(const pixel* y, const pixel* cb, const pixel* cr, intptr_t stride, intptr_t cstride, int width,
                                   int height, int method, int subme, int merange, const int32_t* wp, pixel* oy, pixel* ocb, pixel* ocr)
{
    ensure_init();
    static bool scales = false;
    if (!scales) { MotionEstimate::initScales(); scales = true; }
    x265_param* p = x265_param_alloc();
    x265_param_default(p);
    p->sourceWidth = width; p->sourceHeight = height; p->internalCsp = X265_CSP_I420; p->maxCUSize = 64;
    p->subpelRefine = subme; p->searchMethod = method; p->searchRange = merange; p->maxSlices = 1;
    PicYuv* pic = new PicYuv();
    pic->create(p, true, NULL);
    const pixel* in[3] = { y, cb, cr };
    pixel* out[3] = { oy, ocb, ocr };
    for (int c = 0; c < 3; c++)
    {
        const int ch = c > 0, w = width >> ch, h = height >> ch;
        const intptr_t s = ch ? cstride : stride, ps = ch ? pic->m_strideC : pic->m_stride;
        for (int r = 0; r < h; r++) memcpy(pic->m_picOrg[c] + r * ps, in[c] + r * s, sizeof(pixel) * w);
        extendPicBorder(pic->m_picOrg[c], ps, w, h, ch ? pic->m_chromaMarginX : pic->m_lumaMarginX, ch ? pic->m_chromaMarginY : pic->m_lumaMarginY);
    }
    WeightParam wt[3];
    memset(wt, 0, sizeof(wt));
    for (int c = 0; c < 3; c++)
    {
        wt[c].wtPresent = wp[4 * c]; wt[c].inputWeight = wp[4 * c + 1];
        wt[c].log2WeightDenom = wp[4 * c + 2]; wt[c].inputOffset = wp[4 * c + 3];
    }
    MotionReference mref;
    mref.init(pic, wt[0].wtPresent ? wt : NULL, *p);
    int range = p->searchRange;
    range += !!(p->searchMethod < 2);
    range += NTAPS_LUMA / 2;
    range += 2 + (MotionEstimate::hpelIterationCount(p->subpelRefine) + 1) / 2;
    const int lag = 1 + ((range + p->maxCUSize - 1) / p->maxCUSize);
    const int numRows = (height + p->maxCUSize - 1) / p->maxCUSize;
    for (int i = 0; i < numRows && mref.isWeighted; i++)
        mref.applyWeight(std::min(numRows - 1, i + lag), numRows, numRows, 0);
    for (int c = 0; c < 3; c++)
    {
        const int ch = c > 0, w = width >> ch, h = height >> ch, mx = ch ? 48 : 96, my = ch ? 40 : 80;
        const intptr_t s = ch ? cstride : stride, ps = ch ? pic->m_strideC : pic->m_stride;
        assert(mx <= (ch ? pic->m_chromaMarginX : pic->m_lumaMarginX) && my <= (ch ? pic->m_chromaMarginY : pic->m_lumaMarginY));
        for (int r = -my; r < h + my && out[c]; r++)
            memcpy(out[c] + r * s - mx, mref.fpelPlane[c] + r * ps - mx, sizeof(pixel) * (w + 2 * mx));
    }
    const int weighted = mref.isWeighted;
    pic->destroy();
    delete pic;
    x265_param_free(p);
    return weighted;
}

/* x265ref_analyse_frame_chroma with weighted references: f->refs / refC = what the search reads (x265ref_wref_planes), w =
 * the weights and the unweighted planes */
extern "C" int x265ref_analyse_frame_wref(drv_frame* f, int stages, drv_chroma_resid* cr, const drv_wref* w)
{
    if ((stages & 8) && !f->chroma) return -1;
    x265ref_analyse_frame(f, stages & 5);
    drv_run_wref(f, cr, w, stages);
    return 0;
}
