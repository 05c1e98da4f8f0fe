/* oracle/ref_shim_bidir.cpp -- TEST INFRASTRUCTURE ONLY (never linked into the product).
 * ref_shim_wref.cpp (included whole) plus B slices (frame_bidir.h) on the REAL reference code: the bi-prediction from a real
 * Predict (predInterLumaShort / predInterChromaShort of both lists) and the real Yuv::addAvg, the costs from the real table's
 * cu[].sa8d and chroma[X265_CSP_I420].cu[].sa8d, the zero try's range test from the real MV::checkRange.  Built by
 * Makefile.bidir with the reference objects into oracle/_ref/libx265ref_bidir{8,10}.so. */
#include "ref_shim_wref.cpp"

/* Predict::motionCompensation's two-list path (predict.cpp:168-189) for the CU at (x, y): the real predInterLumaShort /
 * predInterChromaShort of each slot's planes on a PicYuv without a CUData (as ref_wpred drives it), then the real addAvg */
static void ref_bipred(const drv_frame* f, int r0, int mx0, int my0, int r1, int mx1, int my1, int x, int y, int S, pixel* predY,
                       pixel (*predC)[32 * 32], int chroma)
{
    static thread_local Predict* pr = NULL;
    static thread_local ShortYuv* sy[2] = { NULL, NULL };
    static thread_local Yuv* py = NULL;
    if (!pr)
    {
        pr = new Predict(); pr->allocBuffers(X265_CSP_I420);
        for (int l = 0; l < 2; l++) { sy[l] = new ShortYuv(); sy[l]->create(MAX_CU_SIZE, X265_CSP_I420); }
        py = new Yuv(); py->create(MAX_CU_SIZE, X265_CSP_I420);
    }
    const intptr_t stride = f->p.stride, cs = f->cstride;
    const RefPu rpu = { 0, 0, 0, S, S };
    const PredictionUnit& pu = reinterpret_cast<const PredictionUnit&>(rpu);
    const int r[2] = { r0, r1 };
    const MV mv[2] = { MV(mx0, my0), MV(mx1, my1) };
    for (int l = 0; l < 2; l++)
    {
        PicYuv pic;
        intptr_t zero = 0;
        pic.m_cuOffsetY = &zero; pic.m_cuOffsetC = &zero; pic.m_buOffsetY = &zero; pic.m_buOffsetC = &zero;
        pic.m_stride = stride; pic.m_strideC = cs;
        pic.m_picOrg[0] = (pixel*)f->refs[r[l]] + (intptr_t)y * stride + x;
        pic.m_picOrg[1] = chroma ? (pixel*)f->refC[r[l]][0] + (intptr_t)(y / 2) * cs + x / 2 : NULL;
        pic.m_picOrg[2] = chroma ? (pixel*)f->refC[r[l]][1] + (intptr_t)(y / 2) * cs + x / 2 : NULL;
        pr->predInterLumaShort(pu, *sy[l], pic, mv[l]);
        if (chroma) pr->predInterChromaShort(pu, *sy[l], pic, mv[l]);
        pic.m_cuOffsetY = pic.m_cuOffsetC = pic.m_buOffsetY = pic.m_buOffsetC = NULL;
        pic.m_picOrg[0] = pic.m_picOrg[1] = pic.m_picOrg[2] = NULL;
    }
    py->addAvg(*sy[0], *sy[1], 0, S, S, true, chroma != 0);
    for (int i = 0; i < S; i++) memcpy(predY + i * S, py->m_buf[0] + i * py->m_size, sizeof(pixel) * S);
    for (int pl = 0; pl < 2 && chroma; pl++)
        for (int i = 0; i < S / 2; i++) memcpy(predC[pl] + i * (S / 2), py->m_buf[1 + pl] + i * py->m_csize, sizeof(pixel) * (S / 2));
}
#define DRV_BIPRED(f, r0, mx0, my0, r1, mx1, my1, x, y, S, pY, pC, c) ref_bipred(f, r0, mx0, my0, r1, mx1, my1, x, y, S, pY, pC, c)
#define DRV_SA8D_C(a, sa, b, sb, S) g_c.chroma[X265_CSP_I420].cu[lg2(S) - 2].sa8d(a, sa, b, sb)
#define DRV_IN_RANGE(px, py, mnx, mny, mxx, mxy) MV(px, py).checkRange(MV(mnx, mny), MV(mxx, mxy))
#include "frame_bidir.h"

/* x265ref_analyse_frame_chroma with B slices (orc_analyse_frame_bidir's twin) */
extern "C" int x265ref_analyse_frame_bidir(drv_frame* f, int stages, drv_chroma_resid* cr, drv_bidir* b)
{
    if ((stages & 8) && !f->chroma) return -1;
    x265ref_analyse_frame(f, stages & 5);
    drv_run_bidir(f, cr, b, stages);
    return 0;
}
