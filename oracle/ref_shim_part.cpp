/* oracle/ref_shim_part.cpp -- TEST INFRASTRUCTURE ONLY (never linked into the product).
 * ref_shim_bidir.cpp (included whole) plus the PART stage (frame_part.h) on the REAL reference code: every PU predicted by a
 * real Predict (predInterLumaPixel / predInterChromaPixel, or predInterLumaShort / predInterChromaShort + addWeightUni for a
 * weighted slot) into one real Yuv of the CU, through a PredictionUnit whose puAbsPartIdx is the PU's z-order offset in the CU
 * and a PicYuv whose per-partition offsets are the reference's own z-scan tables, so the reference's PU addressing places
 * each PU; the costs from the real table's cu[].sa8d and chroma[X265_CSP_I420].cu[].sa8d.  Built by Makefile.part with the
 * reference objects into oracle/_ref/libx265ref_part{8,10}.so. */
#include "ref_shim_bidir.cpp"

struct drv_part_pu_s;
static void ref_part_pred(const drv_frame* f, const drv_wref* w, int x, int y, int S, int npu, const struct drv_part_pu_s* pu, pixel* predY,
                          pixel (*predC)[32 * 32], int chroma);
#define DRV_PART_PRED(f, w, x, y, S, npu, pu, pY, pC, c) ref_part_pred(f, w, x, y, S, npu, pu, pY, pC, c)
#include "frame_part.h"

/* Predict::motionCompensation's P-slice path (predict.cpp:82-118) for every PU of the partition, into the CU's Yuv: the CU
 * sits at its CTU's origin (ctuAddr 0, cuAbsPartIdx 0) of a PicYuv whose origin is the CU's pixel in the slot's unweighted
 * planes, m_buOffsetY / m_buOffsetC built from g_zscanToPelX / g_zscanToPelY as PicYuv::createOffsets builds them; the PU's
 * puAbsPartIdx is g_rasterToZscan of its origin's 4x4 unit, the value CUData::getPartIndexAndSize gives it */
static void ref_part_pred(const drv_frame* f, const drv_wref* w, int x, int y, int S, int npu, const struct drv_part_pu_s* pu, pixel* predY,
                          pixel (*predC)[32 * 32], int chroma)
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
    const intptr_t stride = f->p.stride, cs = f->cstride;
    intptr_t buY[MAX_NUM_PARTITIONS], buC[MAX_NUM_PARTITIONS], zero = 0;
    for (uint32_t i = 0; i < MAX_NUM_PARTITIONS; i++)
    {
        buY[i] = g_zscanToPelX[i] + (intptr_t)g_zscanToPelY[i] * stride;
        buC[i] = (g_zscanToPelX[i] >> 1) + (intptr_t)(g_zscanToPelY[i] >> 1) * cs;
    }
    for (int u = 0; u < npu; u++)
    {
        const drv_part_pu& q = pu[u];
        const int r = q.slot;
        PicYuv pic;
        pic.m_cuOffsetY = &zero; pic.m_cuOffsetC = &zero; pic.m_buOffsetY = buY; pic.m_buOffsetC = buC;
        pic.m_stride = stride; pic.m_strideC = cs;
        pic.m_picOrg[0] = (pixel*)w->refs[r] + (intptr_t)y * stride + x;
        pic.m_picOrg[1] = chroma ? (pixel*)w->refC[r][0] + (intptr_t)(y / 2) * cs + x / 2 : NULL;
        pic.m_picOrg[2] = chroma ? (pixel*)w->refC[r][1] + (intptr_t)(y / 2) * cs + x / 2 : NULL;
        const RefPu rpu = { 0, 0, g_rasterToZscan[(q.ry >> 2) * (MAX_CU_SIZE >> 2) + (q.rx >> 2)], q.pw, q.ph };
        const PredictionUnit& p = reinterpret_cast<const PredictionUnit&>(rpu);
        const MV mv(q.mvx, q.mvy);
        if (w->wp[r][0][0])
        {
            Predict::WeightValues wv[3];
            for (int plane = 0; plane < 3; plane++)
            {
                const int32_t* e = w->wp[r][plane];
                wv[plane].w = e[1]; wv[plane].offset = e[3] * (1 << (X265_DEPTH - 8));
                wv[plane].shift = e[2]; wv[plane].round = e[2] >= 1 ? 1 << (e[2] - 1) : 0;
            }
            pr->predInterLumaShort(p, *sy, pic, mv);
            if (chroma) pr->predInterChromaShort(p, *sy, pic, mv);
            pr->addWeightUni(p, *py, *sy, wv, true, chroma != 0);
        }
        else
        {
            pr->predInterLumaPixel(p, *py, pic, mv);
            if (chroma) pr->predInterChromaPixel(p, *py, pic, mv);
        }
        pic.m_cuOffsetY = pic.m_cuOffsetC = pic.m_buOffsetY = pic.m_buOffsetC = NULL;
        pic.m_picOrg[0] = pic.m_picOrg[1] = pic.m_picOrg[2] = NULL;
    }
    for (int i = 0; i < S; i++) memcpy(predY + i * S, py->m_buf[0] + i * py->m_size, sizeof(pixel) * S);
    for (int pl = 0; pl < 2 && chroma; pl++)
        for (int i = 0; i < S / 2; i++) memcpy(predC[pl] + i * (S / 2), py->m_buf[1 + pl] + i * py->m_csize, sizeof(pixel) * (S / 2));
}

/* x265ref_analyse_frame with the PART stage (orc_analyse_frame_part's twin) */
extern "C" int x265ref_analyse_frame_part(drv_frame* f, int stages, drv_part* pt)
{
    x265ref_analyse_frame(f, stages & 7);
    if (stages & 32) drv_run_part(f, pt);
    return 0;
}
