/* oracle/ref_shim_part_b.cpp -- TEST INFRASTRUCTURE ONLY (never linked into the product).
 * ref_shim_part.cpp (included whole) plus the PART_B stage (frame_part_b.h) on the REAL reference code: the bi try through
 * RefPredCtx (ref_shim.cpp: the real setSourcePU / bufSATD / bufChromaSATD, pixelavg_pp from the real table), the final
 * prediction through a real Predict::motionCompensation of a B slice with every PU at its z-order puAbsPartIdx, the zero
 * try's range test through the real MV::checkRange.  Built by Makefile.part_b with the reference objects into
 * oracle/_ref/libx265ref_part_b{8,10}.so. */
#include "ref_shim_part.cpp"

static int ref_part_bi_cost(const drv_frame* f, const drv_wref* w, int px, int py, int pw, int ph, int s0, int mx0, int my0, int s1,
                            int mx1, int my1, int chroma, int avgPP);
#define DRV_PART_BI_COST(f, w, px, py, pw, ph, s0, mx0, my0, s1, mx1, my1, c, a) ref_part_bi_cost(f, w, px, py, pw, ph, s0, mx0, my0, s1, mx1, my1, c, a)
struct drv_part_b_pu_s;
static void ref_part_b_pred(const drv_frame* f, const drv_wref* w, int x, int y, int S, int npu, const struct drv_part_b_pu_s* pu,
                            pixel* predY, pixel (*predC)[32 * 32], int chroma);
#define DRV_PART_B_PRED(f, w, x, y, S, npu, pu, pY, pC, c) ref_part_b_pred(f, w, x, y, S, npu, pu, pY, pC, c)
#include "frame_part_b.h"

/* the bi try's cost on the real classes: RefPredCtx (ref_shim.cpp), the real setSourcePU / bufSATD / bufChromaSATD with
 * pixelavg_pp from the real table when avgPP, else the real motionCompensation's addAvg; its setSourcePU takes subme 3 with
 * `chroma` and 2 without, so the real MotionEstimate decides bChromaSATD from the PU's size */
static int ref_part_bi_cost(const drv_frame* f, const drv_wref* w, int px, int py, int pw, int ph, int s0, int mx0, int my0, int s1,
                            int mx1, int my1, int chroma, int avgPP)
{
    static thread_local RefPredCtx* ctx = NULL;
    if (!ctx) ctx = new RefPredCtx();
    const intptr_t st = f->p.stride, cs = chroma ? f->cstride : st, off = py * st + px, coff = chroma ? (py / 2) * cs + px / 2 : off;
    /* without chroma the luma planes stand in for the chroma ones: run() copies the source's chroma, which is then unused */
    const pixel* fe[3] = { f->fenc + off, (chroma ? f->fencC[0] : f->fenc) + coff, (chroma ? f->fencC[1] : f->fenc) + coff };
    const pixel* r0[3] = { w->refs[s0] + off, (chroma ? w->refC[s0][0] : w->refs[s0]) + coff, (chroma ? w->refC[s0][1] : w->refs[s0]) + coff };
    const pixel* r1[3] = { w->refs[s1] + off, (chroma ? w->refC[s1][0] : w->refs[s1]) + coff, (chroma ? w->refC[s1][1] : w->refs[s1]) + coff };
    const int mv0[2] = { mx0, my0 }, mv1[2] = { mx1, my1 };
    return ctx->run(fe, r0, r1, st, cs, pw, ph, mv0, mv1, 1, chroma, avgPP);
}

/* Predict::motionCompensation's B-slice path (predict.cpp:119-240) for every PU of the partition into the CU's Yuv: a CUData
 * of a B slice without weighted bi-prediction whose m_refIdx / m_mv hold each PU's lists at its z-order puAbsPartIdx (index 0
 * of each list the PicYuv of that list's slot, placed as in ref_part_pred), in a picture large enough that clipMv leaves the
 * vectors alone (as RefPredCtx); an L0 or L1 PU takes predInterLumaPixel / predInterChromaPixel, a bi PU both lists'
 * predInterLumaShort / predInterChromaShort and Yuv::addAvg */
struct RefPartBCtx
{
    Predict pr; Yuv py; PicYuv pic[2];
    x265_param param;
    SPS* sps; PPS* pps; FrameData* fd; Slice* slice; CUData* cu;
    int8_t refIdx[2][MAX_NUM_PARTITIONS]; MV mv[2][MAX_NUM_PARTITIONS];
    intptr_t buY[MAX_NUM_PARTITIONS], buC[MAX_NUM_PARTITIONS], zero;
    RefPartBCtx()
    {
        pr.allocBuffers(X265_CSP_I420); py.create(MAX_CU_SIZE, X265_CSP_I420);
        memset(&param, 0, sizeof(param)); param.maxCUSize = 64;
        sps = (SPS*)calloc(1, sizeof(SPS)); pps = (PPS*)calloc(1, sizeof(PPS)); fd = (FrameData*)calloc(1, sizeof(FrameData));
        slice = (Slice*)calloc(1, sizeof(Slice)); cu = (CUData*)calloc(1, sizeof(CUData));
        sps->picWidthInLumaSamples = 1 << 15; sps->picHeightInLumaSamples = 1 << 15;
        fd->m_param = &param;
        slice->m_sps = sps; slice->m_pps = pps; slice->m_sliceType = B_SLICE;
        slice->m_numRefIdx[0] = slice->m_numRefIdx[1] = 1;
        slice->m_refReconPicList[0][0] = &pic[0]; slice->m_refReconPicList[1][0] = &pic[1];
        cu->m_slice = slice; cu->m_encData = fd;
        cu->m_cuPelX = 1 << 14; cu->m_cuPelY = 1 << 14;
        cu->m_refIdx[0] = refIdx[0]; cu->m_refIdx[1] = refIdx[1]; cu->m_mv[0] = mv[0]; cu->m_mv[1] = mv[1];
        zero = 0;
        for (int l = 0; l < 2; l++)
        {
            pic[l].m_cuOffsetY = &zero; pic[l].m_cuOffsetC = &zero; pic[l].m_buOffsetY = buY; pic[l].m_buOffsetC = buC;
            pic[l].m_stride = pic[l].m_strideC = 0;
        }
    }
    /* the per-partition offsets of the frame's strides, built as PicYuv::createOffsets builds them */
    void place(intptr_t stride, intptr_t cs)
    {
        if (pic[0].m_stride == stride && pic[0].m_strideC == cs) return;
        for (uint32_t i = 0; i < MAX_NUM_PARTITIONS; i++)
        {
            buY[i] = g_zscanToPelX[i] + (intptr_t)g_zscanToPelY[i] * stride;
            buC[i] = (g_zscanToPelX[i] >> 1) + (intptr_t)(g_zscanToPelY[i] >> 1) * cs;
        }
        for (int l = 0; l < 2; l++) { pic[l].m_stride = stride; pic[l].m_strideC = cs; }
    }
};

static void ref_part_b_pred(const drv_frame* f, const drv_wref* w, int x, int y, int S, int npu, const struct drv_part_b_pu_s* pu,
                            pixel* predY, pixel (*predC)[32 * 32], int chroma)
{
    static thread_local RefPartBCtx* ctx = NULL;
    if (!ctx) ctx = new RefPartBCtx();
    const intptr_t stride = f->p.stride, cs = f->cstride;
    ctx->place(stride, cs);
    for (int u = 0; u < npu; u++)
    {
        const drv_part_b_pu& q = pu[u];
        const uint32_t idx = g_rasterToZscan[(q.ry >> 2) * (MAX_CU_SIZE >> 2) + (q.rx >> 2)];
        for (int l = 0; l < 2; l++)
        {
            const int r = q.slot[l];
            PicYuv& pic = ctx->pic[l];
            pic.m_picOrg[0] = (pixel*)w->refs[r] + (intptr_t)y * stride + x;
            pic.m_picOrg[1] = chroma ? (pixel*)w->refC[r][0] + (intptr_t)(y / 2) * cs + x / 2 : NULL;
            pic.m_picOrg[2] = chroma ? (pixel*)w->refC[r][1] + (intptr_t)(y / 2) * cs + x / 2 : NULL;
            ctx->refIdx[l][idx] = (int8_t)((q.dir >> l) & 1 ? 0 : -1);
            ctx->mv[l][idx] = MV(q.mv[l][0], q.mv[l][1]);
        }
        const RefPu rpu = { 0, 0, idx, q.pw, q.ph };
        ctx->pr.motionCompensation(*ctx->cu, reinterpret_cast<const PredictionUnit&>(rpu), ctx->py, true, chroma != 0);
    }
    const Yuv& py = ctx->py;
    for (int i = 0; i < S; i++) memcpy(predY + i * S, py.m_buf[0] + i * py.m_size, sizeof(pixel) * S);
    for (int pl = 0; pl < 2 && chroma; pl++)
        for (int i = 0; i < S / 2; i++) memcpy(predC[pl] + i * (S / 2), py.m_buf[1 + pl] + i * py.m_csize, sizeof(pixel) * (S / 2));
}

/* x265ref_analyse_frame with the PART_B stage (orc_analyse_frame_part_b's twin) */
extern "C" int x265ref_analyse_frame_part_b(drv_frame* f, int stages, drv_part_b* pb)
{
    static bool scales = false;
    x265ref_analyse_frame(f, stages & 5);
    if (!scales) { MotionEstimate::initScales(); scales = true; }
    if (stages & 64) drv_run_part_b(f, pb);
    return 0;
}
