/* oracle/ref_shim_sao.cpp -- TEST INFRASTRUCTURE ONLY (never linked into the product).
 *
 * Frame-level SAO on the REAL Deblock, SAO and FrameFilter::ParallelFilter classes (pins oracle/oracle_sao.c).  Built by
 * Makefile.sao with the reference objects of Makefile.ref into oracle/_ref/libx265ref_sao{8,10}.so.
 *
 * The picture is set up as ref_shim_deblock.cpp sets it up (real CUData CTUs of a real FrameData from the per-4x4 map of
 * x265cu_deblock_frame, the CTU shapes of frameencoder.cpp:205-258), with a source PicYuv next to the reconstruction.  Both
 * are copied into padded planes of the same stride, as the encoder's are (calcSaoStatsCTU reads the source with the
 * reconstruction's stride, sao.cpp:740-808; generateLumaOffsets reads maxCUSize + 1 rows of a CTU, below the picture in the
 * last row).  One ParallelFilter per CTU row holds its SAO: create() for row 0, createFromRootNode() for the others
 * (FrameFilter::init, framefilter.cpp:195-225).
 *
 * run() restates ParallelFilter::processTasks (framefilter.cpp:439-562) and the last-row pass of FrameFilter::processRow
 * (:598-606), single-threaded, row after row.  Deblock::deblockCTU, ParallelFilter::copySaoAboveRef and
 * ParallelFilter::processSaoCTU are the reference's own.  In place of SAO::rdoSaoUnitCu(c - 2) it clears m_count /
 * m_offsetOrg, runs calcSaoStatsCTU for every plane, records the result, and writes the caller's parameters into
 * ctuParam[plane][addr] (the decision's output).  processPostCu only extends the borders into the margins, which nothing
 * here reads back, and is left out.  restoreOrigLosslessYuv is file-static in framefilter.cpp, so the transquant-bypass
 * restoration after each processSaoCTU is its copy, restated over the map's bypass units (flags bit 2): the one piece of
 * code this shim restates.
 */
#include "common.h"
#include "primitives.h"
#include "constants.h"
#include "picyuv.h"
#include "frame.h"
#include "framedata.h"
#include "deblock.h"
#include "slice.h"
#include "sao.h"
#include "framefilter.h"
#include <string.h>
#include <stdlib.h>
#include <vector>

using namespace X265_NS;

namespace X265_NS {
void setupCPrimitives(EncoderPrimitives &p);
void setupAliasPrimitives(EncoderPrimitives &p);
}

static void prim_init()
{
    static bool done = false;
    if (done) return;
    setupCPrimitives(primitives);
    setupAliasPrimitives(primitives);
    done = true;
}

/* reaches SAO's protected statistics the way its friend FrameFilter does */
struct SaoStats : public SAO
{
    static void collect(SAO& s, int addr, int planes, int32_t* out)
    {
        PerPlane& count = s.*(&SaoStats::m_count);
        PerPlane& org = s.*(&SaoStats::m_offsetOrg);
        memset(count, 0, sizeof(PerPlane));
        memset(org, 0, sizeof(PerPlane));
        for (int p = 0; p < planes; p++)
            s.calcSaoStatsCTU(addr, p);
        memcpy(out, count, sizeof(PerPlane));
        memcpy(out + sizeof(PerPlane) / sizeof(int32_t), org, sizeof(PerPlane));
    }
};

extern "C" {

struct ref_dbk_unit { int8_t qp; uint8_t flags, log2CuSize, partSize, tuDepth; int8_t refPic[2]; int16_t mv[2][2]; };
struct ref_sao_ctu { int8_t typeIdx; uint8_t bandPos; int8_t offset[4]; uint8_t pad[2]; };

enum { RUN_DEBLOCK = 1, RUN_STATS = 2, RUN_APPLY = 4 };
static const int PAD_X = 80, PAD_Y = 80;     /* > maxCUSize + 1 rows below the last CTU row */

/* planes: y / cb / cr (cb = cr = NULL: 4:0:0) in-out at pixel (0,0); f*: the source.  units: the x265cu_deblock_unit map (for
 * deblocking, and for the bypass restoration when `restore`).  dprm: x265cu_deblock_params as int32[6] (RUN_DEBLOCK).
 * params: [3][numCtus] records, merge: [3][numCtus] SaoMergeMode (NULL: none) -- what rdoSaoUnitCu would leave.
 * stats: [numCtus][2][3][5][32] (RUN_STATS). */
static int run(int mode, pixel* y, pixel* cb, pixel* cr, intptr_t stride, intptr_t cstride,
               const pixel* fy, const pixel* fcb, const pixel* fcr, intptr_t fstride, intptr_t fcstride,
               int width, int height, int ctuSize, const void* unitsv, const int32_t* dprm, int restore,
               const void* paramsv, const uint8_t* merge, int saoLuma, int saoChroma, int32_t* stats)
{
    prim_init();
    const ref_dbk_unit* units = (const ref_dbk_unit*)unitsv;
    const ref_sao_ctu* params = (const ref_sao_ctu*)paramsv;
    const int csp = cb ? X265_CSP_I420 : X265_CSP_I400, planes = cb ? 3 : 1;
    x265_param param;
    memset(&param, 0, sizeof(param));
    param.sourceWidth = width; param.sourceHeight = height; param.internalCsp = csp;
    param.maxCUSize = ctuSize; param.minCUSize = 8;
    param.maxLog2CUSize = g_log2Size[ctuSize];                                  /* encoder.cpp:4255-4258 */
    param.maxCUDepth = param.maxLog2CUSize - g_log2Size[param.minCUSize];
    param.unitSizeDepth = param.maxLog2CUSize - LOG2_UNIT_SIZE;
    param.num4x4Partitions = 1U << (param.unitSizeDepth << 1);
    param.bEnableLoopFilter = 1;
    param.bEnableSAO = 1;
    param.frameNumThreads = 1;

    SPS* sps = (SPS*)calloc(1, sizeof(SPS));                                   /* encoder.cpp:3355-3363 */
    sps->chromaFormatIdc = csp;
    sps->picWidthInLumaSamples = width; sps->picHeightInLumaSamples = height;
    sps->numCuInWidth = (width + ctuSize - 1) / ctuSize; sps->numCuInHeight = (height + ctuSize - 1) / ctuSize;
    sps->numCUsInFrame = sps->numCuInWidth * sps->numCuInHeight;
    sps->numPartitions = param.num4x4Partitions;
    sps->numPartInCUSize = 1 << param.unitSizeDepth;
    PPS* pps = (PPS*)calloc(1, sizeof(PPS));                                   /* encoder.cpp:3454-3468 */
    if (dprm)
    {
        pps->chromaQpOffset[0] = dprm[3]; pps->chromaQpOffset[1] = dprm[4];
        pps->bTransquantBypassEnabled = dprm[5] != 0;
        pps->deblockingFilterBetaOffsetDiv2 = dprm[1];
        pps->deblockingFilterTcOffsetDiv2 = dprm[2];
    }

    /* padded copies, one stride for source and reconstruction */
    const intptr_t ps = width + 2 * PAD_X, pcs = width / 2 + 2 * PAD_X;
    const size_t prow = height + 2 * PAD_Y, pcrow = height / 2 + 2 * PAD_Y;
    std::vector<pixel> buf[6];
    pixel* org[6];
    const pixel* in[6] = { y, cb, cr, fy, fcb, fcr };
    const intptr_t inStride[6] = { stride, cstride, cstride, fstride, fcstride, fcstride };
    for (int k = 0; k < 6; k++)
    {
        const int p = k % 3;
        if (p && !cb) { org[k] = NULL; continue; }
        const intptr_t s = p ? pcs : ps;
        buf[k].assign((size_t)s * (p ? pcrow : prow), 0);
        org[k] = &buf[k][(size_t)PAD_Y * s + PAD_X];
        const int w = p ? width / 2 : width, h = p ? height / 2 : height;
        if (in[k])
            for (int j = 0; j < h; j++)
                memcpy(org[k] + j * s, in[k] + j * inStride[k], w * sizeof(pixel));
    }

    PicYuv recon, fenc;                                                         /* picyuv.cpp:72-198 */
    PicYuv* pics[2] = { &recon, &fenc };
    for (int i = 0; i < 2; i++)
    {
        PicYuv& pic = *pics[i];
        pic.m_param = &param; pic.m_picWidth = width; pic.m_picHeight = height; pic.m_picCsp = csp;
        pic.m_hChromaShift = pic.m_vChromaShift = cb ? 1 : 0;
        pic.m_stride = ps; pic.m_strideC = cb ? pcs : 0;
        pic.m_lumaMarginX = PAD_X; pic.m_lumaMarginY = PAD_Y;
        pic.m_chromaMarginX = cb ? PAD_X : 0; pic.m_chromaMarginY = cb ? PAD_Y : 0;
        pic.m_picOrg[0] = org[3 * i]; pic.m_picOrg[1] = org[3 * i + 1]; pic.m_picOrg[2] = org[3 * i + 2];
        if (!pic.createOffsets(*sps)) return -1;
    }

    Frame frame;
    Frame* pictures = new Frame[MAX_NUM_REF];                                   /* one per picture id (ref_shim_deblock.cpp) */
    FrameData* fd = new FrameData();
    if (!fd->create(param, *sps, csp)) return -1;
    fd->m_reconPic = &recon;
    frame.m_encData = fd; frame.m_param = &param; frame.m_reconPic = &recon; frame.m_fencPic = &fenc;
    Slice* slice = fd->m_slice;
    slice->m_sps = sps; slice->m_pps = pps; slice->m_param = &param;
    slice->m_sliceType = dprm ? (SliceType)dprm[0] : B_SLICE;
    for (int l = 0; l < 2; l++)
        for (int i = 0; i < MAX_NUM_REF; i++) slice->m_refFrameList[l][i] = &pictures[i];

    const uint32_t cols = sps->numCuInWidth, rows = sps->numCuInHeight, upr = width >> 2;
    const int maxLog2 = param.maxLog2CUSize;
    for (uint32_t addr = 0; addr < sps->numCUsInFrame; addr++)
    {
        CUData* ctu = fd->getPicCTU(addr);
        ctu->initCTU(frame, addr, 0, addr < cols, addr >= cols * (rows - 1), addr == sps->numCUsInFrame - 1);
        const int cx = (addr % cols) * ctuSize, cyy = (addr / cols) * ctuSize;
        if (!units) continue;
        for (int uy = 0; uy < ctuSize / 4 && cyy + 4 * uy < height; uy++)
            for (int ux = 0; ux < ctuSize / 4 && cx + 4 * ux < width; ux++)
            {
                const ref_dbk_unit& u = units[(size_t)((cyy >> 2) + uy) * upr + (cx >> 2) + ux];
                const uint32_t z = g_rasterToZscan[uy * RASTER_SIZE + ux];
                ctu->m_qp[z] = u.qp;
                ctu->m_predMode[z] = (u.flags & 1) ? MODE_INTRA : MODE_INTER;
                ctu->m_cbf[0][z] = (uint8_t)(((u.flags >> 1) & 1) << u.tuDepth);
                ctu->m_tqBypass[z] = (u.flags >> 2) & 1;
                ctu->m_log2CUSize[z] = u.log2CuSize;
                ctu->m_cuDepth[z] = (uint8_t)(maxLog2 - u.log2CuSize);
                ctu->m_partSize[z] = u.partSize;
                ctu->m_tuDepth[z] = u.tuDepth;
                for (int l = 0; l < 2; l++)
                {
                    ctu->m_refIdx[l][z] = u.refPic[l] < 0 ? -1 : u.refPic[l];
                    ctu->m_mv[l][z] = MV(u.mv[l][0], u.mv[l][1]);
                }
            }
    }
    CUGeom* geoms = new CUGeom[4 * CUGeom::MAX_GEOMS];
    const int wRem = width & (ctuSize - 1), hRem = height & (ctuSize - 1);
    for (int g = 0; g < 4; g++)
        CUData::calcCTUGeoms((g & 1) && wRem ? wRem : ctuSize, (g & 2) && hRem ? hRem : ctuSize, ctuSize, 8, geoms + g * CUGeom::MAX_GEOMS);
    auto geomOf = [&](uint32_t addr) -> const CUGeom& {
        const int g = ((addr % cols) == cols - 1 ? 1 : 0) | ((addr / cols) == rows - 1 ? 2 : 0);
        return geoms[g * CUGeom::MAX_GEOMS];
    };

    /* FrameFilter::init / start (framefilter.cpp:176-251) for the fields processSaoCTU and copySaoAboveRef read */
    FrameFilter ff;
    ff.m_param = &param; ff.m_frame = &frame; ff.m_useSao = 1; ff.m_numRows = rows; ff.m_numCols = cols;
    ff.m_hChromaShift = ff.m_vChromaShift = cb ? 1 : 0;
    FrameFilter::ParallelFilter* pf = new FrameFilter::ParallelFilter[rows];
    ff.m_parallelFilter = pf;
    for (uint32_t r = 0; r < rows; r++)
    {
        if (!pf[r].m_sao.create(&param, r == 0 ? 1 : 0)) return -1;
        if (r) pf[r].m_sao.createFromRootNode(&pf[0].m_sao);
        pf[r].m_sao.m_frame = &frame;                                           /* SAO::startSlice (sao.cpp:229) */
        pf[r].m_row = r; pf[r].m_rowAddr = r * cols; pf[r].m_frameFilter = &ff; pf[r].m_encData = fd;
        pf[r].m_prevRow = r ? &pf[r - 1] : NULL;
    }
    SAOParam* saoParam = new SAOParam;
    pf[0].m_sao.allocSaoParam(saoParam);
    saoParam->bSaoFlag[0] = saoLuma != 0;
    saoParam->bSaoFlag[1] = saoChroma != 0;
    const int n = sps->numCUsInFrame;

    /* the transquant-bypass restoration of one CTU after its SAO (restoreOrigLosslessYuv over the map's bypass units) */
    auto restoreCtu = [&](uint32_t addr) {
        if (!restore || !units) return;
        const int cx = (addr % cols) * ctuSize, cyy = (addr / cols) * ctuSize;
        for (int uy = cyy / 4; uy < (cyy + ctuSize) / 4 && uy < height / 4; uy++)
            for (int ux = cx / 4; ux < (cx + ctuSize) / 4 && ux < (int)upr; ux++)
                if (units[(size_t)uy * upr + ux].flags & 4)
                {
                    primitives.cu[BLOCK_4x4].copy_pp(org[0] + 4 * uy * ps + 4 * ux, ps, org[3] + 4 * uy * ps + 4 * ux, ps);
                    if (cb)
                        for (int k = 1; k < 3; k++)
                            for (int j = 0; j < 2; j++)
                                memcpy(org[k] + (2 * uy + j) * pcs + 2 * ux, org[3 + k] + (2 * uy + j) * pcs + 2 * ux, 2 * sizeof(pixel));
                }
    };
    /* in place of SAO::rdoSaoUnitCu(addr): the statistics, then the decision's output */
    auto decide = [&](FrameFilter::ParallelFilter& row, uint32_t addr) {
        if (mode & RUN_STATS)
            SaoStats::collect(row.m_sao, addr, planes, stats + (size_t)addr * 2 * 3 * 5 * 32);
        for (int p = 0; p < planes; p++)
        {
            SaoCtuParam& d = saoParam->ctuParam[p][addr];
            const ref_sao_ctu& s = params[(size_t)p * n + addr];
            d.mergeMode = merge ? (SaoMergeMode)merge[(size_t)p * n + addr] : SAO_MERGE_NONE;
            d.typeIdx = s.typeIdx; d.bandPos = s.bandPos;
            for (int i = 0; i < SAO_NUM_OFFSET; i++) d.offset[i] = s.offset[i];
        }
    };
    auto sao = [&](FrameFilter::ParallelFilter& row, int col) {
        if (!(mode & RUN_APPLY)) return;
        const bool bypass = pps->bTransquantBypassEnabled;     /* processSaoCTU's own restoration needs FrameEncoder's geoms */
        pps->bTransquantBypassEnabled = false;
        row.processSaoCTU(saoParam, col);
        pps->bTransquantBypassEnabled = bypass;
        restoreCtu(row.m_rowAddr + col);
    };
    auto deblock = [&](uint32_t addr, int dir) {
        if (mode & RUN_DEBLOCK) Deblock::deblockCTU(fd->getPicCTU(addr), geomOf(addr), dir);
    };

    for (uint32_t r = 0; r < rows; r++)
    {
        FrameFilter::ParallelFilter& row = pf[r];
        const bool first = r == 0;
        /* processTasks, colStart 0 .. colEnd numCols (framefilter.cpp:457-505) */
        for (uint32_t col = 0; col < cols; col++)
        {
            const uint32_t cuAddr = row.m_rowAddr + col;
            deblock(cuAddr, Deblock::EDGE_VER);
            if (col >= 1)
            {
                deblock(cuAddr - 1, Deblock::EDGE_HOR);
                row.copySaoAboveRef(fd->getPicCTU(cuAddr - 1), &recon, cuAddr - 1, col - 1);
                if (col >= 2)
                    decide(row, cuAddr - 2);
                if (!first && col >= 3)
                    sao(*row.m_prevRow, col - 3);
            }
        }
        /* the numCols tail (:507-561) */
        const uint32_t cuAddr = row.m_rowAddr + cols - 1;
        deblock(cuAddr, Deblock::EDGE_HOR);
        row.copySaoAboveRef(fd->getPicCTU(cuAddr), &recon, cuAddr, cols - 1);
        if (cols >= 2)
            decide(row, cuAddr - 1);
        if (cols >= 1)
            decide(row, cuAddr);
        if (!first && cols >= 3)
            sao(*row.m_prevRow, cols - 3);
        if (!first && cols >= 2)
            sao(*row.m_prevRow, cols - 2);
        if (!first && cols >= 1)
            sao(*row.m_prevRow, cols - 1);
        /* the last row (FrameFilter::processRow :598-606) */
        if (r == rows - 1)
            for (uint32_t col = 0; col < cols; col++)
                sao(row, col);
    }

    for (int k = 0; k < 3; k++)
    {
        pixel* out[3] = { y, cb, cr };
        if (!org[k]) continue;
        const intptr_t s = k ? pcs : ps;
        const int w = k ? width / 2 : width, h = k ? height / 2 : height;
        for (int j = 0; j < h; j++)
            memcpy(out[k] + j * (k ? cstride : stride), org[k] + j * s, w * sizeof(pixel));
    }

    for (uint32_t r = 0; r < rows; r++)
        pf[r].m_sao.destroy(r == 0 ? 1 : 0);
    ff.m_parallelFilter = NULL;
    delete[] pf;
    delete saoParam;
    delete[] geoms;
    fd->m_reconPic = NULL;
    fd->destroy();
    delete fd;
    delete[] pictures;
    for (int i = 0; i < 2; i++)
    {
        PicYuv& pic = *pics[i];
        X265_FREE(pic.m_cuOffsetY); X265_FREE(pic.m_cuOffsetC); X265_FREE(pic.m_buOffsetY); X265_FREE(pic.m_buOffsetC);
        pic.m_cuOffsetY = pic.m_cuOffsetC = NULL; pic.m_buOffsetY = pic.m_buOffsetC = NULL;
        pic.m_picOrg[0] = pic.m_picOrg[1] = pic.m_picOrg[2] = NULL;
    }
    free(sps); free(pps);
    return 0;
}

/* deblocking, statistics and apply interleaved in FrameFilter's order: the decomposition pin */
int x265ref_sao_frame(pixel* y, pixel* cb, pixel* cr, intptr_t stride, intptr_t cstride,
                      const pixel* fy, const pixel* fcb, const pixel* fcr, intptr_t fstride, intptr_t fcstride,
                      int width, int height, int ctuSize, const void* units, const int32_t* dprm,
                      const void* params, const uint8_t* merge, int saoLuma, int saoChroma, int32_t* stats)
{
    return run(RUN_DEBLOCK | RUN_STATS | RUN_APPLY, y, cb, cr, stride, cstride, fy, fcb, fcr, fstride, fcstride, width, height,
               ctuSize, units, dprm, dprm[5], params, merge, saoLuma, saoChroma, stats);
}

/* the statistics alone, of a picture taken as deblocked */
int x265ref_sao_stats_frame(const pixel* y, const pixel* cb, const pixel* cr, intptr_t stride, intptr_t cstride,
                            const pixel* fy, const pixel* fcb, const pixel* fcr, intptr_t fstride, intptr_t fcstride,
                            int width, int height, int ctuSize, int32_t* stats)
{
    const int n = ((width + ctuSize - 1) / ctuSize) * ((height + ctuSize - 1) / ctuSize);
    std::vector<ref_sao_ctu> off(3 * (size_t)n);
    for (auto& p : off) { memset(&p, 0, sizeof(p)); p.typeIdx = -1; }
    const int w = width, h = height;
    std::vector<pixel> copy[3];                            /* run() writes the planes back: keep the caller's const */
    pixel* pl[3] = { NULL, NULL, NULL };
    const pixel* src[3] = { y, cb, cr };
    for (int k = 0; k < (cb ? 3 : 1); k++)
    {
        const int pw = k ? w / 2 : w, ph = k ? h / 2 : h;
        copy[k].resize((size_t)pw * ph);
        for (int j = 0; j < ph; j++)
            memcpy(&copy[k][(size_t)j * pw], src[k] + j * (k ? cstride : stride), pw * sizeof(pixel));
        pl[k] = copy[k].data();
    }
    return run(RUN_STATS, pl[0], pl[1], pl[2], w, w / 2, fy, fcb, fcr, fstride, fcstride, width, height, ctuSize, NULL, NULL, 0,
               off.data(), NULL, 0, 0, stats);
}

/* the apply alone, on a picture taken as deblocked; units: NULL, or the map whose bypass units are restored */
int x265ref_sao_apply_frame(pixel* y, pixel* cb, pixel* cr, intptr_t stride, intptr_t cstride, int width, int height, int ctuSize,
                            const void* params, const uint8_t* merge, int saoLuma, int saoChroma, const void* units,
                            const pixel* fy, const pixel* fcb, const pixel* fcr, intptr_t fstride, intptr_t fcstride)
{
    return run(RUN_APPLY, y, cb, cr, stride, cstride, fy, fcb, fcr, fstride, fcstride, width, height, ctuSize, units, NULL,
               units != NULL, params, merge, saoLuma, saoChroma, NULL);
}

} // extern "C"
