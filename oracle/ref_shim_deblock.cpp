/* oracle/ref_shim_deblock.cpp -- TEST INFRASTRUCTURE ONLY (never linked into the product).
 *
 * Frame-level deblocking on the REAL Deblock class (pins oracle/oracle_deblock.c).  Built by Makefile.deblock with the
 * reference objects of Makefile.ref into oracle/_ref/libx265ref_deblock{8,10}.so.  The per-4x4 decision map of
 * x265cu_deblock_frame (include/x265_b200.h, raster order) is written into real CUData CTUs of a real FrameData, built as
 * the encoder builds them: CUData::calcCTUGeoms per CTU shape (frameencoder.cpp:205-258), initCTU, the PPS fields of
 * encoder.cpp:3454-3468, and m_refFrameList[l][id] = one shared dummy Frame per picture id, so that equal ids compare as
 * the reference compares Frame pointers.  Deblock::deblockCTU then runs in FrameFilter's single-thread order
 * (framefilter.cpp:457-516): per CTU row, EDGE_VER of CTU c then EDGE_HOR of CTU c - 1, then EDGE_HOR of the last column.
 * Planes are the caller's, at pixel (0,0) (deblocking never reads outside the picture); cb = cr = NULL: 4:0:0.
 * params as x265cu_deblock_params: {sliceType, betaOffsetDiv2, tcOffsetDiv2, cbQpOffset, crQpOffset, transquantBypass}.
 * It contains no algorithm of its own: the filtering is the reference's.
 */
#include "common.h"
#include "primitives.h"
#include "constants.h"
#include "picyuv.h"
#include "frame.h"
#include "framedata.h"
#include "deblock.h"
#include "slice.h"
#include <string.h>
#include <stdlib.h>

using namespace X265_NS;

namespace X265_NS {
void setupCPrimitives(EncoderPrimitives &p);
void setupAliasPrimitives(EncoderPrimitives &p);
}

/* Deblock's edge filters go through the global table (primitives.pelFilterLumaStrong / pelFilterChroma): the C one */
static void deblock_init()
{
    static bool done = false;
    if (done) return;
    setupCPrimitives(primitives);
    setupAliasPrimitives(primitives);
    done = true;
}

extern "C" {

struct ref_dbk_unit { int8_t qp; uint8_t flags, log2CuSize, partSize, tuDepth; int8_t refPic[2]; int16_t mv[2][2]; };

int x265ref_deblock_frame(pixel* luma, intptr_t stride, pixel* cb, pixel* cr, intptr_t cstride, int width, int height, int ctuSize,
                          const void* unitsv, const int32_t* prm)
{
    deblock_init();
    const ref_dbk_unit* units = (const ref_dbk_unit*)unitsv;
    const int csp = cb ? X265_CSP_I420 : X265_CSP_I400;
    x265_param param;
    memset(&param, 0, sizeof(param));
    param.sourceWidth = width; param.sourceHeight = height; param.internalCsp = csp;
    param.maxCUSize = ctuSize; param.minCUSize = 8;
    param.maxLog2CUSize = g_log2Size[ctuSize];                                  /* encoder.cpp:4255-4258 */
    param.maxCUDepth = param.maxLog2CUSize - g_log2Size[param.minCUSize];
    param.unitSizeDepth = param.maxLog2CUSize - LOG2_UNIT_SIZE;
    param.num4x4Partitions = 1U << (param.unitSizeDepth << 1);
    param.bEnableLoopFilter = 1;

    SPS* sps = (SPS*)calloc(1, sizeof(SPS));                                   /* encoder.cpp:3355-3363 */
    sps->chromaFormatIdc = csp;
    sps->picWidthInLumaSamples = width; sps->picHeightInLumaSamples = height;
    sps->numCuInWidth = (width + ctuSize - 1) / ctuSize; sps->numCuInHeight = (height + ctuSize - 1) / ctuSize;
    sps->numCUsInFrame = sps->numCuInWidth * sps->numCuInHeight;
    sps->numPartitions = param.num4x4Partitions;
    sps->numPartInCUSize = 1 << param.unitSizeDepth;
    PPS* pps = (PPS*)calloc(1, sizeof(PPS));                                   /* encoder.cpp:3454-3468 */
    pps->chromaQpOffset[0] = prm[3]; pps->chromaQpOffset[1] = prm[4];
    pps->bTransquantBypassEnabled = prm[5] != 0;
    pps->deblockingFilterBetaOffsetDiv2 = prm[1];
    pps->deblockingFilterTcOffsetDiv2 = prm[2];

    PicYuv recon;                                                               /* the caller's planes, picyuv.cpp:72-198 */
    recon.m_param = &param; recon.m_picWidth = width; recon.m_picHeight = height; recon.m_picCsp = csp;
    recon.m_hChromaShift = recon.m_vChromaShift = cb ? 1 : 0;
    recon.m_stride = stride; recon.m_strideC = cb ? cstride : 0;
    recon.m_picOrg[0] = luma; recon.m_picOrg[1] = cb; recon.m_picOrg[2] = cr;
    if (!recon.createOffsets(*sps)) return -1;

    Frame frame;
    Frame* pictures = new Frame[MAX_NUM_REF];                                   /* one per picture id */
    FrameData* fd = new FrameData();
    if (!fd->create(param, *sps, csp)) return -1;
    fd->m_reconPic = &recon;
    frame.m_encData = fd; frame.m_param = &param; frame.m_reconPic = &recon;
    Slice* slice = fd->m_slice;
    slice->m_sps = sps; slice->m_pps = pps; slice->m_param = &param;
    slice->m_sliceType = (SliceType)prm[0];
    for (int l = 0; l < 2; l++)
        for (int i = 0; i < MAX_NUM_REF; i++) slice->m_refFrameList[l][i] = &pictures[i];

    const uint32_t cols = sps->numCuInWidth, rows = sps->numCuInHeight, upr = width >> 2;
    const int maxLog2 = param.maxLog2CUSize;
    for (uint32_t addr = 0; addr < sps->numCUsInFrame; addr++)
    {
        CUData* ctu = fd->getPicCTU(addr);
        ctu->initCTU(frame, addr, 0, addr < cols, addr >= cols * (rows - 1), addr == sps->numCUsInFrame - 1);
        const int cx = (addr % cols) * ctuSize, cy = (addr / cols) * ctuSize;
        for (int uy = 0; uy < ctuSize / 4 && cy + 4 * uy < height; uy++)
            for (int ux = 0; ux < ctuSize / 4 && cx + 4 * ux < width; ux++)
            {
                const ref_dbk_unit& u = units[(size_t)((cy >> 2) + uy) * upr + (cx >> 2) + ux];
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

    /* CTU shapes: body, right, bottom, corner (frameencoder.cpp:205-258) */
    CUGeom* geoms = new CUGeom[4 * CUGeom::MAX_GEOMS];
    const int wRem = width & (ctuSize - 1), hRem = height & (ctuSize - 1);
    for (int g = 0; g < 4; g++)
        CUData::calcCTUGeoms((g & 1) && wRem ? wRem : ctuSize, (g & 2) && hRem ? hRem : ctuSize, ctuSize, 8, geoms + g * CUGeom::MAX_GEOMS);
    auto geomOf = [&](uint32_t addr) -> const CUGeom& {
        const int g = ((addr % cols) == cols - 1 ? 1 : 0) | ((addr / cols) == rows - 1 ? 2 : 0);
        return geoms[g * CUGeom::MAX_GEOMS];
    };
    for (uint32_t r = 0; r < rows; r++)
    {
        for (uint32_t c = 0; c < cols; c++)
        {
            Deblock::deblockCTU(fd->getPicCTU(r * cols + c), geomOf(r * cols + c), Deblock::EDGE_VER);
            if (c >= 1)
                Deblock::deblockCTU(fd->getPicCTU(r * cols + c - 1), geomOf(r * cols + c - 1), Deblock::EDGE_HOR);
        }
        Deblock::deblockCTU(fd->getPicCTU(r * cols + cols - 1), geomOf(r * cols + cols - 1), Deblock::EDGE_HOR);
    }

    delete[] geoms;
    fd->m_reconPic = NULL;
    fd->destroy();
    delete fd;
    delete[] pictures;
    X265_FREE(recon.m_cuOffsetY); X265_FREE(recon.m_cuOffsetC); X265_FREE(recon.m_buOffsetY); X265_FREE(recon.m_buOffsetC);
    recon.m_cuOffsetY = recon.m_cuOffsetC = NULL; recon.m_buOffsetY = recon.m_buOffsetC = NULL;
    recon.m_picOrg[0] = recon.m_picOrg[1] = recon.m_picOrg[2] = NULL;
    free(sps); free(pps);
    return 0;
}

} // extern "C"
