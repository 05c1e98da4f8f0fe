/* oracle/ref_shim_aq.cpp -- TEST INFRASTRUCTURE ONLY (never linked into the product).
 *
 * The REAL LookaheadTLD::calcAdaptiveQuantFrame (encoder/slicetype.cpp:444-694) on a real Frame (pins oracle/oracle_aq.c).
 * Built by Makefile.aq with the reference objects of Makefile.ref into oracle/_ref/libx265ref_aq{8,10}.so.
 *
 * The Frame is created as the encoder creates it (Frame::create with or without quantOffsets, frame.cpp:141-146), for
 * 4:2:0 or 4:0:0; the caller's planes are copied into its PicYuv and the borders replicated (extendPicBorder), as
 * copyFromPicture and the lookahead leave them.  Before the call every qpAqOffset / qpCuTreeOffset entry holds
 * -1000 - i, every invQscaleFactor 7 + 3 i and every blockVariance 0x5a5a0000 + i, so the results also pin which words the
 * reference leaves alone. */
#include "common.h"
#include "primitives.h"
#include "frame.h"
#include "picyuv.h"
#include "lowres.h"
#include "slicetype.h"
#include <string.h>

using namespace X265_NS;

namespace X265_NS {
void setupCPrimitives(EncoderPrimitives &p);
void setupAliasPrimitives(EncoderPrimitives &p);
void extendPicBorder(pixel* recon, intptr_t stride, int width, int height, int marginX, int marginY);
}

/* the parameter record of oracle/oracle_aq.c (x265cu_aq_params) */
struct AqParams
{
    int32_t aqMode, qgSize, weightp, variance, hevcAq, hdr10Opt, aqMotion, reserved;
    double aqStrength;
    const float* quantOffsets;
};

static void prim_init()
{
    static bool done = false;
    if (done) return;
    setupCPrimitives(primitives);
    setupAliasPrimitives(primitives);
    done = true;
}

extern "C" {
/* y: W x H, cb / cr: (W / 2) x (H / 2) (NULL: 4:0:0), contiguous rows.  Outputs, blockCount long (4 * w8 * h8 at qgSize 8,
 * else w8 * h8; left untouched where the Lowres array is not allocated, i.e. aqMode 0 / without variance):
 * qpAqOffset, qpCuTreeOffset, invQscaleFactor, blockVariance; invq8 (w8 * h8); wp[6] = wp_sum[3], wp_ssd[3];
 * frameVariance. */
void x265ref_aq(const pixel* y, const pixel* cb, const pixel* cr, int W, int H, const AqParams* a, double* qpAqOffset,
                double* qpCuTreeOffset, int32_t* invq, int32_t* invq8, uint32_t* blockVariance, uint64_t* wp, double* frameVariance)
{
    prim_init();
    x265_param* p = x265_param_alloc();
    x265_param_default(p);
    p->sourceWidth = W; p->sourceHeight = H; p->internalCsp = cb ? X265_CSP_I420 : X265_CSP_I400;
    p->rc.aqMode = a->aqMode; p->rc.aqStrength = a->aqStrength; p->rc.qgSize = a->qgSize; p->rc.hevcAq = 0;
    p->bEnableWeightedPred = a->weightp; p->bEnableWeightedBiPred = 0; p->bEnableFades = a->variance; p->bDynamicRefine = 0;
    p->bAQMotion = 0; p->bHDR10Opt = 0; p->rc.cuTree = 0; p->rc.bStatRead = 0; p->maxCUSize = 64;
    Frame* fr = new Frame();
    fr->m_param = p;
    float dummy = 0;
    fr->create(p, a->quantOffsets ? &dummy : NULL);
    Lowres& lr = fr->m_lowres;
    const int w8 = lr.maxBlocksInRow, h8 = lr.maxBlocksInCol;
    const int blockCount = a->qgSize == 8 ? 4 * w8 * h8 : w8 * h8;
    if (a->quantOffsets)
        memcpy(fr->m_quantOffsets, a->quantOffsets, blockCount * sizeof(float));
    PicYuv* pic = fr->m_fencPic;
    for (int r = 0; r < H; r++)
        memcpy(pic->m_picOrg[0] + (intptr_t)r * pic->m_stride, y + (intptr_t)r * W, W * sizeof(pixel));
    extendPicBorder(pic->m_picOrg[0], pic->m_stride, W, H, pic->m_lumaMarginX, pic->m_lumaMarginY);
    if (cb)
    {
        for (int c = 1; c < 3; c++)
        {
            const pixel* src = c == 1 ? cb : cr;
            for (int r = 0; r < H / 2; r++)
                memcpy(pic->m_picOrg[c] + (intptr_t)r * pic->m_strideC, src + (intptr_t)r * (W / 2), (W / 2) * sizeof(pixel));
            extendPicBorder(pic->m_picOrg[c], pic->m_strideC, W / 2, H / 2, pic->m_chromaMarginX, pic->m_chromaMarginY);
        }
    }
    for (int i = 0; i < blockCount; i++)
    {
        if (lr.qpAqOffset) { lr.qpAqOffset[i] = -1000.0 - i; lr.qpCuTreeOffset[i] = -1000.0 - i; lr.invQscaleFactor[i] = 7 + 3 * i; }
        if (lr.blockVariance) lr.blockVariance[i] = 0x5a5a0000u + i;
    }
    LookaheadTLD tld;
    tld.init(w8, h8, w8 * h8);
    tld.calcAdaptiveQuantFrame(fr, p);
    if (lr.qpAqOffset)
    {
        memcpy(qpAqOffset, lr.qpAqOffset, blockCount * sizeof(double));
        memcpy(qpCuTreeOffset, lr.qpCuTreeOffset, blockCount * sizeof(double));
        memcpy(invq, lr.invQscaleFactor, blockCount * sizeof(int32_t));
        if (a->qgSize == 8) memcpy(invq8, lr.invQscaleFactor8x8, w8 * h8 * sizeof(int32_t));
    }
    if (lr.blockVariance)
    {
        memcpy(blockVariance, lr.blockVariance, blockCount * sizeof(uint32_t));
        *frameVariance = lr.frameVariance;
    }
    for (int i = 0; i < 3; i++) { wp[i] = lr.wp_sum[i]; wp[3 + i] = lr.wp_ssd[i]; }
    fr->destroy();
    delete fr;
    x265_param_free(p);
}
}
