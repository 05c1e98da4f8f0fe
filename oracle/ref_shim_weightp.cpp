/* oracle/ref_shim_weightp.cpp -- TEST INFRASTRUCTURE ONLY (never linked into the product).
 *
 * The REAL weightAnalyse (encoder/weightPrediction.cpp:222-539) on real Frames and a real Slice (pins
 * oracle/oracle_weightp.c).  Built by Makefile.weightp with the reference objects of Makefile.ref into
 * oracle/_ref/libx265ref_weightp{8,10}.so.
 *
 * Frame 0 is the picture being encoded, frame 1 m_refFrameList[0][0] and frame 2 m_refFrameList[1][0] (B slices).  Each is
 * created as the encoder creates it (Frame::create), for 4:2:0 or 4:0:0; the caller's planes are copied into its PicYuv
 * and the borders replicated (extendPicBorder), Lowres::init builds the lowres planes and the real lowresIntraEstimate
 * fills frame 0's intraCost.  The picture statistics wp_sum / wp_ssd are the caller's (calcAdaptiveQuantFrame accumulates
 * them; they are inputs of the analysis, as in x265ref_la_weights), and so are the motion fields: per list either NULL
 * (the field keeps Lowres::init's 0x7FFF "not searched" marker) or lowresMvs[list][diffPoc] as int32 pairs.
 *
 * x265ref_weightp_costs pins the candidate costs themselves: weightPrediction.cpp is compiled into this file (Makefile.weightp
 * links the reference objects without weightPrediction.o), so its file-local mcLuma, mcChroma and weightCost are called on
 * the same Frames, with the set-up weightAnalyse gives them (:228-246, 291-403). */
#include "weightPrediction.cpp"
#include "common.h"
#include "primitives.h"
#include "frame.h"
#include "picyuv.h"
#include "lowres.h"
#include "slice.h"
#include "slicetype.h"
#include <string.h>

using namespace X265_NS;

namespace X265_NS {
void setupCPrimitives(EncoderPrimitives &p);
void setupAliasPrimitives(EncoderPrimitives &p);
void extendPicBorder(pixel* recon, intptr_t stride, int width, int height, int marginX, int marginY);
}

/* the parameter record of oracle/oracle_weightp.c (x265cu_wp_params) */
struct WpParams
{
    int32_t sliceType, numRefIdx[2], bframes, width, height, csp;
};

static void prim_init()
{
    static bool done = false;
    if (done) return;
    setupCPrimitives(primitives);
    setupAliasPrimitives(primitives);
    done = true;
}

struct Setup
{
    x265_param* p;
    Frame* fr[3];
    int nfr, w8, h8;
    Slice slice;
};

static void setup(Setup& su, const pixel* const* y, const pixel* const* cb, const pixel* const* cr, const WpParams* a,
                  const int32_t* poc, const uint64_t* wp, const int32_t* const* mvs)
{
    prim_init();
    const int W = a->width, H = a->height;
    x265_param* p = x265_param_alloc();
    x265_param_default(p);
    p->sourceWidth = W; p->sourceHeight = H; p->internalCsp = a->csp ? X265_CSP_I420 : X265_CSP_I400;
    p->bframes = a->bframes; p->rc.aqMode = 0; p->rc.hevcAq = 0; p->bAQMotion = 0; p->rc.cuTree = 0; p->bEnableHME = 0;
    p->rc.qgSize = 32; p->maxCUSize = 64; p->logLevel = X265_LOG_NONE;
    su.p = p;
    su.nfr = a->sliceType == P_SLICE ? 2 : 3;
    su.fr[0] = su.fr[1] = su.fr[2] = NULL;
    for (int f = 0; f < su.nfr; f++)
    {
        Frame* fr = su.fr[f] = new Frame();
        fr->m_param = p;
        fr->create(p, NULL);
        fr->m_poc = poc[f];
        PicYuv* pic = fr->m_fencPic;
        for (int r = 0; r < H; r++)
            memcpy(pic->m_picOrg[0] + (intptr_t)r * pic->m_stride, y[f] + (intptr_t)r * W, W * sizeof(pixel));
        extendPicBorder(pic->m_picOrg[0], pic->m_stride, W, H, pic->m_lumaMarginX, pic->m_lumaMarginY);
        if (a->csp)
        {
            for (int c = 1; c < 3; c++)
            {
                const pixel* src = c == 1 ? cb[f] : cr[f];
                for (int r = 0; r < H / 2; r++)
                    memcpy(pic->m_picOrg[c] + (intptr_t)r * pic->m_strideC, src + (intptr_t)r * (W / 2), (W / 2) * sizeof(pixel));
                extendPicBorder(pic->m_picOrg[c], pic->m_strideC, W / 2, H / 2, pic->m_chromaMarginX, pic->m_chromaMarginY);
            }
        }
        fr->m_lowres.init(pic, poc[f]);
        for (int i = 0; i < 3; i++) { fr->m_lowres.wp_sum[i] = wp[6 * f + i]; fr->m_lowres.wp_ssd[i] = wp[6 * f + 3 + i]; }
    }
    Lowres& lr = su.fr[0]->m_lowres;
    su.w8 = lr.maxBlocksInRow; su.h8 = lr.maxBlocksInCol;
    LookaheadTLD tld;
    tld.init(su.w8, su.h8, su.w8 * su.h8);
    tld.lowresIntraEstimate(lr, p->rc.qgSize);
    Slice& slice = su.slice;
    slice.m_sliceType = a->sliceType == P_SLICE ? P_SLICE : B_SLICE;
    slice.m_poc = poc[0];
    slice.m_numRefIdx[0] = a->numRefIdx[0];
    slice.m_numRefIdx[1] = a->numRefIdx[1];
    for (int list = 0; list < su.nfr - 1; list++)
    {
        for (int r = 0; r < MAX_NUM_REF; r++)
            slice.m_refFrameList[list][r] = su.fr[1 + list];
        const int diffPoc = abs(poc[0] - poc[1 + list]);
        if (mvs[list] && diffPoc <= a->bframes + 1)
            for (int i = 0; i < su.w8 * su.h8; i++)
            {
                lr.lowresMvs[list][diffPoc][i].x = mvs[list][2 * i];
                lr.lowresMvs[list][diffPoc][i].y = mvs[list][2 * i + 1];
            }
    }
}

static void teardown(Setup& su)
{
    for (int f = 0; f < su.nfr; f++)
    {
        su.fr[f]->destroy();
        delete su.fr[f];
    }
    x265_param_free(su.p);
}

extern "C" {
/* y[3] / cb[3] / cr[3]: W x H and (W / 2) x (H / 2) contiguous planes of frames 0..2 (cb = cr = NULL: 4:0:0; frame 2
 * unused, may be NULL, for P slices); poc[3]; wp[3][6] = per frame {wp_sum[3], wp_ssd[3]}; mvs[2] as above.
 * Outputs: out[2][16][3][4] = {wtPresent, inputWeight, log2WeightDenom, inputOffset} of every slot of
 * Slice::m_weightPredTable (only slots with list < numPredDir and ref < numRefIdx[list] are written by the reference:
 * the others hold whatever the reference's stack held); intraCost[w8 * h8] of frame 0. */
void x265ref_weightp(const pixel* const* y, const pixel* const* cb, const pixel* const* cr, const WpParams* a,
                     const int32_t* poc, const uint64_t* wp, const int32_t* const* mvs, int32_t* out, int32_t* intraCost)
{
    Setup su;
    setup(su, y, cb, cr, a, poc, wp, mvs);
    memcpy(intraCost, su.fr[0]->m_lowres.intraCost, sizeof(int32_t) * su.w8 * su.h8);
    weightAnalyse(su.slice, *su.fr[0], *su.p);
    for (int list = 0; list < 2; list++)
        for (int r = 0; r < MAX_NUM_REF; r++)
            for (int pl = 0; pl < 3; pl++)
            {
                const WeightParam& w = su.slice.m_weightPredTable[list][r][pl];
                int32_t* o = out + ((list * MAX_NUM_REF + r) * 3 + pl) * 4;
                o[0] = w.wtPresent; o[1] = w.inputWeight; o[2] = (int32_t)w.log2WeightDenom; o[3] = w.inputOffset;
            }
    teardown(su);
}

/* The same frames; weightCost of each candidate cands[n][4] = {weighted, w0, denom, offset} for plane `plane` (0 luma,
 * 1 Cb, 2 Cr) of list `list`, after mcLuma / mcChroma with lowresMvs[list][diffPoc] when use_mvs, as weightAnalyse
 * prepares its inputs (:228-246, 347-403).  costs[n]: the uint32 sums, without sliceHeaderCost. */
void x265ref_weightp_costs(const pixel* const* y, const pixel* const* cb, const pixel* const* cr, const WpParams* a,
                           const int32_t* poc, const uint64_t* wp, const int32_t* const* mvs, int list, int plane, int use_mvs,
                           const int32_t* cands, int n, uint32_t* costs)
{
    Setup su;
    setup(su, y, cb, cr, a, poc, wp, mvs);
    Frame& frame = *su.fr[0];
    PicYuv* fencPic = frame.m_fencPic;
    Lowres& fenc = frame.m_lowres;
    Cache cache;
    memset(&cache, 0, sizeof(cache));
    cache.intraCost = fenc.intraCost;
    cache.numPredDir = su.slice.isInterP() ? 1 : 2;
    cache.lowresWidthInCU = fenc.width >> 3;
    cache.lowresHeightInCU = fenc.lines >> 3;
    cache.csp = su.p->internalCsp;
    cache.hshift = CHROMA_H_SHIFT(cache.csp);
    cache.vshift = CHROMA_V_SHIFT(cache.csp);
    pixel* mcbuf = X265_MALLOC(pixel, 2 * fencPic->m_stride * fencPic->m_picHeight);
    pixel* weightTemp = mcbuf + fencPic->m_stride * fencPic->m_picHeight;
    Frame* refFrame = su.slice.m_refFrameList[list][0];
    Lowres& refLowres = refFrame->m_lowres;
    const int diffPoc = abs(su.slice.m_poc - refFrame->m_poc);
    const MV* mv = use_mvs ? fenc.lowresMvs[list][diffPoc] : NULL;
    pixel *orig, *fref;
    intptr_t stride;
    int width, height;
    if (plane == 0)
    {
        orig = fenc.lowresPlane[0]; stride = fenc.lumaStride; width = fenc.width; height = fenc.lines;
        fref = refLowres.lowresPlane[0];
        if (mv) { mcLuma(mcbuf, refLowres, mv); fref = mcbuf; }
    }
    else
    {
        orig = fencPic->m_picOrg[plane]; stride = fencPic->m_strideC; fref = refFrame->m_fencPic->m_picOrg[plane];
        width = ((fencPic->m_picWidth >> 4) << 4) >> cache.hshift;
        height = ((fencPic->m_picHeight >> 4) << 4) >> cache.vshift;
        if (mv) { mcChroma(mcbuf, fref, stride, mv, cache, height, width); fref = mcbuf; }
    }
    for (int i = 0; i < n; i++)
    {
        WeightParam w;
        SET_WEIGHT(w, true, cands[4 * i + 1], cands[4 * i + 2], cands[4 * i + 3]);
        costs[i] = weightCost(orig, fref, weightTemp, stride, cache, width, height, cands[4 * i] ? &w : NULL, !plane);
    }
    X265_FREE(mcbuf);
    teardown(su);
}
}
