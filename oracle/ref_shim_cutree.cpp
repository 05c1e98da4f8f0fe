/* oracle/ref_shim_cutree.cpp -- TEST INFRASTRUCTURE ONLY (never linked into the product).
 *
 * The REAL Lookahead::cuTree (encoder/slicetype.cpp:2538-2639, with estimateCUPropagate and cuTreeFinish) over caller arrays
 * (pins oracle/oracle_cutree.c).  Built by Makefile.cutree with the reference objects of Makefile.ref into
 * oracle/_ref/libx265ref_cutree{8,10}.so.
 *
 * Each frame is a real Lowres whose cuTree fields point at the caller's arrays: intraCost, invQscaleFactor (or
 * invQscaleFactor8x8 when rc.qgSize == 8), lowresCosts[d0][d1], lowresMvs[list][dist] (converted from int32 pairs),
 * qpAqOffset and weightedCostDelta.  The caller's estimates are marked computed (costEst >= 0 and rowSatds[..][0] != -1,
 * slicetype.cpp:3121), so that singleCost returns them without a search.  propagateCost and qpCuTreeOffset are the shim's
 * own: before the call every frame's propagateCost holds cutree_pattern() and every qpCuTreeOffset -1000 - frame, so the
 * results also pin which words the reference leaves alone.  cuTree and cuTreeFinish are protected; a derived struct reaches
 * them, as ref_shim_sao.cpp reaches SAO. */
#include "common.h"
#include "primitives.h"
#include "lowres.h"
#include "slicetype.h"
#include <string.h>
#include <vector>

using namespace X265_NS;

namespace X265_NS {
void setupCPrimitives(EncoderPrimitives &p);
void setupAliasPrimitives(EncoderPrimitives &p);
}

#define DIST 18

/* the record layout of oracle/oracle_cutree.c */
struct CutreeFrame
{
    const int32_t* intraCost; const int32_t* invQscale; uint16_t* propagateCost;
    const uint16_t* lowresCosts[DIST][DIST];
    const int32_t* mvs[2][DIST];
    int32_t sliceType, reserved;
    const double* qpAqOffset; double* qpCuTreeOffset;
    double weightedCostDelta[DIST];
};
struct CutreeParams
{
    int32_t bIntra, lookaheadDepth, bBPyramid, bEnableWeightedBiPred, vbv, fpsNum, fpsDenom, qgSize;
    double qCompress;
};

struct CuTreeAccess : public Lookahead
{
    static void run(Lookahead& la, Lowres** frames, int numframes, bool bIntra)
    {
        (la.*(&CuTreeAccess::cuTree))(frames, numframes, bIntra);
    }
    static void finish(Lookahead& la, Lowres* frame, double averageDuration, int ref0Distance)
    {
        (la.*(&CuTreeAccess::cuTreeFinish))(frame, averageDuration, ref0Distance);
    }
};

static void prim_init()
{
    static bool done = false;
    if (done) return;
    setupCPrimitives(primitives);
    setupAliasPrimitives(primitives);
    done = true;
}

struct CtWindow
{
    x265_param* param;
    Lookahead* la;
    std::vector<Lowres*> fr;
    std::vector<std::vector<uint16_t> > prop;
    std::vector<std::vector<MV> > mvs;
    std::vector<std::vector<int32_t> > invq;
    std::vector<std::vector<double> > aq, qp;
    int32_t rowSatd0;
    int ncu, nfull;
};

static CtWindow* make_window(const CutreeFrame* in, int numframes, const CutreeParams* p, int w8, int h8)
{
    prim_init();
    CtWindow* w = new CtWindow();
    x265_param* param = x265_param_alloc();
    x265_param_default(param);
    param->sourceWidth = w8 * 16; param->sourceHeight = h8 * 16;
    param->bframes = 16; param->lookaheadDepth = p->lookaheadDepth; param->bBPyramid = p->bBPyramid;
    param->bEnableWeightedBiPred = p->bEnableWeightedBiPred; param->rc.vbvBufferSize = p->vbv ? 1000 : 0;
    param->fpsNum = p->fpsNum; param->fpsDenom = p->fpsDenom; param->rc.qgSize = p->qgSize; param->rc.hevcAq = 0;
    param->rc.qCompress = p->qCompress; param->rc.cuTree = 1; param->lookaheadSlices = 0; param->gopLookahead = 0;
    w->param = param;
    w->la = new Lookahead(param, NULL);
    w->la->m_tld = new LookaheadTLD[1];
    w->la->m_scratch = X265_MALLOC(int, w->la->m_8x8Width);
    w->ncu = w8 * h8;
    w->nfull = p->qgSize == 8 ? 4 * w->ncu : w->ncu;
    w->rowSatd0 = 0;
    const int n = numframes + 1;
    w->prop.resize(n); w->invq.resize(n); w->aq.resize(n); w->qp.resize(n); w->mvs.resize(n * 2 * DIST);
    for (int f = 0; f < n; f++)
    {
        Lowres* lr = (Lowres*)X265_MALLOC(Lowres, 1);
        memset((void*)lr, 0, sizeof(Lowres));
        const CutreeFrame& c = in[f];
        lr->sliceType = c.sliceType;
        lr->widthFullRes = w8 * 16; lr->heightFullRes = h8 * 16;
        lr->maxBlocksInRow = w8; lr->maxBlocksInCol = h8;
        lr->maxBlocksInRowFullRes = w8 * 2; lr->maxBlocksInColFullRes = h8 * 2;
        lr->intraCost = (int32_t*)c.intraCost;
        w->invq[f].assign(c.invQscale, c.invQscale + w->ncu);
        if (p->qgSize == 8) lr->invQscaleFactor8x8 = w->invq[f].data();
        else lr->invQscaleFactor = w->invq[f].data();
        w->prop[f].resize(w->ncu);
        for (int i = 0; i < w->ncu; i++)
            w->prop[f][i] = (uint16_t)((uint32_t)(f + 1) * 40503u + (uint32_t)i * 9973u);    /* cutree_pattern */
        lr->propagateCost = w->prop[f].data();
        w->aq[f].assign(w->nfull, 0.0);
        if (c.qpAqOffset) w->aq[f].assign(c.qpAqOffset, c.qpAqOffset + w->nfull);
        w->qp[f].assign(w->nfull, -1000.0 - f);
        lr->qpAqOffset = w->aq[f].data(); lr->qpCuTreeOffset = w->qp[f].data();
        for (int d = 0; d < DIST; d++) lr->weightedCostDelta[d] = c.weightedCostDelta[d];
        for (int d0 = 0; d0 < DIST; d0++)
            for (int d1 = 0; d1 < DIST; d1++)
            {
                lr->costEst[d0][d1] = -1;
                if (c.lowresCosts[d0][d1])
                {
                    lr->lowresCosts[d0][d1] = (uint16_t*)c.lowresCosts[d0][d1];
                    lr->costEst[d0][d1] = 0;                           /* computed: singleCost returns it */
                    lr->rowSatds[d0][d1] = &w->rowSatd0;
                }
            }
        for (int l = 0; l < 2; l++)
            for (int d = 0; d < DIST; d++)
            {
                if (!c.mvs[l][d]) continue;
                std::vector<MV>& v = w->mvs[(f * 2 + l) * DIST + d];
                v.resize(w->ncu);
                for (int i = 0; i < w->ncu; i++) { v[i].x = (int16_t)c.mvs[l][d][2 * i]; v[i].y = (int16_t)c.mvs[l][d][2 * i + 1]; }
                lr->lowresMvs[l][d] = v.data();
            }
        w->fr.push_back(lr);
    }
    w->fr.push_back(NULL);
    return w;
}

static void release(CtWindow* w)
{
    for (Lowres* lr : w->fr) if (lr) X265_FREE(lr);
    X265_FREE(w->la->m_scratch);
    delete[] w->la->m_tld;
    w->la->m_tld = NULL;
    delete w->la;
    x265_param_free(w->param);
    delete w;
}

extern "C" {
/* Runs the real cuTree on the window.  prop_out: (numframes + 1) x ncu, every frame's propagateCost after the call (as the
 * frame's pointer then points, swaps included); qp_out: (numframes + 1) x (ncu, or 4 ncu when qgSize == 8) qpCuTreeOffset. */
void x265ref_cutree(const CutreeFrame* frames, int numframes, const CutreeParams* p, int w8, int h8, uint16_t* prop_out, double* qp_out)
{
    CtWindow* w = make_window(frames, numframes, p, w8, h8);
    CuTreeAccess::run(*w->la, w->fr.data(), numframes, p->bIntra != 0);
    for (int f = 0; f <= numframes; f++)
    {
        memcpy(prop_out + (size_t)f * w->ncu, w->fr[f]->propagateCost, w->ncu * sizeof(uint16_t));
        memcpy(qp_out + (size_t)f * w->nfull, w->fr[f]->qpCuTreeOffset, w->nfull * sizeof(double));
    }
    release(w);
}

/* The real cuTreeFinish of frame f on the caller's propagateCost (frames[f].propagateCost), averageDuration as cuTree
 * computes it for the window; qp_out receives its qpCuTreeOffset (prefilled -1000 - f). */
void x265ref_cutree_finish(const CutreeFrame* frames, int numframes, const CutreeParams* p, int w8, int h8, int f, int ref0Distance,
                           double* qp_out)
{
    CtWindow* w = make_window(frames, numframes, p, w8, h8);
    memcpy(w->fr[f]->propagateCost, frames[f].propagateCost, w->ncu * sizeof(uint16_t));
    double totalDuration = 0.0;
    for (int j = 0; j <= numframes; j++)
        totalDuration += (double)p->fpsDenom / p->fpsNum;
    CuTreeAccess::finish(*w->la, w->fr[f], totalDuration / (numframes + 1), ref0Distance);
    memcpy(qp_out, w->fr[f]->qpCuTreeOffset, w->nfull * sizeof(double));
    release(w);
}
}
