/* oracle/oracle_weightp.c -- TEST INFRASTRUCTURE ONLY: the frame encoder's weighted-prediction analysis, weightAnalyse
 * (encoder/weightPrediction.cpp:222-539), restated in plain C from the pixels: mcLuma (:60-89, with Lowres::lowresMC,
 * common/lowres.h), mcChroma (:93-163), weightCost (:169-218), sliceHeaderCost (:49-56) and the search (:260-501).
 * Pinned to the real function by oracle/ref_shim_weightp.cpp (tests/test_weightp_oracle_vs_ref.py); the device cost
 * kernel and the library's host decision are compared with it.  8 and 10 bit in one library (runtime depth), 4:2:0 and
 * 4:0:0.  Built by Makefile.weightp with -ffp-contract=off and without fast-math. */
#include <limits.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* the records of include/x265_b200.h (x265cu_wp_frame / _params / _cand / _entry), here with host pointers */
typedef struct {
    const void* lowres[4];          /* the 4 lowres hpel planes at picture origin, margins extended */
    const void* cb;                 /* full-resolution source Cb / Cr at (0,0), margins extended; NULL for 4:0:0 */
    const void* cr;
    int32_t lowresStride, chromaStride;
    uint64_t wp_sum[3], wp_ssd[3];
    int32_t poc, reserved;
} OrcWpFrame;
typedef struct {
    int32_t sliceType;              /* 0 B, 1 P */
    int32_t numRefIdx[2];
    int32_t bframes;
    int32_t width, height;          /* m_picWidth / m_picHeight */
    int32_t csp;                    /* 0 = 4:0:0, 1 = 4:2:0 */
} OrcWpParams;
typedef struct { int32_t weighted, w0, denom, offset; } OrcWpCand;
typedef struct { int32_t wtPresent, inputWeight, log2WeightDenom, inputOffset; } OrcWpEntry;

/* decision counters (branch reach) */
enum {
    WPC_EARLY, WPC_CHROMA_DENOM, WPC_CHROMA_SCALE_SKIP, WPC_OFFSET_RESCALE, WPC_RESCALE_REFMEAN0, WPC_DELTA_SKIP,
    WPC_OFFSET_BREAK, WPC_LUMA_DENOM, WPC_REJECT_0998, WPC_CHROMA_FIXUP, WPC_LIST1, WPC_PATH_COPY, WPC_PATH_HPP,
    WPC_PATH_VPP, WPC_PATH_HV, WPC_MC_BLOCK, WPC_COPY_BLOCK, WPC_ORIG_ZERO, WPC_WEIGHTED, WPC_N
};
static int64_t g_cnt[WPC_N];
void orc_wp_counters(int64_t* out, int reset)
{
    if (out) memcpy(out, g_cnt, sizeof(g_cnt));
    if (reset) memset(g_cnt, 0, sizeof(g_cnt));
}
int orc_wp_num_counters(void) { return WPC_N; }

static const int16_t chromaFilter[8][4] = {     /* g_chromaFilter (common/constants.cpp) */
    { 0, 64, 0, 0 }, { -2, 58, 10, -2 }, { -4, 54, 16, -2 }, { -6, 46, 28, -4 },
    { -4, 36, 36, -4 }, { -4, 28, 46, -6 }, { -2, 16, 54, -4 }, { -2, 10, 58, -2 }
};

static inline int rd(const void* p, int depth, intptr_t i)
{
    return depth == 8 ? ((const uint8_t*)p)[i] : ((const uint16_t*)p)[i];
}
static inline int clip3(int lo, int hi, int v) { return v < lo ? lo : (v > hi ? hi : v); }

/* (int) of a float as x86's cvttss2si computes it: NaN and values outside the int range give INT_MIN (refMean == 0
 * divides by zero in the offset rescale, :436) */
static inline int cvt(float v) { return (v >= -2147483648.f && v < 2147483648.f) ? (int)v : INT_MIN; }

/* bitSize (common/bitstream.h:94-112) and the sizes built on it */
static int bitsize(unsigned v) { int n = 0; while (v >> (n + 1)) n++; return v ? 2 * n + 1 : 1; }
static int bs_size_ue(unsigned v) { return bitsize(v + 1); }
static int bs_size_se(int val)
{
    int tmp = 1 - val * 2;
    if (tmp < 0) tmp = val * 2;
    return tmp < 256 ? bitsize((unsigned)tmp) : bitsize((unsigned)tmp >> 8) + 16;
}
static int slice_header_cost(const OrcWpEntry* w, int lambda, int bChroma)
{
    if (bChroma) lambda *= 4;
    int denomCost = bs_size_ue((unsigned)w->log2WeightDenom) * (2 - bChroma);
    return lambda * (10 + denomCost + 2 * (bs_size_se(w->inputWeight) + bs_size_se(w->inputOffset)));
}

/* SATD of an 8x8 block of differences: two 8x4 tiles, each the halved sum of its two 4x4 Hadamard sums (pixel.cpp) */
static int satd8x8(const int* d)
{
    int total = 0;
    for (int t = 0; t < 2; t++)
    {
        int s = 0;
        for (int h = 0; h < 2; h++)
        {
            int m[4][4];
            for (int y = 0; y < 4; y++)
                for (int x = 0; x < 4; x++) m[y][x] = d[(4 * t + y) * 8 + 4 * h + x];
            for (int y = 0; y < 4; y++)
            {
                int a0 = m[y][0] + m[y][1], a1 = m[y][0] - m[y][1], a2 = m[y][2] + m[y][3], a3 = m[y][2] - m[y][3];
                m[y][0] = a0 + a2; m[y][1] = a1 + a3; m[y][2] = a0 - a2; m[y][3] = a1 - a3;
            }
            for (int x = 0; x < 4; x++)
            {
                int a0 = m[0][x] + m[1][x], a1 = m[0][x] - m[1][x], a2 = m[2][x] + m[3][x], a3 = m[2][x] - m[3][x];
                s += abs(a0 + a2) + abs(a1 + a3) + abs(a0 - a2) + abs(a1 - a3);
            }
        }
        total += s >> 1;
    }
    return total;
}

typedef struct {
    int depth, plane, width, height;        /* width / height of the analysed area (lowres w8 * 8 x h8 * 8, or cw x ch) */
    int w8, h8;                             /* lowresWidthInCU / lowresHeightInCU */
    const OrcWpFrame* fenc; const OrcWpFrame* ref;
    const int32_t* mvs;                     /* NULL: no motion compensation */
} Ctx;

/* one 8x8 block of the (motion-compensated) reference at (x, y): mcLuma / Lowres::lowresMC, mcChroma, or the plane */
static void ref_block(const Ctx* c, int x, int y, int* out)
{
    const int D = c->depth;
    if (c->plane == 0)
    {
        const intptr_t s = c->ref->lowresStride;
        if (!c->mvs)
        {
            for (int r = 0; r < 8; r++)
                for (int k = 0; k < 8; k++) out[r * 8 + k] = rd(c->ref->lowres[0], D, (intptr_t)(y + r) * s + x + k);
            return;
        }
        const int cu = (y >> 3) * c->w8 + (x >> 3);
        int qx = c->mvs[2 * cu], qy = c->mvs[2 * cu + 1];
        qx = clip3((-x - 8) * 4, (c->width - x - 1 + 8) * 4, qx);     /* MV::clipped (:79-84) */
        qy = clip3((-y - 8) * 4, (c->height - y - 1 + 8) * 4, qy);
        const int ha = (qy & 2) | ((qx & 2) >> 1);
        const intptr_t oa = (intptr_t)(y + (qy >> 2)) * s + x + (qx >> 2);
        if ((qx | qy) & 1)
        {
            const int rx = qx + (qx & 1), ry = qy + (qy & 1);
            const int hb = (ry & 2) | ((rx & 2) >> 1);
            const intptr_t ob = (intptr_t)(y + (ry >> 2)) * s + x + (rx >> 2);
            for (int r = 0; r < 8; r++)
                for (int k = 0; k < 8; k++)
                    out[r * 8 + k] = (rd(c->ref->lowres[ha], D, oa + r * s + k) + rd(c->ref->lowres[hb], D, ob + r * s + k) + 1) >> 1;
        }
        else
            for (int r = 0; r < 8; r++)
                for (int k = 0; k < 8; k++) out[r * 8 + k] = rd(c->ref->lowres[ha], D, oa + r * s + k);
        return;
    }
    const void* src = c->plane == 1 ? c->ref->cb : c->ref->cr;
    const intptr_t s = c->ref->chromaStride;
    const intptr_t pixoff = (intptr_t)y * s + x;
    if (!c->mvs || !(x < c->w8 && y < c->h8))
    {
        if (c->mvs) g_cnt[WPC_COPY_BLOCK]++;
        for (int r = 0; r < 8; r++)
            for (int k = 0; k < 8; k++) out[r * 8 + k] = rd(src, D, pixoff + r * s + k);
        return;
    }
    g_cnt[WPC_MC_BLOCK]++;
    const int cu = y * c->w8 + (x >> 3);            /* y is a pixel row (:114) */
    int mx = c->mvs[2 * cu], my = c->mvs[2 * cu + 1];
    mx = (int)((unsigned)mx << 1) >> 1;             /* mv <<= 1, then >>= hshift / vshift (4:2:0) */
    my = (int)((unsigned)my << 1) >> 1;
    mx = clip3((-x - 8) * 4, (c->width - x - 1 + 8) * 4, mx);
    my = clip3((-y - 8) * 4, (c->height - y - 1 + 8) * 4, my);
    const intptr_t t = pixoff + (intptr_t)(my >> 2) * s + (mx >> 2);
    const int xf = mx & 7, yf = my & 7, maxv = (1 << D) - 1;
    const int16_t* cx = chromaFilter[xf];
    const int16_t* cy = chromaFilter[yf];
    if (!(xf | yf))
    {
        g_cnt[WPC_PATH_COPY]++;
        for (int r = 0; r < 8; r++)
            for (int k = 0; k < 8; k++) out[r * 8 + k] = rd(src, D, t + r * s + k);
    }
    else if (!yf)
    {
        g_cnt[WPC_PATH_HPP]++;                      /* interp_horiz_pp (ipfilter.cpp) */
        for (int r = 0; r < 8; r++)
            for (int k = 0; k < 8; k++)
            {
                int sum = 0;
                for (int i = 0; i < 4; i++) sum += rd(src, D, t + r * s + k - 1 + i) * cx[i];
                out[r * 8 + k] = clip3(0, maxv, (int16_t)((sum + 32) >> 6));
            }
    }
    else if (!xf)
    {
        g_cnt[WPC_PATH_VPP]++;                      /* interp_vert_pp */
        for (int r = 0; r < 8; r++)
            for (int k = 0; k < 8; k++)
            {
                int sum = 0;
                for (int i = 0; i < 4; i++) sum += rd(src, D, t + (r - 1 + i) * s + k) * cy[i];
                out[r * 8 + k] = clip3(0, maxv, (int16_t)((sum + 32) >> 6));
            }
    }
    else
    {
        g_cnt[WPC_PATH_HV]++;                       /* interp_horiz_ps (isRowExt) + interp_vert_sp */
        const int head = 14 - D, hs = 6 - head, vs = 6 + head;
        const int hoff = (int)((unsigned)-8192 << hs), voff = (1 << (vs - 1)) + (8192 << 6);
        int16_t imm[11][8];
        for (int r = 0; r < 11; r++)
            for (int k = 0; k < 8; k++)
            {
                int sum = 0;
                for (int i = 0; i < 4; i++) sum += rd(src, D, t + (r - 1) * s + k - 1 + i) * cx[i];
                imm[r][k] = (int16_t)((sum + hoff) >> hs);
            }
        for (int r = 0; r < 8; r++)
            for (int k = 0; k < 8; k++)
            {
                int sum = 0;
                for (int i = 0; i < 4; i++) sum += imm[r + i][k] * cy[i];
                out[r * 8 + k] = clip3(0, maxv, (int16_t)((sum + voff) >> vs));
            }
    }
}

static void ctx_init(Ctx* c, int depth, const OrcWpParams* p, const OrcWpFrame* fenc, const OrcWpFrame* ref,
                     const int32_t* mvs, int plane)
{
    c->depth = depth; c->plane = plane; c->fenc = fenc; c->ref = ref; c->mvs = mvs;
    c->w8 = ((p->width / 2) + 7) >> 3; c->h8 = ((p->height / 2) + 7) >> 3;
    if (plane == 0) { c->width = c->w8 * 8; c->height = c->h8 * 8; }
    else { c->width = ((p->width >> 4) << 4) >> 1; c->height = ((p->height >> 4) << 4) >> 1; }   /* :377-378 */
}

/* weightCost (:169-218) of every candidate of one plane; costs[i] is the wrapping uint32 sum, without sliceHeaderCost */
static void costs_ctx(const Ctx* c, const int32_t* intraCost, const OrcWpCand* cands, int n, uint32_t* costs)
{
    const int D = c->depth, maxv = (1 << D) - 1, corr = 14 - D;
    const void* fp = c->plane == 0 ? c->fenc->lowres[0] : (c->plane == 1 ? c->fenc->cb : c->fenc->cr);
    const intptr_t fs = c->plane == 0 ? c->fenc->lowresStride : c->fenc->chromaStride;
    for (int i = 0; i < n; i++) costs[i] = 0;
    int refb[64], fb[64], d[64];
    int cu = 0;
    for (int y = 0; y < c->height; y += 8)
        for (int x = 0; x < c->width; x += 8, cu++)
        {
            ref_block(c, x, y, refb);
            for (int r = 0; r < 8; r++)
                for (int k = 0; k < 8; k++) fb[r * 8 + k] = rd(fp, D, (intptr_t)(y + r) * fs + x + k);
            for (int i = 0; i < n; i++)
            {
                const OrcWpCand* w = &cands[i];
                const int round = w->denom ? 1 << (w->denom - 1) : 0;
                for (int j = 0; j < 64; j++)
                {
                    int rv = refb[j];
                    if (w->weighted)
                    {
                        /* weight_pp (pixel.cpp:518-543) with round << correction, denom + correction, offset << (D - 8) */
                        int16_t v = (int16_t)(rv << corr);
                        rv = clip3(0, maxv, ((w->w0 * v + (round << corr)) >> (w->denom + corr)) + (w->offset << (D - 8)));
                    }
                    d[j] = rv - fb[j];
                }
                int cmp = satd8x8(d);
                /* the reference passes (ref, fenc) to satd: |H(r - f)| == |H(f - r)| */
                if (c->plane == 0) cmp = cmp < intraCost[cu] ? cmp : intraCost[cu];
                costs[i] += (uint32_t)cmp;
            }
        }
}

/* one plane's candidate costs, as x265cu_weightp_costs computes them */
void orc_wp_costs(int depth, const OrcWpParams* p, const OrcWpFrame* fenc, const OrcWpFrame* ref, const int32_t* intraCost,
                  const int32_t* mvs, int plane, const OrcWpCand* cands, int n, uint32_t* costs)
{
    Ctx c;
    ctx_init(&c, depth, p, fenc, ref, mvs, plane);
    costs_ctx(&c, intraCost, cands, n, costs);
}

static void set_w(OrcWpEntry* w, int present, int scale, int denom, int off)
{
    w->wtPresent = present; w->inputWeight = scale; w->log2WeightDenom = denom; w->inputOffset = off;
}

/* weightAnalyse (:222-505).  refs[list]: m_refFrameList[list][0]; mvs[list]: lowresMvs[list][diffPoc] as int32 pairs,
 * NULL when that field was not searched (the reference's 0x7FFF marker).  out[2][16][3]: entries the reference writes
 * (list < numPredDir, ref < numRefIdx[list]) are written, the others are left alone.  In 4:0:0 the reference reads
 * guessScale[1] / [2] uninitialised to choose the chroma denominator (:280-286); here they are 0, so chromaDenom stays 7. */
void orc_wp_analyse(int depth, const OrcWpParams* p, const OrcWpFrame* fenc, const int32_t* intraCost,
                    const OrcWpFrame* const* refs, const int32_t* const* mvsIn, OrcWpEntry* out)
{
    OrcWpEntry (*wp)[16][3] = (OrcWpEntry (*)[16][3])out;
    const int numPredDir = p->sliceType == 1 ? 1 : 2;
    const int nplanes = p->csp ? 3 : 1;
    const int lambda = depth == 8 ? 1 : 16;          /* (int)x265_lambda_tab[X265_LOOKAHEAD_QP] */
    const float epsilon = 1.f / 128.f;
    int chromaDenom = 7, lumaDenom = 7, denom;
    int numpixels[3];
    const int w16 = ((p->width + 15) >> 4) << 4, h16 = ((p->height + 15) >> 4) << 4;
    numpixels[0] = w16 * h16;
    numpixels[1] = numpixels[2] = numpixels[0] >> 2;
    for (int list = 0; list < numPredDir; list++)
    {
        OrcWpEntry* weights = wp[list][0];
        const OrcWpFrame* ref = refs[list];
        const int diffPoc = abs(fenc->poc - ref->poc);
        if (list) g_cnt[WPC_LIST1]++;
        float guessScale[3] = { 0, 0, 0 }, fencMean[3] = { 0, 0, 0 }, refMean[3] = { 0, 0, 0 };
        for (int plane = 0; plane < nplanes; plane++)
        {
            set_w(&weights[plane], 0, 1, 0, 0);
            uint64_t fencVar = fenc->wp_ssd[plane] + !ref->wp_ssd[plane];
            uint64_t refVar = ref->wp_ssd[plane] + !ref->wp_ssd[plane];
            guessScale[plane] = sqrtf((float)fencVar / refVar);
            fencMean[plane] = (float)fenc->wp_sum[plane] / (numpixels[plane]) / (1 << (depth - 8));
            refMean[plane] = (float)ref->wp_sum[plane] / (numpixels[plane]) / (1 << (depth - 8));
        }
        while (!list && chromaDenom > 0)
        {
            float thresh = 127.f / (1 << chromaDenom);
            if (guessScale[1] < thresh && guessScale[2] < thresh)
                break;
            chromaDenom--;
            g_cnt[WPC_CHROMA_DENOM]++;
        }
        set_w(&weights[1], 0, 1 << chromaDenom, chromaDenom, 0);
        set_w(&weights[2], 0, 1 << chromaDenom, chromaDenom, 0);
        const int32_t* mvs = NULL;
        for (int plane = 0; plane < nplanes; plane++)
        {
            denom = plane ? chromaDenom : lumaDenom;
            if (plane && !weights[0].wtPresent)
                break;
            if (fabsf(refMean[plane] - fencMean[plane]) < 0.5f && fabsf(1.f - guessScale[plane]) < epsilon)
            {
                g_cnt[WPC_EARLY]++;
                set_w(&weights[plane], 0, 1 << denom, denom, 0);
                continue;
            }
            if (plane)
            {
                int scale = clip3(0, 255, cvt(guessScale[plane] * (1 << denom) + 0.5f));
                if (scale > 127) { g_cnt[WPC_CHROMA_SCALE_SKIP]++; continue; }
                weights[plane].inputWeight = scale;
            }
            else
            {
                /* setFromWeightAndOffset(w, 0, denom, bNormalize = !list) (slice.h:304-316) */
                OrcWpEntry* w = &weights[plane];
                w->inputOffset = 0; w->log2WeightDenom = denom; w->inputWeight = cvt(guessScale[plane] * (1 << denom) + 0.5f);
                while (!list && w->log2WeightDenom > 0 && w->inputWeight > 127) { w->log2WeightDenom--; w->inputWeight >>= 1; }
                if (w->inputWeight > 127) w->inputWeight = 127;
            }
            int mindenom = weights[plane].log2WeightDenom;
            int minscale = weights[plane].inputWeight;
            int minoff = 0;
            if (!plane && diffPoc <= p->bframes + 1)
                mvs = mvsIn[list];
            Ctx c;
            ctx_init(&c, depth, p, fenc, ref, mvs, plane);
            /* every candidate of the search, in the reference's order: they depend on the estimates only */
            OrcWpCand cand[1 + 9 * 5];
            int nc = 0, scaleOf[9], offOf[9], firstOf[9], nsc = 0;
            cand[nc++] = (OrcWpCand){ 0, 0, 0, 0 };
            const int startScale = clip3(0, 127, minscale - 4), endScale = clip3(0, 127, minscale + 4);
            for (int scale = startScale; scale <= endScale; scale++)
            {
                int deltaWeight = scale - (1 << mindenom);
                if (deltaWeight > 127 || deltaWeight <= -128) { g_cnt[WPC_DELTA_SKIP]++; continue; }
                int curScale = scale;
                int curOffset = cvt(fencMean[plane] - refMean[plane] * curScale / (1 << mindenom) + 0.5f);
                if (curOffset < -128 || curOffset > 127)
                {
                    g_cnt[WPC_OFFSET_RESCALE]++;
                    if (refMean[plane] == 0) g_cnt[WPC_RESCALE_REFMEAN0]++;
                    curOffset = clip3(-128, 127, curOffset);
                    curScale = cvt((1 << mindenom) * (fencMean[plane] - curOffset) / refMean[plane] + 0.5f);
                    curScale = clip3(0, 127, curScale);
                }
                scaleOf[nsc] = curScale; offOf[nsc] = curOffset; firstOf[nsc] = nc; nsc++;
                const int so = clip3(-128, 127, curOffset - 2), eo = clip3(-128, 127, curOffset + 2);
                for (int off = so; off <= eo; off++) cand[nc++] = (OrcWpCand){ 1, curScale, mindenom, off };
            }
            uint32_t costs[1 + 9 * 5];
            costs_ctx(&c, intraCost, cand, nc, costs);
            uint32_t origscore = costs[0];
            if (!origscore)
            {
                g_cnt[WPC_ORIG_ZERO]++;
                set_w(&weights[plane], 0, 1 << denom, denom, 0);
                continue;
            }
            uint32_t minscore = origscore;
            int bFound = 0;
            for (int k = 0; k < nsc; k++)
            {
                const int curOffset = offOf[k], curScale = scaleOf[k];
                const int so = clip3(-128, 127, curOffset - 2), eo = clip3(-128, 127, curOffset + 2);
                for (int off = so, i = firstOf[k]; off <= eo; off++, i++)
                {
                    OrcWpEntry wsp;
                    set_w(&wsp, 1, curScale, mindenom, off);
                    uint32_t s = costs[i] + (uint32_t)slice_header_cost(&wsp, lambda, !!plane);
                    if (s < minscore) { minscore = s; minscale = curScale; minoff = off; bFound = 1; }
                    if (minoff == so && off != so) { g_cnt[WPC_OFFSET_BREAK]++; break; }
                }
            }
            if (!(plane || list))
            {
                if (mindenom > 0 && !(minscale & 1))
                {
                    /* CTZ (common.h): tzcnt semantics, 32 for a zero scale */
                    int idx = minscale ? __builtin_ctz((unsigned)minscale) : 32;
                    int shift = idx < mindenom ? idx : mindenom;
                    mindenom -= shift;
                    minscale >>= shift;
                    g_cnt[WPC_LUMA_DENOM]++;
                }
            }
            const int reject = (float)minscore / origscore > 0.998f;
            if (!bFound || (minscale == (1 << mindenom) && minoff == 0) || reject)
            {
                if (bFound && !(minscale == (1 << mindenom) && minoff == 0)) g_cnt[WPC_REJECT_0998]++;
                set_w(&weights[plane], 0, 1 << denom, denom, 0);
            }
            else
            {
                g_cnt[WPC_WEIGHTED]++;
                set_w(&weights[plane], 1, minscale, mindenom, minoff);
            }
        }
        if (weights[0].wtPresent && weights[1].wtPresent != weights[2].wtPresent)
        {
            g_cnt[WPC_CHROMA_FIXUP]++;
            if (weights[1].wtPresent) weights[2] = weights[1];
            else weights[1] = weights[2];
        }
        lumaDenom = weights[0].log2WeightDenom;
        chromaDenom = weights[1].log2WeightDenom;
        for (int r = 1; r < p->numRefIdx[list]; r++)
        {
            set_w(&wp[list][r][0], 0, 1 << lumaDenom, lumaDenom, 0);
            set_w(&wp[list][r][1], 0, 1 << chromaDenom, chromaDenom, 0);
            set_w(&wp[list][r][2], 0, 1 << chromaDenom, chromaDenom, 0);
        }
    }
}
