/* oracle/frame_wref.h -- TEST INFRASTRUCTURE ONLY.
 * Weighted P-slice references of the frame-level CTU-analysis driver (x265cu_analyser_set_ref_weights), written once and
 * instantiated twice: by oracle_frame_wref.c over the oracle's plain-C primitives and by ref_shim_wref.cpp over the REAL
 * reference code.  Include it after frame_chroma.h with DRV_WPRED defined.
 *
 * The existing ME stage runs unchanged with drv_frame.refs / refC pointing at what the search reads: the weighted planes of
 * a weighted reference (MotionReference::fpelPlane, reference.cpp:51-185), the reference's planes otherwise.  The weighted
 * RESID and CHROMA RESID stages below read the unweighted planes from drv_wref: a CU whose reference is weighted takes the
 * weighted uni-prediction of Predict::motionCompensation (predict.cpp:82-112): the 14-bit prediction of the unweighted
 * planes, then addWeightUni (predict.cpp:525-578).  A CU whose reference is not weighted runs RESID / CHROMA RESID as they are.
 * DRV_WPRED(w, ref, x, y, S, qmvx, qmvy, stride, cstride, predY, predC, luma, chroma): that weighted prediction of the luma
 * S x S CU at (x, y) into predY (pitch S, when luma) and of its (S/2) x (S/2) chroma blocks into predC[2] (pitch S/2, when
 * chroma); w is a `const struct drv_wref_s*`. */
#ifndef X265_FRAME_WREF_H
#define X265_FRAME_WREF_H
typedef struct drv_wref_s {
    int32_t wp[16][3][4];             /* m_weightPredTable[0][r][plane] = {wtPresent, inputWeight, log2WeightDenom, inputOffset} */
    const DRV_PIXEL* refs[16];        /* the unweighted reference planes (origin pixels, the luma geometry) */
    const DRV_PIXEL* refC[16][2];     /* their Cb, Cr planes (the chroma geometry) */
} drv_wref;

/* MotionReference::applyWeight once every CTU row of the picture is weighted (reference.cpp:126-185): weight_pp of the
 * picture area with w = inputWeight, offset = inputOffset << (depth - 8), round = (denom ? 1 << (denom - 1) : 0) << (14 -
 * depth), shift = denom + 14 - depth (MotionReference::init, reference.cpp:98-101), then the left / right borders extended
 * and the top / bottom rows copied into the margins.  src / dst are origin pixels of planes with the given margins. */
static void drv_wref_plane(const DRV_PIXEL* src, DRV_PIXEL* dst, intptr_t stride, int width, int height, int marginX, int marginY,
                           const int32_t e[4])
{
    const int corr = 14 - DRV_DEPTH, denom = e[2];
    const int round = (denom ? 1 << (denom - 1) : 0) << corr, shift = denom + corr, offset = e[3] * (1 << (DRV_DEPTH - 8));
    const int maxv = (1 << DRV_DEPTH) - 1;
    for (int y = 0; y < height; y++)
    {
        const DRV_PIXEL* s = src + (intptr_t)y * stride;
        DRV_PIXEL* d = dst + (intptr_t)y * stride;
        for (int x = 0; x < width; x++)
        {
            const int16_t v = (int16_t)(s[x] << corr);
            int o = ((e[1] * v + round) >> shift) + offset;
            d[x] = (DRV_PIXEL)(o < 0 ? 0 : (o > maxv ? maxv : o));
        }
        for (int x = 0; x < marginX; x++) { d[-marginX + x] = d[0]; d[width + x] = d[width - 1]; }
    }
    for (int y = 1; y <= marginY; y++)
    {
        memcpy(dst - marginX - y * stride, dst - marginX, sizeof(DRV_PIXEL) * (width + 2 * marginX));
        memcpy(dst - marginX + (intptr_t)(height - 1 + y) * stride, dst - marginX + (intptr_t)(height - 1) * stride,
               sizeof(DRV_PIXEL) * (width + 2 * marginX));
    }
}

/* the transform chain of RESID / CHROMA RESID over the TUs (T x T, raster order) of one plane of a CU (S x S in the plane):
 * fe / rc = the CU's origin in the source / recon plane, pred = the prediction (pitch S), q = the CU's levels in the plane */
static void drv_wref_tus(const DRV_PIXEL* fe0, DRV_PIXEL* rc0, intptr_t stride, const DRV_PIXEL* pred, int S, int T, int qp, int16_t* q0,
                         uint64_t* sseOut, uint32_t* nsOut)
{
    const int lg = T == 32 ? 5 : (T == 16 ? 4 : (T == 8 ? 3 : 2));
    assert(qp >= 0 && qp <= 51 + 6 * (DRV_DEPTH - 8));
    static const int quantScales[6] = { 26214, 23302, 20560, 18396, 16384, 14564 };   /* scalinglist.cpp:129 */
    static const int invQuantScales[6] = { 40, 45, 51, 57, 64, 72 };                  /* scalinglist.cpp:130 */
    const int per = qp / 6, rem = qp % 6;
    const int transformShift = 15 - DRV_DEPTH - lg;
    const int qbits = 14 + per + transformShift, add = 85 << (qbits - 9);
    const int dqshift = 20 - 14 - transformShift, dqscale = invQuantScales[rem] << per;
    int32_t qc[32 * 32];
    for (int i = 0; i < T * T; i++) qc[i] = quantScales[rem];
    uint64_t sse = 0; uint32_t nsig = 0;
    int t = 0;
    for (int ty = 0; ty < S; ty += T)
        for (int tx = 0; tx < S; tx += T, t++)
        {
            int16_t resi[32 * 32], coefd[32 * 32], deq[32 * 32];
            int32_t deltaU[32 * 32];
            int16_t* q = q0 + (size_t)t * T * T;
            const DRV_PIXEL* fe = fe0 + (intptr_t)ty * stride + tx;
            const DRV_PIXEL* pr = pred + ty * S + tx;
            DRV_PIXEL* rc = rc0 + (intptr_t)ty * stride + tx;
            DRV_SUB_PS(resi, T, fe, pr, stride, S, T);
            DRV_DCT(resi, coefd, T, T);
            uint32_t ns = DRV_QUANT(coefd, qc, deltaU, q, qbits, add, T * T);
            if (ns)
            {
                DRV_DEQUANT(q, deq, T * T, dqscale, dqshift);
                if (ns == 1 && q[0] != 0)
                {   /* DC-only shortcut (quant.cpp:588-598) */
                    const int shift_2nd = 12 - (DRV_DEPTH - 8) - 3;
                    int dc = (((deq[0] * (64 >> 6) + 1) >> 1) * (64 >> 3) + (1 << (shift_2nd - 1))) >> shift_2nd;
                    DRV_BLOCKFILL(resi, T, (int16_t)dc, T);
                }
                else
                    DRV_IDCT(deq, resi, T, T);
                DRV_ADD_PS(rc, stride, pr, resi, S, T, T);
            }
            else
                DRV_COPY_PP(rc, stride, pr, S, T);
            sse += DRV_SSE(fe, stride, rc, stride, T);
            nsig += ns;
        }
    *sseOut = sse; *nsOut = nsig;
}

/* RESID (luma) and / or CHROMA RESID of CU c with the weights of its reference */
static void drv_wref_one(drv_frame* f, drv_chroma_resid* cr, const drv_wref* w, int c, int luma, int chroma)
{
    const fs_params* p = &f->p;
    const int x = f->cus[c][0], y = f->cus[c][1], S = f->cus[c][2];
    int best = 0, bcost = 0x7fffffff;
    for (int r = 0; r < p->numRefs; r++)
    {
        int cost = f->me_out[(size_t)f->cu_jobs[c * p->numRefs + r] * 4];
        if (cost < bcost) { bcost = cost; best = r; }
    }
    if (!w->wp[best][0][0])
    {
        if (luma) drv_resid_one(f, c);
        if (chroma) drv_chroma_one(f, cr, c);
        return;
    }
    const int32_t* mo = f->me_out + (size_t)f->cu_jobs[c * p->numRefs + best] * 4;
    DRV_PIXEL predY[64 * 64], predC[2][32 * 32];
    DRV_WPRED(w, best, x, y, S, mo[1], mo[2], p->stride, f->cstride, predY, predC, luma, chroma);
    const int T = S > 32 ? 32 : S, d = drv_depth_idx(S);
    if (luma)
    {
        const intptr_t off = (intptr_t)y * p->stride + x;
        f->cu_ref[c] = best;
        drv_wref_tus(f->fenc + off, f->recon[d] + off, p->stride, predY, S, T, p->qp, f->coef + f->cu_coef_off[c], &f->cu_sse[c],
                     &f->cu_numsig[c]);
    }
    for (int pl = 0; pl < 2 && chroma; pl++)
    {
        const intptr_t off = (intptr_t)(y / 2) * f->cstride + x / 2;
        drv_wref_tus(f->fencC[pl] + off, cr->recon[d][pl] + off, f->cstride, predC[pl], S / 2, T / 2, cr->qpc[pl],
                     cr->coef[pl] + f->cu_coef_off[c] / 4, &cr->cu_sse[2 * c + pl], &cr->cu_numsig[2 * c + pl]);
    }
}

typedef struct { drv_frame* f; drv_chroma_resid* cr; const drv_wref* w; int luma, chroma; volatile int next; } drv_wref_run;

static void* drv_wref_worker(void* arg)
{
    drv_wref_run* r = (drv_wref_run*)arg;
    for (;;)
    {
        int b = __sync_fetch_and_add(&r->next, 16);
        if (b >= r->f->ncu_run) break;
        int e = b + 16 < r->f->ncu_run ? b + 16 : r->f->ncu_run;
        for (int i = b; i < e; i++) drv_wref_one(r->f, r->cr, r->w, i, r->luma, r->chroma);
    }
    return NULL;
}

/* the weighted RESID (stage bit 1) and CHROMA RESID (bit 3) over the CUs of drv_prepare's rows, after the ME stage */
static void drv_run_wref(drv_frame* f, drv_chroma_resid* cr, const drv_wref* w, int stages)
{
    drv_wref_run r;
    r.f = f; r.cr = cr; r.w = w; r.luma = (stages & 2) != 0; r.chroma = (stages & 8) != 0; r.next = 0;
    if (!r.luma && !r.chroma) return;
    cr->qpc[0] = drv_chroma_qp(f->p.qp, cr->offset[0]);
    cr->qpc[1] = drv_chroma_qp(f->p.qp, cr->offset[1]);
    int nt = f->threads < 1 ? 1 : f->threads;
    if (nt == 1) { drv_wref_worker(&r); return; }
    pthread_t* th = (pthread_t*)malloc(sizeof(pthread_t) * nt);
    for (int t = 0; t < nt; t++) pthread_create(&th[t], NULL, drv_wref_worker, &r);
    for (int t = 0; t < nt; t++) pthread_join(th[t], NULL);
    free(th);
}
#endif
