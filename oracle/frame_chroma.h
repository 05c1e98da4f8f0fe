/* oracle/frame_chroma.h -- TEST INFRASTRUCTURE ONLY.
 * The 4:2:0 chroma residual stage of the frame-level CTU-analysis driver (analyser stage bit 3), written once and
 * instantiated twice: by oracle_frame_chroma.c over the oracle's plain-C primitives and by ref_shim_chroma.cpp over the
 * REAL reference table.  Include it after frame_driver.h (drv_frame, the DRV_* residual macros) with DRV_MC_C defined.
 */
#ifndef X265_FRAME_CHROMA_H
#define X265_FRAME_CHROMA_H
/* ---- CHROMA RESID (stage bit 3): the 4:2:0 chroma residual chain of every CU's best inter prediction ----
 * The luma RESID stage's reference and vector (lowest ME cost of the CU's 2Nx2N jobs, ties to the lowest index); chroma MC of
 * the CU's (S/2) x (S/2) block (Predict::predInterChromaPixel, predict.cpp:306-353: the luma quarter-pel vector read as
 * eighth-pel), then per luma TU (T = min(S, 32)) one (T/2) x (T/2) TU per plane through RESID's chain with the plane's QP
 * (search.cpp:2990-3080, Search::residualTransformQuantInter).  The including file defines
 * DRV_MC_C(src, ss, dst, ds, S, xf, yf): the chroma prediction of the luma S x S PU (copy_pp / filter_hpp / filter_vpp /
 * filter_hps(rowExt) + filter_vsp).  Outputs go to a drv_chroma_resid, so drv_frame keeps its layout. */
typedef struct {
    int offset[2];                    /* in: Cb, Cr chroma QP offset (PPS + slice), -12..12 */
    int qpc[2];                       /* out: the quantiser QP of each plane */
    int16_t* coef[2];                 /* [ncoef / 4] levels per plane: CU c's from cu_coef_off[c] / 4, TUs in RESID's order */
    DRV_PIXEL* recon[4][2];           /* per depth (64,32,16,8) and plane: origin pixels, cstride elements per row */
    uint64_t* cu_sse; uint32_t* cu_numsig;                /* [ncu][2] */
} drv_chroma_resid;

/* Quant::setChromaQP (quant.cpp:221-244) for 4:2:0 with qp = the slice QP + QP_BD_OFFSET (the analyser's quantiser QP) */
static int drv_chroma_qp(int qp, int offset)
{
    static const uint8_t chromaScale[58] = {              /* g_chromaScale (constants.cpp:346) */
        0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28, 29,
        29, 30, 31, 32, 33, 33, 34, 34, 35, 35, 36, 36, 37, 37, 38, 39, 40, 41, 42, 43, 44, 45, 46, 47, 48, 49, 50, 51 };
    const int bd = 6 * (DRV_DEPTH - 8);
    int q = qp - bd + offset;
    q = q < -bd ? -bd : (q > 57 ? 57 : q);
    if (q >= 30) q = chromaScale[q];
    return q + bd;
}

static void drv_chroma_one(drv_frame* f, drv_chroma_resid* cr, int c)
{
    const fs_params* p = &f->p;
    const int x = f->cus[c][0], y = f->cus[c][1], S = f->cus[c][2];
    const int cs = f->cstride, Sc = S / 2;
    int best = 0, bcost = 0x7fffffff;
    for (int r = 0; r < p->numRefs; r++)
    {
        int cost = f->me_out[(size_t)f->cu_jobs[c * p->numRefs + r] * 4];
        if (cost < bcost) { bcost = cost; best = r; }
    }
    const int32_t* mo = f->me_out + (size_t)f->cu_jobs[c * p->numRefs + best] * 4;
    const int qx = mo[1], qy = mo[2];
    const int T = S > 32 ? 32 : S, Tc = T / 2;
    const int lg = Tc == 16 ? 4 : (Tc == 8 ? 3 : 2);
    static const int quantScales[6] = { 26214, 23302, 20560, 18396, 16384, 14564 };   /* scalinglist.cpp:129 */
    static const int invQuantScales[6] = { 40, 45, 51, 57, 64, 72 };                  /* scalinglist.cpp:130 */
    for (int pl = 0; pl < 2; pl++)
    {
        const int qp = cr->qpc[pl];
        assert(qp >= 0 && qp <= 51 + 6 * (DRV_DEPTH - 8));
        const int per = qp / 6, rem = qp % 6;
        const int transformShift = 15 - DRV_DEPTH - lg;
        const int qbits = 14 + per + transformShift, add = 85 << (qbits - 9);
        const int dqshift = 20 - 14 - transformShift, dqscale = invQuantScales[rem] << per;
        int32_t qc[16 * 16];
        for (int i = 0; i < Tc * Tc; i++) qc[i] = quantScales[rem];
        /* chroma MC of the CU's 2Nx2N PU */
        DRV_PIXEL pred[32 * 32];
        const DRV_PIXEL* src = f->refC[best][pl] + (ptrdiff_t)(y / 2) * cs + x / 2 + (qx >> 3) + (ptrdiff_t)(qy >> 3) * cs;
        DRV_MC_C(src, cs, pred, Sc, S, qx & 7, qy & 7);
        const DRV_PIXEL* fenc = f->fencC[pl];
        DRV_PIXEL* recon = cr->recon[drv_depth_idx(S)][pl];
        uint64_t sse = 0; uint32_t nsig = 0;
        int t = 0;
        for (int ty = 0; ty < S; ty += T)
            for (int tx = 0; tx < S; tx += T, t++)
            {
                int16_t resi[16 * 16], coefd[16 * 16], deq[16 * 16];
                int32_t deltaU[16 * 16];
                const int cx = (x + tx) / 2, cy = (y + ty) / 2;
                int16_t* q = cr->coef[pl] + f->cu_coef_off[c] / 4 + (size_t)t * Tc * Tc;
                const DRV_PIXEL* fe = fenc + (ptrdiff_t)cy * cs + cx;
                const DRV_PIXEL* pr = pred + (ty / 2) * Sc + tx / 2;
                DRV_PIXEL* rc = recon + (ptrdiff_t)cy * cs + cx;
                DRV_SUB_PS(resi, Tc, fe, pr, cs, Sc, Tc);
                DRV_DCT(resi, coefd, Tc, Tc);
                uint32_t ns = DRV_QUANT(coefd, qc, deltaU, q, qbits, add, Tc * Tc);
                if (ns)
                {
                    DRV_DEQUANT(q, deq, Tc * Tc, dqscale, dqshift);
                    if (ns == 1 && q[0] != 0)
                    {   /* DC-only shortcut (quant.cpp:588-598) */
                        const int shift_2nd = 12 - (DRV_DEPTH - 8) - 3;
                        int dc = (((deq[0] * (64 >> 6) + 1) >> 1) * (64 >> 3) + (1 << (shift_2nd - 1))) >> shift_2nd;
                        DRV_BLOCKFILL(resi, Tc, (int16_t)dc, Tc);
                    }
                    else
                        DRV_IDCT(deq, resi, Tc, Tc);
                    DRV_ADD_PS(rc, cs, pr, resi, Sc, Tc, Tc);
                }
                else
                    DRV_COPY_PP(rc, cs, pr, Sc, Tc);
                sse += DRV_SSE(fe, cs, rc, cs, Tc);
                nsig += ns;
            }
        cr->cu_sse[2 * c + pl] = sse; cr->cu_numsig[2 * c + pl] = nsig;
    }
}

typedef struct { drv_frame* f; drv_chroma_resid* cr; volatile int next; } drv_chroma_run;

static void* drv_chroma_worker(void* arg)
{
    drv_chroma_run* r = (drv_chroma_run*)arg;
    for (;;)
    {
        int b = __sync_fetch_and_add(&r->next, 16);
        if (b >= r->f->ncu_run) break;
        int e = b + 16 < r->f->ncu_run ? b + 16 : r->f->ncu_run;
        for (int i = b; i < e; i++) drv_chroma_one(r->f, r->cr, i);
    }
    return NULL;
}

/* runs CHROMA RESID over the CUs of drv_prepare's rows (after the ME stage); needs f->chroma planes */
static void drv_run_chroma(drv_frame* f, drv_chroma_resid* cr)
{
    drv_chroma_run r;
    r.f = f; r.cr = cr; r.next = 0;
    cr->qpc[0] = drv_chroma_qp(f->p.qp, cr->offset[0]);
    cr->qpc[1] = drv_chroma_qp(f->p.qp, cr->offset[1]);
    int nt = f->threads < 1 ? 1 : f->threads;
    if (nt == 1) { drv_chroma_worker(&r); return; }
    pthread_t* th = (pthread_t*)malloc(sizeof(pthread_t) * nt);
    for (int t = 0; t < nt; t++) pthread_create(&th[t], NULL, drv_chroma_worker, &r);
    for (int t = 0; t < nt; t++) pthread_join(th[t], NULL);
    free(th);
}
#endif
