/* oracle/frame_bidir.h -- TEST INFRASTRUCTURE ONLY.
 * B slices of the frame-level CTU-analysis driver (x265cu_analyser_set_lists, stage bit 4), written once and instantiated
 * twice: by oracle_frame_bidir.c over the oracle's plain-C primitives and by ref_shim_bidir.cpp over the REAL reference code.
 * Include it after frame_wref.h (drv_wref_tus) with these macros defined:
 *   DRV_BIPRED(f, r0, mx0, my0, r1, mx1, my1, x, y, S, predY, predC, chroma): the bi-prediction of the S x S CU at (x, y),
 *     Predict::motionCompensation's two-list path (predict.cpp:168-189): predInterLumaShort / predInterChromaShort of slot r0
 *     at (mx0, my0) and of slot r1 at (mx1, my1), then Yuv::addAvg, into predY (pitch S) and, when chroma, predC[2] (pitch S/2);
 *   DRV_SA8D_C(a, sa, b, sb, S): primitives.chroma[X265_CSP_I420].cu[log2(S) - 2].sa8d of the chroma block of a luma S x S CU;
 *   DRV_IN_RANGE(px, py, mnx, mny, mxx, mxy): MV(px, py).checkRange(MV(mnx, mny), MV(mxx, mxy)).
 * The uni prediction is the residual stages' own (DRV_MC, DRV_MC_C), the luma cost DRV_SA8D (cu[].sa8d).
 *
 * BIDIR restates checkInter_rd0_4 for 2Nx2N and Analysis::checkBidir2Nx2N (analysis.cpp:3062-3071, 3145-3265) on the
 * analyser's cost model (include/x265_b200.h): per list the lowest ME cost of the CU's 2Nx2N jobs over the list's slots (ties
 * to the lowest), the uni winner list 0 iff cost0 <= cost1; uniCost, biCost and the zero pair's cost are sa8d (+ chroma sa8d)
 * plus the ME's mvcost of each vector against its job's MVP; the CU is bi-predicted iff biCost < uniCost.  The bi RESID /
 * CHROMA RESID of a bi-predicted CU code that bi-prediction with RESID's chain; every other CU runs RESID / CHROMA RESID as
 * they are, whose reference choice is the uni winner. */
#ifndef X265_FRAME_BIDIR_H
#define X265_FRAME_BIDIR_H
typedef struct {
    uint32_t uniCost, biCost;
    int8_t interDir, ref[2];
    uint8_t zero;
    int16_t mv[2][2];
} drv_bidir_cu;                       /* layout == x265cu_bidir_cu */

/* decision counters of a run */
enum { DRV_BD_BI, DRV_BD_UNI_L0, DRV_BD_UNI_L1, DRV_BD_TIE_L0, DRV_BD_ZERO_TRIED, DRV_BD_ZERO_TAKEN, DRV_BD_ZERO_OUT_OF_RANGE,
       DRV_BD_ZERO_SKIPPED, DRV_BD_NCOUNT };

typedef struct {
    int numRefL0;                     /* in: slots [0, numRefL0) are list 0, the rest list 1 */
    drv_bidir_cu* out;                /* [ncu] */
    int counts[DRV_BD_NCOUNT];
} drv_bidir;

static uint32_t drv_bd_mvcost(const drv_frame* f, int mvx, int mvy, int px, int py)
{
    return (uint16_t)(f->mvcost[mvx - px] + f->mvcost[mvy - py]);
}

/* sa8d of the CU's prediction (luma, + Cb and Cr when the frame has chroma) */
static uint32_t drv_bd_sa8d(const drv_frame* f, int x, int y, int S, const DRV_PIXEL* predY, DRV_PIXEL (*predC)[32 * 32])
{
    uint32_t cost = (uint32_t)DRV_SA8D(f->fenc + (intptr_t)y * f->p.stride + x, f->p.stride, predY, S, S);
    for (int pl = 0; pl < 2 && f->chroma; pl++)
        cost += (uint32_t)DRV_SA8D_C(f->fencC[pl] + (intptr_t)(y / 2) * f->cstride + x / 2, f->cstride, predC[pl], S / 2, S);
    return cost;
}

static void drv_bidir_one(drv_frame* f, drv_chroma_resid* cr, drv_bidir* b, int c, int luma, int chroma)
{
    const fs_params* p = &f->p;
    const int x = f->cus[c][0], y = f->cus[c][1], S = f->cus[c][2], nr = p->numRefs;
    int best[2] = { 0, b->numRefL0 }, bc[2] = { 0x7fffffff, 0x7fffffff };
    for (int r = 0; r < nr; r++)
    {
        const int l = r >= b->numRefL0, cost = f->me_out[(size_t)f->cu_jobs[c * nr + r] * 4];
        if (cost < bc[l]) { bc[l] = cost; best[l] = r; }
    }
    int mv[2][2], mvp[2][2];
    for (int l = 0; l < 2; l++)
    {
        const int j = f->cu_jobs[c * nr + best[l]];
        mv[l][0] = f->me_out[(size_t)j * 4 + 1]; mv[l][1] = f->me_out[(size_t)j * 4 + 2];
        mvp[l][0] = f->jobs[j].qmvp[0]; mvp[l][1] = f->jobs[j].qmvp[1];
    }
    const int u = bc[0] <= bc[1] ? 0 : 1;
    DRV_PIXEL predY[64 * 64], predC[2][32 * 32];
    /* uni: the pixel prediction of the residual stages */
    {
        const int qx = mv[u][0], qy = mv[u][1];
        DRV_MC(f->refs[best[u]] + (intptr_t)y * p->stride + x + (qx >> 2) + (intptr_t)(qy >> 2) * p->stride, p->stride, predY, S, S, qx & 3, qy & 3);
        for (int pl = 0; pl < 2 && f->chroma; pl++)
            DRV_MC_C(f->refC[best[u]][pl] + (intptr_t)(y / 2) * f->cstride + x / 2 + (qx >> 3) + (intptr_t)(qy >> 3) * f->cstride, f->cstride,
                     predC[pl], S / 2, S, qx & 7, qy & 7);
    }
    const uint32_t uniCost = drv_bd_sa8d(f, x, y, S, predY, predC) + drv_bd_mvcost(f, mv[u][0], mv[u][1], mvp[u][0], mvp[u][1]);
    DRV_BIPRED(f, best[0], mv[0][0], mv[0][1], best[1], mv[1][0], mv[1][1], x, y, S, predY, predC, f->chroma);
    uint32_t biCost = drv_bd_sa8d(f, x, y, S, predY, predC) + drv_bd_mvcost(f, mv[0][0], mv[0][1], mvp[0][0], mvp[0][1]) +
                      drv_bd_mvcost(f, mv[1][0], mv[1][1], mvp[1][0], mvp[1][1]);
    /* the zero pair: setSearchRange(cu, 0, max(width, height)) with fs_build_me_jobs' clip and the maxMvLen clamp
     * (search.cpp:2724-2768), then mvmax.y += 2 and both bounds << 2 (analysis.cpp:3204-3212) */
    int tryZero = (mv[0][0] | mv[0][1] | mv[1][0] | mv[1][1]) != 0, zero = 0;
    if (!tryZero) __sync_fetch_and_add(&b->counts[DRV_BD_ZERO_SKIPPED], 1);
    else
    {
        const int dist = (p->width > p->height ? p->width : p->height) << 2;
        const int xmax = (p->width + 8 - x - 1) << 2, xmin = -((64 + 8 + x - 1) << 2);
        const int ymax = (p->height + 8 - y - 1) << 2, ymin = -((64 + 8 + y - 1) << 2);
        int mnx = fs_clampi(-dist, xmin, xmax), mxx = fs_clampi(dist, xmin, xmax);
        int mny = fs_clampi(-dist, ymin, ymax), mxy = fs_clampi(dist, ymin, ymax);
        mnx = mnx < -32767 ? -32767 : mnx; mny = mny < -32767 ? -32767 : mny;
        mxx = mxx > 32767 ? 32767 : mxx; mxy = mxy > 32767 ? 32767 : mxy;
        mnx >>= 2; mny >>= 2; mxx >>= 2; mxy >>= 2;
        if (mxy < mny) mxy = mny;
        mxy += 2;
        mnx *= 4; mny *= 4; mxx *= 4; mxy *= 4;
        tryZero = DRV_IN_RANGE(mvp[0][0], mvp[0][1], mnx, mny, mxx, mxy) && DRV_IN_RANGE(mvp[1][0], mvp[1][1], mnx, mny, mxx, mxy);
        __sync_fetch_and_add(&b->counts[tryZero ? DRV_BD_ZERO_TRIED : DRV_BD_ZERO_OUT_OF_RANGE], 1);
    }
    if (tryZero)
    {
        DRV_PIXEL zY[64 * 64], zC[2][32 * 32];
        DRV_BIPRED(f, best[0], 0, 0, best[1], 0, 0, x, y, S, zY, zC, f->chroma);
        const uint32_t zCost = drv_bd_sa8d(f, x, y, S, zY, zC) + drv_bd_mvcost(f, 0, 0, mvp[0][0], mvp[0][1]) +
                               drv_bd_mvcost(f, 0, 0, mvp[1][0], mvp[1][1]);
        if (zCost < biCost)
        {
            biCost = zCost; zero = 1;
            mv[0][0] = mv[0][1] = mv[1][0] = mv[1][1] = 0;
            memcpy(predY, zY, sizeof(zY)); memcpy(predC, zC, sizeof(zC));
            __sync_fetch_and_add(&b->counts[DRV_BD_ZERO_TAKEN], 1);
        }
    }
    drv_bidir_cu* o = &b->out[c];
    o->uniCost = uniCost; o->biCost = biCost;
    o->interDir = (int8_t)(biCost < uniCost ? 3 : u + 1);
    o->ref[0] = (int8_t)best[0]; o->ref[1] = (int8_t)best[1]; o->zero = (uint8_t)zero;
    for (int l = 0; l < 2; l++) { o->mv[l][0] = (int16_t)mv[l][0]; o->mv[l][1] = (int16_t)mv[l][1]; }
    __sync_fetch_and_add(&b->counts[o->interDir == 3 ? DRV_BD_BI : (u ? DRV_BD_UNI_L1 : DRV_BD_UNI_L0)], 1);
    if (o->interDir == 1 && bc[0] == bc[1]) __sync_fetch_and_add(&b->counts[DRV_BD_TIE_L0], 1);
    /* the residual stages */
    if (o->interDir != 3)
    {
        if (luma) drv_resid_one(f, c);
        if (chroma) drv_chroma_one(f, cr, c);
        return;
    }
    const int T = S > 32 ? 32 : S, d = drv_depth_idx(S);
    if (luma)
    {
        const intptr_t off = (intptr_t)y * p->stride + x;
        f->cu_ref[c] = best[0];
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

typedef struct { drv_frame* f; drv_chroma_resid* cr; drv_bidir* b; int luma, chroma; volatile int next; } drv_bidir_run;

static void* drv_bidir_worker(void* arg)
{
    drv_bidir_run* r = (drv_bidir_run*)arg;
    for (;;)
    {
        int b = __sync_fetch_and_add(&r->next, 16);
        if (b >= r->f->ncu_run) break;
        int e = b + 16 < r->f->ncu_run ? b + 16 : r->f->ncu_run;
        for (int i = b; i < e; i++) drv_bidir_one(r->f, r->cr, r->b, i, r->luma, r->chroma);
    }
    return NULL;
}

/* BIDIR (stage bit 4) and the RESID (bit 1) / CHROMA RESID (bit 3) of a B slice over the CUs of drv_prepare's rows, after
 * the ME stage */
static void drv_run_bidir(drv_frame* f, drv_chroma_resid* cr, drv_bidir* b, int stages)
{
    drv_bidir_run r;
    r.f = f; r.cr = cr; r.b = b; r.luma = (stages & 2) != 0; r.chroma = (stages & 8) != 0; r.next = 0;
    memset(b->counts, 0, sizeof(b->counts));
    cr->qpc[0] = drv_chroma_qp(f->p.qp, cr->offset[0]);
    cr->qpc[1] = drv_chroma_qp(f->p.qp, cr->offset[1]);
    int nt = f->threads < 1 ? 1 : f->threads;
    if (nt == 1) { drv_bidir_worker(&r); return; }
    pthread_t* th = (pthread_t*)malloc(sizeof(pthread_t) * nt);
    for (int t = 0; t < nt; t++) pthread_create(&th[t], NULL, drv_bidir_worker, &r);
    for (int t = 0; t < nt; t++) pthread_join(th[t], NULL);
    free(th);
}
#endif
