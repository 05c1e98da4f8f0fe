/* oracle/frame_part_b.h -- TEST INFRASTRUCTURE ONLY.
 * The PART_B stage of the frame-level CTU-analysis driver (stage bit 6, a B slice: the inter estimate of every partition of
 * every CU with predInterSearch's per-PU list choice and bi-prediction), written once and instantiated twice: by
 * oracle_frame_part_b.c over the oracle's plain-C primitives and by ref_shim_part_b.cpp over the REAL reference code.
 * Include it after frame_part.h (drv_wref, drv_bd_sa8d, drv_bd_mvcost, DRV_IN_RANGE) with these macros defined:
 *   DRV_PART_BI_COST(f, w, px, py, pw, ph, s0, mx0, my0, s1, mx1, my1, chroma, avgPP): predInterSearch's bi try of the pw x ph
 *     PU at (px, py) (search.cpp:2486-2511): bufSATD of the bi-prediction of slots s0 / s1 at the pair, pixelavg_pp of the two
 *     pixel predictions when avgPP, else addAvg of the two 14-bit predictions + bufChromaSATD; `chroma` is the chroma
 *     enable and subme > 2, which with the PU's size makes the search's bChromaSATD, and avgPP its negation;
 *   DRV_PART_B_PRED(f, w, x, y, S, npu, pu, predY, predC, chroma): the final prediction of the partition's PUs pu[0 .. npu)
 *     (drv_part_b_pu) into the CU's prediction predY (pitch S) and, when chroma, predC[2] (pitch S/2): a uni PU's pixel
 *     prediction from its list's slot, a bi PU's addAvg of both lists' 14-bit predictions (Predict::motionCompensation's
 *     B-slice path, predict.cpp:119-240).
 * The costs are DRV_SA8D / DRV_SA8D_C through drv_bd_sa8d, as in PART.
 *
 * PART_B restates PART (frame_part.h) for a B slice with predInterSearch's B-slice path (search.cpp:2473-2644) per PU
 * (include/x265_b200.h, x265cu_part_b_cu): per list the slot of lowest ME cost among the PU's jobs in that list, the bi try
 * (not 2Nx2N, not a CU 8) with the zero pair against the CU's BIDIR range, bi iff biCost < cost0 and biCost < cost1, else list
 * 0 iff cost0 <= cost1; the CU's cost is sa8d of the final prediction plus every PU's mvcost. */
#ifndef X265_FRAME_PART_B_H
#define X265_FRAME_PART_B_H
typedef struct {
    uint32_t cost[8], sa8d[8], biCost[8][2];
    int8_t interDir[8][2], ref[8][2][2];
    uint8_t zero[8][2];
    int16_t mv[8][2][2][2];
} drv_part_b_cu;                      /* layout == x265cu_part_b_cu */

/* decision counters of a run, per PU: its direction (and uni L0 by a tie), the bi try refused to a CU 8's PU, the bi try's
 * cost path, the zero pair's fate */
enum { DRV_PB_BI, DRV_PB_UNI_L0, DRV_PB_UNI_L1, DRV_PB_TIE_L0, DRV_PB_BI_CU8, DRV_PB_CHROMA_SATD, DRV_PB_AVG_PP, DRV_PB_ZERO_TRIED,
       DRV_PB_ZERO_TAKEN, DRV_PB_ZERO_OUT_OF_RANGE, DRV_PB_ZERO_SKIPPED, DRV_PB_NCOUNT };

/* one PU of a B partition: its place and size in the CU, each list's slot, its direction (1 L0, 2 L1, 3 bi) and the vectors
 * its prediction uses (a bi PU's pair after the zero try) */
typedef struct drv_part_b_pu_s { int rx, ry, pw, ph, slot[2], dir, mv[2][2]; } drv_part_b_pu;

typedef struct {
    drv_wref w;                       /* in: the unweighted planes (a B slice has no weighted slot) */
    int numRefL0;                     /* in: slots [0, numRefL0) are list 0, the rest list 1 */
    drv_part_b_cu* out;               /* [ncu] */
    int counts[DRV_PB_NCOUNT];
} drv_part_b;

static void drv_part_b_one(drv_frame* f, drv_part_b* pb, int c)
{
    const fs_params* p = &f->p;
    const int x = f->cus[c][0], y = f->cus[c][1], S = f->cus[c][2], nr = p->numRefs;
    drv_part_b_cu* o = &pb->out[c];
    memset(o, 0, sizeof(*o));
    memset(o->ref, -1, sizeof(o->ref));
    for (int ps = 0; ps < 8; ps++)
    {
        o->cost[ps] = o->sa8d[ps] = 0xffffffffu;
        o->biCost[ps][0] = o->biCost[ps][1] = 0xffffffffu;
    }
    /* the zero try's range: BIDIR's, per CU (search.cpp:2515-2529) */
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
    int k = 0;                        /* PU index in the CU's jobs */
    for (int ps = 0; ps < 8; ps++)
    {
        if (!(ps == 0 || ((ps == 1 || ps == 2) && p->rect) || (ps >= 4 && p->amp && S >= 16))) continue;
        const int npu = ps ? 2 : 1;
        drv_part_b_pu pu[2];
        uint32_t mvcost = 0;
        for (int u = 0; u < npu; u++, k++)
        {
            /* 1. per list the best job */
            int best[2] = { 0, pb->numRefL0 }, bc[2] = { 0x7fffffff, 0x7fffffff }, mv[2][2], mvp[2][2];
            for (int r = 0; r < nr; r++)
            {
                const int l = r >= pb->numRefL0, cost = f->me_out[(size_t)(f->cu_jobs[c * nr + r] + k) * 4];
                if (cost < bc[l]) { bc[l] = cost; best[l] = r; }
            }
            for (int l = 0; l < 2; l++)
            {
                const int j = f->cu_jobs[c * nr + best[l]] + k;
                mv[l][0] = f->me_out[(size_t)j * 4 + 1]; mv[l][1] = f->me_out[(size_t)j * 4 + 2];
                mvp[l][0] = f->jobs[j].qmvp[0]; mvp[l][1] = f->jobs[j].qmvp[1];
            }
            const fs_me_job* jb = &f->jobs[f->cu_jobs[c * nr + best[0]] + k];
            drv_part_b_pu* q = &pu[u];
            q->pw = jb->pw; q->ph = jb->ph;
            q->rx = jb->offset % p->stride - x; q->ry = jb->offset / p->stride - y;
            assert(q->rx >= 0 && q->ry >= 0 && q->rx + q->pw <= S && q->ry + q->ph <= S);
            q->slot[0] = best[0]; q->slot[1] = best[1];
            /* 2. the bi try (search.cpp:2478-2591) */
            uint32_t biCost = 0xffffffffu;
            int zero = 0, bv[2][2] = { { mv[0][0], mv[0][1] }, { mv[1][0], mv[1][1] } };
            if (ps && S == 8) __sync_fetch_and_add(&pb->counts[DRV_PB_BI_CU8], 1);
            if (ps && S > 8)
            {
                const int chroma = f->chroma && p->subme > 2;
                const int chromaSatd = chroma && !((q->pw / 2) & 3) && !((q->ph / 2) & 3);
                __sync_fetch_and_add(&pb->counts[chromaSatd ? DRV_PB_CHROMA_SATD : DRV_PB_AVG_PP], 1);
                biCost = (uint32_t)DRV_PART_BI_COST(f, &pb->w, x + q->rx, y + q->ry, q->pw, q->ph, best[0], mv[0][0], mv[0][1], best[1], mv[1][0],
                                                    mv[1][1], chroma, !chromaSatd) +
                         drv_bd_mvcost(f, mv[0][0], mv[0][1], mvp[0][0], mvp[0][1]) + drv_bd_mvcost(f, mv[1][0], mv[1][1], mvp[1][0], mvp[1][1]);
                int tryZero = (mv[0][0] | mv[0][1] | mv[1][0] | mv[1][1]) != 0;
                if (!tryZero) __sync_fetch_and_add(&pb->counts[DRV_PB_ZERO_SKIPPED], 1);
                else
                {
                    tryZero = DRV_IN_RANGE(mvp[0][0], mvp[0][1], mnx, mny, mxx, mxy) && DRV_IN_RANGE(mvp[1][0], mvp[1][1], mnx, mny, mxx, mxy);
                    __sync_fetch_and_add(&pb->counts[tryZero ? DRV_PB_ZERO_TRIED : DRV_PB_ZERO_OUT_OF_RANGE], 1);
                }
                if (tryZero)
                {
                    const uint32_t zCost = (uint32_t)DRV_PART_BI_COST(f, &pb->w, x + q->rx, y + q->ry, q->pw, q->ph, best[0], 0, 0, best[1], 0, 0,
                                                                      chroma, !chromaSatd) +
                                           drv_bd_mvcost(f, 0, 0, mvp[0][0], mvp[0][1]) + drv_bd_mvcost(f, 0, 0, mvp[1][0], mvp[1][1]);
                    if (zCost < biCost)
                    {
                        biCost = zCost; zero = 1;
                        memset(bv, 0, sizeof(bv));
                        __sync_fetch_and_add(&pb->counts[DRV_PB_ZERO_TAKEN], 1);
                    }
                }
            }
            /* 3. the direction (search.cpp:2593-2642) */
            q->dir = biCost < (uint32_t)bc[0] && biCost < (uint32_t)bc[1] ? 3 : bc[0] <= bc[1] ? 1 : 2;
            __sync_fetch_and_add(&pb->counts[q->dir == 3 ? DRV_PB_BI : q->dir == 1 ? DRV_PB_UNI_L0 : DRV_PB_UNI_L1], 1);
            if (q->dir == 1 && bc[0] == bc[1]) __sync_fetch_and_add(&pb->counts[DRV_PB_TIE_L0], 1);
            for (int l = 0; l < 2; l++)
            {
                const int* v = q->dir == 3 ? bv[l] : mv[l];
                q->mv[l][0] = v[0]; q->mv[l][1] = v[1];
                if (q->dir == 3 || q->dir == l + 1) mvcost += drv_bd_mvcost(f, v[0], v[1], mvp[l][0], mvp[l][1]);
                o->ref[ps][u][l] = (int8_t)best[l];
                o->mv[ps][u][l][0] = (int16_t)bv[l][0]; o->mv[ps][u][l][1] = (int16_t)bv[l][1];
            }
            o->biCost[ps][u] = biCost; o->interDir[ps][u] = (int8_t)q->dir; o->zero[ps][u] = (uint8_t)zero;
        }
        /* 4. the CU's prediction and costs */
        DRV_PIXEL predY[64 * 64], predC[2][32 * 32];
        DRV_PART_B_PRED(f, &pb->w, x, y, S, npu, pu, predY, predC, f->chroma);
        const uint32_t sa8d = drv_bd_sa8d(f, x, y, S, predY, predC);
        o->cost[ps] = sa8d + mvcost; o->sa8d[ps] = sa8d;
    }
}

typedef struct { drv_frame* f; drv_part_b* pb; volatile int next; } drv_part_b_run;

static void* drv_part_b_worker(void* arg)
{
    drv_part_b_run* r = (drv_part_b_run*)arg;
    for (;;)
    {
        int b = __sync_fetch_and_add(&r->next, 16);
        if (b >= r->f->ncu_run) break;
        int e = b + 16 < r->f->ncu_run ? b + 16 : r->f->ncu_run;
        for (int i = b; i < e; i++) drv_part_b_one(r->f, r->pb, i);
    }
    return NULL;
}

/* PART_B (stage bit 6) over the CUs of drv_prepare's rows, after the ME stage, threaded as drv_run_part */
static void drv_run_part_b(drv_frame* f, drv_part_b* pb)
{
    drv_part_b_run r;
    r.f = f; r.pb = pb; r.next = 0;
    memset(pb->counts, 0, sizeof(pb->counts));
    const int nt = f->threads < 1 ? 1 : f->threads;
    pthread_t* th = nt > 1 ? (pthread_t*)malloc(sizeof(pthread_t) * (nt - 1)) : NULL;
    int started = 0;
    for (int t = 0; th && t < nt - 1; t++)
        if (pthread_create(&th[started], NULL, drv_part_b_worker, &r) == 0) started++;
    drv_part_b_worker(&r);
    for (int t = 0; t < started; t++) pthread_join(th[t], NULL);
    free(th);
}
#endif
