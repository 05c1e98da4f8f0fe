/* oracle/frame_part.h -- TEST INFRASTRUCTURE ONLY.
 * The PART stage of the frame-level CTU-analysis driver (stage bit 5, a P slice: the inter estimate of every partition of every
 * CU), written once and instantiated twice: by oracle_frame_part.c over the oracle's plain-C primitives and by ref_shim_part.cpp
 * over the REAL reference code.  Include it after frame_wref.h (drv_wref) and frame_bidir.h (drv_bd_sa8d, drv_bd_mvcost) with
 * this macro defined:
 *   DRV_PART_PRED(f, w, x, y, S, npu, pu, predY, predC, chroma): the prediction of the partition's PUs pu[0 .. npu) of the S x S CU
 *     at (x, y) into the CU's prediction predY (pitch S) and, when chroma, predC[2] (pitch S/2), each PU from its slot's
 *     unweighted planes in w (a `const drv_wref*`): predInterLumaPixel / predInterChromaPixel, or for a slot whose luma entry
 *     has wtPresent predInterLumaShort / predInterChromaShort + addWeightUni (Predict::motionCompensation, predict.cpp:82-118).
 * The costs are DRV_SA8D (cu[].sa8d) and DRV_SA8D_C (chroma[I420].cu[].sa8d) through drv_bd_sa8d.
 *
 * PART restates checkInter_rd0_4's sa8dCost (analysis.cpp:3023-3071) for every partition the geometry emits (2Nx2N; 2NxN and
 * Nx2N with rect; 2NxnU, 2NxnD, nLx2N and nRx2N with amp at CU >= 16) on the analyser's cost model (include/x265_b200.h,
 * x265cu_part_cu): each PU takes the slot of lowest ME cost over its jobs (ties to the lowest), its vector is that job's ME
 * result; sa8d of the CU's prediction (+ Cb and Cr with chroma) plus the ME's mvcost of every PU against its job's MVP.  The
 * PUs of a CU's partitions are the jobs that follow its 2Nx2N job in the job list (frame_spec.h), and their geometry is read
 * from those jobs. */
#ifndef X265_FRAME_PART_H
#define X265_FRAME_PART_H
typedef struct {
    uint32_t cost[8], sa8d[8];
    int8_t ref[8][2];
    int16_t mv[8][2][2];
} drv_part_cu;                        /* layout == x265cu_part_cu */

/* one PU of a partition: its slot, its place (rx, ry) and size in the CU, its quarter-pel vector */
typedef struct drv_part_pu_s { int slot, rx, ry, pw, ph, mvx, mvy; } drv_part_pu;

typedef struct {
    drv_wref w;                       /* in: the weights of every slot and the unweighted planes */
    drv_part_cu* out;                 /* [ncu] */
} drv_part;

static void drv_part_one(drv_frame* f, const drv_part* pt, int c)
{
    const fs_params* p = &f->p;
    const int x = f->cus[c][0], y = f->cus[c][1], S = f->cus[c][2], nr = p->numRefs;
    drv_part_cu* o = &pt->out[c];
    for (int ps = 0; ps < 8; ps++)
    {
        o->cost[ps] = o->sa8d[ps] = 0xffffffffu;
        o->ref[ps][0] = o->ref[ps][1] = -1;
        o->mv[ps][0][0] = o->mv[ps][0][1] = o->mv[ps][1][0] = o->mv[ps][1][1] = 0;
    }
    int k = 0;                        /* PU index in the CU's jobs */
    for (int ps = 0; ps < 8; ps++)
    {
        if (!(ps == 0 || ((ps == 1 || ps == 2) && p->rect) || (ps >= 4 && p->amp && S >= 16))) continue;
        const int npu = ps ? 2 : 1;
        drv_part_pu pu[2];
        uint32_t mvcost = 0;
        for (int u = 0; u < npu; u++, k++)
        {
            int best = 0, bc = 0x7fffffff;
            for (int r = 0; r < nr; r++)
            {
                const int cost = f->me_out[(size_t)(f->cu_jobs[c * nr + r] + k) * 4];
                if (cost < bc) { bc = cost; best = r; }
            }
            const int j = f->cu_jobs[c * nr + best] + k;
            const fs_me_job* jb = &f->jobs[j];
            pu[u].slot = best; pu[u].pw = jb->pw; pu[u].ph = jb->ph;
            pu[u].rx = jb->offset % p->stride - x; pu[u].ry = jb->offset / p->stride - y;
            assert(jb->ref == best && pu[u].rx >= 0 && pu[u].ry >= 0 && pu[u].rx + pu[u].pw <= S && pu[u].ry + pu[u].ph <= S);
            pu[u].mvx = f->me_out[(size_t)j * 4 + 1]; pu[u].mvy = f->me_out[(size_t)j * 4 + 2];
            mvcost += drv_bd_mvcost(f, pu[u].mvx, pu[u].mvy, jb->qmvp[0], jb->qmvp[1]);
        }
        DRV_PIXEL predY[64 * 64], predC[2][32 * 32];
        DRV_PART_PRED(f, &pt->w, x, y, S, npu, pu, predY, predC, f->chroma);
        const uint32_t sa8d = drv_bd_sa8d(f, x, y, S, predY, predC);
        o->cost[ps] = sa8d + mvcost; o->sa8d[ps] = sa8d;
        for (int u = 0; u < npu; u++)
        {
            o->ref[ps][u] = (int8_t)pu[u].slot;
            o->mv[ps][u][0] = (int16_t)pu[u].mvx; o->mv[ps][u][1] = (int16_t)pu[u].mvy;
        }
    }
}

typedef struct { drv_frame* f; const drv_part* pt; volatile int next; } drv_part_run;

static void* drv_part_worker(void* arg)
{
    drv_part_run* r = (drv_part_run*)arg;
    for (;;)
    {
        int b = __sync_fetch_and_add(&r->next, 16);
        if (b >= r->f->ncu_run) break;
        int e = b + 16 < r->f->ncu_run ? b + 16 : r->f->ncu_run;
        for (int i = b; i < e; i++) drv_part_one(r->f, r->pt, i);
    }
    return NULL;
}

/* PART (stage bit 5) over the CUs of drv_prepare's rows, after the ME stage.  The calling thread takes CUs too, so the stage
 * completes with whatever helper threads could be started (none where the process may not create more) and joins only those. */
static void drv_run_part(drv_frame* f, const drv_part* pt)
{
    drv_part_run r;
    r.f = f; r.pt = pt; r.next = 0;
    const int nt = f->threads < 1 ? 1 : f->threads;
    pthread_t* th = nt > 1 ? (pthread_t*)malloc(sizeof(pthread_t) * (nt - 1)) : NULL;
    int started = 0;
    for (int t = 0; th && t < nt - 1; t++)
        if (pthread_create(&th[started], NULL, drv_part_worker, &r) == 0) started++;
    drv_part_worker(&r);
    for (int t = 0; t < started; t++) pthread_join(th[t], NULL);
    free(th);
}
#endif
