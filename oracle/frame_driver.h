/* oracle/frame_driver.h -- TEST INFRASTRUCTURE ONLY.
 * CPU driver of the frame-level CTU-analysis workload (see frame_spec.h / DESIGN.md), written once
 * and instantiated twice: by oracle_frame.c over the oracle's plain-C primitives, and by
 * ref_shim.cpp over the REAL reference primitive table + MotionEstimate class (oracle/_ref), which
 * is the "reference" CPU arm of bench.py.  The including file defines the DRV_* macros.
 *
 * Stages (each is what the corresponding x265 caller does with the primitives):
 *   ME      per PU x ref: MotionEstimate::motionEstimate                       (motion.cpp:739)
 *   RESID   per CU: best ref by ME cost, luma MC (predict.cpp:245-266), then per TU
 *           sub_ps -> dct -> quant -> dequant_normal -> idct (DC shortcut) -> add_ps -> sse_pp
 *           (search.cpp:3178 estimateResidualQT, quant.cpp:397-470 and :543-605, non-RDOQ path)
 *   INTRA   per CU (8..32): neighbours from the source plane (slicetype.cpp:729-733 style),
 *           intra_filter, 35 predictions, sa8d each                              (search.cpp:1358-1444)
 */
#ifndef X265_FRAME_DRIVER_H
#define X265_FRAME_DRIVER_H
#include "frame_spec.h"
#include <assert.h>
#include <pthread.h>
#include <stdlib.h>
#include <string.h>

typedef struct {
    fs_params p;
    const DRV_PIXEL* fenc;            /* origin pixel (0,0) of the source plane (margins extended) */
    const DRV_PIXEL* refs[16];        /* origin pixels of the reference planes */
    const int16_t* field;             /* predictor field */
    const uint16_t* mvcost;           /* centred mvcost table */
    /* outputs */
    int njobs; fs_me_job* jobs; int32_t* me_out;          /* [njobs][4] cost, qmvx, qmvy, 0 */
    int ncu; int16_t (*cus)[3]; int32_t* cu_jobs;         /* [ncu][numRefs] job index of the CU's 2Nx2N PU */
    int64_t* cu_coef_off;                                 /* [ncu] offset into coef */
    int16_t* coef;                                        /* quantised levels, per CU contiguous, TU raster */
    DRV_PIXEL* recon[4];                                  /* per depth (64,32,16,8) planes, same geometry as fenc */
    uint64_t* cu_sse; uint32_t* cu_numsig; int32_t* cu_ref;  /* [ncu] */
    uint32_t* intra_cost;                                 /* [ncu][36]: 35 mode costs + best mode (0 for 64x64 CUs) */
    int threads;
    volatile int next;
    int stage;
    /* 4:2:0 chroma for the chroma-SATD term of subpelCompare (motion.cpp:204-212, 1601-1661; MotionEstimate::bChromaSATD).
     * chroma != 0: every ME job runs as the encoder runs it for a 4:2:0 source (setSourcePU with bChroma = true).
     * Planes are half resolution, origin pixels, `cstride` elements per row, margins = half the luma margins. */
    int chroma, cstride;
    const DRV_PIXEL* fencC[2];        /* source Cb, Cr */
    const DRV_PIXEL* refC[16][2];     /* reference Cb, Cr */
    /* bounded samples (bench.py cpu_baseline): analyse only the CTU rows [0, maxCtuRows) of the FULL-frame geometry
     * (0 = all rows).  The lists are in CTU raster order, so these rows are a prefix of every list and their results are
     * what a full-frame run produces for them. */
    int maxCtuRows, njobs_run, ncu_run;
} drv_frame;

static inline int drv_depth_idx(int size) { return size == 64 ? 0 : (size == 32 ? 1 : (size == 16 ? 2 : 3)); }

static void drv_me_one(drv_frame* f, int i);
static void drv_resid_one(drv_frame* f, int i);
static void drv_intra_one(drv_frame* f, int i);

static void* drv_worker(void* arg)
{
    drv_frame* f = (drv_frame*)arg;
    const int total = f->stage == 0 ? f->njobs_run : f->ncu_run;
    const int chunk = f->stage == 0 ? 64 : 16;
    for (;;)
    {
        int b = __sync_fetch_and_add(&f->next, chunk);
        if (b >= total) break;
        int e = b + chunk < total ? b + chunk : total;
        for (int i = b; i < e; i++)
        {
            if (f->stage == 0) drv_me_one(f, i);
            else if (f->stage == 1) drv_resid_one(f, i);
            else drv_intra_one(f, i);
        }
    }
    return NULL;
}

static void drv_run_stage(drv_frame* f, int stage)
{
    f->stage = stage; f->next = 0;
    int nt = f->threads < 1 ? 1 : f->threads;
    if (nt == 1) { drv_worker(f); return; }
    pthread_t* th = (pthread_t*)malloc(sizeof(pthread_t) * nt);
    for (int t = 0; t < nt; t++) pthread_create(&th[t], NULL, drv_worker, f);
    for (int t = 0; t < nt; t++) pthread_join(th[t], NULL);
    free(th);
}

/* build job list, CU list and the CU -> 2Nx2N job map */
static void drv_prepare(drv_frame* f)
{
    const fs_params* p = &f->p;
    f->njobs = fs_build_me_jobs(p, f->field, f->jobs);
    f->ncu = fs_build_cus(p->width, p->height, f->cus);
    /* map: walk jobs; a job is a CU's 2Nx2N PU iff pw == ph and its origin/size equals a CU */
    int64_t off = 0;
    for (int c = 0; c < f->ncu; c++) { f->cu_coef_off[c] = off; off += (int64_t)f->cus[c][2] * f->cus[c][2]; }
    /* index CUs by (x, y, size) through a direct table on the 8x8 grid */
    const int gw = (p->width + 7) / 8, gh = (p->height + 7) / 8;
    int32_t* grid = (int32_t*)malloc(sizeof(int32_t) * gw * gh * 4);
    memset(grid, 0xff, sizeof(int32_t) * gw * gh * 4);
    for (int c = 0; c < f->ncu; c++)
        grid[((f->cus[c][1] / 8) * gw + f->cus[c][0] / 8) * 4 + drv_depth_idx(f->cus[c][2])] = c;
    for (int i = 0; i < f->njobs; i++)
    {
        const fs_me_job* j = &f->jobs[i];
        if (j->pw != j->ph) continue;
        int x = j->offset % p->stride, y = j->offset / p->stride;
        int c = grid[((y / 8) * gw + x / 8) * 4 + drv_depth_idx(j->pw)];
        f->cu_jobs[c * p->numRefs + j->ref] = i;
    }
    free(grid);
    f->njobs_run = f->njobs; f->ncu_run = f->ncu;
    if (f->maxCtuRows > 0)
    {
        const int ylim = 64 * f->maxCtuRows;
        int nj = 0, nc = 0;
        while (nj < f->njobs && f->jobs[nj].offset / p->stride < ylim) nj++;
        while (nc < f->ncu && f->cus[nc][1] < ylim) nc++;
        f->njobs_run = nj; f->ncu_run = nc;
    }
}

static void drv_me_one(drv_frame* f, int i)
{
    int32_t* o = f->me_out + (size_t)i * 4;
    int qmv[2];
    o[0] = DRV_ME(f, &f->jobs[i], qmv);
    o[1] = qmv[0]; o[2] = qmv[1]; o[3] = 0;
}

static void drv_resid_one(drv_frame* f, int c)
{
    const fs_params* p = &f->p;
    const int x = f->cus[c][0], y = f->cus[c][1], S = f->cus[c][2];
    const int stride = p->stride;
    /* best reference by ME cost (ties: lowest index) */
    int best = 0, bcost = 0x7fffffff;
    for (int r = 0; r < p->numRefs; r++)
    {
        int cost = f->me_out[(size_t)f->cu_jobs[c * p->numRefs + r] * 4];
        if (cost < bcost) { bcost = cost; best = r; }
    }
    const int32_t* mo = f->me_out + (size_t)f->cu_jobs[c * p->numRefs + best] * 4;
    const int qx = mo[1], qy = mo[2];
    f->cu_ref[c] = best;
    /* luma MC (predict.cpp:245-266) */
    DRV_PIXEL pred[64 * 64];
    const DRV_PIXEL* src = f->refs[best] + (size_t)y * stride + x + (qx >> 2) + (ptrdiff_t)(qy >> 2) * stride;
    DRV_MC(src, stride, pred, S, S, qx & 3, qy & 3);
    /* TUs */
    const int T = S > 32 ? 32 : S;
    const int lg = T == 32 ? 5 : (T == 16 ? 4 : (T == 8 ? 3 : 2));
    /* the quantiser's QPs are 0..51 + QP_BD_OFFSET (quant.cpp:224); a negative QP would index the tables at rem < 0 */
    assert(p->qp >= 0 && p->qp <= 51 + 6 * (DRV_DEPTH - 8));
    const int per = p->qp / 6, rem = p->qp % 6;
    static const int quantScales[6] = { 26214, 23302, 20560, 18396, 16384, 14564 };   /* scalinglist.cpp:129 */
    static const int invQuantScales[6] = { 40, 45, 51, 57, 64, 72 };                  /* scalinglist.cpp:130 */
    const int transformShift = 15 - DRV_DEPTH - lg;                                    /* quant.cpp:411 */
    const int qbits = 14 + per + transformShift;                                       /* quant.cpp:465 */
    const int add = 85 << (qbits - 9);                                                 /* quant.cpp:466 (non-I slice) */
    const int dqshift = 20 - 14 - transformShift;                                      /* quant.cpp:556 */
    const int dqscale = invQuantScales[rem] << per;                                    /* quant.cpp:567 */
    int32_t qc[32 * 32];
    for (int i = 0; i < T * T; i++) qc[i] = quantScales[rem];
    DRV_PIXEL* recon = f->recon[drv_depth_idx(S)];
    uint64_t sse = 0; uint32_t nsig = 0;
    int t = 0;
    for (int ty = 0; ty < S; ty += T)
        for (int tx = 0; tx < S; tx += T, t++)
        {
            int16_t resi[32 * 32], coefd[32 * 32], deq[32 * 32];
            int32_t deltaU[32 * 32];
            int16_t* q = f->coef + f->cu_coef_off[c] + (size_t)t * T * T;
            const DRV_PIXEL* fe = f->fenc + (size_t)(y + ty) * stride + x + tx;
            const DRV_PIXEL* pr = pred + ty * S + tx;
            DRV_PIXEL* rc = recon + (size_t)(y + ty) * stride + x + tx;
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
    f->cu_sse[c] = sse; f->cu_numsig[c] = nsig;
}

static void drv_intra_one(drv_frame* f, int c)
{
    const fs_params* p = &f->p;
    const int x = f->cus[c][0], y = f->cus[c][1], S = f->cus[c][2];
    uint32_t* out = f->intra_cost + (size_t)c * 36;
    if (S == 64) { memset(out, 0, 36 * sizeof(uint32_t)); return; }
    const int stride = p->stride;
    const DRV_PIXEL* o = f->fenc + (size_t)y * stride + x;
    DRV_PIXEL nb[129], filt[129], pred[32 * 32];
    nb[0] = o[-stride - 1];
    for (int i = 0; i < 2 * S; i++) { nb[1 + i] = o[-stride + i]; nb[2 * S + 1 + i] = o[(ptrdiff_t)i * stride - 1]; }
    DRV_INTRA_FILTER(nb, filt, S);
    uint32_t bestc = 0xffffffffu; int bestm = 0;
    for (int mode = 0; mode < 35; mode++)
    {
        int useF = DRV_USE_FILTERED(mode, S);
        DRV_INTRA_PRED(pred, S, useF ? filt : nb, mode, S <= 16, S);
        uint32_t cost = (uint32_t)DRV_SA8D(o, stride, pred, S, S);
        out[mode] = cost;
        if (cost < bestc) { bestc = cost; bestm = mode; }
    }
    out[35] = (uint32_t)bestm;
}

static void drv_analyse(drv_frame* f)
{
    drv_prepare(f);
    drv_run_stage(f, 0);
    drv_run_stage(f, 1);
    drv_run_stage(f, 2);
}
#endif
