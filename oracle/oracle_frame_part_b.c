/* oracle/oracle_frame_part_b.c -- TEST INFRASTRUCTURE ONLY (see frame_part_b.h).
 * The frame-level driver with the PART stage (oracle_frame_part.c, included whole) plus the PART_B stage, over the oracle's
 * plain-C primitives.  Built by Makefile.part_b into liboracle_part_b{8,10}.so. */
#include "oracle_frame_part.c"

static int orc_part_bi_cost(const drv_frame* f, const drv_wref* w, int px, int py, int pw, int ph, int s0, int mx0, int my0, int s1,
                            int mx1, int my1, int chroma, int avgPP);
#define DRV_PART_BI_COST(f, w, px, py, pw, ph, s0, mx0, my0, s1, mx1, my1, c, a) orc_part_bi_cost(f, w, px, py, pw, ph, s0, mx0, my0, s1, mx1, my1, c, a)
struct drv_part_b_pu_s;
static void orc_part_b_pred(const drv_frame* f, const drv_wref* w, int x, int y, int S, int npu, const struct drv_part_b_pu_s* pu,
                            pixel* predY, pixel (*predC)[32 * 32], int chroma);
#define DRV_PART_B_PRED(f, w, x, y, S, npu, pu, pY, pC, c) orc_part_b_pred(f, w, x, y, S, npu, pu, pY, pC, c)
#include "frame_part_b.h"

/* the bi try's cost: orc_pred_cost (oracle_pred.c), the two-list SATD of predInterSearch, on the PU's planes */
struct orc_pred_job_s
{
    const pixel* fenc[3]; const pixel* ref0[3]; const pixel* ref1[3];
    intptr_t stride, cstride;
    int w, h, mv0[2], mv1[2], cost, chroma, biAvgPP;
};                                    /* layout == oracle_pred.c's orc_pred_job */

static int orc_part_bi_cost(const drv_frame* f, const drv_wref* w, int px, int py, int pw, int ph, int s0, int mx0, int my0, int s1,
                            int mx1, int my1, int chroma, int avgPP)
{
    const intptr_t st = f->p.stride, cs = f->cstride, off = py * st + px, coff = (py / 2) * cs + px / 2;
    struct orc_pred_job_s j;
    j.fenc[0] = f->fenc + off; j.ref0[0] = w->refs[s0] + off; j.ref1[0] = w->refs[s1] + off;
    for (int pl = 0; pl < 2; pl++)
    {
        j.fenc[1 + pl] = chroma ? f->fencC[pl] + coff : NULL;
        j.ref0[1 + pl] = chroma ? w->refC[s0][pl] + coff : NULL;
        j.ref1[1 + pl] = chroma ? w->refC[s1][pl] + coff : NULL;
    }
    j.stride = st; j.cstride = cs; j.w = pw; j.h = ph;
    j.mv0[0] = mx0; j.mv0[1] = my0; j.mv1[0] = mx1; j.mv1[1] = my1;
    j.cost = 1; j.chroma = chroma; j.biAvgPP = avgPP;
    return orc_pred_cost(&j);
}

/* the final prediction of a B partition: the uni PUs through orc_part_pred, each bi PU the rectangle of frame_bidir.h's CU
 * bi-prediction (orc_bipred) at its pair that the PU covers */
static void orc_part_b_pred(const drv_frame* f, const drv_wref* w, int x, int y, int S, int npu, const struct drv_part_b_pu_s* pu,
                            pixel* predY, pixel (*predC)[32 * 32], int chroma)
{
    for (int u = 0; u < npu; u++)
    {
        const drv_part_b_pu* q = &pu[u];
        if (q->dir != 3)
        {
            const int l = q->dir - 1;
            const drv_part_pu up = { q->slot[l], q->rx, q->ry, q->pw, q->ph, q->mv[l][0], q->mv[l][1] };
            orc_part_pred(f, w, x, y, S, 1, &up, predY, predC, chroma);
            continue;
        }
        pixel bY[64 * 64], bC[2][32 * 32];
        orc_bipred(f, q->slot[0], q->mv[0][0], q->mv[0][1], q->slot[1], q->mv[1][0], q->mv[1][1], x, y, S, bY, bC, chroma);
        for (int i = 0; i < q->ph; i++) memcpy(predY + (q->ry + i) * S + q->rx, bY + (q->ry + i) * S + q->rx, sizeof(pixel) * q->pw);
        for (int pl = 0; pl < 2 && chroma; pl++)
            for (int i = 0; i < q->ph / 2; i++)
                memcpy(predC[pl] + (q->ry / 2 + i) * (S / 2) + q->rx / 2, bC[pl] + (q->ry / 2 + i) * (S / 2) + q->rx / 2, sizeof(pixel) * (q->pw / 2));
    }
}

/* orc_analyse_frame with the PART_B stage: ME (bit 0) and intra (bit 2) as they are, then PART_B (bit 6) into `pb` */
int orc_analyse_frame_part_b(drv_frame* f, int stages, drv_part_b* pb)
{
    orc_analyse_frame(f, stages & 5);
    if (stages & 64) drv_run_part_b(f, pb);
    return 0;
}
