/* oracle/oracle_frame_part.c -- TEST INFRASTRUCTURE ONLY (see frame_part.h).
 * The frame-level driver with the chroma residual stage, weighted references and B slices (oracle_frame_bidir.c, included
 * whole) plus the PART stage, over the oracle's plain-C primitives.  Built by Makefile.part into liboracle_part{8,10}.so. */
#include "oracle_frame_bidir.c"

struct drv_part_pu_s;
static void orc_part_pred(const drv_frame* f, const drv_wref* w, int x, int y, int S, int npu, const struct drv_part_pu_s* pu, pixel* predY,
                          pixel (*predC)[32 * 32], int chroma);
#define DRV_PART_PRED(f, w, x, y, S, npu, pu, pY, pC, c) orc_part_pred(f, w, x, y, S, npu, pu, pY, pC, c)
#include "frame_part.h"

/* one plane of one PU (w x h, NT taps) into dst: the pixel path of predInterLumaPixel / predInterChromaPixel (predict.cpp:
 * 245-266, 306-353), or with a weight entry e the 14-bit path of predInterLumaShort / predInterChromaShort (predict.cpp:
 * 268-304, 355-407) and addWeightUni's weight_sp (predict.cpp:525-578) */
static void orc_part_plane(const pixel* src, intptr_t ss, pixel* dst, intptr_t ds, int w, int h, int xf, int yf, int nt, const int32_t* e)
{
    int16_t im[64 * (64 + 7)], sh[64 * 64];
    if (!e)
    {
        if (!(xf | yf)) orc_copy_pp(dst, ds, src, ss, w, h);
        else if (!yf) orc_interp_hpp(src, ss, dst, ds, xf, nt, w, h);
        else if (!xf) orc_interp_vpp(src, ss, dst, ds, yf, nt, w, h);
        else if (nt == 8) orc_interp_hvpp(src, ss, dst, ds, xf, yf, 8, w, h);
        else { orc_interp_hps(src, ss, im, w, xf, 1, nt, w, h); orc_interp_vsp(im + (nt / 2 - 1) * w, w, dst, ds, yf, nt, w, h); }
        return;
    }
    if (!(xf | yf)) orc_p2s(src, ss, sh, w, w, h);
    else if (!yf) orc_interp_hps(src, ss, sh, w, xf, 0, nt, w, h);
    else if (!xf) orc_interp_vps(src, ss, sh, w, yf, nt, w, h);
    else { orc_interp_hps(src, ss, im, w, xf, 1, nt, w, h); orc_interp_vss(im + (nt / 2 - 1) * w, w, sh, w, yf, nt, w, h); }
    const int shift = e[2] + 14 - ORC_DEPTH;
    orc_weight_sp(sh, dst, w, ds, w, h, e[1], 1 << (shift - 1), shift, e[3] * (1 << (ORC_DEPTH - 8)));
}

static void orc_part_pred(const drv_frame* f, const drv_wref* w, int x, int y, int S, int npu, const struct drv_part_pu_s* pu, pixel* predY,
                          pixel (*predC)[32 * 32], int chroma)
{
    const intptr_t st = f->p.stride, cs = f->cstride;
    for (int u = 0; u < npu; u++)
    {
        const drv_part_pu* q = &pu[u];
        const int wt = w->wp[q->slot][0][0] != 0, px = x + q->rx, py = y + q->ry;
        orc_part_plane(w->refs[q->slot] + py * st + px + (q->mvx >> 2) + (q->mvy >> 2) * st, st, predY + q->ry * S + q->rx, S,
                       q->pw, q->ph, q->mvx & 3, q->mvy & 3, 8, wt ? w->wp[q->slot][0] : NULL);
        for (int pl = 0; pl < 2 && chroma; pl++)
            orc_part_plane(w->refC[q->slot][pl] + (py / 2) * cs + px / 2 + (q->mvx >> 3) + (q->mvy >> 3) * cs, cs,
                           predC[pl] + (q->ry / 2) * (S / 2) + q->rx / 2, S / 2, q->pw / 2, q->ph / 2, q->mvx & 7, q->mvy & 7, 4,
                           wt ? w->wp[q->slot][1 + pl] : NULL);
    }
}


/* orc_analyse_frame with the PART stage: ME (bit 0), RESID (bit 1) and intra (bit 2) as they are, then PART (bit 5) into `pt` */
int orc_analyse_frame_part(drv_frame* f, int stages, drv_part* pt)
{
    orc_analyse_frame(f, stages & 7);
    if (stages & 32) drv_run_part(f, pt);
    return 0;
}
