/* oracle/oracle_frame_bidir.c -- TEST INFRASTRUCTURE ONLY (see frame_bidir.h).
 * The frame-level driver with the chroma residual stage and weighted references (oracle_frame_wref.c, included whole) plus
 * B slices, over the oracle's plain-C primitives.  Built by Makefile.bidir into liboracle_bidir{8,10}.so. */
#include "oracle_frame_wref.c"

/* predict.cpp:168-189: both lists through predInterLumaShort / predInterChromaShort (predict.cpp:268-304, 355-407), addAvg */
static void orc_short(const pixel* src, intptr_t ss, int16_t* d, int w, int xf, int yf, int nt)
{
    int16_t im[64 * (64 + 7)];
    if (!(xf | yf)) orc_p2s(src, ss, d, w, w, w);
    else if (!yf) orc_interp_hps(src, ss, d, w, xf, 0, nt, w, w);
    else if (!xf) orc_interp_vps(src, ss, d, w, yf, nt, w, w);
    else { orc_interp_hps(src, ss, im, w, xf, 1, nt, w, w); orc_interp_vss(im + (nt / 2 - 1) * w, w, d, w, yf, nt, w, w); }
}

static void orc_bipred(const drv_frame* f, int r0, int mx0, int my0, int r1, int mx1, int my1, int x, int y, int S, pixel* predY,
                       pixel (*predC)[32 * 32], int chroma)
{
    int16_t s0[64 * 64], s1[64 * 64];
    const intptr_t st = f->p.stride, cs = f->cstride;
    const int r[2] = { r0, r1 }, mv[2][2] = { { mx0, my0 }, { mx1, my1 } };
    for (int l = 0; l < 2; l++)
        orc_short(f->refs[r[l]] + y * st + x + (mv[l][0] >> 2) + (mv[l][1] >> 2) * st, st, l ? s1 : s0, S, mv[l][0] & 3, mv[l][1] & 3, 8);
    orc_addAvg(s0, s1, predY, S, S, S, S, S);
    for (int pl = 0; pl < 2 && chroma; pl++)
    {
        for (int l = 0; l < 2; l++)
            orc_short(f->refC[r[l]][pl] + (y / 2) * cs + x / 2 + (mv[l][0] >> 3) + (mv[l][1] >> 3) * cs, cs, l ? s1 : s0, S / 2,
                      mv[l][0] & 7, mv[l][1] & 7, 4);
        orc_addAvg(s0, s1, predC[pl], S / 2, S / 2, S / 2, S / 2, S / 2);
    }
}
#define DRV_BIPRED(f, r0, mx0, my0, r1, mx1, my1, x, y, S, pY, pC, c) orc_bipred(f, r0, mx0, my0, r1, mx1, my1, x, y, S, pY, pC, c)
#define DRV_SA8D_C(a, sa, b, sb, S) orc_sa8d(a, sa, b, sb, (S) / 2, (S) / 2)
#define DRV_IN_RANGE(px, py, mnx, mny, mxx, mxy) ((px) >= (mnx) && (px) <= (mxx) && (py) >= (mny) && (py) <= (mxy))
#include "frame_bidir.h"

/* orc_analyse_frame_chroma with B slices: ME (bit 0) and intra (bit 2) as they are, then BIDIR (bit 4) with RESID (bit 1) /
 * CHROMA RESID (bit 3) coding its decision */
int orc_analyse_frame_bidir(drv_frame* f, int stages, drv_chroma_resid* cr, drv_bidir* b)
{
    if ((stages & 8) && !f->chroma) return -1;
    orc_analyse_frame(f, stages & 5);
    drv_run_bidir(f, cr, b, stages);
    return 0;
}
