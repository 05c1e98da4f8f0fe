/* oracle/oracle_frame_wref.c -- TEST INFRASTRUCTURE ONLY (see frame_wref.h).
 * The frame-level driver with the chroma residual stage (oracle_frame_chroma.c, included whole) plus weighted P-slice
 * references, over the oracle's plain-C primitives.  Built by Makefile.wref into liboracle_wref{8,10}.so. */
#include "oracle_frame_chroma.c"

struct drv_wref_s;
static void orc_wpred(const struct drv_wref_s* w, int r, int x, int y, int S, int qx, int qy, intptr_t stride, intptr_t cs, pixel* predY,
                      pixel (*predC)[32 * 32], int luma, int chroma);
#define DRV_WPRED(w, r, x, y, S, qx, qy, st, cs, pY, pC, l, c) orc_wpred(w, r, x, y, S, qx, qy, st, cs, pY, pC, l, c)
#include "frame_wref.h"

/* Predict::motionCompensation's weighted P path (predict.cpp:82-112): predInterLumaShort / predInterChromaShort (predict.cpp:
 * 268-304, 355-407) of the unweighted planes, then addWeightUni (predict.cpp:525-578) with the WeightValues of predict.cpp:96-102 */
static void orc_wpred(const struct drv_wref_s* w, int r, int x, int y, int S, int qx, int qy, intptr_t stride, intptr_t cs, pixel* predY,
                      pixel (*predC)[32 * 32], int luma, int chroma)
{
    int16_t sh[64 * 64], im[64 * (64 + 7)];
    const int corr = 14 - ORC_DEPTH;
    if (luma)
    {
        const int32_t* e = w->wp[r][0];
        const pixel* src = w->refs[r] + (intptr_t)y * stride + x + (qx >> 2) + (intptr_t)(qy >> 2) * stride;
        const int xf = qx & 3, yf = qy & 3;
        if (!(xf | yf)) orc_p2s(src, stride, sh, S, S, S);
        else if (!yf) orc_interp_hps(src, stride, sh, S, xf, 0, 8, S, S);
        else if (!xf) orc_interp_vps(src, stride, sh, S, yf, 8, S, S);
        else { orc_interp_hps(src, stride, im, S, xf, 1, 8, S, S); orc_interp_vss(im + 3 * S, S, sh, S, yf, 8, S, S); }
        const int shift = e[2] + corr;
        orc_weight_sp(sh, predY, S, S, S, S, e[1], 1 << (shift - 1), shift, e[3] * (1 << (ORC_DEPTH - 8)));
    }
    for (int pl = 0; pl < 2 && chroma; pl++)
    {
        const int32_t* e = w->wp[r][1 + pl];
        const int Sc = S / 2, xf = qx & 7, yf = qy & 7;
        const pixel* src = w->refC[r][pl] + (intptr_t)(y / 2) * cs + x / 2 + (qx >> 3) + (intptr_t)(qy >> 3) * cs;
        if (!(xf | yf)) orc_p2s(src, cs, sh, Sc, Sc, Sc);
        else if (!yf) orc_interp_hps(src, cs, sh, Sc, xf, 0, 4, Sc, Sc);
        else if (!xf) orc_interp_vps(src, cs, sh, Sc, yf, 4, Sc, Sc);
        else { orc_interp_hps(src, cs, im, Sc, xf, 1, 4, Sc, Sc); orc_interp_vss(im + Sc, Sc, sh, Sc, yf, 4, Sc, Sc); }
        const int shift = e[2] + corr;
        orc_weight_sp(sh, predC[pl], Sc, Sc, Sc, Sc, e[1], 1 << (shift - 1), shift, e[3] * (1 << (ORC_DEPTH - 8)));
    }
}

/* the search planes of one reference as MotionReference::init + applyWeight leave them (frame_wref.h drv_wref_plane): luma
 * weighted when wp[0] has wtPresent, each chroma plane when its own entry has it too and subme > 2 (numInterpPlanes = 3,
 * reference.cpp:57); other planes are copied.  Planes are origin pointers with the analyser's margins (96 x 80, 48 x 40).
 * Returns whether the reference is weighted.  The arguments are x265ref_wref_planes'. */
int orc_wref_planes(const pixel* y, const pixel* cb, const pixel* cr, intptr_t stride, intptr_t cstride, int width, int height,
                    int method, int subme, int merange, const int32_t* wp, pixel* oy, pixel* ocb, pixel* ocr)
{
    (void)method; (void)merange;                  /* they set applyWeight's row lag, which does not change the result */
    const pixel* in[3] = { y, cb, cr };
    pixel* out[3] = { oy, ocb, ocr };
    const int on = wp[0] != 0;
    for (int c = 0; c < 3; c++)
    {
        const int ch = c > 0, mx = ch ? 48 : 96, my = ch ? 40 : 80, w = width >> ch, h = height >> ch;
        const intptr_t s = ch ? cstride : stride;
        if (!out[c]) continue;
        if (on && wp[4 * c] && (c == 0 || subme > 2))
            drv_wref_plane(in[c], out[c], s, w, h, mx, my, wp + 4 * c);
        else
            for (int r = -my; r < h + my; r++) memcpy(out[c] + r * s - mx, in[c] + r * s - mx, sizeof(pixel) * (w + 2 * mx));
    }
    return on;
}

/* orc_analyse_frame_chroma with weighted references: f->refs / refC = what the search reads, w = weights + unweighted planes */
int orc_analyse_frame_wref(drv_frame* f, int stages, drv_chroma_resid* cr, const drv_wref* w)
{
    if ((stages & 8) && !f->chroma) return -1;
    orc_analyse_frame(f, stages & 5);
    drv_run_wref(f, cr, w, stages);
    return 0;
}
