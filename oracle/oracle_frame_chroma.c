/* oracle/oracle_frame_chroma.c -- TEST INFRASTRUCTURE ONLY (see frame_chroma.h).
 * The frame-level driver over the oracle's plain-C primitives (oracle_frame.c, included whole) plus its 4:2:0 chroma
 * residual stage.  Built by Makefile.chroma into liboracle_chroma{8,10}.so in place of oracle_frame.c. */
#include "oracle_frame.c"

/* predInterChromaPixel (predict.cpp:306-353) of the luma S x S PU: an (S/2) x (S/2) block, 4-tap eighth-pel filters */
#define DRV_MC_C(src, ss, dst, ds, S, xf, yf) do { const int w_ = (S) / 2; \
        if (!((xf) | (yf))) orc_copy_pp(dst, ds, src, ss, w_, w_); \
        else if (!(yf)) orc_interp_hpp(src, ss, dst, ds, xf, 4, w_, w_); \
        else if (!(xf)) orc_interp_vpp(src, ss, dst, ds, yf, 4, w_, w_); \
        else { int16_t im_[32 * (32 + 3)]; orc_interp_hps(src, ss, im_, w_, xf, 1, 4, w_, w_); \
               orc_interp_vsp(im_ + w_, w_, dst, ds, yf, 4, w_, w_); } } while (0)
#include "frame_chroma.h"

/* orc_analyse_frame with bit 3: the 4:2:0 chroma residual stage into `cr` (needs the frame's chroma planes) */
int orc_analyse_frame_chroma(drv_frame* f, int stages, drv_chroma_resid* cr)
{
    if ((stages & 8) && !f->chroma) return -1;
    orc_analyse_frame(f, stages & 7);
    if (stages & 8) drv_run_chroma(f, cr);
    return 0;
}

/* the quantiser QP of a chroma plane (Quant::setChromaQP restated, drv_chroma_qp) */
int orc_chroma_qp(int qp, int offset) { return drv_chroma_qp(qp, offset); }
