/* oracle/ref_shim_chroma.cpp -- TEST INFRASTRUCTURE ONLY (never linked into the product).
 * ref_shim.cpp (included whole) plus the 4:2:0 chroma residual stage of the frame driver (frame_chroma.h) on the REAL
 * reference table, and the real Quant::setChromaQP.  Built by Makefile.chroma with the reference objects into
 * oracle/_ref/libx265ref_chroma{8,10}.so. */
#include "ref_shim.cpp"
#include "quant.h"

/* Predict::predInterChromaPixel (predict.cpp:306-353) of the luma S x S PU, 4:2:0: the real chroma pu[partEnum] entries */
#define DRV_MC_C(src, ss, dst, ds, S, xf, yf) do { int part_ = partitionFromSizes(S, S); \
        const auto& cp_ = g_c.chroma[X265_CSP_I420].pu[part_]; \
        if (!((xf) | (yf))) cp_.copy_pp(dst, ds, src, ss); \
        else if (!(yf)) cp_.filter_hpp(src, ss, dst, ds, xf); \
        else if (!(xf)) cp_.filter_vpp(src, ss, dst, ds, yf); \
        else { ALIGN_VAR_32(int16_t, im_[MAX_CU_SIZE * (MAX_CU_SIZE + NTAPS_CHROMA - 1)]); const intptr_t is_ = (S) / 2; \
               cp_.filter_hps(src, ss, im_, is_, xf, 1); cp_.filter_vsp(im_ + (NTAPS_CHROMA / 2 - 1) * is_, is_, dst, ds, yf); } } while (0)
#include "frame_chroma.h"

/* x265ref_analyse_frame with bit 3: the 4:2:0 chroma residual stage on the real table into `cr` */
extern "C" int x265ref_analyse_frame_chroma(drv_frame* f, int stages, drv_chroma_resid* cr)
{
    if ((stages & 8) && !f->chroma) return -1;
    x265ref_analyse_frame(f, stages & 7);
    if (stages & 8) drv_run_chroma(f, cr);
    return 0;
}

/* the REAL Quant::setChromaQP (quant.cpp:221-244, protected) for 4:2:0, as Quant::setQPforQuant calls it: qp = the slice QP
 * + QP_BD_OFFSET, offset = PPS + slice offset.  Returns the quantiser QP it sets for Cb. */
struct QuantPeek : public Quant
{
    int chroma(int qpin) { setChromaQP(qpin, TEXT_CHROMA_U, X265_CSP_I420); return m_qpParam[TEXT_CHROMA_U].qp; }
};
extern "C" int x265ref_chroma_qp(int qp, int offset)
{
    QuantPeek q;
    return q.chroma(qp - QP_BD_OFFSET + offset);
}
