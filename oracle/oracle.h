/* oracle/oracle.h -- TEST INFRASTRUCTURE ONLY.
 *
 * Plain-C CPU restatement of x265's block-primitive hot path (the C entries of
 * EncoderPrimitives, /root/reference/source/common/primitives.h:237-429) and of the callers
 * whose semantics the batched device kernels reproduce (motion.cpp, slicetype.cpp, lowres.h).
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
 * load this library; the product (x265_b200/csrc, libx265cu.so) never links or calls it.
 *
 * Parity status: PINNED.  tests/test_oracle_vs_ref.py compares every function here against the
 * real reference C table compiled from /root/reference (oracle/_ref/libx265ref{8,10}.so) and
 * tests/golden/ holds vectors generated from that reference (tests/golden/make_golden.py).
 *
 * Compile with -DORC_DEPTH=8 or 10 (pixel = uint8_t / uint16_t, common/common.h:126-148).
 * Unlike the reference's templates, block sizes are runtime arguments.
 */
#ifndef X265_ORACLE_H
#define X265_ORACLE_H
#include <stdint.h>
#include <stddef.h>

#ifndef ORC_DEPTH
#define ORC_DEPTH 8
#endif
#if ORC_DEPTH == 8
typedef uint8_t  pixel;
typedef uint32_t sse_t;
#else
typedef uint16_t pixel;
typedef uint64_t sse_t;
#endif

#ifdef __cplusplus
extern "C" {
#endif

int orc_depth(void);

/* ---- pixel compare (pixel.cpp:40-377) ---- */
int  orc_sad(const pixel* a, intptr_t sa, const pixel* b, intptr_t sb, int w, int h);
void orc_sad_x3(const pixel* fenc, const pixel* r0, const pixel* r1, const pixel* r2, intptr_t rs, int32_t* res, int w, int h);
void orc_sad_x4(const pixel* fenc, const pixel* r0, const pixel* r1, const pixel* r2, const pixel* r3, intptr_t rs, int32_t* res, int w, int h);
int  orc_ads(const int* encDC, const uint32_t* sums, int delta, const uint16_t* costMvX, int16_t* mvs, int width, int thresh, int w, int h);
int  orc_satd(const pixel* a, intptr_t sa, const pixel* b, intptr_t sb, int w, int h);
int  orc_sa8d(const pixel* a, intptr_t sa, const pixel* b, intptr_t sb, int w, int h);
sse_t orc_sse_pp(const pixel* a, intptr_t sa, const pixel* b, intptr_t sb, int w, int h);
sse_t orc_sse_ss(const int16_t* a, intptr_t sa, const int16_t* b, intptr_t sb, int w, int h);
sse_t orc_ssd_s(const int16_t* a, intptr_t sa, int n);
uint64_t orc_var(const pixel* a, intptr_t sa, int n);
int  orc_psy_cost_pp(const pixel* src, intptr_t ss, const pixel* rec, intptr_t rs, int n);

/* ---- block ops (pixel.cpp:379-862) ---- */
void orc_copy_pp(pixel* d, intptr_t ds, const pixel* s, intptr_t ss, int w, int h);
void orc_copy_ss(int16_t* d, intptr_t ds, const int16_t* s, intptr_t ss, int w, int h);
void orc_copy_sp(pixel* d, intptr_t ds, const int16_t* s, intptr_t ss, int w, int h);
void orc_copy_ps(int16_t* d, intptr_t ds, const pixel* s, intptr_t ss, int w, int h);
void orc_sub_ps(int16_t* d, intptr_t ds, const pixel* a, const pixel* b, intptr_t sa, intptr_t sb, int w, int h);
void orc_add_ps(pixel* d, intptr_t ds, const pixel* a, const int16_t* r, intptr_t sa, intptr_t sr, int w, int h);
void orc_calcresidual(const pixel* fenc, const pixel* pred, int16_t* resi, intptr_t stride, int n);
void orc_pixelavg_pp(pixel* d, intptr_t ds, const pixel* a, intptr_t sa, const pixel* b, intptr_t sb, int w, int h);
void orc_addAvg(const int16_t* a, const int16_t* b, pixel* d, intptr_t sa, intptr_t sb, intptr_t ds, int w, int h);
void orc_transpose(pixel* d, const pixel* s, intptr_t stride, int n);
void orc_blockfill_s(int16_t* d, intptr_t ds, int16_t val, int n);
void orc_cpy2Dto1D_shl(int16_t* d, const int16_t* s, intptr_t ss, int shift, int n);
void orc_cpy2Dto1D_shr(int16_t* d, const int16_t* s, intptr_t ss, int shift, int n);
void orc_cpy1Dto2D_shl(int16_t* d, const int16_t* s, intptr_t ds, int shift, int n);
void orc_cpy1Dto2D_shr(int16_t* d, const int16_t* s, intptr_t ds, int shift, int n);
uint32_t orc_copy_cnt(int16_t* coeff, const int16_t* resi, intptr_t rs, int n);
int  orc_count_nonzero(const int16_t* q, int n);
void orc_scale2D_64to32(pixel* d, const pixel* s, intptr_t stride);
void orc_scale1D_128to64(pixel* d, const pixel* s);
void orc_weight_pp(const pixel* s, pixel* d, intptr_t stride, int width, int height, int w0, int round, int shift, int offset);
void orc_weight_sp(const int16_t* s, pixel* d, intptr_t ss, intptr_t ds, int width, int height, int w0, int round, int shift, int offset);
void orc_frame_init_lowres(const pixel* src0, pixel* dst0, pixel* dsth, pixel* dstv, pixel* dstc,
                           intptr_t src_stride, intptr_t dst_stride, int width, int height);
void orc_extend_pic_border(pixel* pic, intptr_t stride, int width, int height, int marginX, int marginY);

/* ---- SEA integral planes (framefilter.cpp:39-143) ---- */
void orc_integral_inith(uint32_t* sum, const pixel* pix, intptr_t stride, int n);
void orc_integral_initv(uint32_t* sum, intptr_t stride, int n);

/* ---- interpolation (ipfilter.cpp:40-369); ntaps = 8 (luma) or 4 (chroma) ---- */
void orc_p2s(const pixel* s, intptr_t ss, int16_t* d, intptr_t ds, int w, int h);
void orc_interp_hpp(const pixel* s, intptr_t ss, pixel* d, intptr_t ds, int coeffIdx, int ntaps, int w, int h);
void orc_interp_hps(const pixel* s, intptr_t ss, int16_t* d, intptr_t ds, int coeffIdx, int isRowExt, int ntaps, int w, int h);
void orc_interp_vpp(const pixel* s, intptr_t ss, pixel* d, intptr_t ds, int coeffIdx, int ntaps, int w, int h);
void orc_interp_vps(const pixel* s, intptr_t ss, int16_t* d, intptr_t ds, int coeffIdx, int ntaps, int w, int h);
void orc_interp_vsp(const int16_t* s, intptr_t ss, pixel* d, intptr_t ds, int coeffIdx, int ntaps, int w, int h);
void orc_interp_vss(const int16_t* s, intptr_t ss, int16_t* d, intptr_t ds, int coeffIdx, int ntaps, int w, int h);
void orc_interp_hvpp(const pixel* s, intptr_t ss, pixel* d, intptr_t ds, int idxX, int idxY, int ntaps, int w, int h);

/* ---- prediction costs around the motion search (oracle_pred.c: search.cpp:1901-2023, 2474-2607; predict.cpp:76-420) ---- */
struct orc_pred_job_s;
int orc_pred_cost(const struct orc_pred_job_s* j);      /* the job struct is defined in oracle_pred.c / tests/pred_helpers.py */
/* orc_pred_cost over x265cu_pred_job records, planes and tables as x265ref_pred_cost_batch (oracle/ref_shim.cpp) takes them */
int orc_pred_cost_batch(const pixel* fenc, const pixel* fencCb, const pixel* fencCr, const pixel* const* refs, const pixel* const* refCb,
                        const pixel* const* refCr, intptr_t stride, intptr_t cstride, const void* jobs, int n, int32_t* out);

/* ---- transforms / quant (dct.cpp:43-742) ---- */
const int16_t* orc_dct_matrix(int n);        /* n x n HEVC matrix, regenerated from the 32-pt basis */
void orc_dct(const int16_t* src, int16_t* dst, intptr_t srcStride, int n);
void orc_idct(const int16_t* src, int16_t* dst, intptr_t dstStride, int n);
void orc_dst4(const int16_t* src, int16_t* dst, intptr_t srcStride);
void orc_idst4(const int16_t* src, int16_t* dst, intptr_t dstStride);
uint32_t orc_quant(const int16_t* coef, const int32_t* quantCoeff, int32_t* deltaU, int16_t* qCoef, int qBits, int add, int numCoeff);
uint32_t orc_nquant(const int16_t* coef, const int32_t* quantCoeff, int16_t* qCoef, int qBits, int add, int numCoeff);
void orc_dequant_normal(const int16_t* q, int16_t* coef, int num, int scale, int shift);
void orc_dequant_scaling(const int16_t* q, const int32_t* dq, int16_t* coef, int num, int per, int shift);
void orc_denoise_dct(int16_t* dctCoef, uint32_t* resSum, const uint16_t* offset, int numCoeff);
void orc_propagate_cost(int* dst, const uint16_t* propagateIn, const int32_t* intraCosts, const uint16_t* interCosts,
                        const int32_t* invQscales, const double* fpsFactor, int len);

/* ---- intra (intrapred.cpp:31-234); srcPix = [topLeft, top 2N, left 2N] ---- */
void orc_intra_filter(const pixel* samples, pixel* filtered, int n);
void orc_intra_pred(pixel* dst, intptr_t dstStride, const pixel* srcPix, int dirMode, int bFilter, int n);
void orc_intra_pred_allangs(pixel* dst, const pixel* refPix, const pixel* filtPix, int bLuma, int n);

/* ---- callers: mvcost, motionEstimate, lowres (frame level) -- see oracle_me.c ---- */
void orc_mvcost_table(double lambda, int range, uint16_t* out /* 2*range+1, centred */);

typedef struct {
    const pixel* fenc;      /* source plane */
    intptr_t fencStride;
    intptr_t offset;        /* block origin, same offset in fenc and ref planes (element units) */
    const pixel* ref[4];    /* full-res: ref[0]; lowres: the 4 hpel planes */
    intptr_t refStride;
    int lowres;             /* 1: lowres.h:67-120 qpel-by-averaging path */
    int pw, ph;             /* PU size */
    int method;             /* 0 DIA, 1 HEX, 2 UMH, 3 STAR, 4 SEA (needs `integral`), 5 FULL (x265.h X265_*_SEARCH) */
    int subme;              /* 0..7 (motion.cpp:48-58) */
    int mvmin[2], mvmax[2]; /* full-pel */
    int qmvp[2];            /* qpel predictor */
    int numCand; const int* mvc; /* qpel candidates (x,y pairs) */
    int merange;
    const uint16_t* mvcost; /* centred table (index 0 = mvd 0), qpel units */
    /* chroma-SATD term of subpelCompare (motion.cpp:1601-1661), 4:2:0: when `chroma` != 0, subme > 2 and the chroma
     * block has a SATD (motion.cpp:204-212: pw and ph multiples of 8), every subpelCompare adds the Cb and Cr SATD.
     * Planes are half resolution, `cstride` pixels per row; the PU's chroma origin is
     * ((offset / fencStride) >> 1) * cstride + ((offset % fencStride) >> 1) from the pointers given. */
    int chroma;
    const pixel* fencC[2];  /* source Cb, Cr (origin pixel) */
    const pixel* refC[2];   /* reference Cb, Cr (origin pixel) */
    intptr_t cstride;
    /* X265_SEA (method 4; motion.cpp:1242-1395): the 12 integral planes of the reference picture (FrameFilter::computeMEIntegral,
     * framefilter.cpp:725-822; orc_build_integral) at pixel (0, 0); the search adds `offset` as Search::predInterSearch does
     * (search.cpp:2264).  NULL for the other methods. */
    const uint32_t* const* integral;
} orc_me_job;
int orc_motion_estimate(const orc_me_job* job, int* outQMv);
/* planes[k] = pixel (0, 0) of integral plane k in a buffer of the picture plane's geometry (same stride, >= padY + 1 rows above,
 * >= padX columns left); picHeightCtu = picture height in 64-pixel CTU rows.  k: 0 32x32, 1 32x24, 2 32x8, 3 24x32, 4 16x16,
 * 5 16x12, 6 16x4, 7 12x16, 8 8x32, 9 8x8, 10 4x16, 11 4x4 (width x height of the box sums). */
void orc_build_integral(const pixel* picOrg, intptr_t stride, int picHeightCtu, uint32_t* const* planes);

#ifdef __cplusplus
}
#endif
#endif
