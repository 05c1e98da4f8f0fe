/* include/x265_b200.h -- C ABI of libx265cu.so, the H100-native (sm_90a) implementation of x265's
 * block-primitive hot path.  Plain C: pointers and sizes only, no CUDA/torch types.
 *
 * Two levels, both replacing entries of the reference's EncoderPrimitives table
 * (/root/reference/source/common/primitives.h:237-429):
 *
 *  (1) PER-CALL TABLE  -- x265cu_get_primitive() hands out C function pointers with EXACTLY the
 *      reference typedefs (primitives.h:133-234): host pointers, strides in elements, caller-owned
 *      buffers, outputs fully overwritten, nothing retained.  setupCudaPrimitives() (the drop-in
 *      sibling of setupAssemblyPrimitives(), primitives.h:470, call site primitives.cpp:260-265)
 *      fills an EncoderPrimitives from these; see INTEGRATION.md.  Each call stages the block to the
 *      device, runs the same kernels as (2) with a batch of one, and copies the result back.
 *
 *  (2) BATCHED API     -- one launch per primitive class over a job list (all candidates x all CTUs
 *      of a frame / row), on device-resident planes.  This is what the batching hooks at
 *      CostEstimateGroup::finishBatch (slicetype.cpp:1942-2009) and FrameEncoder::processRowEncoder
 *      (frameencoder.cpp:1340) call.  `_dev` arguments are device pointers obtained from
 *      x265cu_malloc(); every function returns 0 on success, -1 on a CUDA error (message via
 *      x265cu_last_error()); there is NO CPU fallback.
 *
 * depth is 8 (pixel = uint8_t) or 10 (pixel = uint16_t), cf. common/common.h:126-148.
 */
#ifndef X265_B200_H
#define X265_B200_H
#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct x265cu_ctx x265cu_ctx;

/* ---------- context / memory ---------- */
int  x265cu_device_count(void);
x265cu_ctx* x265cu_create(int device);                 /* NULL if no CUDA device (never falls back) */
void x265cu_destroy(x265cu_ctx*);
const char* x265cu_last_error(void);
int  x265cu_sync(x265cu_ctx*);
void* x265cu_stream(x265cu_ctx*);                       /* cudaStream_t the ctx launches on */
void* x265cu_malloc(x265cu_ctx*, size_t bytes);
void  x265cu_free(x265cu_ctx*, void* dev);
void* x265cu_host_alloc(size_t bytes);                  /* pinned host memory */
void  x265cu_host_free(void* p);
int  x265cu_h2d(x265cu_ctx*, void* dev, const void* host, size_t bytes);   /* async on ctx stream */
int  x265cu_d2h(x265cu_ctx*, void* host, const void* dev, size_t bytes);   /* async on ctx stream */
int  x265cu_memset(x265cu_ctx*, void* dev, int value, size_t bytes);
/* strided 2-D copy on the context's stream (asynchronous): kind 0 = host->device, 1 = device->host, 2 = device->device */
int  x265cu_copy2d(x265cu_ctx*, void* dst, size_t dpitch, const void* src, size_t spitch, size_t widthBytes, size_t rows, int kind);
/* timing on the ctx stream (cudaEvent): returns ms between begin/end, <0 on error */
int  x265cu_timer_begin(x265cu_ctx*);
float x265cu_timer_end(x265cu_ctx*);
/* number of kernels this library has launched since the ctx was created */
uint64_t x265cu_launch_count(x265cu_ctx*);   /* kernel launches of the whole process so far (all contexts, per-call table included) */
/* device ms of the three launches of the last motion-estimation batch: pre-checks, integer search, sub-pel */
int x265cu_me_phase_ms(x265cu_ctx*, float ms[3]);

/* ---------- (1) per-call table ---------- */
/* name / i / j / k exactly as the fields of EncoderPrimitives: "pu.sad" (i = LumaPU),
 * "cu.dct" (i = LumaCU), "cu.intra_pred" (i = LumaCU, j = mode), "quant",
 * "chroma.pu.filter_hpp" (k = csp, i = LumaPU) ...  Returns NULL for entries we do not provide. */
void* x265cu_get_primitive(int depth, const char* name, int i, int j, int k);
/* Error convention of the per-call table (SURVEY 8b): the reference's primitives are void / value-returning and cannot
 * fail, so a CUDA failure inside a thunk never kills the process: the thunk logs, returns zeros and latches this flag.
 * The encoder-side hook polls it after x265_encoder_encode() and sets m_aborted (encoder/api.cpp:179-180, 222-229), so the
 * next x265_encoder_encode() returns < 0.  X265CU_DEVICE (environment) selects the GPU of the per-call table. */
int x265cu_primitive_error(void);
const char* x265cu_primitive_error_string(void);
void x265cu_primitive_error_clear(void);
uint64_t x265cu_primitive_calls(void);     /* per-call table invocations of this process so far (diagnostics) */

/* ---------- (2) batched API ---------- */

/* pixel-compare class: sad / satd / sa8d / sse / var / psy   (pixel.cpp:40-377, 167-186, 703-757) */
enum { X265CU_SAD = 0, X265CU_SATD = 1, X265CU_SA8D = 2, X265CU_SSE_PP = 3, X265CU_SSE_SS = 4,
       X265CU_SSD_S = 5, X265CU_VAR = 6, X265CU_PSY = 7 };
typedef struct {
    int64_t a_off, b_off;      /* element offsets into plane A / plane B */
    int32_t a_stride, b_stride;
    int16_t w, h;
    int32_t pad;
} x265cu_cmp_job;
/* out_dev[n] : uint64 (sse_t / var packing as in the reference; int costs zero-extended) */
int x265cu_pixelcmp_batch(x265cu_ctx*, int depth, int op, const void* planeA_dev, const void* planeB_dev,
                          const x265cu_cmp_job* jobs_dev, int n, uint64_t* out_dev);
/* Same costs over a regular grid: block (bx,by) compares A + by*bh*a_stride + bx*bw with the same
 * offset from B (the displacement of a whole-frame compare is baked into B); strides in pixels;
 * op = SAD / SATD / SA8D / SSE_PP; out_dev[by*nbx + bx].  This is the shape of the frame-level cost
 * passes (lowres SATD maps, slicetype.cpp:640-700; weightp cost, slicetype.cpp:462-520): no job list,
 * one lane per 16-byte column so plane reads are fully coalesced. */
int x265cu_pixelcmp_grid(x265cu_ctx*, int depth, int op, const void* A_dev, int64_t a_stride, const void* B_dev, int64_t b_stride,
                         int bw, int bh, int nbx, int nby, uint64_t* out_dev);

/* elementwise block-op class (pixel.cpp:379-862, ipfilter.cpp:40-57) */
enum { X265CU_COPY_PP = 0, X265CU_COPY_SS, X265CU_COPY_SP, X265CU_COPY_PS, X265CU_SUB_PS, X265CU_ADD_PS,
       X265CU_PIXELAVG_PP, X265CU_ADDAVG, X265CU_P2S, X265CU_TRANSPOSE, X265CU_BLOCKFILL_S,
       X265CU_CPY2DTO1D_SHL, X265CU_CPY2DTO1D_SHR, X265CU_CPY1DTO2D_SHL, X265CU_CPY1DTO2D_SHR,
       X265CU_WEIGHT_PP, X265CU_WEIGHT_SP, X265CU_SCALE2D_64TO32, X265CU_DEQUANT_NORMAL };
typedef struct {
    int64_t d_off, a_off, b_off;        /* element offsets into dst / srcA / srcB buffers */
    int32_t d_stride, a_stride, b_stride;
    int16_t w, h;
    int32_t p0, p1, p2, p3;             /* op parameters (shift / value / weights) */
} x265cu_blk_job;
int x265cu_blockop_batch(x265cu_ctx*, int depth, int op, void* dst_dev, const void* a_dev, const void* b_dev,
                         const x265cu_blk_job* jobs_dev, int n);

/* interpolation class (ipfilter.cpp:79-369) */
enum { X265CU_HPP = 0, X265CU_HPS, X265CU_VPP, X265CU_VPS, X265CU_VSP, X265CU_VSS, X265CU_HVPP };
typedef struct {
    int64_t s_off, d_off;
    int32_t s_stride, d_stride;
    int16_t w, h;
    int8_t  idxX, idxY, rowExt, ntaps;   /* ntaps 8 (luma) / 4 (chroma) */
} x265cu_interp_job;
int x265cu_interp_batch(x265cu_ctx*, int depth, int op, const void* src_dev, void* dst_dev,
                        const x265cu_interp_job* jobs_dev, int n);

/* transform / quant class (dct.cpp:43-742).  Blocks are n contiguous TUs. */
enum { X265CU_DCT = 0, X265CU_IDCT = 1, X265CU_DST4 = 2, X265CU_IDST4 = 3 };
/* src: strided 2-D (stride elements between rows, tu_pitch elements between TUs) for DCT;
 * dst contiguous N*N per TU.  For IDCT the roles swap (dst strided). */
int x265cu_transform_batch(x265cu_ctx*, int depth, int op, int size, const int16_t* src_dev, int16_t* dst_dev,
                           int stride, int64_t tu_pitch, int n);
/* quant over n TUs of numCoeff each; quantCoeff shared by all TUs (numCoeff entries).
 * numSig_dev[n] receives the per-TU return value.  deltaU_dev may be NULL (nquant semantics when
 * `nquant` != 0: |level| stored). */
int x265cu_quant_batch(x265cu_ctx*, const int16_t* coef_dev, const int32_t* quantCoeff_dev, int32_t* deltaU_dev,
                       int16_t* qCoef_dev, int qBits, int add, int numCoeff, int n, int nquant, uint32_t* numSig_dev);
int x265cu_dequant_normal_batch(x265cu_ctx*, const int16_t* q_dev, int16_t* coef_dev, int64_t num, int scale, int shift);
int x265cu_dequant_scaling_batch(x265cu_ctx*, const int16_t* q_dev, const int32_t* dq_dev, int16_t* coef_dev,
                                 int numCoeff, int n, int per, int shift);

/* intra class (intrapred.cpp:31-234): n jobs, each with its own 4N+1 neighbour array
 * (nb_dev + job*nb_pitch), mode, filter flag; dst block at dst_dev + job*dst_pitch, row stride dst_stride */
typedef struct { int32_t mode, bFilter; } x265cu_intra_job;
int x265cu_intra_pred_batch(x265cu_ctx*, int depth, int size, const void* nb_dev, int64_t nb_pitch,
                            void* dst_dev, int64_t dst_pitch, int dst_stride,
                            const x265cu_intra_job* jobs_dev, int n);
int x265cu_intra_filter_batch(x265cu_ctx*, int depth, int size, const void* nb_dev, void* filt_dev, int64_t pitch, int n);
int x265cu_intra_allangs_batch(x265cu_ctx*, int depth, int size, const void* ref_dev, const void* filt_dev, int64_t nb_pitch,
                               void* dst_dev, int bLuma, int n);

/* lowres (pixel.cpp:604-628 + :1027-1041): full frame -> 4 half-pel planes, margins extended */
int x265cu_frame_init_lowres(x265cu_ctx*, int depth, const void* src_dev, int src_stride,
                             void* dst0_dev, void* dsth_dev, void* dstv_dev, void* dstc_dev,
                             int dst_stride, int width, int height, int marginX, int marginY);
int x265cu_extend_border(x265cu_ctx*, int depth, void* plane_dev, int stride, int width, int height, int marginX, int marginY);

/* mvcost table (bitcost.cpp:33-110): host helper, out[2*range+1] centred */
void x265cu_mvcost_table(double lambda, int range, uint16_t* out_host);

/* motion estimation class: one job = one MotionEstimate::motionEstimate() call
 * (motion.cpp:739-1569; DIA / HEX / STAR / FULL integer search + sub-pel refine, luma).  All jobs of a
 * launch share fenc plane, stride and mvcost table; results: out_dev[job] = {cost, qmv.x, qmv.y, 0}.
 * Methods 2 (UMH) and 4 (SEA) are not run on the device: the job list is not validated, and such a job is searched as
 * STAR.  The caller keeps method in {0, 1, 3, 5}. */
typedef struct {
    int32_t offset;             /* block origin (element offset, same in fenc and ref planes) */
    int16_t ref;                /* index into the ref plane table */
    int8_t  pw, ph;             /* PU size */
    int16_t mvmin[2], mvmax[2]; /* full-pel */
    int16_t qmvp[2];            /* qpel predictor */
    int16_t mvc[8];             /* up to 4 qpel candidates */
    int8_t  numCand, method, subme, merange;
} x265cu_me_job;
int x265cu_me_batch(x265cu_ctx*, int depth, const void* fenc_dev, int fencStride,
                    const void* const* refplanes_dev /* device array of plane ptrs */, int refStride, int lowres,
                    const uint16_t* mvcost_dev /* centred table base */, int mvcost_range,
                    const x265cu_me_job* jobs_dev, int n, int32_t* out_dev);

/* The same call with the chroma-SATD term of subpelCompare (motion.cpp:1601-1661) for 4:2:0 sources: with
 * MotionEstimate::bChromaSATD (motion.cpp:204-212: subme > 2 and PU width and height multiples of 8, so that the
 * chroma block has a SATD primitive, primitives.cpp:139-158) every sub-pel compare -- the clipped MVP, the MV
 * candidates and all refinement points -- adds SATD(Cb) + SATD(Cr) of the chroma block predicted at the eighth-pel
 * vector with the 4-tap filters.  Other jobs of the launch behave exactly as in x265cu_me_batch.
 * Chroma planes are half resolution, `cstride` pixels per row for source and references alike; the chroma pixel of the
 * luma position (x, y) = (offset % fencStride, offset / fencStride) is at (y >> 1) * cstride + (x >> 1) from the
 * pointers given.  `chroma` is a host struct of device pointers. */
typedef struct {
    const void* fencCb_dev; const void* fencCr_dev;
    const void* const* refCb_dev; const void* const* refCr_dev;   /* device arrays of plane pointers, indexed by job.ref */
    int cstride;
} x265cu_me_chroma;
int x265cu_me_batch_chroma(x265cu_ctx*, int depth, const void* fenc_dev, int fencStride,
                           const void* const* refplanes_dev, int refStride, const x265cu_me_chroma* chroma,
                           const uint16_t* mvcost_dev, int mvcost_range, const x265cu_me_job* jobs_dev, int n, int32_t* out_dev);

/* ---------- prediction costs around the motion search ----------
 * The motion-compensated prediction + cost evaluations Search::predInterSearch makes besides motionEstimate:
 *   - Search::selectMVP (encoder/search.cpp:1992-2023): SAD of the luma prediction at each AMVP candidate
 *     (predInterLumaPixel + MotionEstimate::bufSAD)                              -> cost = X265CU_PRED_SAD, one list;
 *   - Search::mergeEstimation (search.cpp:1901-1960): Predict::motionCompensation of the merge candidate (uni or bi),
 *     bufSATD + bufChromaSATD                                                     -> X265CU_PRED_SATD | X265CU_PRED_CHROMA;
 *   - the bi-directional estimate (search.cpp:2474-2607): with bChromaSATD the same motionCompensation(bi) path
 *     (addAvg of the two 14-bit intermediates, luma + chroma), without it pixelavg_pp of the two pixel predictions
 *     (luma only)                                                                -> X265CU_PRED_AVG_PP.
 * Prediction = the unweighted paths of common/predict.cpp:76-420 (4:2:0; eighth-pel chroma vector = the luma vector).
 * Vectors are quarter-pel and already clipped (CUData::clipMv, cudata.cpp:1915-1928).  The chroma term needs a chroma block
 * that is a multiple of 4x4 (motion.cpp:204-212) and chroma planes; it is skipped otherwise.  out_dev[n]: the distortion
 * (the caller adds the bit costs).  `chroma` may be NULL (no X265CU_PRED_CHROMA jobs). */
enum { X265CU_PRED_SAD = 0, X265CU_PRED_SATD = 1 };
enum { X265CU_PRED_CHROMA = 1, X265CU_PRED_AVG_PP = 2 };
typedef struct {
    int32_t offset;            /* PU origin: element offset into the luma planes (source and references share the geometry) */
    int16_t pw, ph;
    int8_t  ref0, ref1;        /* index into refplanes_dev / the chroma tables; -1 = list unused */
    uint8_t cost;              /* X265CU_PRED_SAD / X265CU_PRED_SATD */
    uint8_t flags;             /* X265CU_PRED_CHROMA | X265CU_PRED_AVG_PP */
    int16_t mv0[2], mv1[2];    /* quarter-pel */
} x265cu_pred_job;
int x265cu_pred_cost_batch(x265cu_ctx*, int depth, const void* fenc_dev, int fencStride, const void* const* refplanes_dev, int refStride,
                           const x265cu_me_chroma* chroma, const x265cu_pred_job* jobs_dev, int n, int32_t* out_dev);

/* ---------- frame-level CTU analysis (DESIGN.md "Frame analysis workload") ----------
 * One analyser = one picture geometry.  Reference planes stay resident in HBM (x265cu_analyser_set_ref
 * = what the recon-row broadcast feeds); per frame the host passes the source luma and the 16x16
 * predictor field (AMVP / lowres MVs, search.cpp:1968-2023, 2406-2410) and gets back, for every PU x
 * reference, the motionEstimate() result (motion.cpp:739), for every CU the residual-coding stats of
 * its best 2Nx2N prediction (search.cpp:3178; quant.cpp:397-470, 543-605) and its 35 intra SA8D costs
 * (search.cpp:1358-1444).  stages: bit0 ME, bit1 residual, bit2 intra, bit3 chroma residual (see
 * x265cu_analyser_enable_chroma_residual), bit4 BIDIR of a B slice (see x265cu_analyser_set_lists), bit5 PART of a P slice
 * (see x265cu_analyser_part_results), bit6 PART_B of a B slice (see x265cu_analyser_part_b_results). */
typedef struct x265cu_analyser x265cu_analyser;
typedef struct {
    int width, height, depth, numRefs;
    int method, subme, merange, rect;     /* X265_*_SEARCH, subpel refine level, range, rect PUs */
    int qp; double lambda;                /* quant QP, 0..51 + 6 * (depth - 8) (the slice QP plus QP_BD_OFFSET);
                                             mvcost lambda (x265_lambda_tab[qp]), finite and >= 0 */
    int amp;                              /* AMP PUs (2NxnU/nD, nLx2N/nRx2N at CU >= 16; presets slower+, param.cpp:494-520) */
} x265cu_analysis_params;
typedef struct {                          /* host destinations (any may be NULL) */
    int32_t*  me_packed;                  /* [njobs][2]: cost, (mvx | mvy << 16) */
    uint64_t* cu_sse; uint32_t* cu_numsig; int32_t* cu_ref;   /* [ncu] */
    uint32_t* intra_cost;                 /* [ncu][36]: 35 costs + best mode */
} x265cu_analysis_out;
/* Returns NULL, with the reason in x265cu_last_error(), for parameters the device cannot run as the reference does:
 * method not 0 (DIA), 1 (HEX), 3 (STAR) or 5 (FULL); merange outside 0..127 (x265cu_me_job holds it in 8 bits); subme
 * outside 0..7; width or height not a positive multiple of 8; qp outside 0..51 + 6 * (depth - 8), the QPs the quantiser
 * has; lambda negative, infinite or NaN.  Also NULL without a message when numRefs is not 1..16 or depth not 8 or 10. */
x265cu_analyser* x265cu_analyser_create(x265cu_ctx*, const x265cu_analysis_params*);
void x265cu_analyser_destroy(x265cu_analyser*);
int x265cu_analyser_counts(x265cu_analyser*, int* njobs, int* ncu, int* ntu, int64_t* ncoef, int* stride);
int x265cu_analyser_set_ref(x265cu_analyser*, int idx, const void* host_luma, int host_stride);
int x265cu_analyser_load_inputs(x265cu_analyser*, const void* fenc_host, int host_stride, const int16_t* field_host);
int x265cu_analyser_run_resident(x265cu_analyser*, int stages);       /* kernels only, inputs resident */
int x265cu_analyser_analyse(x265cu_analyser*, const void* fenc_host, int host_stride, const int16_t* field_host,
                            int stages, x265cu_analysis_out* out);    /* H2D + kernels + D2H, synchronous */
int x265cu_analyser_stage_ms(x265cu_analyser*, float ms[4]);          /* device ms of the last run: ME stage, residual, intra, ME kernel */
void* x265cu_analyser_ref_plane(x265cu_analyser*, int idx, int* stride); /* device address of ref idx's pixel (0,0) */
int x265cu_analyser_ref_updated(x265cu_analyser*, int idx);            /* re-extend borders after writing the plane in place */
int x265cu_analyser_fetch(x265cu_analyser*, int what, void* host);    /* parity/debug access to resident results; what =
                                                                          16 + 16 * ref + yf * 4 + xf: the whole allocation of
                                                                          reference ref's quarter-pel phase plane (xf, yf), of
                                                                          its weighted plane when it is weighted
                                                                          (x265cu_analyser_set_ref_weights) */
/* Every reference of an analyser is stored with its 15 quarter-pel phase planes, which every ME run rebuilds for the
 * sub-pel refinement: 15 planes of (width + 192, 64-aligned) x (height + 160) pixels per reference, e.g. 561 MB at
 * 3840x2160 8-bit with 4 references, 1.40 GB at 3840x2160 10-bit with 5, 5.3 GB at 7680x4320 10-bit with 5.  A weighted
 * reference adds a second block of 16 (x265cu_analyser_set_ref_weights). */
/* CTU-row shards (BASELINE configs[4]: WPP CTU rows sharded per GPU; the reference enables row r once the reference
 * rows it needs are reconstructed, frameencoder.cpp:850-868, producer side framefilter.cpp:664).  All job / CU / TU
 * lists are in CTU raster order, so rows [ctuRow0, ctuRow1) are one contiguous slice of every result array
 * (x265cu_analyser_row_range); run_rows / analyse_rows compute exactly that slice, bit-identical to the same
 * entries of a full-frame run.  `out` arrays stay full-frame sized. */
int x265cu_analyser_ctu_rows(x265cu_analyser*);
int x265cu_analyser_row_range(x265cu_analyser*, int ctuRow0, int ctuRow1, int* job0, int* njobs, int* cu0, int* ncu);
int x265cu_analyser_run_rows(x265cu_analyser*, int stages, int ctuRow0, int ctuRow1);
int x265cu_analyser_analyse_rows(x265cu_analyser*, const void* fenc_host, int host_stride, const int16_t* field_host,
                                 int stages, int ctuRow0, int ctuRow1, x265cu_analysis_out* out);
/* 4:2:0 chroma for the chroma-SATD term of subpelCompare (MotionEstimate::bChromaSATD, motion.cpp:204-212, 1601-1661): after
 * enable_chroma() the ME stage of every run adds SATD(Cb) + SATD(Cr) to every sub-pel compare of the PUs that have a chroma
 * SATD, as the encoder does for a 4:2:0 source at subme > 2 (x265cu_me_batch_chroma's kernels on resident planes).  Upload
 * the source's chroma with load_chroma() before analyse() / run_*(), each reference's with set_ref_chroma(); host planes are
 * (width / 2) x (height / 2), host_stride in pixels. */
int x265cu_analyser_enable_chroma(x265cu_analyser*);
int x265cu_analyser_set_ref_chroma(x265cu_analyser*, int idx, const void* cb_host, const void* cr_host, int host_stride);
int x265cu_analyser_load_chroma(x265cu_analyser*, const void* cb_host, const void* cr_host, int host_stride);
void* x265cu_analyser_recon_plane(x265cu_analyser*, int depthIdx /* 0..3 = CU 64,32,16,8 */, int* stride);
int x265cu_analyser_recon_to_ref(x265cu_analyser*, int depthIdx, int refIdx, int ctuRow0, int ctuRow1);
/* 4:2:0 chroma residual chain, stage bit 3 (value 8): for every CU, on the reference and vector the residual stage picks (lowest
 * ME cost of the CU's 2Nx2N jobs, ties to the lowest index), and for each luma TU (T = min(S, 32)) one (T/2) x (T/2) TU per
 * chroma plane at half the luma coordinates: predInterChromaPixel (predict.cpp:306-353) over the vector read as eighth-pel,
 * sub_ps, dct, quant (flat lists, no RDOQ / sign hiding), dequant_normal, idct or the DC-only shortcut, add_ps with the
 * recon clip, sse_pp (search.cpp:2990-3080).  The plane's quantiser QP is Quant::setChromaQP of qp - QP_BD_OFFSET + offset
 * (quant.cpp:221-244).  Outputs: per CU and plane the SSE and the number of nonzero levels ([ncu][2]); per plane the levels
 * (ncoef / 4: CU c's from its luma level offset / 4, TUs in the luma TU order); four recon planes per chroma plane, one per
 * CU size, in the chroma geometry (stride / 2, margins 48 x 40).
 * enable_chroma_residual() returns -1 (reason in x265cu_last_error) before enable_chroma() or for an offset outside -12..12
 * (the HEVC range of the PPS + slice offset); a run with bit 3 returns -1 before any launch unless it has run. */
int x265cu_analyser_enable_chroma_residual(x265cu_analyser*, int cbQpOffset, int crQpOffset);
int x265cu_analyser_chroma_qp(x265cu_analyser*, int qp[2]);             /* quantiser QP of Cb, Cr */
int x265cu_analyser_chroma_results(x265cu_analyser*, int ctuRow0, int ctuRow1, uint64_t* sse, uint32_t* numsig);
                                                                       /* [ncu][2] full-frame host arrays, rows' slice filled */
int x265cu_analyser_fetch_chroma(x265cu_analyser*, int what, void* host); /* 0 / 1: Cb / Cr levels; 2 + 2 * depthIdx + plane:
                                                                          recon plane allocation; 10 + 2 * ref + plane: the
                                                                          reference's chroma plane allocation */
void* x265cu_analyser_recon_plane_chroma(x265cu_analyser*, int depthIdx, int plane, int* cstride);
int x265cu_analyser_recon_to_ref_chroma(x265cu_analyser*, int depthIdx, int refIdx, int ctuRow0, int ctuRow1);
int x265cu_analyser_ref_chroma_updated(x265cu_analyser*, int idx);     /* re-extend the chroma borders of ref idx */
/* device address of chroma plane `plane` (0 Cb, 1 Cr) of ref idx at pixel (0,0) and its stride in elements (NULL before
 * enable_chroma()); the chroma twin of x265cu_analyser_ref_plane */
void* x265cu_analyser_ref_plane_chroma(x265cu_analyser*, int idx, int plane, int* cstride);
/* device address of the resident source plane `plane` (0 luma, 1 Cb, 2 Cr) at pixel (0,0) and its stride in elements, as
 * the last load_inputs() / load_chroma() left it (NULL for chroma before enable_chroma()); the source twin of ref_plane /
 * ref_plane_chroma, e.g. for x265cu_sao_stats_frame */
void* x265cu_analyser_src_plane(x265cu_analyser*, int plane, int* stride);

/* ---------- frame-level deblocking (common/deblock.cpp) ----------
 * The host's final decisions, one record per 4x4 luma unit in raster order over the picture (width / 4 records per row),
 * mirroring the CUData fields Deblock reads. */
typedef struct {
    int8_t  qp;             /* CUData::m_qp (spec QP, -QpBdOffset..51) */
    uint8_t flags;          /* bit 0 intra (isIntra), bit 1 luma cbf of the unit's TU (getCbf(.., TEXT_LUMA, tuDepth)),
                               bit 2 cu_transquant_bypass (m_tqBypass) */
    uint8_t log2CuSize;     /* 3..6 */
    uint8_t partSize;       /* PartSize: SIZE_2Nx2N 0 .. SIZE_nRx2N 7 */
    uint8_t tuDepth;        /* m_tuDepth */
    int8_t  refPic[2];      /* identity of the L0 / L1 reference PICTURE, -1 = list unused.  Deblock compares Frame pointers,
                               not indices (deblock.cpp:210-225): equal ids = the same picture, in either list */
    int16_t mv[2][2];       /* quarter-pel m_mv[list] */
} x265cu_deblock_unit;      /* 16 bytes */

typedef struct {
    int32_t sliceType;                      /* B_SLICE 0, P_SLICE 1, I_SLICE 2 (slice.h) */
    int32_t betaOffsetDiv2, tcOffsetDiv2;   /* PPS, -6..6 */
    int32_t cbQpOffset, crQpOffset;         /* PPS chromaQpOffset[2], -12..12 (the slice offsets do not enter deblocking) */
    int32_t transquantBypass;               /* PPS bTransquantBypassEnabled, 0 or 1 */
} x265cu_deblock_params;

/* Deblocks one picture (a single slice: only picture borders are unfiltered edges) in place on the context's stream, as
 * Deblock::deblockCTU over every CTU in FrameFilter's order does (framefilter.cpp:457-516): every vertical edge, then every
 * horizontal edge of the result; luma edges on the 8x8 grid, 4:2:0 chroma edges every 8 chroma samples.  Planes point at
 * pixel (0,0), strides in elements; cb_dev == cr_dev == NULL filters luma only (4:0:0).  units_dev: (width / 4) x
 * (height / 4) records.  Returns -1 with x265cu_last_error(), before any launch, for depth not 8 or 10, width or height not a
 * positive multiple of 8, a stride smaller than the row, parameters outside the ranges above, a NULL luma or unit pointer,
 * or only one NULL chroma pointer.  Any byte values in the map are read safely: a unit outside the documented ranges gives
 * unspecified pixels, never a fault. */
int x265cu_deblock_frame(x265cu_ctx*, int depth, void* luma_dev, int stride, void* cb_dev, void* cr_dev, int cstride,
                         int width, int height, const x265cu_deblock_unit* units_dev, const x265cu_deblock_params* params);

/* ---------- the in-loop filters over a band of CTU rows [ctuRow0, ctuRow1) (row shards, row-by-row filtering) ----------
 * Y0 = ctuRow0 * ctuSize and Y1 = min(height, ctuRow1 * ctuSize) are the band's luma rows, C0 = Y0 / 2 and C1 = Y1 / 2 its
 * 4:2:0 chroma rows; every range below is clipped to the picture.  The arguments are those of the frame calls, with the
 * same checks, plus ctuSize (16, 32 or 64; deblocking uses it only for the band's rows) and 0 <= ctuRow0 < ctuRow1 <=
 * ceil(height / ctuSize); a call that breaks one returns -1 with x265cu_last_error() before any launch.  Records are read
 * exactly as the frame calls read them.  Each band call is a pure function of the pre-deblock picture, so any partition of
 * the CTU rows, on one plane or on separate per-GPU copies, in any order, gives the whole-picture result (INTEGRATION.md,
 * "Row-range filtering"). */

/* Writes dst luma rows [Y0-4, Y1+4) and chroma rows [C0-4, C1+4), full width, with the values x265cu_deblock_frame gives over
 * the whole picture; reads src rows in the same ranges and unit rows [Y0/4-2, Y1/4+2).  src == dst (in place) is allowed
 * when those src rows are still pre-deblock; otherwise the planes must not overlap. */
int x265cu_deblock_rows(x265cu_ctx*, int depth, int width, int height, int ctuSize, int ctuRow0, int ctuRow1,
                        const void* src_y, const void* src_cb, const void* src_cr, int sstride, int scstride,
                        void* dst_y, void* dst_cb, void* dst_cr, int stride, int cstride,
                        const x265cu_deblock_unit* units_dev, const x265cu_deblock_params* params);

/* ---------- frame-level SAO (encoder/sao.cpp): statistics and apply; the decision stays on the host ----------
 * One slice per picture; 4:2:0, or 4:0:0 when every chroma pointer is NULL; CTU 16, 32 or 64.  Planes are device pointers at
 * pixel (0,0), strides in elements; both calls run on the context's stream.  Both read the deblocked, not-yet-SAO'd
 * picture only, as FrameFilter's interleaved order does (the statistics skip the samples the next CTU row's deblocking still
 * changes; the apply of a CTU reads its neighbours from copies taken before any SAO), so a picture is: x265cu_deblock_frame,
 * x265cu_sao_stats_frame, the host's SAO decision, x265cu_sao_apply_frame.  Each call returns -1 with x265cu_last_error(),
 * before any launch, for depth not 8 or 10, width or height not a positive multiple of 8, another CTU size, a stride smaller
 * than the row, a NULL luma / stats / parameter pointer, only some chroma pointers, saoChroma without chroma planes, flags
 * other than 0 or 1, or bypass units without source planes. */
typedef struct {
    int8_t  typeIdx;        /* SaoCtuParam as rdoSaoUnitCu leaves it (merged CTUs hold the copied parameters): -1 off,
                               0..3 SAO_EO_0..3, 4 SAO_BO; any other value is off */
    uint8_t bandPos;        /* 0..31, read & 31 */
    int8_t  offset[4];      /* any value: the result is clipped to the pixel range */
    uint8_t pad[2];
} x265cu_sao_ctu;           /* 8 bytes; arrays [3][numCtus], CTU raster order */

/* SAO::calcSaoStatsCTU of every CTU and plane (sao.cpp:735-917), all five types (bLimitSAO is the caller's: INTEGRATION.md).
 * stats_dev: int32 [numCtus][2: count, offsetOrg][3][5][32], i.e. two SAO::PerPlane per CTU (types in SaoType order, edge
 * classes through s_eoTable), ready to memcpy into m_count / m_offsetOrg.  Every entry is written; entries the reference never
 * writes (classes >= 5 of the edge types, chroma of a 4:0:0 call) are 0. */
int x265cu_sao_stats_frame(x265cu_ctx*, int depth, int width, int height, int ctuSize,
                           const void* fenc_y, const void* fenc_cb, const void* fenc_cr, int fstride, int fcstride,
                           const void* rec_y, const void* rec_cb, const void* rec_cr, int stride, int cstride, int32_t* stats_dev);
/* The records of the CTUs in rows [ctuRow0, ctuRow1) of the full-picture stats array; no other record is written.  Reads
 * deblocked rows [Y0-1, Y1) / [C0-1, C1) (the statistics skip the bottom 4 luma / 2 chroma rows of a CTU above the picture
 * bottom) and the same source rows. */
int x265cu_sao_stats_rows(x265cu_ctx*, int depth, int width, int height, int ctuSize, int ctuRow0, int ctuRow1,
                          const void* fenc_y, const void* fenc_cb, const void* fenc_cr, int fstride, int fcstride,
                          const void* rec_y, const void* rec_cb, const void* rec_cr, int stride, int cstride, int32_t* stats_dev);

/* FrameFilter's processSaoCTU over every CTU (generateLumaOffsets / generateChromaOffsets / applyPixelOffsets, sao.cpp:274-732),
 * in place.  saoLuma / saoChroma: SAOParam::bSaoFlag[0 / 1].  Cr is filtered with Cb's type and its own offsets, and only
 * when both types are >= 0 (sao.cpp:727; x265's decision gives both the same type; an EO record of one and a BO record of the
 * other give unspecified Cr pixels).  bypass_units_dev: NULL, or the x265cu_deblock_unit map, whose transquant-bypass units
 * (flags bit 2) then get the source samples back (origCUSampleRestoration).  Out-of-range records give unspecified pixels,
 * never a fault. */
int x265cu_sao_apply_frame(x265cu_ctx*, int depth, int width, int height, int ctuSize,
                           void* y, void* cb, void* cr, int stride, int cstride,
                           const x265cu_sao_ctu* params_dev, int saoLuma, int saoChroma,
                           const x265cu_deblock_unit* bypass_units_dev,
                           const void* fenc_y, const void* fenc_cb, const void* fenc_cr, int fstride, int fcstride);
/* Out of place: reads deblocked src rows [Y0-1, Y1+1) / [C0-1, C1+1); writes EVERY sample of dst rows [Y0, Y1) / [C0, C1)
 * (filtered, copied where SAO is off, or restored from the source for bypass units) and nothing else.  Also returns -1 for
 * src and dst planes that are the same. */
int x265cu_sao_apply_rows(x265cu_ctx*, int depth, int width, int height, int ctuSize, int ctuRow0, int ctuRow1,
                          const void* src_y, const void* src_cb, const void* src_cr, int sstride, int scstride,
                          void* dst_y, void* dst_cb, void* dst_cr, int stride, int cstride,
                          const x265cu_sao_ctu* params_dev, int saoLuma, int saoChroma, const x265cu_deblock_unit* bypass_units_dev,
                          const void* fenc_y, const void* fenc_cb, const void* fenc_cr, int fstride, int fcstride);

/* ---------- lookahead frame costs (BASELINE configs[1]; slicetype.cpp:696-805, 3115-3388) ----------
 * All pointers are device pointers.  Planes are the 4 lowres hpel planes of a frame (origin pixel,
 * margins extended: x265cu_frame_init_lowres).  One launch handles n frames / n (p0,p1,b) triples. */
typedef struct {
    const void* plane0; const int32_t* invQscale;            /* invQscale NULL when AQ is off */
    int32_t* intraCost; uint8_t* intraMode; uint16_t* lowresCosts; int32_t* rowSatds; int64_t* out; /* out[2]: costEst, costEstAq */
} x265cu_la_intra_job;
int x265cu_lowres_intra_batch(x265cu_ctx*, int depth, const x265cu_la_intra_job* jobs_dev, int n, int stride, int w8, int h8, int lambda);
typedef struct {
    const void* fenc[4]; const void* ref0[4]; const void* ref1[4];
    int32_t* mvs[2]; int32_t* mvcosts[2];                    /* [cu][2] qpel MVs and [cu] costs per list, in/out */
    const int32_t* intraCost; const int32_t* invQscale;
    uint16_t* lowresCosts; int32_t* rowSatds; int64_t* out;  /* out[3]: costEst, costEstAq, intraMbs */
    int32_t bidir, doSearch0, doSearch1;
    int32_t rows;                                            /* 0: whole frame; else a cooperative slice (slicetype.cpp:3075-3112): CU rows [rows & 0xffff, rows >> 16) */
} x265cu_la_job;
int x265cu_lookahead_cost_batch(x265cu_ctx*, int depth, const x265cu_la_job* jobs_dev, int n, int stride, int w8, int h8,
                                const uint16_t* mvcost_dev /* centred table base, lambda of X265_LOOKAHEAD_QP */);

/* cuTree: estimateCUPropagateCost (common/pixel.cpp:914-940; EncoderPrimitives::propagateCost, primitives.h:212, 356) over
 * `len` lowres CUs -- a whole frame in one launch instead of one call per CU row (slicetype.cpp:2654-2664).  Device arrays;
 * fpsFactor as the reference passes it (slicetype.cpp:2652).  Double precision, bit-exact to the C primitive. */
int x265cu_propagate_cost_batch(x265cu_ctx*, int* dst_dev, const uint16_t* propagateIn_dev, const int32_t* intraCosts_dev,
                                const uint16_t* interCosts_dev, const int32_t* invQscales_dev, double fpsFactor, int64_t len);

/* cuTree's propagation chain: Lookahead::cuTree (slicetype.cpp:2538-2639) with every estimateCUPropagate step
 * (:2641-2747) on the device, in stream order, without a host round trip.  What stays with the caller: the singleCost
 * calls (the estimates must exist before the call; x265cu_cutree_estimates lists them) and cuTreeFinish, which the host
 * runs, in the order of `finish`, on the propagateCost of the listed frames (its log2 is the host's libm).
 *
 * frames[0..numframes] are HOST records of device pointers, the reference's Lowres fields:
 *   intraCost, invQscale    Lowres::intraCost / invQscaleFactor (invQscaleFactor8x8 when rc.qgSize == 8), per lowres CU
 *   propagateCost           in / out (2-byte aligned); cleared, accumulated and swapped as the reference does: on return
 *                           the pointers of frames[0] and frames[lastnonb] are exchanged where :2572 / :2633 exchange them
 *   lowresCosts[d0][d1]     the estimate (b - d0, b + d1, b) of this frame (LOWRES_COST_SHIFT list bits); NULL: not supplied
 *   mvs[list][dist]         Lowres::lowresMvs[list][dist] as int32 (x, y) pairs, the layout of x265cu_la_job
 *   sliceType               X265_TYPE_* (only X265_TYPE_B = 5 against the rest matters)
 * A P estimate (b == p1) must carry list-0 bits only, as every estimate of the lookahead does.
 * finish (2 * maxFinish ints) receives (frame, ref0Distance) per cuTreeFinish call, in the reference's order (with VBV the
 * in-chain calls of :2745-2746 first).  ref0Distance -1 marks the lookahead-less intra case (:2561-2571): the host copies
 * qpAqOffset to qpCuTreeOffset instead.  Returns the number of finish entries, or -1 before any launch (x265cu_last_error)
 * when an estimate or motion field the chain reads was not supplied, an invQscale / propagateCost pointer is NULL, or the
 * window reaches the reference's estimateCUPropagate(0, 0, 0) (lookaheadDepth 0 without an anchor after frame 0). */
#define X265CU_CUTREE_DIST 18                                /* X265_BFRAME_MAX + 2 */
typedef struct {
    const int32_t* intraCost; const int32_t* invQscale; uint16_t* propagateCost;
    const uint16_t* lowresCosts[X265CU_CUTREE_DIST][X265CU_CUTREE_DIST];
    const int32_t* mvs[2][X265CU_CUTREE_DIST];
    int32_t sliceType, reserved;
} x265cu_cutree_frame;
typedef struct {
    int32_t bIntra, lookaheadDepth, bBPyramid, bEnableWeightedBiPred, vbv;   /* vbv: rc.vbvBufferSize != 0 */
    int32_t fpsNum, fpsDenom;
} x265cu_cutree_params;
int x265cu_cutree(x265cu_ctx*, x265cu_cutree_frame* frames, int numframes, const x265cu_cutree_params* params, int w8, int h8,
                  int32_t* finish, int maxFinish);
/* The (p0, p1, b) estimates x265cu_cutree reads for these slice types (sliceTypes[0..numframes]), in the order the
 * reference's singleCost calls them: 3 ints each into triples (room for maxTriples).  Returns the count, or -1. */
int x265cu_cutree_estimates(const int32_t* sliceTypes, int numframes, const x265cu_cutree_params* params, int32_t* triples,
                            int maxTriples);

/* Lookahead weighted-prediction analysis: LookaheadTLD::weightsAnalyse + weightCostLuma (slicetype.cpp:807-840, 860-961), the
 * call estimateFrameCost makes before the L0 search when --weightp is on (slicetype.cpp:3137).  Planes are whole padded
 * lowres buffers (Lowres::buffer[i], lowres.cpp:132-139: `planesize` pixels each, picture origin at `padoffset`), device
 * resident; refBuf_dev4 is a HOST array of the 4 device plane pointers; wbuf_dev (4 * planesize pixels) is
 * LookaheadTLD::wbuffer.  Host inputs: intraCost_host[CUs] (Lowres::intraCost) and stats = {fenc wp_sum, fenc wp_ssd,
 * ref wp_sum, ref wp_ssd} (Lowres::wp_sum[0] / wp_ssd[0], slicetype.cpp:49-57, 665-676).  wp_out = {isWeighted, scale,
 * log2 denominator, offset}; when isWeighted, wbuf_dev holds the 4 re-weighted planes for x265cu_lookahead_cost_batch's
 * ref0 (slicetype.cpp:3222).  The decision logic runs on the host as in the reference; the plane passes (weight_pp over
 * the padded plane, 8x8 SATD map) are launches of the block-op and grid pixel-compare kernels. */
int x265cu_lookahead_weights_analyse(x265cu_ctx*, int depth, const void* fencBuf_dev, const void* const* refBuf_dev4,
                                     void* wbuf_dev, int64_t planesize, int stride, int width, int lines, int64_t padoffset,
                                     const int32_t* intraCost_host, const uint64_t* stats, int* wp_out);

/* Adaptive quantisation: LookaheadTLD::calcAdaptiveQuantFrame (slicetype.cpp:444-694), split as cuTree is.  The per-block
 * integer work (acEnergyCu, :49-84, 256-275) is x265cu_aq_energy on the device, exact in any order; the float decision is
 * x265cu_aq_finish, a literal restatement on the host (its pow / log2 are the host's libm, and the library's host code is
 * compiled without FMA contraction or fast-math, so it equals a reference built with the same libm bit for bit).
 *
 * Geometry, with L = 8 at qgSize 8 and 16 otherwise, w8 = (W / 2 + 7) >> 3, h8 = (H / 2 + 7) >> 3 (Lowres::maxBlocksInRow /
 * maxBlocksInCol):
 *   energy grid   ceil(W / L) x ceil(H / L) blocks, raster order: the reference's loops over blockY / blockX step L
 *   blockCount    4 * w8 * h8 at qgSize 8, else w8 * h8: the length of qpAqOffset / invQscaleFactor / blockVariance /
 *                 quantOffsets (Lowres::create, Frame::create); it can exceed the energy grid at qgSize 8 */

/* energy[ceil(W / L) * ceil(H / L)] (uint32, device) receives acEnergyCu of every block; totals[3][2] (uint64, device)
 * receives, per plane, the sums of var's `sum` and `ssd` over all blocks: what one acEnergyCu pass adds to wp_sum[plane] /
 * wp_ssd[plane].  Luma is var 16x16 (shift 8), or 8x8 (shift 6) at qgSize 8; 4:2:0 chroma is var 8x8 (shift 6), or 4x4
 * (shift 4), at (blockX >> 1, blockY >> 1).  Planes are device pointers at pixel (0,0), strides in elements; cb = cr = NULL
 * is 4:0:0 (luma only, chroma totals 0).  Edge blocks: reads past the picture take the nearest in-picture sample (clamped
 * coordinates), which is what the reference reads from PicYuv's replicated padding (picyuv.cpp:209-234), so the planes
 * need no margins.  Returns -1 before any launch (x265cu_last_error) for a depth other than 8 / 10, a qgSize other than
 * 8 / 16 / 32 / 64, a non-positive or odd width or height, a stride smaller than the row, a NULL luma or output pointer, or
 * only one NULL chroma pointer.  Runs on the context's stream. */
int x265cu_aq_energy(x265cu_ctx*, int depth, const void* luma, int stride, const void* cb, const void* cr, int cstride,
                     int width, int height, int qgSize, uint32_t* energy_dev, uint64_t* totals_dev);

typedef struct {
    int32_t aqMode;             /* rc.aqMode: 0 NONE, 1 VARIANCE, 2 AUTO_VARIANCE, 3 AUTO_VARIANCE_BIASED (4 EDGE refused) */
    int32_t qgSize;             /* rc.qgSize: 8, 16, 32 or 64 */
    int32_t weightp;            /* bEnableWeightedPred || bEnableWeightedBiPred */
    int32_t variance;           /* bDynamicRefine || bEnableFades: blockVariance / frameVariance */
    int32_t hevcAq, hdr10Opt, aqMotion;   /* rc.hevcAq, bHDR10Opt, bAQMotion: refused when set (they stay on the host) */
    int32_t reserved;
    double aqStrength;          /* rc.aqStrength */
    const float* quantOffsets;  /* x265_picture::quantOffsets (blockCount floats, frame.cpp:141-146) or NULL */
} x265cu_aq_params;

/* Host outputs of x265cu_aq_finish; each may be NULL.  The arrays are in / out: entries the reference does not write keep
 * their contents (aqMode 0 writes no offsets; the main path writes only the energy grid's entries).  qpAqOffset holds what
 * the reference stores in both Lowres::qpAqOffset and qpCuTreeOffset.  invQscaleFactor8x8 (w8 * h8, qgSize 8) is the
 * reduction of :637-650, which reads invQscaleFactor with the reference's stride widthInCU * 2; it needs invQscaleFactor. */
typedef struct {
    double* qpAqOffset;             /* blockCount */
    int32_t* invQscaleFactor;       /* blockCount, x265_exp2fix8 of the offsets */
    int32_t* invQscaleFactor8x8;    /* w8 * h8, qgSize 8 only */
    uint64_t* wp_sum;               /* [3]: Lowres::wp_sum after the call */
    uint64_t* wp_ssd;               /* [3]: Lowres::wp_ssd after the call (weightp's correction applied, :653-676) */
    uint32_t* blockVariance;        /* blockCount, with variance */
    double* frameVariance;          /* with variance */
} x265cu_aq_out;

/* calcAdaptiveQuantFrame's decision (:466-693) on x265cu_aq_energy's energies and totals (host copies); needs no device.
 * The caller skips the reference's `rc.bStatRead && cuTree && IS_REFERENCED` case (:473), which computes no offsets.
 * Returns -1 with x265cu_last_error for aq-mode 4 (EDGE: Sobel and atan2 in float), hevc-aq, HDR10 opt and aq-motion,
 * which stay on the host; for bad depth / qgSize / geometry; for NULL energy or totals; for invQscaleFactor8x8 without
 * invQscaleFactor; and for variance with weightp when weightp's rounding of the picture to ((W + 8) >> 4) << 4 columns /
 * rows changes the grid the fades pass walks (:664-665, 678-693; for sides that are multiples of 8, qgSize 8 with W or
 * H % 16 == 8). */
int x265cu_aq_finish(int depth, int width, int height, const x265cu_aq_params* params, const uint32_t* energy,
                     const uint64_t* totals, const x265cu_aq_out* out);

/* The whole of calcAdaptiveQuantFrame for one picture: x265cu_aq_energy, the download of energies and totals, x265cu_aq_finish
 * into `out` (may be NULL) and, when aqMode != 0 and invQscale_dev is not NULL, the upload of invQscaleFactor (w8 * h8
 * entries, or invQscaleFactor8x8 at qgSize 8) into invQscale_dev: the array x265cu_la_intra_job.invQscale,
 * x265cu_la_job.invQscale and x265cu_cutree_frame.invQscale read.  Synchronises the context's stream. */
int x265cu_aq_frame(x265cu_ctx*, int depth, const void* luma, int stride, const void* cb, const void* cr, int cstride,
                    int width, int height, const x265cu_aq_params* params, int32_t* invQscale_dev, const x265cu_aq_out* out);

/* Weighted-prediction analysis of a P / B slice: weightAnalyse (encoder/weightPrediction.cpp:222-539), the frame encoder's
 * choice of the slice's pred_weight_table for luma and both chroma planes, on the lookahead's device-resident lowres
 * planes, intra costs and motion fields and the source chroma.  The candidate costs (weightCost, :169-218, after mcLuma /
 * mcChroma, :60-163) are k_weightp_costs on the device: one warp per 8x8 block, the motion-compensated reference block
 * formed in shared memory (no weighted or compensated plane is written), every candidate scored from it with the
 * reference's 8x4-tiled SATD and wrapping uint32 sums.  The search (:260-501) is a literal restatement on the host: its
 * candidates depend on the picture statistics only, so one launch and one download per plane and list serve it.
 * Refs 1..numRefIdx-1 of each list are reset as the reference resets them; entries past numRefIdx[list], and list 1 of
 * a P slice, are left untouched (the reference never writes them).  8 and 10 bit; 4:2:0 and 4:0:0.  In 4:0:0 the
 * reference picks the chroma denominator from two uninitialised floats (:280-286); here it stays 7. */
typedef struct {
    const void* lowres[4];      /* the 4 lowres hpel planes (Lowres::lowresPlane) at picture origin, margins extended */
    const void* cb;             /* full-resolution source Cb / Cr at (0,0), margins extended; NULL for 4:0:0 */
    const void* cr;
    int32_t lowresStride, chromaStride;   /* in pixels */
    uint64_t wp_sum[3], wp_ssd[3];        /* Lowres::wp_sum / wp_ssd, as calcAdaptiveQuantFrame leaves them */
    int32_t poc, reserved;
} x265cu_wp_frame;
typedef struct {
    int32_t sliceType;          /* 0 B (two lists), 1 P (list 0) */
    int32_t numRefIdx[2];       /* Slice::m_numRefIdx, 1..16 for each list the slice uses */
    int32_t bframes;            /* param.bframes: motion fields are used for diffPoc <= bframes + 1 */
    int32_t width, height;      /* m_picWidth / m_picHeight, multiples of 8 */
    int32_t csp;                /* 0 = 4:0:0, 1 = 4:2:0 */
} x265cu_wp_params;
typedef struct { int32_t weighted, w0, denom, offset; } x265cu_wp_cand;     /* weighted = 0: the unweighted reference */
typedef struct { int32_t wtPresent, inputWeight, log2WeightDenom, inputOffset; } x265cu_wp_entry;

/* weightCost of each candidate for one plane (0 luma on the lowres planes, 1 Cb, 2 Cr) of fenc against ref, without the
 * slice-header cost: costs[i] = sum over the 8x8 blocks of satd (luma: min(satd, intraCost[cu])) in wrapping uint32.  A
 * weighted candidate weights each reference pixel as weight_pp does, offset = candidate offset << (depth - 8).
 * mvs_dev: lowresMvs[list][diffPoc] as int32 pairs (w8 * h8, device) or NULL for no motion compensation.  intraCost_dev
 * (w8 * h8, device) is read for luma.  Records are host structs holding device pointers.  Chroma motion compensation
 * reads the reference chroma from column / row -9 to cw + 16 / ch + 16, where cw = ((width >> 4) << 4) >> 1 and
 * ch = ((height >> 4) << 4) >> 1: the caller extends the borders at least that far (PicYuv's 48 x 40 chroma margins
 * do); luma reads within 8 + 8 lowres pixels of the lowres picture.  1..48 candidates (w0 0..127, denom 0..7, offset
 * -128..127).  Returns -1 before any launch (x265cu_last_error) on bad arguments.  Synchronises the context's stream. */
int x265cu_weightp_costs(x265cu_ctx*, int depth, const x265cu_wp_params* params, const x265cu_wp_frame* fenc,
                         const x265cu_wp_frame* ref, const int32_t* intraCost_dev, const int32_t* mvs_dev, int plane,
                         const x265cu_wp_cand* cands, int ncand, uint32_t* costs);

/* The cost provider of x265cu_weightp_decide: fill costs[0..n) for the candidates of (list, plane), with motion
 * compensation when use_mvs.  Returns 0, or -1 to abort the decision. */
typedef int (*x265cu_wp_cost_fn)(void* user, int list, int plane, int use_mvs, const x265cu_wp_cand* cands, int n,
                                 uint32_t* costs);
/* The search of weightAnalyse on costs from `cost` (needs no device).  fenc / refs[list] give poc and the picture
 * statistics; has_mvs[list] says whether lowresMvs[list][diffPoc] was searched.  out: [2][16][3] entries. */
int x265cu_weightp_decide(int depth, const x265cu_wp_params* params, const x265cu_wp_frame* fenc,
                          const x265cu_wp_frame* const* refs, const int32_t* has_mvs, x265cu_wp_cost_fn cost, void* user,
                          x265cu_wp_entry* out);
/* The whole analysis on the device: refs[list] = m_refFrameList[list][0], mvs_dev[list] = lowresMvs[list][diffPoc]
 * (NULL: not searched), intraCost_dev of fenc.  One cost launch and one download per analysed plane and list. */
int x265cu_weightp_analyse(x265cu_ctx*, int depth, const x265cu_wp_params* params, const x265cu_wp_frame* fenc,
                           const int32_t* intraCost_dev, const x265cu_wp_frame* const* refs, const int32_t* const* mvs_dev,
                           x265cu_wp_entry* out);

/* ---------- weighted P-slice references of the frame analyser ----------
 * Applies one reference's weights, as x265cu_weightp_analyse's [0][idx] row gives them (m_weightPredTable[0][idx][0..2]:
 * luma, Cb, Cr), to the analyses of a P slice whose list 0 is the analyser's references.  The reference is weighted iff
 * w[0].wtPresent (frameencoder.cpp:550, predict.cpp:94); w == NULL or w[0].wtPresent == 0 makes it unweighted again, and the
 * results are then those of an analyser that was never weighted.  For a weighted reference:
 *   - the motion search (pre-checks, integer search, sub-pel phases) reads a weighted copy of its luma plane, and the
 *     chroma-SATD term a weighted copy of each chroma plane whose own wtPresent is set (at subme > 2): MotionReference::init
 *     and applyWeight (reference.cpp:51-185), weight_pp with w = inputWeight, offset = inputOffset << (depth - 8), shift =
 *     denom + 14 - depth, round = (denom ? 1 << (denom - 1) : 0) << (14 - depth), borders replicated;
 *   - the residual stages (bits 1 and 3) predict a CU that chose it from its unweighted planes in 14-bit precision, then
 *     weight_sp with addWeightUni's shift = denom + 14 - depth and round = 1 << (shift - 1) (predict.cpp:82-112, 525-578);
 *     chroma uses entries 1 and 2 whatever their wtPresent.  The choice of reference is unchanged.
 * ref_plane / ref_plane_chroma, recon_to_ref* and ref_updated / ref_chroma_updated keep addressing the unweighted planes; the
 * weighted copies are rebuilt from them at the start of the next run after any change.  They cover the whole picture and
 * its margins, so row runs give the entries of a full-frame run.  x265cu_analyser_fetch code 16 + 16 * ref + phase returns
 * what the search reads (the weighted block of a weighted reference), x265cu_analyser_fetch_chroma code 10 + 2 * numRefs +
 * 2 * ref + plane the chroma plane the chroma-SATD term reads.
 * Memory: a weighted reference gets its own block of 16 luma planes (the weighted plane and its 15 phases), allocated on first
 * use and kept until destroy: 150 MB at 3840x2160 8-bit, 300 MB at 10-bit; plus one chroma plane (2.3 / 4.7 MB) per weighted
 * chroma plane.
 * Returns -1 before any state change (x265cu_last_error) for idx outside 0..numRefs - 1 or an entry with wtPresent not 0 / 1,
 * log2WeightDenom outside 0..7, inputWeight outside -128..255 or inputOffset outside -128..127.  Only P slices: B-slice
 * weights (weightb, addWeightBi) are not applied, and a run of a B slice (x265cu_analyser_set_lists) is refused while any
 * reference is weighted. */
int x265cu_analyser_set_ref_weights(x265cu_analyser*, int idx, const x265cu_wp_entry w[3]);

/* ---------- B slices of the frame analyser ----------
 * x265cu_analyser_set_lists splits the analyser's numRefs reference slots into the slice's two lists: slots [0, numRefL0)
 * are list-0 refIdx 0..numRefL0 - 1, slots [numRefL0, numRefs) list-1 refIdx 0..numRefL1 - 1.  A picture in both lists (GPB,
 * low-delay B) is loaded into two slots, each with its own predictor plane, as the encoder searches it twice.  numRefL1 == 0
 * is a P slice: the state at creation, whose results are those of an analyser that never saw a B slice.  The ME stage and
 * its job list do not change: every slot is searched.  Returns -1 before any state change (x265cu_last_error) unless
 * numRefL0 >= 1, numRefL1 >= 0 and numRefL0 + numRefL1 == numRefs.
 *
 * Stage bit 4 (value 16), BIDIR: Analysis::checkInter_rd0_4 for 2Nx2N and checkBidir2Nx2N (analysis.cpp:3062-3071,
 * 3145-3265) for every CU (8 to 64), on the analyser's own cost model:
 *   1. per list, the CU's 2Nx2N job of lowest ME cost over that list's slots (ties to the lowest slot); the uni-directional
 *      winner is list 0 if cost0 <= cost1, else list 1 (search.cpp:2611);
 *   2. uniCost = sa8d of the winner's pixel prediction (predInterLumaPixel), + sa8d(Cb) + sa8d(Cr) of its chroma prediction
 *      when chroma is enabled (x265cu_analyser_enable_chroma; the chroma SA8D of a CU 8 is satd 4x4, primitives.cpp:185-188),
 *      + mvcost(mv - mvp) of the winner;
 *   3. biCost = sa8d of addAvg(predInterLumaShort(L0 best), predInterLumaShort(L1 best)) (+ the chroma twin) + mvcost0(mv0 -
 *      mvp0) + mvcost1(mv1 - mvp1), each MVP the MVP of that job;
 *   4. the zero pair is tried if either vector is nonzero and both MVPs lie in setSearchRange(cu, 0, max(width, height)) (the
 *      clip of the ME job build, then mvmax.y += 2 and both bounds << 2); zCost, the same formula with both vectors zero,
 *      replaces biCost and the pair if zCost < biCost;
 *   5. the CU is bi-predicted iff biCost < uniCost.
 * The bits model is the analyser's: the only bits term is the ME's mvcost table (x265cu_mvcost_table at the analyser's lambda,
 * the sum of the two components truncated to 16 bits as the ME's).  No reference-index, list-selection or MVP-index bits and
 * no checkBestMVP: those belong to the host's AMVP and CABAC state.
 * On a B slice the residual stages (bits 1 and 3) code the decision: a CU with interDir 1 or 2 takes its winning slot as on
 * a P slice; a CU with interDir 3 predicts every TU through the two 14-bit predictions and addAvg (predict.cpp:168-189), then
 * runs the unchanged chain, and its cu_ref is its list-0 slot.
 * Refused with -1 before any launch: value 16 on a P slice; value 2 or 8 on a B slice without value 16 in the same call; any
 * run of a B slice while a reference is weighted (x265cu_analyser_set_ref_weights). */
typedef struct {
    uint32_t uniCost, biCost;   /* step 2, and step 3 after the zero try */
    int8_t   interDir;          /* 1 L0, 2 L1, 3 bi */
    int8_t   ref[2];            /* slot of the best L0 / L1 2Nx2N job */
    uint8_t  zero;              /* 1: the zero pair replaced the searched pair */
    int16_t  mv[2][2];          /* the bi pair's quarter-pel vectors */
} x265cu_bidir_cu;
int x265cu_analyser_set_lists(x265cu_analyser*, int numRefL0, int numRefL1);
/* the BIDIR records of the CTU rows [ctuRow0, ctuRow1) into `out`, a full-frame host array of ncu records (synchronous) */
int x265cu_analyser_bidir_results(x265cu_analyser*, int ctuRow0, int ctuRow1, x265cu_bidir_cu* out);

/* ---------- inter estimate of every partition of a P slice's CUs ----------
 * Stage bit 5 (value 32), PART: the sa8dCost of checkInter_rd0_4 (analysis.cpp:3023-3071) for every partition the analyser's
 * geometry emits for every CU (8 to 64): 2Nx2N always, 2NxN and Nx2N with rect, 2NxnU, 2NxnD, nLx2N and nRx2N with amp at
 * CU >= 16 -- what compressInterCU_rd0_4 compares (analysis.cpp:1439-1593).  On the analyser's cost model:
 *   1. each PU takes the slot of lowest ME cost among its jobs, ties to the lowest slot (PU k of CU c for slot r is job
 *      cu_jobs[c * numRefs + r] + k, k in the geometry's order: 2Nx2N; 2NxN x2; Nx2N x2; 2NxnU x2; 2NxnD x2; nLx2N x2;
 *      nRx2N x2), so the 2Nx2N entry's slot is the residual stage's cu_ref;
 *   2. each PU is predicted at its ME vector into the CU's S x S prediction: predInterLumaPixel, and with chroma enabled
 *      (x265cu_analyser_enable_chroma) predInterChromaPixel of its (pw/2) x (ph/2) chroma block (the vector read as eighth-pel);
 *      a weighted slot (x265cu_analyser_set_ref_weights) takes predInterLumaShort / predInterChromaShort of its unweighted
 *      planes and addWeightUni, as the residual stages do (predict.cpp:82-112);
 *   3. sa8d = cu[S].sa8d of the luma prediction, + chroma[I420].cu[S].sa8d of Cb and of Cr when chroma is enabled (satd 4x4
 *      for a CU 8); cost = sa8d + the sum over the partition's PUs of mvcost(mv - mvp), the MVP the job's, each PU's two
 *      components summed to 16 bits as in the ME.
 * As in BIDIR there are no reference-index, MVP-index or list bits, no checkBestMVP and no merge estimation of the rect /
 * AMP PUs, and nothing is gated by split cost or thresholds: every emitted partition is evaluated and the host decides.
 * One record per CU, read with x265cu_analyser_part_results; the records are allocated zeroed by the first value-32 run.
 * Refused with -1 before any launch: value 32 on a B slice (numRefL1 > 0: a B slice's rect / AMP PUs need predInterSearch's
 * per-PU list choice and bi-prediction, which stage bit 6 below computes).  Every vector used is the ME result of one of the CU's PU jobs, which
 * k_build_me_jobs' clip bounds relative to the CU origin, and every PU lies inside its CU, so the reads stay inside what
 * an_planes_cover (luma) and an_chroma_reach_ok (chroma) check; a value-32 run where either fails is refused too. */
typedef struct {
    uint32_t cost[8];      /* indexed by PartSize (SIZE_2Nx2N 0 .. SIZE_nRx2N 7); UINT32_MAX where not evaluated (NxN always) */
    uint32_t sa8d[8];      /* the distortion part of cost; UINT32_MAX where not evaluated */
    int8_t   ref[8][2];    /* slot of PU 0 / PU 1; -1 where there is no such PU */
    int16_t  mv[8][2][2];  /* quarter-pel vector of each PU; 0 where there is no such PU */
} x265cu_part_cu;          /* 144 bytes */
/* the PART records of the CTU rows [ctuRow0, ctuRow1) into `out`, a full-frame host array of ncu records (synchronous);
 * refused before any value-32 run and for a bad row range */
int x265cu_analyser_part_results(x265cu_analyser*, int ctuRow0, int ctuRow1, x265cu_part_cu* out);

/* ---------- inter estimate of every partition of a B slice's CUs ----------
 * Stage bit 6 (value 64), PART_B: stage bit 5 for a B slice (x265cu_analyser_set_lists with numRefL1 > 0), i.e. checkInter_rd0_4
 * (analysis.cpp:3023-3071) with predInterSearch's B-slice path (search.cpp:2473-2644) for every partition the geometry emits
 * for every CU (8 to 64), in the same set and order as stage bit 5.  Per PU of the partition, on the analyser's cost model:
 *   1. per list, the slot of lowest ME cost among the PU's jobs in that list (list 0 = slots [0, numRefL0)), ties to the
 *      lowest slot; cost0 / cost1 are those jobs' ME costs (me_packed), mv0 / mv1 their vectors, mvp0 / mvp1 their MVPs;
 *   2. the bi try, iff the partition is not 2Nx2N and the CU is not 8x8 (isBipredRestriction): bChromaSATD is chroma enabled,
 *      subme > 2 and the PU's (pw/2) x (ph/2) chroma block has both sides a multiple of 4 (motion.cpp:212).  biCost = bufSATD of
 *      the bi-prediction (addAvg of the two 14-bit predictions with bChromaSATD, else pixelavg_pp of the two pixel predictions),
 *      + bufChromaSATD of the addAvg chroma with bChromaSATD, + mvcost(mv0 - mvp0) + mvcost(mv1 - mvp1).  The zero pair is
 *      tried iff either vector is nonzero and both MVPs lie in the CU's setSearchRange(cu, 0, max(width, height)) (mvmax.y += 2,
 *      both bounds << 2, as in BIDIR); its cost, the same formula at zero vectors, replaces biCost and the pair iff lower;
 *   3. the PU is bi iff biCost < cost0 and biCost < cost1, else list 0 iff cost0 <= cost1, else list 1.
 * The CU's prediction places each PU's final prediction: a uni PU's pixel prediction (as stage bit 5), a bi PU's addAvg of its
 * two 14-bit predictions, luma and, with chroma enabled, Cb and Cr (predict.cpp:168-189), whichever path its biCost took.
 * sa8d is the CU's sa8d over that prediction (+ Cb and Cr with chroma), cost = sa8d + every PU's mvcost: one vector for a uni
 * PU, two for a bi PU.  As in BIDIR and PART there are no list-selection, reference-index or MVP-index bits, no checkBestMVP,
 * no merge estimation of the rect / AMP PUs and no gating: the host adds its bits and decides.  Every PU keeps both lists'
 * slot and vector, a uni PU too, so that the host can redo the decision with its own bits.
 * One record per CU, read with x265cu_analyser_part_b_results; the records are allocated zeroed by the first value-64 run.
 * Refused with -1 before any launch: value 64 on a P slice; any run of a B slice while a reference is weighted; a value-64 run
 * where an_planes_cover or, with chroma, an_chroma_reach_ok fails (every vector read is a PU job's ME result or zero, inside
 * the reach stage bit 5 checks). */
typedef struct {
    uint32_t cost[8], sa8d[8];     /* indexed by PartSize as x265cu_part_cu; UINT32_MAX where not evaluated */
    uint32_t biCost[8][2];         /* per PU, after the zero try; UINT32_MAX where the bi try did not run or there is no PU */
    int8_t   interDir[8][2];       /* 1 L0, 2 L1, 3 bi; 0 where there is no PU */
    int8_t   ref[8][2][2];         /* [part][pu][list] slot of that list's best job; -1 where there is no PU */
    uint8_t  zero[8][2];           /* 1: the zero pair replaced the searched pair */
    int16_t  mv[8][2][2][2];       /* [part][pu][list] that list's vector (the bi pair after the zero try: both 0 where zero is
                                      set, whatever interDir; the searched vector is then the slot's ME result); 0 where there is
                                      no PU */
} x265cu_part_b_cu;                /* 320 bytes */
/* the PART_B records of the CTU rows [ctuRow0, ctuRow1) into `out`, a full-frame host array of ncu records (synchronous);
 * refused before any value-64 run and for a bad row range */
int x265cu_analyser_part_b_results(x265cu_analyser*, int ctuRow0, int ctuRow1, x265cu_part_b_cu* out);

#ifdef __cplusplus
}
#endif
#endif
