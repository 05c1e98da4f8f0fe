// x265_b200/csrc/x265cu.cu -- the single translation unit of libx265cu.so: context, memory,
// batched C-ABI entry points (include/x265_b200.h) and the per-call primitive table.
#include "common.cuh"
#include "pixelcmp.cuh"
#include "pixelcmp_grid.cuh"
#include "blockops.cuh"
#include "interp.cuh"
#include "transform.cuh"
#include "intra.cuh"
#include "me.cuh"
#include "predcost.cuh"
#include "frame.cuh"
#include "resid.cuh"
#include "lookahead.cuh"
#include "aq.cuh"
#include <math.h>
#include <mutex>
#include <vector>
#include <algorithm>

static thread_local char g_err[512] = "";
unsigned long long g_x265cu_launches = 0;
void x265cu_set_error(const char* what, cudaError_t e, const char* file, int line)
{
    snprintf(g_err, sizeof(g_err), "%s failed: %s (%s:%d)", what, cudaGetErrorString(e), file, line);
    fprintf(stderr, "x265cu: %s\n", g_err);
}

extern "C" {

const char* x265cu_last_error(void) { return g_err; }

int x265cu_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

static void ctx_release(x265cu_ctx* c)
{
    if (c->h_stage) cudaFreeHost(c->h_stage);
    cudaFree(c->d_stage); cudaFree(c->d_counter); cudaFree(c->d_me_state); cudaFree(c->d_sao_lines); cudaFree(c->d_cutree); cudaFree(c->d_aq);
    if (c->ev0) cudaEventDestroy(c->ev0);
    if (c->ev1) cudaEventDestroy(c->ev1);
    for (int i = 0; i < 4; i++) if (c->me_ev[i]) cudaEventDestroy(c->me_ev[i]);
    if (c->stream) cudaStreamDestroy(c->stream);
    delete c;
}

x265cu_ctx* x265cu_create(int device)
{
    if (device < 0 || device >= x265cu_device_count())
    {
        snprintf(g_err, sizeof(g_err), "no CUDA device %d (libx265cu has no CPU fallback)", device);
        return NULL;
    }
    if (cudaSetDevice(device) != cudaSuccess) return NULL;
    x265cu_ctx* c = new x265cu_ctx();
    memset(c, 0, sizeof(*c));
    c->device = device;
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, device);
    c->sm_count = prop.multiProcessorCount;
    c->stage_bytes = 4u << 20;
    bool ok = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) == cudaSuccess;
    ok = ok && cudaEventCreate(&c->ev0) == cudaSuccess && cudaEventCreate(&c->ev1) == cudaSuccess;
    for (int i = 0; i < 4 && ok; i++) ok = cudaEventCreate(&c->me_ev[i]) == cudaSuccess;
    ok = ok && build_dct_tables(device) == 0;
    ok = ok && cudaMallocHost((void**)&c->h_stage, c->stage_bytes) == cudaSuccess &&
         cudaMalloc((void**)&c->d_stage, c->stage_bytes) == cudaSuccess &&
         cudaMalloc((void**)&c->d_counter, 64) == cudaSuccess;
    if (!ok)
    {
        x265cu_set_error("ctx create", cudaGetLastError(), __FILE__, __LINE__);
        ctx_release(c);
        return NULL;
    }
    return c;
}

void x265cu_destroy(x265cu_ctx* c)
{
    cudaSetDevice(c->device);
    if (!c) return;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    ctx_release(c);
}

int x265cu_sync(x265cu_ctx* c) { cudaSetDevice(c->device); CU_CHECK(cudaStreamSynchronize(c->stream)); return 0; }
void* x265cu_stream(x265cu_ctx* c) { cudaSetDevice(c->device); return (void*)c->stream; }
void* x265cu_malloc(x265cu_ctx* c, size_t bytes)
{
    void* p = NULL;
    cudaSetDevice(c->device);
    if (cudaMalloc(&p, bytes) != cudaSuccess) { x265cu_set_error("cudaMalloc", cudaGetLastError(), __FILE__, __LINE__); return NULL; }
    return p;
}
void x265cu_free(x265cu_ctx* c, void* dev) { cudaSetDevice(c->device); cudaFree(dev); }
void* x265cu_host_alloc(size_t bytes) { void* p = NULL; if (cudaMallocHost(&p, bytes) != cudaSuccess) return NULL; return p; }
void x265cu_host_free(void* p) { cudaFreeHost(p); }
int x265cu_h2d(x265cu_ctx* c, void* dev, const void* host, size_t bytes) { cudaSetDevice(c->device); CU_CHECK(cudaMemcpyAsync(dev, host, bytes, cudaMemcpyHostToDevice, c->stream)); return 0; }
int x265cu_d2h(x265cu_ctx* c, void* host, const void* dev, size_t bytes) { cudaSetDevice(c->device); CU_CHECK(cudaMemcpyAsync(host, dev, bytes, cudaMemcpyDeviceToHost, c->stream)); return 0; }
int x265cu_copy2d(x265cu_ctx* c, void* dst, size_t dpitch, const void* src, size_t spitch, size_t widthBytes, size_t rows, int kind)
{
    cudaSetDevice(c->device);
    const cudaMemcpyKind k = kind == 0 ? cudaMemcpyHostToDevice : kind == 1 ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
    CU_CHECK(cudaMemcpy2DAsync(dst, dpitch, src, spitch, widthBytes, rows, k, c->stream));
    return 0;
}
int x265cu_memset(x265cu_ctx* c, void* dev, int value, size_t bytes) { cudaSetDevice(c->device); CU_CHECK(cudaMemsetAsync(dev, value, bytes, c->stream)); return 0; }
int x265cu_timer_begin(x265cu_ctx* c) { cudaSetDevice(c->device); CU_CHECK(cudaEventRecord(c->ev0, c->stream)); return 0; }
float x265cu_timer_end(x265cu_ctx* c)
{
    cudaSetDevice(c->device);
    float ms = -1.f;
    if (cudaEventRecord(c->ev1, c->stream) != cudaSuccess) return -1.f;
    if (cudaEventSynchronize(c->ev1) != cudaSuccess) return -1.f;
    if (cudaEventElapsedTime(&ms, c->ev0, c->ev1) != cudaSuccess) return -1.f;
    return ms;
}
uint64_t x265cu_launch_count(x265cu_ctx* c) { (void)c; return __atomic_load_n(&g_x265cu_launches, __ATOMIC_RELAXED); }
int x265cu_me_phase_ms(x265cu_ctx* c, float* ms)
{
    cudaSetDevice(c->device);
    CU_CHECK(cudaEventSynchronize(c->me_ev[3]));
    for (int i = 0; i < 3; i++) CU_CHECK(cudaEventElapsedTime(&ms[i], c->me_ev[i], c->me_ev[i + 1]));
    return 0;
}

// ---------------- batched API ----------------
int x265cu_pixelcmp_batch(x265cu_ctx* c, int depth, int op, const void* A, const void* B, const x265cu_cmp_job* jobs, int n, uint64_t* out)
{ cudaSetDevice(c->device); return launch_pixelcmp(c, depth, op, A, B, jobs, n, out); }
int x265cu_pixelcmp_grid(x265cu_ctx* c, int depth, int op, const void* A, int64_t a_stride, const void* B, int64_t b_stride,
                         int bw, int bh, int nbx, int nby, uint64_t* out)
{ cudaSetDevice(c->device); return launch_pixelcmp_grid(c, depth, op, A, a_stride, B, b_stride, bw, bh, nbx, nby, out); }

int x265cu_blockop_batch(x265cu_ctx* c, int depth, int op, void* D, const void* A, const void* B, const x265cu_blk_job* jobs, int n)
{ cudaSetDevice(c->device); return launch_blockop(c, depth, op, D, A, B, jobs, n); }

int x265cu_interp_batch(x265cu_ctx* c, int depth, int op, const void* src, void* dst, const x265cu_interp_job* jobs, int n)
{ cudaSetDevice(c->device); return launch_interp(c, depth, op, src, dst, jobs, n); }

int x265cu_transform_batch(x265cu_ctx* c, int depth, int op, int size, const int16_t* src, int16_t* dst, int stride, int64_t tu_pitch, int n)
{ cudaSetDevice(c->device); return launch_transform(c, depth, op, size, src, dst, stride, tu_pitch, n); }

int x265cu_quant_batch(x265cu_ctx* c, const int16_t* coef, const int32_t* qc, int32_t* deltaU, int16_t* qCoef, int qBits, int add,
                       int numCoeff, int n, int nquant, uint32_t* numSig)
{
    cudaSetDevice(c->device);
    if (n <= 0) return 0;
    int blocks = (n + 7) / 8; if (blocks > c->sm_count * 8) blocks = c->sm_count * 8;
    k_quant<<<blocks, 256, 0, c->stream>>>(coef, qc, deltaU, qCoef, qBits, add, numCoeff, n, nquant, numSig);
    CU_LAUNCH_CHECK(c);
    return 0;
}

int x265cu_dequant_normal_batch(x265cu_ctx* c, const int16_t* q, int16_t* coef, int64_t num, int scale, int shift)
{
    cudaSetDevice(c->device);
    if (num <= 0) return 0;
    int64_t blocks = (num + 255) / 256; if (blocks > c->sm_count * 16) blocks = c->sm_count * 16;
    k_dequant_normal<<<(int)blocks, 256, 0, c->stream>>>(q, coef, num, scale, shift);
    CU_LAUNCH_CHECK(c);
    return 0;
}

int x265cu_dequant_scaling_batch(x265cu_ctx* c, const int16_t* q, const int32_t* dq, int16_t* coef, int numCoeff, int n, int per, int shift)
{
    cudaSetDevice(c->device);
    int64_t total = (int64_t)numCoeff * n;
    if (total <= 0) return 0;
    int64_t blocks = (total + 255) / 256; if (blocks > c->sm_count * 16) blocks = c->sm_count * 16;
    k_dequant_scaling<<<(int)blocks, 256, 0, c->stream>>>(q, dq, coef, numCoeff, total, per, shift);
    CU_LAUNCH_CHECK(c);
    return 0;
}

int x265cu_intra_pred_batch(x265cu_ctx* c, int depth, int size, const void* nb, int64_t nb_pitch, void* dst, int64_t dst_pitch, int dst_stride,
                            const x265cu_intra_job* jobs, int n)
{
    cudaSetDevice(c->device);
    if (n <= 0) return 0;
    int blocks = n < c->sm_count * 8 ? n : c->sm_count * 8;
    int threads = size * size < 256 ? (size * size < 32 ? 32 : size * size) : 256;
    if (depth == 8) k_intra_pred<uint8_t><<<blocks, threads, 0, c->stream>>>(size, (const uint8_t*)nb, nb_pitch, (uint8_t*)dst, dst_pitch, dst_stride, jobs, n);
    else            k_intra_pred<uint16_t><<<blocks, threads, 0, c->stream>>>(size, (const uint16_t*)nb, nb_pitch, (uint16_t*)dst, dst_pitch, dst_stride, jobs, n);
    CU_LAUNCH_CHECK(c);
    return 0;
}

int x265cu_intra_filter_batch(x265cu_ctx* c, int depth, int size, const void* nb, void* filt, int64_t pitch, int n)
{
    cudaSetDevice(c->device);
    if (n <= 0) return 0;
    int blocks = (n + 7) / 8 < c->sm_count * 8 ? (n + 7) / 8 : c->sm_count * 8;       // a warp per neighbour array
    if (depth == 8) k_intra_filter<uint8_t><<<blocks, 256, 0, c->stream>>>(size, (const uint8_t*)nb, (uint8_t*)filt, pitch, n);
    else            k_intra_filter<uint16_t><<<blocks, 256, 0, c->stream>>>(size, (const uint16_t*)nb, (uint16_t*)filt, pitch, n);
    CU_LAUNCH_CHECK(c);
    return 0;
}

int x265cu_intra_allangs_batch(x265cu_ctx* c, int depth, int size, const void* ref, const void* filt, int64_t nb_pitch, void* dst, int bLuma, int n)
{
    cudaSetDevice(c->device);
    if (n <= 0) return 0;
    if ((((uintptr_t)dst) & 7) == 0 && size >= 4 && size <= 32)
    {   // vector-store kernel: one CTA per block, all 33 modes
        int blocks = n < c->sm_count * 16 ? n : c->sm_count * 16;
        if (!((uintptr_t)dst & 15))
        {   // packed-pixel kernel (16-byte row pieces): words per item = min(row bytes, 16) / 4
            const int rowBytes = size * (depth == 8 ? 1 : 2), uw = (rowBytes < 16 ? rowBytes : 16) / 4;
            blocks = n < c->sm_count * 8 ? n : c->sm_count * 8;
            if (depth == 8)
            {
                if (uw == 4)      k_intra_allangs_packed<uint8_t, 4><<<blocks, 256, 0, c->stream>>>(size, (const uint8_t*)ref, (const uint8_t*)filt, nb_pitch, (uint8_t*)dst, bLuma, n);
                else if (uw == 2) k_intra_allangs_packed<uint8_t, 2><<<blocks, 256, 0, c->stream>>>(size, (const uint8_t*)ref, (const uint8_t*)filt, nb_pitch, (uint8_t*)dst, bLuma, n);
                else              k_intra_allangs_packed<uint8_t, 1><<<blocks, 256, 0, c->stream>>>(size, (const uint8_t*)ref, (const uint8_t*)filt, nb_pitch, (uint8_t*)dst, bLuma, n);
            }
            else
            {
                if (uw == 4)      k_intra_allangs_packed<uint16_t, 4><<<blocks, 256, 0, c->stream>>>(size, (const uint16_t*)ref, (const uint16_t*)filt, nb_pitch, (uint16_t*)dst, bLuma, n);
                else              k_intra_allangs_packed<uint16_t, 2><<<blocks, 256, 0, c->stream>>>(size, (const uint16_t*)ref, (const uint16_t*)filt, nb_pitch, (uint16_t*)dst, bLuma, n);
            }
            CU_LAUNCH_CHECK(c);
            return 0;
        }
        if (depth == 8) k_intra_allangs_cta<uint8_t><<<blocks, 256, 0, c->stream>>>(size, (const uint8_t*)ref, (const uint8_t*)filt, nb_pitch, (uint8_t*)dst, bLuma, n);
        else            k_intra_allangs_cta<uint16_t><<<blocks, 256, 0, c->stream>>>(size, (const uint16_t*)ref, (const uint16_t*)filt, nb_pitch, (uint16_t*)dst, bLuma, n);
        CU_LAUNCH_CHECK(c);
        return 0;
    }
    dim3 grid(33, n < 4096 ? n : 4096);
    int threads = size * size < 256 ? (size * size < 32 ? 32 : size * size) : 256;
    if (depth == 8) k_intra_allangs<uint8_t><<<grid, threads, 0, c->stream>>>(size, (const uint8_t*)ref, (const uint8_t*)filt, nb_pitch, (uint8_t*)dst, bLuma, n);
    else            k_intra_allangs<uint16_t><<<grid, threads, 0, c->stream>>>(size, (const uint16_t*)ref, (const uint16_t*)filt, nb_pitch, (uint16_t*)dst, bLuma, n);
    CU_LAUNCH_CHECK(c);
    return 0;
}

int x265cu_extend_border(x265cu_ctx* c, int depth, void* plane, int stride, int width, int height, int mx, int my)
{
    cudaSetDevice(c->device);
    if (depth == 8) return extend_border_t<uint8_t>(c, (uint8_t*)plane, stride, width, height, mx, my);
    return extend_border_t<uint16_t>(c, (uint16_t*)plane, stride, width, height, mx, my);
}

int x265cu_frame_init_lowres(x265cu_ctx* c, int depth, const void* src, int sstride, void* d0, void* dh, void* dv, void* dc,
                             int dstride, int width, int height, int mx, int my)
{
    cudaSetDevice(c->device);
    dim3 block(64, 4), grid((width / 4 + 63) / 64 + 1, (height + 3) / 4);
    const uintptr_t dal = (uintptr_t)d0 | (uintptr_t)dh | (uintptr_t)dv | (uintptr_t)dc | (uintptr_t)dstride;
    if (depth == 8 && (width & 7) == 0 && (((uintptr_t)src | (uintptr_t)sstride) & 15) == 0 && (dal & 7) == 0)
    {
        dim3 g8((width / 8 + 63) / 64, (height + 3) / 4);
        k_lowres_init_u8x8<<<g8, block, 0, c->stream>>>((const uint8_t*)src, sstride, (uint8_t*)d0, (uint8_t*)dh, (uint8_t*)dv, (uint8_t*)dc, dstride, width / 8, height);
    }
    else if (depth != 8 && (width & 3) == 0 && (((uintptr_t)src | (uintptr_t)(sstride * 2)) & 15) == 0 && (((uintptr_t)d0 | (uintptr_t)dh | (uintptr_t)dv | (uintptr_t)dc | (uintptr_t)(dstride * 2)) & 7) == 0)
    {
        dim3 g4((width / 4 + 63) / 64, (height + 3) / 4);
        k_lowres_init_u16x4<<<g4, block, 0, c->stream>>>((const uint16_t*)src, sstride, (uint16_t*)d0, (uint16_t*)dh, (uint16_t*)dv, (uint16_t*)dc, dstride, width / 4, height);
    }
    else if (depth == 8)
        k_lowres_init<uint8_t><<<grid, block, 0, c->stream>>>((const uint8_t*)src, sstride, (uint8_t*)d0, (uint8_t*)dh, (uint8_t*)dv, (uint8_t*)dc, dstride, width, height);
    else
        k_lowres_init<uint16_t><<<grid, block, 0, c->stream>>>((const uint16_t*)src, sstride, (uint16_t*)d0, (uint16_t*)dh, (uint16_t*)dv, (uint16_t*)dc, dstride, width, height);
    CU_LAUNCH_CHECK(c);
    if (mx > 0 || my > 0)
    {
        void* planes[4] = { d0, dh, dv, dc };                    // all four planes in one launch
        if (depth == 8) { if (extend_border_n<uint8_t>(c, (uint8_t* const*)planes, 4, dstride, width, height, mx, my)) return -1; }
        else            { if (extend_border_n<uint16_t>(c, (uint16_t* const*)planes, 4, dstride, width, height, mx, my)) return -1; }
    }
    return 0;
}

// bitcost.cpp:95-109 + :49-55 (host helper; double log rounded to a float bit size, double lambda, cap 2^15-1).  The
// logarithm must be the double-precision one: a float logf moves some rounded costs by one (|mvd| = 656 qpel at qp 30, 8 bit).
void x265cu_mvcost_table(double lambda, int range, uint16_t* out)
{
    float log2_2 = (float)(2.0f / log(2.0));
    for (int i = 0; i <= range; i++)
    {
        float bits = i ? (float)(log((double)(i + 1)) * log2_2 + 1.718f) : 0.718f;
        double v = bits * lambda + 0.5f;
        if (v > 32767.0) v = 32767.0;
        out[range + i] = out[range - i] = (uint16_t)v;
    }
}

int x265cu_me_batch(x265cu_ctx* c, int depth, const void* fenc, int fencStride, const void* const* refs, int refStride, int lowres,
                    const uint16_t* mvcost, int mvcost_range, const x265cu_me_job* jobs, int n, int32_t* out)
{
    cudaSetDevice(c->device);
    (void)mvcost_range;
    return launch_me(c, depth, fenc, fencStride, refs, refStride, lowres, mvcost, jobs, n, out, c->d_counter);
}

int x265cu_me_batch_chroma(x265cu_ctx* c, int depth, const void* fenc, int fencStride, const void* const* refs, int refStride,
                           const x265cu_me_chroma* chroma, const uint16_t* mvcost, int mvcost_range, const x265cu_me_job* jobs, int n, int32_t* out)
{
    cudaSetDevice(c->device);
    (void)mvcost_range;
    if (!chroma || !chroma->fencCb_dev || !chroma->fencCr_dev || !chroma->refCb_dev || !chroma->refCr_dev || chroma->cstride <= 0)
    {
        x265cu_set_error("x265cu_me_batch_chroma: chroma planes missing", cudaErrorInvalidValue, __FILE__, __LINE__);
        return -1;
    }
    MeChromaArgs a;
    a.fencCb = chroma->fencCb_dev; a.fencCr = chroma->fencCr_dev; a.refCb = chroma->refCb_dev; a.refCr = chroma->refCr_dev; a.cstride = chroma->cstride;
    return launch_me(c, depth, fenc, fencStride, refs, refStride, 0, mvcost, jobs, n, out, c->d_counter, &a);
}

int x265cu_pred_cost_batch(x265cu_ctx* c, int depth, const void* fenc, int fencStride, const void* const* refs, int refStride,
                           const x265cu_me_chroma* chroma, const x265cu_pred_job* jobs, int n, int32_t* out)
{
    cudaSetDevice(c->device);
    if (n <= 0) return 0;
    PredChroma ch = { NULL, NULL, NULL, NULL, 0 };
    if (chroma && chroma->fencCb_dev && chroma->fencCr_dev && chroma->refCb_dev && chroma->refCr_dev && chroma->cstride > 0)
    {
        ch.fcb = chroma->fencCb_dev; ch.fcr = chroma->fencCr_dev; ch.rcb = chroma->refCb_dev; ch.rcr = chroma->refCr_dev; ch.cstride = chroma->cstride;
    }
    if (depth == 8) return launch_pred_cost_t<uint8_t>(c, fenc, fencStride, refs, refStride, ch, jobs, n, out);
    return launch_pred_cost_t<uint16_t>(c, fenc, fencStride, refs, refStride, ch, jobs, n, out);
}

__global__ void k_la_intra_zero(const x265cu_la_intra_job* jobs, int h8)
{
    const x265cu_la_intra_job jb = jobs[blockIdx.x];
    for (int i = threadIdx.x; i < h8; i += blockDim.x) jb.rowSatds[i] = 0;
    if (threadIdx.x < 2) jb.out[threadIdx.x] = 0;
}

int x265cu_lowres_intra_batch(x265cu_ctx* c, int depth, const x265cu_la_intra_job* jobs, int n, int stride, int w8, int h8, int lambda)
{
    cudaSetDevice(c->device);
    if (n <= 0) return 0;
    k_la_intra_zero<<<n, 128, 0, c->stream>>>(jobs, h8);
    CU_LAUNCH_CHECK(c);
    int bx = (w8 * h8 + 31) / 32; if (bx > c->sm_count * 4) bx = c->sm_count * 4;
    dim3 grid(bx, n);
    if (depth == 8) k_lowres_intra<uint8_t><<<grid, 256, 0, c->stream>>>(jobs, stride, w8, h8, lambda);
    else            k_lowres_intra<uint16_t><<<grid, 256, 0, c->stream>>>(jobs, stride, w8, h8, lambda);
    CU_LAUNCH_CHECK(c);
    return 0;
}

// frame totals of every triple of the batch: zeroed once before the launch (the slices of a triple accumulate into them)
__global__ void k_la_zero_out(const x265cu_la_job* jobs, int n)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const x265cu_la_job jb = jobs[i];
    if (jb.rows == 0 || (jb.rows & 0xffff) == 0) { jb.out[0] = 0; jb.out[1] = 0; jb.out[2] = 0; }
}

int x265cu_lookahead_cost_batch(x265cu_ctx* c, int depth, const x265cu_la_job* jobs, int n, int stride, int w8, int h8, const uint16_t* mvcost)
{
    cudaSetDevice(c->device);
    if (n <= 0) return 0;
    k_la_zero_out<<<(n + 127) / 128, 128, 0, c->stream>>>(jobs, n);
    CU_LAUNCH_CHECK(c);
    const size_t smem = sizeof(MeShared) * LA_WARPS;
    // cluster size: enough CTAs (of LA_WARPS warps) for the longest anti-diagonal in one round, at most 4
    const int maxdiag = h8 < (w8 + 1) / 2 ? h8 : (w8 + 1) / 2;
    int csize = (maxdiag + LA_WARPS - 1) / LA_WARPS;
    csize = csize >= 4 ? 4 : (csize >= 2 ? 2 : 1);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)n * csize); cfg.blockDim = dim3(LA_WARPS * 32); cfg.dynamicSmemBytes = smem; cfg.stream = c->stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = csize; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    if (depth == 8)
    {
        CU_CHECK(cudaFuncSetAttribute(k_lookahead_cost<uint8_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        CU_CHECK(cudaLaunchKernelEx(&cfg, k_lookahead_cost<uint8_t>, jobs, stride, w8, h8, mvcost));
    }
    else
    {
        CU_CHECK(cudaFuncSetAttribute(k_lookahead_cost<uint16_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        CU_CHECK(cudaLaunchKernelEx(&cfg, k_lookahead_cost<uint16_t>, jobs, stride, w8, h8, mvcost));
    }
    CU_LAUNCH_CHECK(c);
    return 0;
}

int x265cu_propagate_cost_batch(x265cu_ctx* c, int* dst, const uint16_t* propagateIn, const int32_t* intraCosts, const uint16_t* interCosts,
                                const int32_t* invQscales, double fpsFactor, int64_t len)
{
    cudaSetDevice(c->device);
    if (len <= 0) return 0;
    int64_t blocks = (len + 255) / 256; if (blocks > c->sm_count * 16) blocks = c->sm_count * 16;
    k_propagate_cost<<<(int)blocks, 256, 0, c->stream>>>(dst, propagateIn, intraCosts, interCosts, invQscales, fpsFactor, len);
    CU_LAUNCH_CHECK(c);
    return 0;
}

} // extern "C"

#include "analyser.cuh"
#include "thunks.cuh"
#include "la_weights.cuh"
#include "weightp.cuh"

static_assert(sizeof(x265cu_wp_frame) == 112 && sizeof(x265cu_wp_params) == 28 && sizeof(x265cu_wp_cand) == 16 &&
              sizeof(x265cu_wp_entry) == 16, "weightp records (include/x265_b200.h)");
static_assert(sizeof(x265cu_deblock_unit) == 16 && sizeof(x265cu_deblock_params) == 24, "deblocking records (include/x265_b200.h)");
static_assert(sizeof(x265cu_bidir_cu) == 20, "BIDIR record (include/x265_b200.h)");
static_assert(sizeof(x265cu_part_cu) == 144, "PART record (include/x265_b200.h)");
static_assert(sizeof(x265cu_part_b_cu) == 320, "PART_B record (include/x265_b200.h)");
static_assert(offsetof(x265cu_part_b_cu, biCost) == 64 && offsetof(x265cu_part_b_cu, interDir) == 128 &&
              offsetof(x265cu_part_b_cu, ref) == 144 && offsetof(x265cu_part_b_cu, zero) == 176 && offsetof(x265cu_part_b_cu, mv) == 192,
              "PART_B record layout (include/x265_b200.h, tests/test_gpu_x_partitions_b.py)");

// the argument rules of the deblocking calls on one set of planes; NULL when they hold
static const char* deblock_check(const char* fn, int depth, int width, int height, const void* luma, const void* cb,
                                 const void* cr, int stride, int cstride, const x265cu_deblock_unit* units,
                                 const x265cu_deblock_params* p)
{
    static char msg[160];
    const bool chroma = cb || cr;
    const char* why = NULL;
    if (depth != 8 && depth != 10) why = "depth must be 8 or 10";
    else if (width <= 0 || height <= 0 || (width & 7) || (height & 7)) why = "width and height must be positive multiples of 8";
    else if (!luma || !units || !p) why = "NULL luma plane, unit map or parameters";
    else if (chroma && (!cb || !cr)) why = "give both chroma planes or neither";
    else if (stride < width || (chroma && cstride < width / 2)) why = "stride smaller than the row";
    else if (p->sliceType < 0 || p->sliceType > 2) why = "sliceType must be 0 (B), 1 (P) or 2 (I)";
    else if (p->betaOffsetDiv2 < -6 || p->betaOffsetDiv2 > 6 || p->tcOffsetDiv2 < -6 || p->tcOffsetDiv2 > 6)
        why = "beta / tc offsets (div 2) must be in -6..6";
    else if (p->cbQpOffset < -12 || p->cbQpOffset > 12 || p->crQpOffset < -12 || p->crQpOffset > 12)
        why = "chroma QP offsets must be in -12..12";
    else if (p->transquantBypass != 0 && p->transquantBypass != 1) why = "transquantBypass must be 0 or 1";
    if (!why) return NULL;
    snprintf(msg, sizeof(msg), "%s: %s", fn, why);
    return msg;
}

// the band rules the three row calls share; NULL when they hold
static const char* rows_check(const char* fn, int height, int ctuSize, int ctuRow0, int ctuRow1)
{
    static char msg[160];
    const char* why = NULL;
    if (ctuSize != 16 && ctuSize != 32 && ctuSize != 64) why = "ctuSize must be 16, 32 or 64";
    else if (ctuRow0 < 0 || ctuRow0 >= ctuRow1) why = "need 0 <= ctuRow0 < ctuRow1";
    else if (height > 0 && ctuRow1 > (height + ctuSize - 1) / ctuSize) why = "ctuRow1 beyond the picture's last CTU row";
    if (!why) return NULL;
    snprintf(msg, sizeof(msg), "%s: %s", fn, why);
    return msg;
}

static lf::DeblockArgs deblock_args(void* luma, void* cb, void* cr, int stride, int cstride, int width, int height,
                                    const x265cu_deblock_unit* units, const x265cu_deblock_params* p, int y0, int y1)
{
    lf::DeblockArgs a;
    a.plane[0] = luma; a.plane[1] = cb; a.plane[2] = cr;
    a.stride = stride; a.cstride = cstride; a.width = width; a.height = height; a.units = units;
    a.sliceType = p->sliceType; a.betaOffset = p->betaOffsetDiv2 * 2; a.tcOffset = p->tcOffsetDiv2 * 2;
    a.cbQpOffset = p->cbQpOffset; a.crQpOffset = p->crQpOffset; a.bypass = p->transquantBypass;
    lf::deblock_window(a, y0, y1);
    return a;
}

extern "C" int x265cu_deblock_frame(x265cu_ctx* c, int depth, void* luma, int stride, void* cb, void* cr, int cstride,
                                    int width, int height, const x265cu_deblock_unit* units, const x265cu_deblock_params* p)
{
    cudaSetDevice(c->device);
    const char* bad = deblock_check("x265cu_deblock_frame", depth, width, height, luma, cb, cr, stride, cstride, units, p);
    if (bad) { x265cu_set_error(bad, cudaErrorInvalidValue, __FILE__, __LINE__); return -1; }
    const lf::DeblockArgs a = deblock_args(luma, cb, cr, stride, cstride, width, height, units, p, 0, height);
    return depth == 8 ? lf::launch_deblock_frame<uint8_t>(c, a, false) : lf::launch_deblock_frame<uint16_t>(c, a, false);
}

extern "C" int x265cu_deblock_rows(x265cu_ctx* c, int depth, int width, int height, int ctuSize, int ctuRow0, int ctuRow1,
                                   const void* src_y, const void* src_cb, const void* src_cr, int sstride, int scstride,
                                   void* dst_y, void* dst_cb, void* dst_cr, int stride, int cstride,
                                   const x265cu_deblock_unit* units, const x265cu_deblock_params* p)
{
    cudaSetDevice(c->device);
    const char* fn = "x265cu_deblock_rows";
    const char* bad = deblock_check(fn, depth, width, height, dst_y, dst_cb, dst_cr, stride, cstride, units, p);
    if (!bad) bad = deblock_check(fn, depth, width, height, src_y, src_cb, src_cr, sstride, scstride, units, p);
    if (!bad && (src_cb != NULL) != (dst_cb != NULL)) bad = "x265cu_deblock_rows: give chroma for both the source and the destination, or for neither";
    if (!bad) bad = rows_check(fn, height, ctuSize, ctuRow0, ctuRow1);
    if (bad) { x265cu_set_error(bad, cudaErrorInvalidValue, __FILE__, __LINE__); return -1; }
    const int y0 = ctuRow0 * ctuSize, y1 = min(height, ctuRow1 * ctuSize), es = depth == 8 ? 1 : 2;
    // out of place: the rows the passes read and write, luma [y0 - 4, y1 + 4) and chroma [y0/2 - 4, y1/2 + 4)
    for (int k = 0; k < 3; k++)
    {
        const void* s = k == 0 ? src_y : k == 1 ? src_cb : src_cr;
        void* d = k == 0 ? dst_y : k == 1 ? dst_cb : dst_cr;
        if (!d || d == s) continue;
        const int sh = k ? 1 : 0, r0 = max(0, (y0 >> sh) - 4), r1 = min(height >> sh, (y1 >> sh) + 4);
        const size_t ss = (size_t)(k ? scstride : sstride) * es, ds = (size_t)(k ? cstride : stride) * es;
        CU_CHECK(cudaMemcpy2DAsync((uint8_t*)d + r0 * ds, ds, (const uint8_t*)s + r0 * ss, ss, (size_t)(width >> sh) * es,
                                   r1 - r0, cudaMemcpyDeviceToDevice, c->stream));
    }
    const lf::DeblockArgs a = deblock_args(dst_y, dst_cb, dst_cr, stride, cstride, width, height, units, p, y0, y1);
    return depth == 8 ? lf::launch_deblock_frame<uint8_t>(c, a, true) : lf::launch_deblock_frame<uint16_t>(c, a, true);
}

static_assert(sizeof(x265cu_sao_ctu) == 8, "SAO record (include/x265_b200.h)");

// the argument rules both SAO calls share; NULL when they hold
static const char* sao_check(const char* fn, int depth, int width, int height, int ctuSize, const void* y, const void* cb,
                             const void* cr, int stride, int cstride)
{
    static char msg[160];
    const char* why = NULL;
    if (depth != 8 && depth != 10) why = "depth must be 8 or 10";
    else if (width <= 0 || height <= 0 || (width & 7) || (height & 7)) why = "width and height must be positive multiples of 8";
    else if (ctuSize != 16 && ctuSize != 32 && ctuSize != 64) why = "ctuSize must be 16, 32 or 64";
    else if (!y) why = "NULL luma plane";
    else if ((cb != NULL) != (cr != NULL)) why = "give both chroma planes or neither";
    else if (stride < width || (cb && cstride < width / 2)) why = "stride smaller than the row";
    if (!why) return NULL;
    snprintf(msg, sizeof(msg), "%s: %s", fn, why);
    return msg;
}

static int ilog2_ctu(int ctuSize) { return ctuSize == 64 ? 6 : ctuSize == 32 ? 5 : 4; }

// x265cu_sao_stats_frame over CTU rows [ctuRow0, ctuRow1); fn names the call in the messages
static int sao_stats(const char* fn, x265cu_ctx* c, int depth, int width, int height, int ctuSize, int ctuRow0, int ctuRow1,
                     const void* fenc_y, const void* fenc_cb, const void* fenc_cr, int fstride, int fcstride,
                     const void* rec_y, const void* rec_cb, const void* rec_cr, int stride, int cstride, int32_t* stats)
{
    static char msg[200];
    cudaSetDevice(c->device);
    const char* bad = sao_check(fn, depth, width, height, ctuSize, rec_y, rec_cb, rec_cr, stride, cstride);
    if (!bad) bad = sao_check(fn, depth, width, height, ctuSize, fenc_y, fenc_cb, fenc_cr, fstride, fcstride);
    if (!bad && (fenc_cb != NULL) != (rec_cb != NULL))
        bad = (snprintf(msg, sizeof(msg), "%s: give chroma for both the source and the reconstruction, or for neither", fn), msg);
    if (!bad && !stats) bad = (snprintf(msg, sizeof(msg), "%s: NULL stats", fn), msg);
    if (!bad) bad = rows_check(fn, height, ctuSize, ctuRow0, ctuRow1);
    if (bad) { x265cu_set_error(bad, cudaErrorInvalidValue, __FILE__, __LINE__); return -1; }
    lf::SaoStatsArgs a;
    a.fenc[0] = fenc_y; a.fenc[1] = fenc_cb; a.fenc[2] = fenc_cr;
    a.rec[0] = rec_y; a.rec[1] = rec_cb; a.rec[2] = rec_cr;
    a.fstride = fstride; a.fcstride = fcstride; a.stride = stride; a.cstride = cstride;
    a.width = width; a.height = height; a.log2Ctu = ilog2_ctu(ctuSize);
    a.cols = (width + ctuSize - 1) / ctuSize; a.planes = rec_cb ? 3 : 1; a.stats = stats; a.row0 = ctuRow0;
    const int n = a.cols * (ctuRow1 - ctuRow0);
    return depth == 8 ? lf::launch_sao_stats_frame<uint8_t>(c, a, n) : lf::launch_sao_stats_frame<uint16_t>(c, a, n);
}

extern "C" int x265cu_sao_stats_frame(x265cu_ctx* c, int depth, int width, int height, int ctuSize,
                                      const void* fenc_y, const void* fenc_cb, const void* fenc_cr, int fstride, int fcstride,
                                      const void* rec_y, const void* rec_cb, const void* rec_cr, int stride, int cstride, int32_t* stats)
{
    const int rows = ctuSize > 0 && height > 0 ? (height + ctuSize - 1) / ctuSize : 1;
    return sao_stats("x265cu_sao_stats_frame", c, depth, width, height, ctuSize, 0, rows, fenc_y, fenc_cb, fenc_cr, fstride,
                     fcstride, rec_y, rec_cb, rec_cr, stride, cstride, stats);
}

extern "C" int x265cu_sao_stats_rows(x265cu_ctx* c, int depth, int width, int height, int ctuSize, int ctuRow0, int ctuRow1,
                                     const void* fenc_y, const void* fenc_cb, const void* fenc_cr, int fstride, int fcstride,
                                     const void* rec_y, const void* rec_cb, const void* rec_cr, int stride, int cstride, int32_t* stats)
{
    return sao_stats("x265cu_sao_stats_rows", c, depth, width, height, ctuSize, ctuRow0, ctuRow1, fenc_y, fenc_cb, fenc_cr,
                     fstride, fcstride, rec_y, rec_cb, rec_cr, stride, cstride, stats);
}

// x265cu_sao_apply_frame (src == dst, every CTU row) and x265cu_sao_apply_rows (src != dst, CTU rows [ctuRow0, ctuRow1))
static int sao_apply(const char* fn, x265cu_ctx* c, int depth, int width, int height, int ctuSize, int ctuRow0, int ctuRow1,
                     const void* sy, const void* scb, const void* scr, int sstride, int scstride,
                     void* y, void* cb, void* cr, int stride, int cstride,
                     const x265cu_sao_ctu* params, int saoLuma, int saoChroma, const x265cu_deblock_unit* units,
                     const void* fenc_y, const void* fenc_cb, const void* fenc_cr, int fstride, int fcstride)
{
    static char msg[200];
    cudaSetDevice(c->device);
    const bool rows = sy != y;
    const char* bad = sao_check(fn, depth, width, height, ctuSize, y, cb, cr, stride, cstride);
    if (!bad && rows) bad = sao_check(fn, depth, width, height, ctuSize, sy, scb, scr, sstride, scstride);
    if (!bad && rows && (scb != NULL) != (cb != NULL))
        bad = (snprintf(msg, sizeof(msg), "%s: give chroma for both the source and the destination, or for neither", fn), msg);
    if (!bad && rows && cb && (scb == cb || scr == cr))
        bad = (snprintf(msg, sizeof(msg), "%s: the source and destination planes must differ", fn), msg);
    if (!bad && !params) bad = (snprintf(msg, sizeof(msg), "%s: NULL parameters", fn), msg);
    if (!bad && (saoLuma != 0 && saoLuma != 1 || saoChroma != 0 && saoChroma != 1))
        bad = (snprintf(msg, sizeof(msg), "%s: saoLuma / saoChroma must be 0 or 1", fn), msg);
    if (!bad && saoChroma && !cb) bad = (snprintf(msg, sizeof(msg), "%s: saoChroma set without chroma planes", fn), msg);
    if (!bad && units)
    {
        bad = sao_check(fn, depth, width, height, ctuSize, fenc_y, fenc_cb, fenc_cr, fstride, fcstride);
        if (!bad && (fenc_cb != NULL) != (cb != NULL))
            bad = (snprintf(msg, sizeof(msg), "%s: bypass units need source planes for every plane filtered", fn), msg);
    }
    if (!bad) bad = rows_check(fn, height, ctuSize, ctuRow0, ctuRow1);
    if (bad) { x265cu_set_error(bad, cudaErrorInvalidValue, __FILE__, __LINE__); return -1; }
    lf::SaoApplyArgs a;
    a.plane[0] = y; a.plane[1] = cb; a.plane[2] = cr;
    a.src[0] = sy; a.src[1] = scb; a.src[2] = scr;
    a.fenc[0] = fenc_y; a.fenc[1] = fenc_cb; a.fenc[2] = fenc_cr;
    a.stride = stride; a.cstride = cstride; a.sstride = sstride; a.scstride = scstride; a.fstride = fstride; a.fcstride = fcstride;
    a.width = width; a.height = height; a.log2Ctu = ilog2_ctu(ctuSize);
    a.cols = (width + ctuSize - 1) / ctuSize; a.rows = (height + ctuSize - 1) / ctuSize; a.planes = cb ? 3 : 1;
    a.row0 = ctuRow0;
    a.on[0] = saoLuma; a.on[1] = a.on[2] = saoChroma;
    a.params = params; a.units = units;
    a.lines[0] = a.lines[1] = a.lines[2] = NULL;
    return depth == 8 ? lf::launch_sao_apply_frame<uint8_t>(c, a, ctuRow1) : lf::launch_sao_apply_frame<uint16_t>(c, a, ctuRow1);
}

extern "C" int x265cu_sao_apply_frame(x265cu_ctx* c, int depth, int width, int height, int ctuSize,
                                      void* y, void* cb, void* cr, int stride, int cstride,
                                      const x265cu_sao_ctu* params, int saoLuma, int saoChroma, const x265cu_deblock_unit* units,
                                      const void* fenc_y, const void* fenc_cb, const void* fenc_cr, int fstride, int fcstride)
{
    const int rows = ctuSize > 0 && height > 0 ? (height + ctuSize - 1) / ctuSize : 1;
    return sao_apply("x265cu_sao_apply_frame", c, depth, width, height, ctuSize, 0, rows, y, cb, cr, stride, cstride, y, cb, cr,
                     stride, cstride, params, saoLuma, saoChroma, units, fenc_y, fenc_cb, fenc_cr, fstride, fcstride);
}

extern "C" int x265cu_sao_apply_rows(x265cu_ctx* c, int depth, int width, int height, int ctuSize, int ctuRow0, int ctuRow1,
                                     const void* src_y, const void* src_cb, const void* src_cr, int sstride, int scstride,
                                     void* dst_y, void* dst_cb, void* dst_cr, int stride, int cstride,
                                     const x265cu_sao_ctu* params, int saoLuma, int saoChroma, const x265cu_deblock_unit* units,
                                     const void* fenc_y, const void* fenc_cb, const void* fenc_cr, int fstride, int fcstride)
{
    if (src_y && src_y == dst_y)
    {
        x265cu_set_error("x265cu_sao_apply_rows: src_y == dst_y (the call is out of place)", cudaErrorInvalidValue, __FILE__, __LINE__);
        return -1;
    }
    return sao_apply("x265cu_sao_apply_rows", c, depth, width, height, ctuSize, ctuRow0, ctuRow1, src_y, src_cb, src_cr, sstride,
                     scstride, dst_y, dst_cb, dst_cr, stride, cstride, params, saoLuma, saoChroma, units, fenc_y, fenc_cb, fenc_cr,
                     fstride, fcstride);
}

// ---------------------------------------------------------------------------------------------
// cuTree's propagation chain (Lookahead::cuTree, slicetype.cpp:2538-2639) on the device
namespace {
enum { CT_EST, CT_CLEAR, CT_STEP, CT_SWAP, CT_FINISH, CT_COPY_AQ };
struct CtOp { int kind, a, b, c, d; };
const int CT_TYPE_B = 5;                                              // X265_TYPE_B

// The reference's control flow as a list of operations: the singleCost calls (CT_EST p0 p1 b), the memsets, the steps
// (CT_STEP p0 p1 b referenced), the pointer swaps and the cuTreeFinish calls (CT_FINISH frame ref0Distance).
const char* cutree_plan(const int32_t* st, int numframes, const x265cu_cutree_params* p, std::vector<CtOp>& ops)
{
    const int idx = !p->bIntra;
    int lastnonb, curnonb = 1, bframes = 0;
    int i = numframes;
    while (i > 0 && st[i] == CT_TYPE_B)
        i--;
    lastnonb = i;
    auto op = [&](int k, int a, int b = 0, int c = 0, int d = 0) { ops.push_back(CtOp{ k, a, b, c, d }); };
    auto step = [&](int p0, int p1, int b, int referenced) {
        op(CT_STEP, p0, p1, b, referenced);
        if (p->vbv && p->lookaheadDepth && referenced)
            op(CT_FINISH, b, b == p1 ? b - p0 : 0);                   // :2745-2746
    };
    if (!p->lookaheadDepth)
    {
        if (p->bIntra)
        {
            op(CT_CLEAR, 0);
            op(CT_COPY_AQ, 0);
            return NULL;
        }
        op(CT_SWAP, lastnonb, 0);
        op(CT_CLEAR, 0);
    }
    else
    {
        if (lastnonb < idx)
            return NULL;
        op(CT_CLEAR, lastnonb);
    }
    while (i-- > idx)
    {
        curnonb = i;
        while (st[curnonb] == CT_TYPE_B && curnonb > 0)
            curnonb--;
        if (curnonb < idx)
            break;
        op(CT_EST, curnonb, lastnonb, lastnonb);
        op(CT_CLEAR, curnonb);
        bframes = lastnonb - curnonb - 1;
        if (p->bBPyramid && bframes > 1)
        {
            const int middle = (bframes + 1) / 2 + curnonb;
            op(CT_EST, curnonb, lastnonb, middle);
            op(CT_CLEAR, middle);
            while (i > curnonb)
            {
                const int p0 = i > middle ? middle : curnonb;
                const int p1 = i < middle ? middle : lastnonb;
                if (i != middle)
                {
                    op(CT_EST, p0, p1, i);
                    step(p0, p1, i, 0);
                }
                i--;
            }
            step(curnonb, lastnonb, middle, 1);
        }
        else
        {
            while (i > curnonb)
            {
                op(CT_EST, curnonb, lastnonb, i);
                step(curnonb, lastnonb, i, 0);
                i--;
            }
        }
        step(curnonb, lastnonb, lastnonb, 1);
        lastnonb = curnonb;
    }
    if (!p->lookaheadDepth)
    {
        if (lastnonb == 0)
            return "the window reaches estimateCUPropagate(0, 0, 0) (lookaheadDepth 0 without an anchor after frame 0)";
        op(CT_EST, 0, lastnonb, lastnonb);
        step(0, lastnonb, lastnonb, 1);
        op(CT_SWAP, lastnonb, 0);
    }
    op(CT_FINISH, lastnonb, lastnonb);
    if (p->bBPyramid && bframes > 1 && !p->vbv)
        op(CT_FINISH, lastnonb + (bframes + 1) / 2, 0);
    for (const CtOp& o : ops)
        if (o.kind == CT_EST && (o.c - o.a >= X265CU_CUTREE_DIST || o.b - o.c >= X265CU_CUTREE_DIST))
            return "a mini-GOP is longer than X265_BFRAME_MAX + 1 frames";
    return NULL;
}

const char* cutree_args(const int32_t* st, int numframes, const x265cu_cutree_params* p, std::vector<CtOp>& ops)
{
    if (!st || !p || numframes < 0)
        return "NULL frames / parameters or numframes < 0";
    if (p->fpsNum <= 0 || p->fpsDenom <= 0)
        return "fpsNum and fpsDenom must be positive";
    return cutree_plan(st, numframes, p, ops);
}

double clip_duration(double f) { return std::min(std::max(0.01, f), 1.00); }   // CLIP_DURATION (ratecontrol.h:42-47)
} // namespace

extern "C" int x265cu_cutree_estimates(const int32_t* sliceTypes, int numframes, const x265cu_cutree_params* params, int32_t* triples,
                                       int maxTriples)
{
    std::vector<CtOp> ops;
    const char* bad = cutree_args(sliceTypes, numframes, params, ops);
    int n = 0;
    for (const CtOp& o : ops)
        if (o.kind == CT_EST)
        {
            if (n >= maxTriples || !triples) { bad = "more estimates than maxTriples"; break; }
            triples[3 * n] = o.a; triples[3 * n + 1] = o.b; triples[3 * n + 2] = o.c;
            n++;
        }
    if (bad)
    {
        static thread_local char msg[256];
        snprintf(msg, sizeof(msg), "x265cu_cutree_estimates: %s", bad);
        x265cu_set_error(msg, cudaErrorInvalidValue, __FILE__, __LINE__);
        return -1;
    }
    return n;
}

extern "C" int x265cu_cutree(x265cu_ctx* c, x265cu_cutree_frame* frames, int numframes, const x265cu_cutree_params* p, int w8, int h8,
                             int32_t* finish, int maxFinish)
{
    static thread_local char msg[256];
    cudaSetDevice(c->device);
    std::vector<CtOp> ops;
    std::vector<int32_t> st(numframes >= 0 && frames ? numframes + 1 : 0);
    for (size_t f = 0; f < st.size(); f++)
        st[f] = frames[f].sliceType;
    const char* bad = frames ? cutree_args(st.data(), numframes, p, ops) : "NULL frames";
    if (!bad && (w8 <= 0 || h8 <= 0))
        bad = "w8 and h8 must be positive";
    int nfinish = 0, nsteps = 0;
    for (size_t k = 0; k < ops.size() && !bad; k++)
    {
        const CtOp& o = ops[k];
        if (o.kind == CT_FINISH || o.kind == CT_COPY_AQ)
            nfinish++;
        if (o.kind == CT_CLEAR && !frames[o.a].propagateCost)
            bad = (snprintf(msg, sizeof(msg), "frame %d: NULL propagateCost", o.a), msg);
        if (o.kind != CT_STEP)
            continue;
        nsteps++;
        const int p0 = o.a, p1 = o.b, b = o.c;
        const x265cu_cutree_frame& f = frames[b];
        if (!frames[p0].propagateCost || !frames[p1].propagateCost || !f.propagateCost)
            bad = (snprintf(msg, sizeof(msg), "step (%d, %d, %d): NULL propagateCost", p0, p1, b), msg);
        else if (!f.intraCost || !f.invQscale)
            bad = (snprintf(msg, sizeof(msg), "frame %d: NULL intraCost or invQscale", b), msg);
        else if (!f.lowresCosts[b - p0][p1 - b])
            bad = (snprintf(msg, sizeof(msg), "estimate (%d, %d, %d) not supplied (lowresCosts[%d][%d])", p0, p1, b, b - p0, p1 - b), msg);
        else if (!f.mvs[0][b - p0] || (p1 > b && !f.mvs[1][p1 - b]))
            bad = (snprintf(msg, sizeof(msg), "estimate (%d, %d, %d): motion field not supplied", p0, p1, b), msg);
    }
    if (!bad && nfinish > maxFinish)
        bad = (snprintf(msg, sizeof(msg), "%d cuTreeFinish calls, room for %d", nfinish, maxFinish), msg);
    if (!bad && nfinish && !finish)
        bad = "NULL finish list";
    const int ncu = w8 * h8;
    const size_t amountBytes = (size_t)CUTREE_MAX_STEPS * ncu * 4, need = amountBytes + (size_t)(nsteps + 1) * 4;
    if (!bad && c->cutree_bytes < need)
    {
        cudaFree(c->d_cutree);
        c->d_cutree = NULL; c->cutree_bytes = 0;
        if (cudaMalloc(&c->d_cutree, need) != cudaSuccess) { x265cu_set_error("x265cu_cutree: scratch", cudaGetLastError(), __FILE__, __LINE__); return -1; }
        c->cutree_bytes = need;
    }
    if (bad)
    {
        static thread_local char full[320];
        snprintf(full, sizeof(full), "x265cu_cutree: %s", bad);
        x265cu_set_error(full, cudaErrorInvalidValue, __FILE__, __LINE__);
        return -1;
    }
    int* amounts = (int*)c->d_cutree;
    int* flags = (int*)((char*)c->d_cutree + amountBytes);
    CU_CHECK(cudaMemsetAsync(flags, 0, (size_t)(nsteps + 1) * 4, c->stream));

    double totalDuration = 0.0;                                       // :2545-2549, the summing loop
    for (int j = 0; j <= numframes; j++)
        totalDuration += (double)p->fpsDenom / p->fpsNum;
    const double averageDuration = totalDuration / (numframes + 1);
    const double fpsFactor = clip_duration((double)p->fpsDenom / p->fpsNum) / clip_duration(averageDuration);   // :2654

    std::vector<uint16_t*> pc(numframes + 1);
    for (int f = 0; f <= numframes; f++)
        pc[f] = frames[f].propagateCost;
    // the pending level: its steps and the arrays they read (their own propagateCost) and add into (p0's, p1's)
    CuTreeLevel L;
    L.n = 0;
    std::vector<const uint16_t*> R, W;
    int level = 0;
    auto has = [](const std::vector<const uint16_t*>& v, const uint16_t* q) { return std::find(v.begin(), v.end(), q) != v.end(); };
    auto flush = [&]() -> int {
        if (!L.n) return 0;
        const dim3 grid((ncu + 255) / 256, L.n);
        int* flag = flags + level++;
        k_cutree_amount<<<grid, 256, 0, c->stream>>>(L, ncu, fpsFactor, amounts, flag);
        CU_LAUNCH_CHECK(c);
        k_cutree_scatter<<<grid, 256, 0, c->stream>>>(L, w8, h8, amounts, flag);
        CU_LAUNCH_CHECK(c);
        L.n = 0; R.clear(); W.clear();
        return 0;
    };
    // a memset runs at once in stream order, after the launched levels and before the pending one: legal when the pending
    // level does not touch the array (the reference's memset precedes every pending step that touches it)
    auto zero = [&](uint16_t* q, size_t n) -> int {
        if ((has(R, q) || has(W, q)) && flush()) return -1;
        CU_CHECK(cudaMemsetAsync(q, 0, n * sizeof(uint16_t), c->stream));
        return 0;
    };
    nfinish = 0;
    for (const CtOp& o : ops)
    {
        switch (o.kind)
        {
        case CT_CLEAR:
            if (zero(pc[o.a], ncu)) return -1;
            break;
        case CT_SWAP:
            std::swap(pc[o.a], pc[o.b]);
            break;
        case CT_FINISH:
        case CT_COPY_AQ:
            finish[2 * nfinish] = o.a; finish[2 * nfinish + 1] = o.kind == CT_FINISH ? o.b : -1;
            nfinish++;
            break;
        case CT_STEP:
        {
            const int p0 = o.a, p1 = o.b, b = o.c, referenced = o.d;
            if (!referenced && zero(pc[b], w8)) return -1;            // :2657-2658, row 0 of b's own array
            const uint16_t* in = referenced ? pc[b] : NULL;
            if (L.n == CUTREE_MAX_STEPS || (in && has(W, in)) || has(R, pc[p0]) || (p1 > b && has(R, pc[p1])))
                if (flush()) return -1;
            const x265cu_cutree_frame& f = frames[b];
            CuTreeStep& s = L.s[L.n++];
            s.intraCost = f.intraCost; s.invQscale = f.invQscale; s.propagateIn = in;
            s.lowresCosts = f.lowresCosts[b - p0][p1 - b];
            s.mvs[0] = f.mvs[0][b - p0];
            s.mvs[1] = p1 > b ? f.mvs[1][p1 - b] : f.mvs[0][b - p0];  // a P estimate has no list-1 CUs
            s.ref[0] = pc[p0]; s.ref[1] = pc[p1];
            const int distScaleFactor = (((b - p0) << 8) + ((p1 - p0) >> 1)) / (p1 - p0);
            const int bipredWeight = p->bEnableWeightedBiPred ? 64 - (distScaleFactor >> 2) : 32;
            s.bipredWeight[0] = bipredWeight; s.bipredWeight[1] = 64 - bipredWeight;
            if (in) R.push_back(in);
            W.push_back(pc[p0]);
            if (p1 > b) W.push_back(pc[p1]);
            break;
        }
        default:
            break;
        }
    }
    if (flush()) return -1;
    for (int f = 0; f <= numframes; f++)
        frames[f].propagateCost = pc[f];
    return nfinish;
}

// ---------------- adaptive quantisation: calcAdaptiveQuantFrame (slicetype.cpp:444-694) ----------------
// the argument rules of x265cu_aq_energy; NULL when they hold
static const char* aq_energy_check(int depth, const void* luma, int stride, const void* cb, const void* cr, int cstride,
                                   int width, int height, int qgSize, const void* energy, const void* totals)
{
    if (depth != 8 && depth != 10) return "depth must be 8 or 10";
    if (qgSize != 8 && qgSize != 16 && qgSize != 32 && qgSize != 64) return "qgSize must be 8, 16, 32 or 64";
    if (width <= 0 || height <= 0 || (width & 1) || (height & 1)) return "width and height must be positive and even";
    if (!luma || !energy || !totals) return "NULL luma plane or output";
    if (!cb != !cr) return "give both chroma planes or neither";
    if (stride < width || (cb && cstride < width / 2)) return "stride smaller than the row";
    return NULL;
}

static int aq_energy_launch(x265cu_ctx* c, int depth, const void* luma, int stride, const void* cb, const void* cr, int cstride,
                            int width, int height, int qgSize, uint32_t* energy, uint64_t* totals)
{
    const int L = qgSize == 8 ? 8 : 16;
    const int bw = (width + L - 1) / L, nb = bw * ((height + L - 1) / L);
    CU_CHECK(cudaMemsetAsync(totals, 0, 6 * sizeof(uint64_t), c->stream));
    const dim3 grid((nb + AQ_WARPS - 1) / AQ_WARPS), block(AQ_WARPS * 32);
    unsigned long long* t = (unsigned long long*)totals;
#define AQ_LAUNCH(P, LB) k_aq_energy<P, LB><<<grid, block, 0, c->stream>>>((const P*)luma, stride, (const P*)cb, (const P*)cr, \
                                                                           cstride, width, height, bw, nb, energy, t)
    if (depth == 8) { if (L == 8) AQ_LAUNCH(uint8_t, 8); else AQ_LAUNCH(uint8_t, 16); }
    else            { if (L == 8) AQ_LAUNCH(uint16_t, 8); else AQ_LAUNCH(uint16_t, 16); }
#undef AQ_LAUNCH
    CU_LAUNCH_CHECK(c);
    return 0;
}

extern "C" int x265cu_aq_energy(x265cu_ctx* c, int depth, const void* luma, int stride, const void* cb, const void* cr, int cstride,
                                int width, int height, int qgSize, uint32_t* energy_dev, uint64_t* totals_dev)
{
    const char* bad = aq_energy_check(depth, luma, stride, cb, cr, cstride, width, height, qgSize, energy_dev, totals_dev);
    if (bad)
    {
        char msg[160];
        snprintf(msg, sizeof(msg), "x265cu_aq_energy: %s", bad);
        x265cu_set_error(msg, cudaErrorInvalidValue, __FILE__, __LINE__);
        return -1;
    }
    cudaSetDevice(c->device);
    return aq_energy_launch(c, depth, luma, stride, cb, cr, cstride, width, height, qgSize, energy_dev, totals_dev);
}

// x265_exp2fix8 (common/common.cpp:96-103); its table is round((2^(i/64) - 1) * 256)
static int aq_exp2fix8(double x)
{
    static const struct Lut { uint8_t v[64]; Lut() { for (int i = 0; i < 64; i++) v[i] = (uint8_t)floor((exp2(i / 64.0) - 1) * 256 + 0.5); } } lut;
    int i = (int)(x * (-64.f / 6.f) + 512.5f);
    if (i < 0) return 0;
    if (i > 1023) return 0xffff;
    return (lut.v[i & 63] + 256) << (i >> 6) >> 8;
}

// the rules of x265cu_aq_finish; NULL when they hold
static const char* aq_finish_check(int depth, int width, int height, const x265cu_aq_params* p, const void* energy,
                                   const void* totals, const x265cu_aq_out* out)
{
    if (!p) return "NULL parameters";
    if (p->aqMode == 4) return "aq-mode 4 (EDGE) stays on the host";
    if (p->aqMode < 0 || p->aqMode > 4) return "aqMode must be 0..3";
    if (p->hevcAq) return "hevc-aq stays on the host";
    if (p->hdr10Opt) return "HDR10 opt stays on the host";
    if (p->aqMotion) return "aq-motion stays on the host";
    if (depth != 8 && depth != 10) return "depth must be 8 or 10";
    if (p->qgSize != 8 && p->qgSize != 16 && p->qgSize != 32 && p->qgSize != 64) return "qgSize must be 8, 16, 32 or 64";
    if (width <= 0 || height <= 0 || (width & 1) || (height & 1)) return "width and height must be positive and even";
    if (!energy || !totals) return "NULL energies or totals";
    if (out && out->invQscaleFactor8x8 && !out->invQscaleFactor) return "invQscaleFactor8x8 needs invQscaleFactor";
    if (p->variance && p->weightp)
    {
        const int L = p->qgSize == 8 ? 8 : 16;
        const int wp = ((width + 8) >> 4) << 4, hp = ((height + 8) >> 4) << 4;
        if ((wp + L - 1) / L != (width + L - 1) / L || (hp + L - 1) / L != (height + L - 1) / L)
            return "with weightp the fades pass walks a grid other than the energy grid; it stays on the host";
    }
    return NULL;
}

// slicetype.cpp:466-693 on the energies (one acEnergyCu per grid block, raster order) and one pass's plane totals
static void aq_finish(int depth, int W, int H, const x265cu_aq_params* p, const uint32_t* energy, const uint64_t* totals,
                      const x265cu_aq_out* o)
{
    const int qg = p->qgSize, L = qg == 8 ? 8 : 16;
    const int bw = (W + L - 1) / L, bh = (H + L - 1) / L, nb = bw * bh;
    const int w8 = ((W / 2) + 7) >> 3, h8 = ((H / 2) + 7) >> 3;
    const int blockCount = qg == 8 ? (2 * w8) * (2 * h8) : w8 * h8;
    const float modeOneConst = qg == 8 ? 11.427f : 14.427f, modeTwoConst = qg == 8 ? 8.f : 11.f;
    const float* quantOffsets = p->quantOffsets;
    std::vector<double> qpBuf, cut;
    std::vector<int32_t> invqBuf;
    double* qpAq = o->qpAqOffset;
    int32_t* invq = o->invQscaleFactor;
    if (!qpAq) { qpBuf.assign(blockCount, 0.0); qpAq = qpBuf.data(); }
    if (!invq) { invqBuf.assign(blockCount, 0); invq = invqBuf.data(); }
    uint64_t wsum[3] = { 0, 0, 0 }, wssd[3] = { 0, 0, 0 };
    auto add_pass = [&]() { for (int i = 0; i < 3; i++) { wsum[i] += totals[2 * i]; wssd[i] += totals[2 * i + 1]; } };

    if (p->aqMode == 0 || p->aqStrength == 0)
    {
        if (p->aqMode && p->aqStrength == 0)
            for (int i = 0; i < blockCount; i++)
            {
                qpAq[i] = quantOffsets ? quantOffsets[i] : 0;
                invq[i] = quantOffsets ? aq_exp2fix8(qpAq[i]) : 256;
            }
        if (p->weightp)
            add_pass();
    }
    else
    {
        add_pass();                                  // modes 2 / 3: the first loop's acEnergyCu; mode 1: the second's
        double avg_adj_pow2 = 0, avg_adj = 0, qp_adj = 0, bias_strength = 0.f, strength = 0.f;
        if (p->aqMode == 2 || p->aqMode == 3)
        {
            cut.resize(nb);
            const double bit_depth_correction = 1.f / (1 << (2 * (depth - 8)));
            for (int b = 0; b < nb; b++)
            {
                qp_adj = pow(energy[b] * bit_depth_correction + 1, 0.1);
                cut[b] = qp_adj;
                avg_adj += qp_adj;
                avg_adj_pow2 += qp_adj * qp_adj;
            }
            avg_adj /= blockCount;                   // blockCount, not the number of loop iterations
            avg_adj_pow2 /= blockCount;
            strength = p->aqStrength * avg_adj;
            avg_adj = avg_adj - 0.5f * (avg_adj_pow2 - modeTwoConst) / avg_adj;
            bias_strength = p->aqStrength;
        }
        else
            strength = p->aqStrength * 1.0397f;
        for (int b = 0; b < nb; b++)
        {
            if (p->aqMode == 3)
            {
                qp_adj = cut[b];
                qp_adj = strength * (qp_adj - avg_adj) + bias_strength * (1.f - modeTwoConst / (qp_adj * qp_adj));
            }
            else if (p->aqMode == 2)
            {
                qp_adj = cut[b];
                qp_adj = strength * (qp_adj - avg_adj);
            }
            else
            {
                const uint32_t e = energy[b];
                qp_adj = strength * (log2(e > 1u ? e : 1u) - (modeOneConst + 2 * (depth - 8)));
            }
            if (quantOffsets)
                qp_adj += quantOffsets[b];
            qpAq[b] = qp_adj;
            invq[b] = aq_exp2fix8(qp_adj);
        }
    }
    if (qg == 8 && o->invQscaleFactor8x8)            // the full-res stride is widthInCU * 2, whatever the loop wrote
        for (int cuY = 0; cuY < h8; cuY++)
            for (int cuX = 0; cuX < w8; cuX++)
            {
                const int i = cuX * 2 + cuY * w8 * 4;
                o->invQscaleFactor8x8[cuX + cuY * w8] = (invq[i] + invq[i + 1] + invq[i + 2 * w8] + invq[i + 2 * w8 + 1]) / 4;
            }
    int maxCol = W, maxRow = H;
    if (p->weightp)
    {
        maxCol = ((maxCol + 8) >> 4) << 4;
        maxRow = ((maxRow + 8) >> 4) << 4;
        const int width[3] = { maxCol, maxCol >> 1, maxCol >> 1 }, height[3] = { maxRow, maxRow >> 1, maxRow >> 1 };
        for (int i = 0; i < 3; i++)                  // uint64, wraps as the reference's does (4:0:0: chroma stays 0)
            wssd[i] = wssd[i] - (wsum[i] * wsum[i] + (width[i] * height[i]) / 2) / (width[i] * height[i]);
    }
    if (p->variance)                                 // the fades pass: a second acEnergyCu pass, after the correction
    {
        uint64_t rowVariance = 0;                    // never reset between rows
        double frameVariance = 0;
        for (int by = 0; by < bh; by++)
        {
            for (int bx = 0; bx < bw; bx++)
            {
                const uint32_t e = energy[by * bw + bx];
                if (o->blockVariance) o->blockVariance[by * bw + bx] = e;
                rowVariance += e;
            }
            frameVariance += (rowVariance / maxCol);
        }
        frameVariance /= maxRow;
        if (o->frameVariance) *o->frameVariance = frameVariance;
        add_pass();
    }
    for (int i = 0; i < 3; i++)
    {
        if (o->wp_sum) o->wp_sum[i] = wsum[i];
        if (o->wp_ssd) o->wp_ssd[i] = wssd[i];
    }
}

static int aq_refuse(const char* fn, const char* why)
{
    char msg[200];
    snprintf(msg, sizeof(msg), "%s: %s", fn, why);
    x265cu_set_error(msg, cudaErrorInvalidValue, __FILE__, __LINE__);
    return -1;
}

extern "C" int x265cu_aq_finish(int depth, int width, int height, const x265cu_aq_params* p, const uint32_t* energy,
                                const uint64_t* totals, const x265cu_aq_out* out)
{
    const char* bad = aq_finish_check(depth, width, height, p, energy, totals, out);
    if (bad) return aq_refuse("x265cu_aq_finish", bad);
    const x265cu_aq_out none = {};
    aq_finish(depth, width, height, p, energy, totals, out ? out : &none);
    return 0;
}

extern "C" int x265cu_aq_frame(x265cu_ctx* c, int depth, const void* luma, int stride, const void* cb, const void* cr, int cstride,
                               int width, int height, const x265cu_aq_params* p, int32_t* invQscale_dev, const x265cu_aq_out* out)
{
    const char* bad = p ? aq_energy_check(depth, luma, stride, cb, cr, cstride, width, height, p->qgSize, luma, luma) : NULL;
    if (!bad) bad = aq_finish_check(depth, width, height, p, luma, luma, out);
    if (bad) return aq_refuse("x265cu_aq_frame", bad);
    cudaSetDevice(c->device);
    const int L = p->qgSize == 8 ? 8 : 16;
    const int nb = ((width + L - 1) / L) * ((height + L - 1) / L);
    const int w8 = ((width / 2) + 7) >> 3, h8 = ((height / 2) + 7) >> 3;
    const int blockCount = p->qgSize == 8 ? 4 * w8 * h8 : w8 * h8;
    const size_t need = 6 * sizeof(uint64_t) + (size_t)nb * sizeof(uint32_t);
    if (c->aq_bytes < need)
    {
        cudaFree(c->d_aq);
        c->d_aq = NULL; c->aq_bytes = 0;
        if (cudaMalloc(&c->d_aq, need) != cudaSuccess) { x265cu_set_error("x265cu_aq_frame: scratch", cudaGetLastError(), __FILE__, __LINE__); return -1; }
        c->aq_bytes = need;
    }
    uint64_t* d_tot = (uint64_t*)c->d_aq;
    uint32_t* d_energy = (uint32_t*)(d_tot + 6);
    if (aq_energy_launch(c, depth, luma, stride, cb, cr, cstride, width, height, p->qgSize, d_energy, d_tot)) return -1;
    std::vector<uint32_t> energy(nb);
    uint64_t totals[6];
    CU_CHECK(cudaMemcpyAsync(totals, d_tot, sizeof(totals), cudaMemcpyDeviceToHost, c->stream));
    CU_CHECK(cudaMemcpyAsync(energy.data(), d_energy, (size_t)nb * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
    CU_CHECK(cudaStreamSynchronize(c->stream));
    x265cu_aq_out o = out ? *out : x265cu_aq_out{};
    std::vector<int32_t> invq, invq8;
    if (!o.invQscaleFactor) { invq.assign(blockCount, 0); o.invQscaleFactor = invq.data(); }       // Lowres::create zeroes it
    if (p->qgSize == 8 && !o.invQscaleFactor8x8) { invq8.assign(w8 * h8, 0); o.invQscaleFactor8x8 = invq8.data(); }
    aq_finish(depth, width, height, p, energy.data(), totals, &o);
    if (p->aqMode != 0 && invQscale_dev)
    {
        const int32_t* src = p->qgSize == 8 ? o.invQscaleFactor8x8 : o.invQscaleFactor;
        CU_CHECK(cudaMemcpyAsync(invQscale_dev, src, (size_t)w8 * h8 * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
        CU_CHECK(cudaStreamSynchronize(c->stream));
    }
    return 0;
}
