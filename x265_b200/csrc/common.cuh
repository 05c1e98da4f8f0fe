// x265_b200/csrc/common.cuh -- shared declarations for the sm_90a kernels and the C ABI.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include "../../include/x265_b200.h"

#define X265CU_FENC_STRIDE 64          // common/common.h:70

struct x265cu_ctx
{
    int device;
    int sm_count;
    cudaStream_t stream;
    cudaEvent_t ev0, ev1;
    uint64_t launches;
    // per-call thunk staging (pinned host + device arenas)
    uint8_t* h_stage; uint8_t* d_stage; size_t stage_bytes;
    int* d_counter;                     // work-queue counters for persistent kernels
    void* d_me_state; size_t me_state_bytes;   // per-job state between the ME phases
    cudaEvent_t me_ev[4];               // boundaries of the three ME launches of the last x265cu_me_batch / analyser run
    void* d_sao_lines; size_t sao_lines_bytes; // CTU edge lines saved by x265cu_sao_apply_frame before it filters in place
    void* d_cutree; size_t cutree_bytes;       // x265cu_cutree: one level's propagate amounts and the levels' overflow flags
    void* d_aq; size_t aq_bytes;               // x265cu_aq_frame: the energies and plane totals of one picture
};

void x265cu_set_error(const char* what, cudaError_t e, const char* file, int line);
// kernel launches of the whole process (every context, the per-call table's per-thread contexts included): what
// x265cu_launch_count() reports
extern unsigned long long g_x265cu_launches;
static inline void x265cu_count_launch(x265cu_ctx* c) { c->launches++; __atomic_fetch_add(&g_x265cu_launches, 1ull, __ATOMIC_RELAXED); }

#define CU_CHECK(expr) do { cudaError_t e__ = (expr); if (e__ != cudaSuccess) { \
    x265cu_set_error(#expr, e__, __FILE__, __LINE__); return -1; } } while (0)
#define CU_LAUNCH_CHECK(ctx) do { x265cu_count_launch(ctx); cudaError_t e__ = cudaGetLastError(); if (e__ != cudaSuccess) { \
    x265cu_set_error("kernel launch", e__, __FILE__, __LINE__); return -1; } } while (0)

template <typename P> struct PixTraits;
template <> struct PixTraits<uint8_t>  { static constexpr int depth = 8;  static constexpr int maxv = 255; };
template <> struct PixTraits<uint16_t> { static constexpr int depth = 10; static constexpr int maxv = 1023; };

__device__ __forceinline__ int clip3i(int lo, int hi, int v) { return min(max(v, lo), hi); }
__device__ __forceinline__ int clip16(int v) { return min(max(v, -32768), 32767); }

__device__ __forceinline__ int warp_sum(int v)
{
    return __reduce_add_sync(0xffffffffu, v);          // REDUX.SUM: one instruction on sm_80+
}
__device__ __forceinline__ unsigned long long warp_sum64(unsigned long long v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Constant tables.  All kernels live in ONE translation unit (x265cu.cu includes the *.cuh class
// files), so plain __constant__ definitions are enough (no -rdc).
// HEVC interpolation taps (spec 8.5.3.3.3; reference copy: common/constants.cpp:250-268)
__constant__ int16_t c_lumaFilter[4][8] = {
    { 0, 0, 0, 64, 0, 0, 0, 0 }, { -1, 4, -10, 58, 17, -5, 1, 0 },
    { -1, 4, -11, 40, 40, -11, 4, -1 }, { 0, 1, -5, 17, 58, -10, 4, -1 } };
__constant__ int16_t c_chromaFilter[8][4] = {
    { 0, 64, 0, 0 }, { -2, 58, 10, -2 }, { -4, 54, 16, -2 }, { -6, 46, 28, -4 },
    { -4, 36, 36, -4 }, { -4, 28, 46, -6 }, { -2, 16, 54, -4 }, { -2, 10, 58, -2 } };
// transform matrices, generated on the host at context creation (transform.cuh: build_dct_tables)
__constant__ int8_t c_dct[4][32 * 32];   // [log2N-2][k*N + j]
// the same matrices in GLOBAL memory for lane-indexed reads (a constant-bank access with 32 different addresses is
// replayed 32 times, which the tensor-core transform's fragment set-up would pay on every TU)
__device__ int8_t d_dct[4][32 * 32];
__constant__ int8_t c_dst4[16];
