// x265_b200/csrc/aq.cuh -- adaptive quantisation's per-block integer pass on the device:
//   k_aq_energy : LookaheadTLD::acEnergyCu (encoder/slicetype.cpp:49-84, 256-275) of every block of one picture, in the
//                 reference's raster loop order, plus the per-plane sums of `sum` and `ssd` that acEnergyVar adds to
//                 Lowres::wp_sum / wp_ssd.  The float decision (calcAdaptiveQuantFrame's pow / log2) is x265cu_aq_finish,
//                 on the host.
// One warp per block, eight consecutive blocks of a block row per CTA, so that a CTA's rows are read as contiguous runs.
// Lanes take consecutive pixels of a block row (k = lane + 32 i), reads clamp to the picture (the replicated padding of
// PicYuv::copyFromPicture, common/picyuv.cpp:209-234).  Per-block sums and ssd fold with REDUX; the CTA's plane totals
// are added with one 64-bit atomicAdd each, exact in any order.
#pragma once
#include "common.cuh"

#define AQ_WARPS 8

// var of one L x L block (pixel.cpp:704-720) at (x0, y0) of a W x H plane with clamped reads; lane 0 gets (sum, ssd)
template <typename P, int L>
__device__ __forceinline__ void aq_block_var(const P* __restrict__ pl, int stride, int W, int H, int x0, int y0, int lane,
                                             uint32_t& sum, uint32_t& ssd)
{
    uint32_t s = 0, q = 0;
#pragma unroll
    for (int k = lane; k < L * L; k += 32)
    {
        const int x = min(x0 + (k % L), W - 1), y = min(y0 + (k / L), H - 1);
        const uint32_t v = pl[(intptr_t)y * stride + x];
        s += v; q += v * v;
    }
    sum = __reduce_add_sync(0xffffffffu, s);
    ssd = __reduce_add_sync(0xffffffffu, q);
}

// acEnergyVar: (uint32)(ssd - ((uint64)sum * sum >> shift))
__device__ __forceinline__ uint32_t aq_ac_energy(uint32_t sum, uint32_t ssd, int shift)
{
    return (uint32_t)(ssd - ((uint64_t)sum * sum >> shift));
}

// LB: luma block (16, or 8 at qgSize 8); the 4:2:0 chroma block is LB / 2 at (blockX >> 1, blockY >> 1)
template <typename P, int LB>
__global__ void __launch_bounds__(AQ_WARPS * 32) k_aq_energy(const P* __restrict__ y, int ystride, const P* __restrict__ cb,
                                                             const P* __restrict__ cr, int cstride, int W, int H, int bw, int nblocks,
                                                             uint32_t* __restrict__ energy, unsigned long long* __restrict__ totals)
{
    constexpr int CB = LB / 2;
    constexpr int LSHIFT = LB == 16 ? 8 : 6, CSHIFT = LB == 16 ? 6 : 4;
    __shared__ unsigned long long s_tot[6];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x < 6) s_tot[threadIdx.x] = 0;
    __syncthreads();
    const int b = blockIdx.x * AQ_WARPS + warp;
    if (b < nblocks)
    {
        const int bx = (b % bw) * LB, by = (b / bw) * LB;
        uint32_t sum, ssd;
        aq_block_var<P, LB>(y, ystride, W, H, bx, by, lane, sum, ssd);
        uint32_t e = aq_ac_energy(sum, ssd, LSHIFT);
        if (lane == 0) { atomicAdd(&s_tot[0], (unsigned long long)sum); atomicAdd(&s_tot[1], (unsigned long long)ssd); }
        if (cb)
        {
            aq_block_var<P, CB>(cb, cstride, W >> 1, H >> 1, bx >> 1, by >> 1, lane, sum, ssd);
            e += aq_ac_energy(sum, ssd, CSHIFT);
            if (lane == 0) { atomicAdd(&s_tot[2], (unsigned long long)sum); atomicAdd(&s_tot[3], (unsigned long long)ssd); }
            aq_block_var<P, CB>(cr, cstride, W >> 1, H >> 1, bx >> 1, by >> 1, lane, sum, ssd);
            e += aq_ac_energy(sum, ssd, CSHIFT);
            if (lane == 0) { atomicAdd(&s_tot[4], (unsigned long long)sum); atomicAdd(&s_tot[5], (unsigned long long)ssd); }
        }
        if (lane == 0) energy[b] = e;
    }
    __syncthreads();
    if (threadIdx.x < 6 && s_tot[threadIdx.x]) atomicAdd(&totals[threadIdx.x], s_tot[threadIdx.x]);
}
