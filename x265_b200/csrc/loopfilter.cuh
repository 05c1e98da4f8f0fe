// x265_b200/csrc/loopfilter.cuh -- in-loop filter class (SURVEY 8f.1): deblocking edge filters and SAO.
// Semantics: /root/reference/source/common/loopfilter.cpp:39-200 (calSign, processSaoCUE0/E1/E1_2Rows/E2/E3/B0,
// pelFilterLumaStrong_c, pelFilterChroma_c) and /root/reference/source/encoder/sao.cpp:1762-1927 (saoCuStatsBO/E0..E3).
// The reference walks every row left to right and carries the edge sign of the previous sample / row in a scalar or in the
// upBuff arrays; every sign is a function of ORIGINAL samples only (a sample is modified after its last use as a neighbour),
// so all kernels read an unmodified input block and write a separate output block: one thread per sample, rows that pass
// signs to the next row (E1 / E2 / E3 and the statistics) synchronise once per row.
// Blocks are staged compactly by the per-call thunks (thunks.cuh); each kernel documents its layout.
// The frame-level deblocking (k_deblock_frame, x265cu_deblock_frame / _rows) is the exception: it filters whole planes, or a
// window of CTU rows, in place, since the edges of one direction touch disjoint samples (see there).
#pragma once
#include "common.cuh"

namespace lf {

__device__ __forceinline__ int sgn(int x) { return (x > 0) - (x < 0); }
template <typename P> __device__ __forceinline__ int clipP(int v) { return min(max(v, 0), PixTraits<P>::maxv); }

// calSign (loopfilter.cpp:39-43)
template <typename P>
__global__ void k_sign(int8_t* __restrict__ dst, const P* __restrict__ a, const P* __restrict__ b, int n)
{
    for (int i = threadIdx.x; i < n; i += blockDim.x) dst[i] = (int8_t)sgn((int)a[i] - (int)b[i]);
}

// processSaoCUE0 (:45-63).  in: 2 rows x (width + 1) samples, pitch = width + 1.  out: 2 rows x width.
template <typename P>
__global__ void k_sao_e0(const P* __restrict__ in, P* __restrict__ out, const int8_t* __restrict__ off, int width, const int8_t* __restrict__ signLeft)
{
    for (int i = threadIdx.x; i < 2 * width; i += blockDim.x)
    {
        const int y = i / width, x = i - y * width;
        const P* r = in + y * (width + 1);
        const int c = r[x];
        const int sr = sgn(c - (int)r[x + 1]);
        const int sl = x ? sgn(c - (int)r[x - 1]) : (int)signLeft[y];       // signLeft0 = -signRight of the sample before
        out[y * width + x] = (P)clipP<P>(c + off[sr + sl + 2]);
    }
}

// processSaoCUE1 / E1_2Rows (:65-98).  in: (rows + 1) x width.  out: rows x width; up: upBuff1 in/out (width).
template <typename P>
__global__ void k_sao_e1(const P* __restrict__ in, P* __restrict__ out, int8_t* __restrict__ up, const int8_t* __restrict__ off, int width, int rows)
{
    for (int x = threadIdx.x; x < width; x += blockDim.x)
    {
        int u = up[x];
        for (int y = 0; y < rows; y++)
        {
            const int c = in[y * width + x];
            const int sd = sgn(c - (int)in[(y + 1) * width + x]);
            out[y * width + x] = (P)clipP<P>(c + off[sd + u + 2]);
            u = -sd;
        }
        up[x] = (int8_t)u;
    }
}

// processSaoCUE2 (:100-110).  in: row 0 = rec[0 .. width), row 1 = rec[stride + 1 .. stride + 1 + width).  buff1 read,
// bufft[1 .. width] written (passed as bufft + 1).
template <typename P>
__global__ void k_sao_e2(const P* __restrict__ in, P* __restrict__ out, int8_t* __restrict__ bufft1, const int8_t* __restrict__ buff1,
                         const int8_t* __restrict__ off, int width)
{
    for (int x = threadIdx.x; x < width; x += blockDim.x)
    {
        const int c = in[x];
        const int sd = sgn(c - (int)in[width + x]);
        bufft1[x] = (int8_t)(-sd);
        out[x] = (P)clipP<P>(c + off[sd + buff1[x] + 2]);
    }
}

// processSaoCUE3 (:112-124).  n = endX - startX - 1 samples x = startX + 1 ..: in row 0 = rec[x], row 1 = rec[x + stride];
// up = upBuff1 + startX (n + 1 entries): reads up[1 + i], writes up[i].
template <typename P>
__global__ void k_sao_e3(const P* __restrict__ in, P* __restrict__ out, const int8_t* __restrict__ upIn, int8_t* __restrict__ upOut,
                         const int8_t* __restrict__ off, int n)
{
    for (int i = threadIdx.x; i < n; i += blockDim.x)
    {
        const int c = in[i];
        const int sd = sgn(c - (int)in[n + i]);
        out[i] = (P)clipP<P>(c + off[sd + upIn[1 + i] + 2]);
        upOut[i] = (int8_t)(-sd);
    }
}

// processSaoCUB0 (:126-138).  w x h block, compact.
template <typename P>
__global__ void k_sao_b0(const P* __restrict__ in, P* __restrict__ out, const int8_t* __restrict__ off, int n)
{
    constexpr int boShift = PixTraits<P>::depth - 5;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    {
        const int c = in[i];
        out[i] = (P)clipP<P>(c + off[c >> boShift]);
    }
}

// ---- deblocking, one line across an edge: m[0..7] = the samples p3 p2 p1 p0 | q0 q1 q2 q3 (m[4] = src[0] of the reference),
// read as int16_t of the pixel as the reference does.  Each helper replaces the samples its filter writes.

// pelFilterLumaStrong_c (loopfilter.cpp:140-160): m[1..6], no pixel clip (the tc bounds keep them in range)
__device__ __forceinline__ void luma_strong_line(int* m, int tcP, int tcQ)
{
    const int m0 = m[0], m1 = m[1], m2 = m[2], m3 = m[3], m4 = m[4], m5 = m[5], m6 = m[6], m7 = m[7];
    m[1] = clip3i(-tcP, tcP, ((2 * m0 + 3 * m1 + m2 + m3 + m4 + 4) >> 3) - m1) + m1;
    m[2] = clip3i(-tcP, tcP, ((m1 + m2 + m3 + m4 + 2) >> 2) - m2) + m2;
    m[3] = clip3i(-tcP, tcP, ((m1 + 2 * m2 + 2 * m3 + 2 * m4 + m5 + 4) >> 3) - m3) + m3;
    m[4] = clip3i(-tcQ, tcQ, ((m2 + 2 * m3 + 2 * m4 + 2 * m5 + m6 + 4) >> 3) - m4) + m4;
    m[5] = clip3i(-tcQ, tcQ, ((m3 + m4 + m5 + m6 + 2) >> 2) - m5) + m5;
    m[6] = clip3i(-tcQ, tcQ, ((m3 + m4 + m5 + 3 * m6 + 2 * m7 + 4) >> 3) - m6) + m6;
}

// pelFilterLuma (deblock.cpp:278-315), the normal filter: m[2..5].  maskP1 / maskQ1 already include maskP / maskQ.
template <typename P>
__device__ __forceinline__ void luma_normal_line(int* m, int tc, int maskP, int maskQ, int maskP1, int maskQ1)
{
    const int m1 = m[1], m2 = m[2], m3 = m[3], m4 = m[4], m5 = m[5], m6 = m[6];
    int delta = (9 * (m4 - m3) - 3 * (m5 - m2) + 8) >> 4;
    if (abs(delta) >= tc * 10) return;
    delta = clip3i(-tc, tc, delta);
    const int tc2 = tc >> 1;
    m[3] = clipP<P>(m3 + (delta & maskP));
    m[4] = clipP<P>(m4 - (delta & maskQ));
    if (maskP1) m[2] = clipP<P>(m2 + clip3i(-tc2, tc2, (((m1 + m3 + 1) >> 1) - m2 + delta) >> 1));
    if (maskQ1) m[5] = clipP<P>(m5 + clip3i(-tc2, tc2, (((m6 + m4 + 1) >> 1) - m5 - delta) >> 1));
}

// pelFilterChroma_c (loopfilter.cpp:167-181): m[3], m[4] from m[2..5]
template <typename P>
__device__ __forceinline__ void chroma_line(int* m, int tc, int maskP, int maskQ)
{
    const int delta = clip3i(-tc, tc, ((((m[4] - m[3]) * 4) + m[2] - m[5] + 4) >> 3));
    m[3] = clipP<P>(m[3] + (delta & maskP));
    m[4] = clipP<P>(m[4] - (delta & maskQ));
}

// Per-call table entries pelFilterLumaStrong / pelFilterChroma.  in / out: 4 lines x 8 samples m0..m7 (m4 = src[0]).
template <typename P>
__global__ void k_deblock_luma_strong(const P* __restrict__ in, P* __restrict__ out, int tcP, int tcQ)
{
    const int i = threadIdx.x;
    if (i >= 4) return;
    int m[8];
#pragma unroll
    for (int k = 0; k < 8; k++) m[k] = (int)(int16_t)in[i * 8 + k];
    luma_strong_line(m, tcP, tcQ);
#pragma unroll
    for (int k = 0; k < 8; k++) out[i * 8 + k] = (P)m[k];
}
template <typename P>
__global__ void k_deblock_chroma(const P* __restrict__ in, P* __restrict__ out, int tc, int maskP, int maskQ)
{
    const int i = threadIdx.x;
    if (i >= 4) return;
    int m[8];
#pragma unroll
    for (int k = 0; k < 8; k++) m[k] = (int)(int16_t)in[i * 8 + k];
    chroma_line<P>(m, tc, maskP, maskQ);
#pragma unroll
    for (int k = 0; k < 8; k++) out[i * 8 + k] = (P)m[k];
}

// ---- frame-level deblocking (deblock.cpp, driven by the per-4x4 decision map of x265cu_deblock_frame) ----
// Deblock::s_tcTable / s_betaTable (deblock.cpp:499-509) and g_chromaScale (constants.cpp:346), in global memory: the frame
// kernels index them per lane.
__device__ const uint8_t d_tcTable[54] = {
    0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 1, 1, 1, 1, 2,
    2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 5, 5, 6, 6, 7, 8, 9, 10, 11, 13, 14, 16, 18, 20, 22, 24 };
__device__ const uint8_t d_betaTable[52] = {
    0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17,
    18, 20, 22, 24, 26, 28, 30, 32, 34, 36, 38, 40, 42, 44, 46, 48, 50, 52, 54, 56, 58, 60, 62, 64 };
__device__ const uint8_t d_chromaScale[70] = {
    0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28, 29, 29, 30, 31,
    32, 33, 33, 34, 34, 35, 35, 36, 36, 37, 37, 38, 39, 40, 41, 42, 43, 44, 45, 46, 47, 48, 49, 50, 51,
    51, 51, 51, 51, 51, 51, 51, 51, 51, 51, 51, 51 };

struct DeblockArgs
{
    void* plane[3];                 // luma, Cb, Cr at pixel (0,0); plane[1] == NULL: luma only
    int stride, cstride, width, height;
    const x265cu_deblock_unit* units;
    int sliceType, betaOffset, tcOffset, cbQpOffset, crQpOffset, bypass;   // offsets already doubled (deblock.cpp:328-329)
    // The window (deblock_window): vertical pass over unit rows [s0, s1), filtering luma on [l0, l1) of them (the others
    // only carry a chroma segment); horizontal pass over the edges [e0, e1) (luma y = 8e).
    int s0, s1, l0, l1, e0, e1;
};

// The window of luma rows [y0, y1) (CTU-row aligned, y1 == height or a multiple of 16): the vertical pass covers unit rows
// [y0/4 - 1, y1/4 + 1) in luma and the chroma segments of chroma rows [y0/2 - 4, y1/2 + 4), whose threads are the even unit
// rows [y0/4 - 2, y1/4 + 2); the horizontal pass every edge y with y0 <= y <= y1 inside the picture.  Then luma rows
// [y0 - 4, y1 + 4) and chroma rows [y0/2 - 4, y1/2 + 4) hold their whole-picture values and no other sample is written.
// y0 = 0, y1 = height is the whole picture.
__host__ __device__ inline void deblock_window(DeblockArgs& a, int y0, int y1)
{
    const int nu = a.height >> 2;
    a.s0 = max(0, y0 / 4 - 2); a.s1 = min(nu, y1 / 4 + 2);
    a.l0 = y0 / 4 - 1;         a.l1 = y1 / 4 + 1;
    a.e0 = max(1, y0 / 8);     a.e1 = min(a.height >> 3, y1 / 8 + 1);
}

// Edge flag of the 8-sample edge at `pos` (x for vertical edges, y for horizontal ones) as Deblock::deblockCU leaves it at the Q
// unit (deblock.cpp:90-93): the CU edge 2 (never the picture border: pos > 0 here), else a TU edge 2 (setEdgefilterTU), else an
// internal PU edge 1 (setEdgefilterPU), else 0.
template <int DIR>
__device__ __forceinline__ int edge_flag(const x265cu_deblock_unit& q, int pos)
{
    const int log2S = min(max((int)q.log2CuSize, 3), 6), S = 1 << log2S;
    const int o = pos & (S - 1);
    if (o == 0) return 2;
    const int T = S >> min((int)q.tuDepth, 3);
    if ((o & (T - 1)) == 0) return 2;
    const int ps = q.partSize, h = S >> 1, qu = S >> 2;
    bool pu;
    if (DIR == 0) pu = ((ps == 2 || ps == 3) && o == h) || (ps == 6 && o == qu) || (ps == 7 && o == S - qu);
    else          pu = ((ps == 1 || ps == 3) && o == h) || (ps == 4 && o == qu) || (ps == 5 && o == S - qu);
    return pu ? 1 : 0;
}

__device__ __forceinline__ bool mv_far(int ax, int ay, int bx, int by) { return abs(ax - bx) >= 4 || abs(ay - by) >= 4; }

// Deblock::getBoundaryStrength (deblock.cpp:191-247) for an edge with flag != 0.  refPic ids stand for the Frame pointers the
// reference compares; an id < 0 is an unused list (NULL, zero vector).
__device__ __forceinline__ int boundary_strength(const x265cu_deblock_unit& p, const x265cu_deblock_unit& q, int flag, int sliceType)
{
    if ((p.flags | q.flags) & 1) return 2;
    if (flag > 1 && ((p.flags | q.flags) & 2)) return 1;
    const int rP0 = p.refPic[0] < 0 ? -1 : p.refPic[0], rQ0 = q.refPic[0] < 0 ? -1 : q.refPic[0];
    const int rP1 = p.refPic[1] < 0 ? -1 : p.refPic[1], rQ1 = q.refPic[1] < 0 ? -1 : q.refPic[1];
    const int p0x = rP0 >= 0 ? p.mv[0][0] : 0, p0y = rP0 >= 0 ? p.mv[0][1] : 0, q0x = rQ0 >= 0 ? q.mv[0][0] : 0, q0y = rQ0 >= 0 ? q.mv[0][1] : 0;
    if (sliceType == 1) return (rP0 != rQ0 || mv_far(q0x, q0y, p0x, p0y)) ? 1 : 0;
    const int p1x = rP1 >= 0 ? p.mv[1][0] : 0, p1y = rP1 >= 0 ? p.mv[1][1] : 0, q1x = rQ1 >= 0 ? q.mv[1][0] : 0, q1y = rQ1 >= 0 ? q.mv[1][1] : 0;
    if ((rP0 == rQ0 && rP1 == rQ1) || (rP0 == rQ1 && rP1 == rQ0))
    {
        if (rP0 != rP1)
        {
            if (rP0 == rQ0) return (mv_far(q0x, q0y, p0x, p0y) || mv_far(q1x, q1y, p1x, p1y)) ? 1 : 0;
            return (mv_far(q1x, q1y, p0x, p0y) || mv_far(q0x, q0y, p1x, p1y)) ? 1 : 0;
        }
        return ((mv_far(q0x, q0y, p0x, p0y) || mv_far(q1x, q1y, p1x, p1y)) && (mv_far(q1x, q1y, p0x, p0y) || mv_far(q0x, q0y, p1x, p1y))) ? 1 : 0;
    }
    return 1;
}

// One 4-line segment of every 8-sample edge of one direction, one thread each, in place (the filters of neighbouring edges
// touch disjoint samples: reads 4 / writes 3 per side, 2 / 1 for chroma).  DIR 0 (EDGE_VER): x = edge index e (luma x = 8e,
// e >= 1), y = unit row a.  DIR 1 (EDGE_HOR): x = unit column a, y = edge index e (luma y = 8e).  The thread of an even e and
// an even a also filters the chroma segment of that edge (4:2:0: chroma edges every 8 chroma samples, 4 chroma lines = the
// 8 luma lines from unit a; deblock.cpp:104-113, 456-460).  BAND: the launch covers the window of `a` (deblock_window);
// otherwise the whole picture, and the window fields are not read (the frame call's code stays that of a whole-picture pass).
template <typename P, int DIR, bool BAND>
__global__ void __launch_bounds__(256) k_deblock_frame(const DeblockArgs a)
{
    const int gx = blockIdx.x * blockDim.x + threadIdx.x, gy = blockIdx.y * blockDim.y + threadIdx.y;
    const int e = DIR == 0 ? gx + 1 : gy + (BAND ? a.e0 : 1), s = DIR == 0 ? gy + (BAND ? a.s0 : 0) : gx;
    if (DIR == 0 ? (e >= (a.width >> 3) || s >= (BAND ? a.s1 : a.height >> 2))
                 : (e >= (BAND ? a.e1 : a.height >> 3) || s >= (a.width >> 2))) return;
    const int upr = a.width >> 2;
    const size_t iq = DIR == 0 ? (size_t)s * upr + 2 * e : (size_t)(2 * e) * upr + s;
    const size_t ip = DIR == 0 ? iq - 1 : iq - upr;
    const x265cu_deblock_unit uq = a.units[iq], up = a.units[ip];
    const int flag = edge_flag<DIR>(uq, 8 * e);
    if (!flag) return;
    const int bs = boundary_strength(up, uq, flag, a.sliceType);
    if (!bs) return;
    int maskP = -1, maskQ = -1;
    if (a.bypass)
    {   // deblock.cpp:358-365, 469-476
        maskP = (up.flags & 4) ? 0 : -1; maskQ = (uq.flags & 4) ? 0 : -1;
        if (!(maskP | maskQ)) return;
    }
    constexpr int shift = PixTraits<P>::depth - 8;
    const int qpA = ((int)up.qp + (int)uq.qp + 1) >> 1;

    // luma (edgeFilterLuma, deblock.cpp:317-415); a vertical-pass thread outside [l0, l1) only filters its chroma segment
    if (DIR == 1 || !BAND || (s >= a.l0 && s < a.l1))
    {
        P* src = (P*)a.plane[0];
        const ptrdiff_t across = DIR == 0 ? 1 : a.stride, along = DIR == 0 ? a.stride : 1;
        src += DIR == 0 ? (ptrdiff_t)(4 * s) * a.stride + 8 * e : (ptrdiff_t)(8 * e) * a.stride + 4 * s;
        int m[4][8];
#pragma unroll
        for (int i = 0; i < 4; i++)
#pragma unroll
            for (int k = 0; k < 8; k++) m[i][k] = (int)(int16_t)src[i * along + (k - 4) * across];
        const int beta = d_betaTable[clip3i(0, 51, qpA + a.betaOffset)] << shift;
        const int dp0 = abs(m[0][1] - 2 * m[0][2] + m[0][3]), dq0 = abs(m[0][4] - 2 * m[0][5] + m[0][6]);
        const int dp3 = abs(m[3][1] - 2 * m[3][2] + m[3][3]), dq3 = abs(m[3][4] - 2 * m[3][5] + m[3][6]);
        const int d0 = dp0 + dq0, d3 = dp3 + dq3;
        if (d0 + d3 < beta)
        {
            const int tc = d_tcTable[clip3i(0, 53, qpA + 2 * (bs - 1) + a.tcOffset)] << shift;
            const int sb = beta >> 3, st = (tc * 5 + 1) >> 1;
            const bool sw = 2 * d0 < (beta >> 2) && 2 * d3 < (beta >> 2) &&
                            abs(m[0][0] - m[0][3]) + abs(m[0][7] - m[0][4]) < sb && abs(m[0][3] - m[0][4]) < st &&
                            abs(m[3][0] - m[3][3]) + abs(m[3][7] - m[3][4]) < sb && abs(m[3][3] - m[3][4]) < st;
            if (sw)
            {
#pragma unroll
                for (int i = 0; i < 4; i++)
                {
                    luma_strong_line(m[i], (2 * tc) & maskP, (2 * tc) & maskQ);
#pragma unroll
                    for (int k = 1; k < 7; k++) src[i * along + (k - 4) * across] = (P)m[i][k];
                }
            }
            else
            {
                const int side = (beta + (beta >> 1)) >> 3;
                const int maskP1 = (dp0 + dp3 < side ? -1 : 0) & maskP, maskQ1 = (dq0 + dq3 < side ? -1 : 0) & maskQ;
#pragma unroll
                for (int i = 0; i < 4; i++)
                {
                    luma_normal_line<P>(m[i], tc, maskP, maskQ, maskP1, maskQ1);
#pragma unroll
                    for (int k = 2; k < 6; k++) src[i * along + (k - 4) * across] = (P)m[i][k];
                }
            }
        }
    }

    // chroma (edgeFilterChroma, deblock.cpp:417-497): bs 2 only, the BS and QPs of the segment's first luma unit
    if (a.plane[1] && bs == 2 && !(e & 1) && !(s & 1))
    {
        const ptrdiff_t across = DIR == 0 ? 1 : a.cstride, along = DIR == 0 ? a.cstride : 1;
        const ptrdiff_t org = DIR == 0 ? (ptrdiff_t)(2 * s) * a.cstride + 4 * e : (ptrdiff_t)(4 * e) * a.cstride + 2 * s;
#pragma unroll
        for (int c = 0; c < 2; c++)
        {
            int qp = qpA + (c ? a.crQpOffset : a.cbQpOffset);
            if (qp >= 30) qp = d_chromaScale[min(qp, 69)];
            const int tc = d_tcTable[clip3i(0, 53, qp + 2 + a.tcOffset)] << shift;
            P* src = (P*)a.plane[1 + c] + org;
#pragma unroll
            for (int i = 0; i < 4; i++)
            {
                int m[8];
#pragma unroll
                for (int k = 2; k < 6; k++) m[k] = (int)(int16_t)src[i * along + (k - 4) * across];
                chroma_line<P>(m, tc, maskP, maskQ);
                src[i * along - across] = (P)m[3];
                src[i * along] = (P)m[4];
            }
        }
    }
}

// the two passes of x265cu_deblock_frame / x265cu_deblock_rows over the window in `a`; band: a window that is not the whole
// picture (arguments validated by the caller)
template <typename P>
static int launch_deblock_frame(x265cu_ctx* c, const DeblockArgs& a, bool band)
{
    const dim3 block(32, 8);
    const int ne = (a.width >> 3) - 1, ns = a.s1 - a.s0;               // vertical: edges x segments
    if (ne > 0 && ns > 0)
    {
        const dim3 grid((ne + 31) / 32, (ns + 7) / 8);
        if (band) k_deblock_frame<P, 0, true><<<grid, block, 0, c->stream>>>(a);
        else      k_deblock_frame<P, 0, false><<<grid, block, 0, c->stream>>>(a);
        CU_LAUNCH_CHECK(c);
    }
    const int nh = a.e1 - a.e0, nc = a.width >> 2;                     // horizontal: segments x edges
    if (nh > 0)
    {
        const dim3 grid((nc + 31) / 32, (nh + 7) / 8);
        if (band) k_deblock_frame<P, 1, true><<<grid, block, 0, c->stream>>>(a);
        else      k_deblock_frame<P, 1, false><<<grid, block, 0, c->stream>>>(a);
        CU_LAUNCH_CHECK(c);
    }
    return 0;
}

// ---- SAO statistics (sao.cpp:1762-1927).  stats / count: in/out (32 classes for BO, 5 for the edge types through s_eoTable).
__constant__ int c_eoTable[5] = { 1, 2, 0, 3, 4 };                 // SAO::s_eoTable (sao.cpp)

// block accumulation helper: every thread adds into shared bins, thread 0..n-1 flush
template <int NB>
__device__ __forceinline__ void stats_flush(int* s_st, int* s_ct, int32_t* stats, int32_t* count, bool viaEoTable)
{
    __syncthreads();
    if (threadIdx.x < NB)
    {
        const int dst = viaEoTable ? c_eoTable[threadIdx.x] : threadIdx.x;
        stats[dst] += s_st[threadIdx.x]; count[dst] += s_ct[threadIdx.x];
    }
}

// saoCuStatsBO: diff pitch 64, rec compact pitch `rp`
template <typename P>
__global__ void k_sao_stats_bo(const int16_t* __restrict__ diff, const P* __restrict__ rec, int rp, int endX, int endY, int32_t* stats, int32_t* count)
{
    constexpr int boShift = PixTraits<P>::depth - 5;
    __shared__ int s_st[32], s_ct[32];
    if (threadIdx.x < 32) { s_st[threadIdx.x] = 0; s_ct[threadIdx.x] = 0; }
    __syncthreads();
    for (int i = threadIdx.x; i < endX * endY; i += blockDim.x)
    {
        const int y = i / endX, x = i - y * endX;
        const int cls = rec[y * rp + x] >> boShift;
        atomicAdd(&s_st[cls], (int)diff[y * 64 + x]); atomicAdd(&s_ct[cls], 1);
    }
    stats_flush<32>(s_st, s_ct, stats, count, false);
}

// saoCuStatsE0: rec rows with one sample to the left and one to the right: compact pitch rp, row origin at column 1
template <typename P>
__global__ void k_sao_stats_e0(const int16_t* __restrict__ diff, const P* __restrict__ rec, int rp, int endX, int endY, int32_t* stats, int32_t* count)
{
    __shared__ int s_st[5], s_ct[5];
    if (threadIdx.x < 5) { s_st[threadIdx.x] = 0; s_ct[threadIdx.x] = 0; }
    __syncthreads();
    for (int i = threadIdx.x; i < endX * endY; i += blockDim.x)
    {
        const int y = i / endX, x = i - y * endX;
        const P* r = rec + y * rp + 1;
        const int c = r[x];
        const int et = sgn(c - (int)r[x + 1]) + sgn(c - (int)r[x - 1]) + 2;
        atomicAdd(&s_st[et], (int)diff[y * 64 + x]); atomicAdd(&s_ct[et], 1);
    }
    stats_flush<5>(s_st, s_ct, stats, count, true);
}

// saoCuStatsE1: rec (endY + 1) rows x endX compact; up = upBuff1 in/out
template <typename P>
__global__ void k_sao_stats_e1(const int16_t* __restrict__ diff, const P* __restrict__ rec, int8_t* __restrict__ up, int endX, int endY, int32_t* stats, int32_t* count)
{
    __shared__ int s_st[5], s_ct[5];
    if (threadIdx.x < 5) { s_st[threadIdx.x] = 0; s_ct[threadIdx.x] = 0; }
    __syncthreads();
    for (int x = threadIdx.x; x < endX; x += blockDim.x)
    {
        int u = up[x];
        for (int y = 0; y < endY; y++)
        {
            const int sd = sgn((int)rec[y * endX + x] - (int)rec[(y + 1) * endX + x]);
            atomicAdd(&s_st[sd + u + 2], (int)diff[y * 64 + x]); atomicAdd(&s_ct[sd + u + 2], 1);
            u = -sd;
        }
        up[x] = (int8_t)u;
    }
    stats_flush<5>(s_st, s_ct, stats, count, true);
}

// saoCuStatsE2: rec block rows 0 .. endY, columns -1 .. endX (pitch rp = endX + 2, origin at column 1).
// bufA / bufB: the caller's upBuff1 / upBufft INCLUDING their [-1] element (so index 1 + x); the reference swaps the two
// pointers after every row: row y reads from buffer (y & 1 ? B : A) and writes into the other one.
template <typename P>
__global__ void k_sao_stats_e2(const int16_t* __restrict__ diff, const P* __restrict__ rec, int rp, int8_t* __restrict__ bufA, int8_t* __restrict__ bufB,
                               int endX, int endY, int32_t* stats, int32_t* count)
{
    __shared__ int s_st[5], s_ct[5];
    __shared__ int8_t s_b[2][80];
    if (threadIdx.x < 5) { s_st[threadIdx.x] = 0; s_ct[threadIdx.x] = 0; }
    for (int i = threadIdx.x; i < endX + 2; i += blockDim.x) { s_b[0][i] = bufA[i]; s_b[1][i] = bufB[i]; }
    __syncthreads();
    for (int y = 0; y < endY; y++)
    {
        int8_t* b1 = s_b[y & 1] + 1;       // upBuff1 of this row
        int8_t* bt = s_b[(y & 1) ^ 1] + 1; // upBufft of this row
        const P* r = rec + y * rp + 1;
        if (threadIdx.x == 0) bt[0] = (int8_t)sgn((int)r[rp] - (int)r[-1]);
        for (int x = threadIdx.x; x < endX; x += blockDim.x)
        {
            const int sd = sgn((int)r[x] - (int)r[x + rp + 1]);
            const int et = sd + b1[x] + 2;
            atomicAdd(&s_st[et], (int)diff[y * 64 + x]); atomicAdd(&s_ct[et], 1);
            // bt[x + 1] is written here and bt[0] above: distinct entries; b1 is only read in this row
            bt[x + 1] = (int8_t)(-sd);
        }
        __syncthreads();
    }
    for (int i = threadIdx.x; i < endX + 2; i += blockDim.x) { bufA[i] = s_b[0][i]; bufB[i] = s_b[1][i]; }
    stats_flush<5>(s_st, s_ct, stats, count, true);
}

// saoCuStatsE3: rec block rows 0 .. endY, columns -1 .. endX (pitch rp, origin at column 1); up = upBuff1 INCLUDING [-1].
template <typename P>
__global__ void k_sao_stats_e3(const int16_t* __restrict__ diff, const P* __restrict__ rec, int rp, int8_t* __restrict__ up, int endX, int endY,
                               int32_t* stats, int32_t* count)
{
    __shared__ int s_st[5], s_ct[5];
    __shared__ int8_t s_u[2][80];
    if (threadIdx.x < 5) { s_st[threadIdx.x] = 0; s_ct[threadIdx.x] = 0; }
    for (int i = threadIdx.x; i < endX + 1; i += blockDim.x) { s_u[0][i] = up[i]; s_u[1][i] = up[i]; }
    __syncthreads();
    for (int y = 0; y < endY; y++)
    {
        const int8_t* cur = s_u[y & 1] + 1;
        int8_t* nxt = s_u[(y & 1) ^ 1] + 1;
        const P* r = rec + y * rp + 1;
        for (int x = threadIdx.x; x < endX; x += blockDim.x)
        {
            const int sd = sgn((int)r[x] - (int)r[x + rp - 1]);
            const int et = sd + cur[x] + 2;
            atomicAdd(&s_st[et], (int)diff[y * 64 + x]); atomicAdd(&s_ct[et], 1);
            nxt[x - 1] = (int8_t)(-sd);                            // upBuff1[x - 1] for the next row
        }
        if (threadIdx.x == 0) nxt[endX - 1] = (int8_t)sgn((int)r[endX - 1 + rp] - (int)r[endX]);
        __syncthreads();
    }
    for (int i = threadIdx.x; i < endX + 1; i += blockDim.x) up[i] = s_u[endY & 1][i];
    stats_flush<5>(s_st, s_ct, stats, count, true);
}

// ---- frame-level SAO (x265cu_sao_stats_frame / x265cu_sao_apply_frame): whole planes, one CTA per (CTU, plane) ----
// Both read the deblocked, not-yet-SAO'd picture only (include/x265_b200.h; pinned by tests/test_sao_oracle_vs_ref.py).

// the edge class of sample c between its neighbours a and b (edgeType of sao.cpp / loopfilter.cpp: 0..4, 2 = neither)
__device__ __forceinline__ int sao_edge_type(int c, int a, int b) { return sgn(c - a) + sgn(c - b) + 2; }
// the band of sample c (SAO_BO_BITS = 5)
template <typename P> __device__ __forceinline__ int sao_band(int c) { return c >> (PixTraits<P>::depth - 5); }

// The geometry of CTU `addr` in plane p (calcSaoStatsCTU / applyPixelOffsets, sao.cpp:274-308, 735-767): origin, size
// clipped to the picture, and whether it touches each picture border.
struct SaoCtuGeom
{
    int picW, picH, lpelx, tpely, w, h;
    bool left, top, right, bottom;
};
__device__ __forceinline__ SaoCtuGeom sao_ctu_geom(int width, int height, int log2Ctu, int cols, int addr, int p)
{
    SaoCtuGeom g;
    const int s = p ? 1 : 0, log2S = log2Ctu - s;
    g.picW = width >> s; g.picH = height >> s;
    g.lpelx = (addr % cols) << log2S; g.tpely = (addr / cols) << log2S;
    g.w = min(1 << log2S, g.picW - g.lpelx); g.h = min(1 << log2S, g.picH - g.tpely);
    g.left = g.lpelx == 0; g.top = g.tpely == 0;
    g.right = g.lpelx + g.w == g.picW; g.bottom = g.tpely + g.h == g.picH;
    return g;
}

struct SaoStatsArgs
{
    const void* fenc[3]; const void* rec[3];   // at pixel (0,0); planes = 1: luma only
    int fstride, fcstride, stride, cstride, width, height, log2Ctu, cols, planes;
    int row0;                                  // CTU row of blockIdx.x == 0: the grid covers CTU rows from row0 on
    int32_t* stats;                            // [numCtus][2][3][5][32]
};

// SAO::calcSaoStatsCTU (sao.cpp:735-917) of CTU row0 * cols + blockIdx.x, plane blockIdx.y: every sample of the CTU once, classified for
// each type inside that type's region (skipB 4 / skipR 5 away from the picture's right / bottom border, 2 / 3 in chroma; the
// E0 rows ignore the picture bottom, sao.cpp:836).  Neighbour coordinates are clamped to the picture: the regions only hold
// samples whose neighbours lie inside it.  Edge-type counts and sums stay in registers, band histograms in per-warp shared
// bins; warp reductions, then one sum over the warps.  The CTA writes its plane's whole record (320 entries), zeros included.
template <typename P>
__global__ void __launch_bounds__(256) k_sao_stats_frame(const SaoStatsArgs a)
{
    constexpr int NW = 8;
    __shared__ int s_bo[NW][2][32];
    __shared__ int s_eo[NW][2][4][5];
    const int addr = a.row0 * a.cols + blockIdx.x, p = blockIdx.y, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    for (int i = tid; i < NW * 2 * 32; i += blockDim.x) (&s_bo[0][0][0])[i] = 0;
    __syncthreads();
    int ec[4][5], es[4][5];
#pragma unroll
    for (int t = 0; t < 4; t++)
#pragma unroll
        for (int k = 0; k < 5; k++) { ec[t][k] = 0; es[t][k] = 0; }
    if (p < a.planes)
    {
        const SaoCtuGeom g = sao_ctu_geom(a.width, a.height, a.log2Ctu, a.cols, addr, p);
        const int po = p ? 2 : 0, log2S = a.log2Ctu - (p ? 1 : 0), S = 1 << log2S;
        const int boX = g.right ? g.w : g.w - 5 + po, boY = g.bottom ? g.h : g.h - 4 + po;
        const int sx = g.left, sy = g.top;
        const int eX = g.right ? g.w - 1 : g.w - 5 + po, e0Y = g.h - 4 + po, e1Y = g.bottom ? g.h - 1 : g.h - 4 + po;
        const P* rec = (const P*)(p == 0 ? a.rec[0] : p == 1 ? a.rec[1] : a.rec[2]);     // constant indices: no stack copy
        const P* fenc = (const P*)(p == 0 ? a.fenc[0] : p == 1 ? a.fenc[1] : a.fenc[2]);
        const ptrdiff_t rs = p ? a.cstride : a.stride, fs = p ? a.fcstride : a.fstride;
        for (int i = tid; i < S * S; i += blockDim.x)
        {
            const int x = i & (S - 1), y = i >> log2S;
            const bool inBo = x < boX && y < boY;
            const bool inE0 = x >= sx && x < eX && y < e0Y;
            const bool inE1 = x < boX && y >= sy && y < e1Y;
            const bool inE23 = x >= sx && x < eX && y >= sy && y < e1Y;
            if (!(inBo || inE0 || inE1 || inE23)) continue;
            const int px = g.lpelx + x, py = g.tpely + y;
            const int xl = max(px - 1, 0), xr = min(px + 1, g.picW - 1);
            const P* r0 = rec + (ptrdiff_t)max(py - 1, 0) * rs;
            const P* r1 = rec + (ptrdiff_t)py * rs;
            const P* r2 = rec + (ptrdiff_t)min(py + 1, g.picH - 1) * rs;
            const int c = r1[px], diff = (int)fenc[(ptrdiff_t)py * fs + px] - c;
            if (inBo)
            {
                const int b = sao_band<P>(c);
                atomicAdd(&s_bo[warp][0][b], 1);
                atomicAdd(&s_bo[warp][1][b], diff);
            }
            int et[4];
            et[0] = inE0 ? sao_edge_type(c, r1[xl], r1[xr]) : -1;
            et[1] = inE1 ? sao_edge_type(c, r0[px], r2[px]) : -1;
            et[2] = inE23 ? sao_edge_type(c, r0[xl], r2[xr]) : -1;
            et[3] = inE23 ? sao_edge_type(c, r0[xr], r2[xl]) : -1;
#pragma unroll
            for (int t = 0; t < 4; t++)
#pragma unroll
                for (int k = 0; k < 5; k++)
                {
                    ec[t][k] += et[t] == k;
                    es[t][k] += et[t] == k ? diff : 0;
                }
        }
    }
#pragma unroll
    for (int t = 0; t < 4; t++)
#pragma unroll
        for (int k = 0; k < 5; k++)
        {
            const int n = warp_sum(ec[t][k]), d = warp_sum(es[t][k]);
            if (lane == 0) { s_eo[warp][0][t][k] = n; s_eo[warp][1][t][k] = d; }
        }
    __syncthreads();
    // [count / offsetOrg][type][class]: BO classes are bands; edge class k is edgeType eoInv[k] (s_eoTable = {1, 2, 0, 3, 4})
    int32_t* rec = a.stats + (size_t)addr * (2 * 3 * 5 * 32) + p * (5 * 32);
    for (int i = tid; i < 2 * 5 * 32; i += blockDim.x)
    {
        const int kind = i / (5 * 32), t = (i >> 5) % 5, k = i & 31;
        int v = 0;
        if (t == 4)
            for (int w = 0; w < NW; w++) v += s_bo[w][kind][k];
        else if (k < 5)
        {
            const int e = k == 0 ? 2 : k == 1 ? 0 : k == 2 ? 1 : k;
            for (int w = 0; w < NW; w++) v += s_eo[w][kind][t][e];
        }
        rec[kind * (3 * 5 * 32) + t * 32 + k] = v;
    }
}

struct SaoApplyArgs
{
    void* plane[3]; const void* fenc[3];       // at pixel (0,0); planes = 1: luma only
    const void* src[3];                        // the deblocked input: == plane (in place, through `lines`) or a separate plane
    int stride, cstride, fstride, fcstride, sstride, scstride, width, height, log2Ctu, cols, rows, planes;
    int row0;                                  // CTU row of blockIdx.x == 0: the grid covers CTU rows from row0 on
    int on[3];                                 // SAOParam::bSaoFlag per plane
    const x265cu_sao_ctu* params;              // [3][numCtus]
    const x265cu_deblock_unit* units;          // NULL: no transquant-bypass restoration
    void* lines[3];                            // per plane: [rows][2: top, bottom][picW], then [cols][2: left, right][picH]
};

// Saves the edge lines of every CTU of the planes with SAO on (the reference's m_tmpU / m_tmpL at picture scope), so that
// k_sao_apply_frame can filter in place: thread i of plane blockIdx.y copies entry i of that plane's line store.
template <typename P>
__global__ void __launch_bounds__(256) k_sao_save_lines(const SaoApplyArgs a)
{
    const int p = blockIdx.y;
    if (p >= a.planes || !a.on[p]) return;
    const int s = p ? 1 : 0, picW = a.width >> s, picH = a.height >> s, S = 1 << (a.log2Ctu - s);
    const P* src = (const P*)a.plane[p];
    const ptrdiff_t st = p ? a.cstride : a.stride;
    P* dst = (P*)a.lines[p];
    const long nRow = (long)a.rows * 2 * picW, nAll = nRow + (long)a.cols * 2 * picH;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < nAll; i += (long)gridDim.x * blockDim.x)
    {
        int x, y;
        if (i < nRow)
        {
            const int r = (int)(i / (2 * picW)), side = (int)(i / picW) & 1;
            x = (int)(i % picW);
            y = side ? min((r + 1) * S, picH) - 1 : r * S;
        }
        else
        {
            const long j = i - nRow;
            const int c = (int)(j / (2 * picH)), side = (int)(j / picH) & 1;
            y = (int)(j % picH);
            x = side ? min((c + 1) * S, picW) - 1 : c * S;
        }
        dst[i] = src[(ptrdiff_t)y * st + x];
    }
}

// processSaoCTU of CTU row0 * cols + blockIdx.x, plane blockIdx.y (sao.cpp:274-732, framefilter.cpp:324-343).  In place
// (src == plane): the CTA stages its CTU from the plane and a one-sample ring from the saved lines into shared memory, then
// writes the filtered samples of its own CTU only.  Out of place: it stages the CTU and the ring from src, which is never
// written, and writes every sample of its CTU (filtered, else copied from src).  Which samples a type changes: BO all; EO_0 not the picture's left / right column; EO_1 not its top /
// bottom row; EO_2 / EO_3 neither.  Cr uses Cb's type and its own offsets, and is filtered only when both types are >= 0
// (sao.cpp:704-728).  Types outside -1..4 are off, bandPos is read & 31, offsets are any int8 (the result is clipped).
// Transquant-bypass units (flags bit 2) then get the source samples back, whatever the SAO flags (origCUSampleRestoration).
template <typename P>
__global__ void __launch_bounds__(256) k_sao_apply_frame(const SaoApplyArgs a)
{
    __shared__ P s_t[66 * 66];
    const int addr = a.row0 * a.cols + blockIdx.x, p = blockIdx.y, tid = threadIdx.x;
    if (p >= a.planes) return;
    const int n = a.cols * a.rows;
    const x265cu_sao_ctu prm = a.params[(size_t)p * n + addr];
    int type = prm.typeIdx;
    if (p == 2)
    {
        const int tcb = a.params[(size_t)n + addr].typeIdx;
        type = type >= 0 && type <= 4 ? tcb : -1;
    }
    const bool sao = a.on[p] && type >= 0 && type <= 4;
    const P* src = (const P*)(p == 0 ? a.src[0] : p == 1 ? a.src[1] : a.src[2]);
    P* plane = (P*)(p == 0 ? a.plane[0] : p == 1 ? a.plane[1] : a.plane[2]);
    const bool copy = src != plane;
    if (!sao && !a.units && !copy) return;
    const SaoCtuGeom g = sao_ctu_geom(a.width, a.height, a.log2Ctu, a.cols, addr, p);
    const int log2S = a.log2Ctu - (p ? 1 : 0), S = 1 << log2S, T = g.w + 2;
    const ptrdiff_t st = p ? a.cstride : a.stride, sst = p ? a.scstride : a.sstride;
    if (sao && copy)
    {
        for (int i = tid; i < T * (g.h + 2); i += blockDim.x)
        {
            const int tx = i % T, ty = i / T, px = g.lpelx + tx - 1, py = g.tpely + ty - 1;
            s_t[ty * T + tx] = px >= 0 && px < g.picW && py >= 0 && py < g.picH ? src[(ptrdiff_t)py * sst + px] : (P)0;
        }
        __syncthreads();
    }
    else if (sao)
    {
        const P* lines = (const P*)a.lines[p];
        const long rowLines = (long)a.rows * 2 * g.picW;
        const int r = addr / a.cols, c = addr % a.cols;
        for (int i = tid; i < T * (g.h + 2); i += blockDim.x)
        {
            const int tx = i % T, ty = i / T, px = g.lpelx + tx - 1, py = g.tpely + ty - 1;
            P v = 0;
            if (px >= 0 && px < g.picW && py >= 0 && py < g.picH)
            {
                if (ty == 0)               v = lines[((long)(r - 1) * 2 + 1) * g.picW + px];      // bottom row of the row above
                else if (ty == g.h + 1)    v = lines[((long)(r + 1) * 2) * g.picW + px];          // top row of the row below
                else if (tx == 0)          v = lines[rowLines + ((long)(c - 1) * 2 + 1) * g.picH + py];   // right column, left CTU
                else if (tx == g.w + 1)    v = lines[rowLines + ((long)(c + 1) * 2) * g.picH + py];       // left column, right CTU
                else                       v = plane[(ptrdiff_t)py * st + px];
            }
            s_t[ty * T + tx] = v;
        }
        __syncthreads();
    }
    const int x0 = type != 4 && type != 1 ? g.left : 0, x1 = type != 4 && type != 1 && g.right ? g.w - 1 : g.w;
    const int y0 = type != 4 && type != 0 ? g.top : 0, y1 = type != 4 && type != 0 && g.bottom ? g.h - 1 : g.h;
    const int dxa = type == 1 ? 0 : type == 3 ? 1 : -1, dya = type == 0 ? 0 : -1;   // neighbour a; b is the mirror
    const int bandPos = prm.bandPos & 31, o0 = prm.offset[0], o1 = prm.offset[1], o2 = prm.offset[2], o3 = prm.offset[3];
    const P* fenc = (const P*)a.fenc[p];
    const ptrdiff_t fs = p ? a.fcstride : a.fstride;
    const int us = p ? 1 : 2, upr = a.width >> 2;
    for (int i = tid; i < S * S; i += blockDim.x)
    {
        const int x = i & (S - 1), y = i >> log2S;
        if (x >= g.w || y >= g.h) continue;
        const int px = g.lpelx + x, py = g.tpely + y;
        if (a.units && (a.units[(size_t)(py >> us) * upr + (px >> us)].flags & 4))
        {
            plane[(ptrdiff_t)py * st + px] = fenc[(ptrdiff_t)py * fs + px];
            continue;
        }
        if (!sao || x < x0 || x >= x1 || y < y0 || y >= y1)
        {
            if (copy) plane[(ptrdiff_t)py * st + px] = sao ? s_t[(y + 1) * T + x + 1] : src[(ptrdiff_t)py * sst + px];
            continue;
        }
        const P* t = s_t + (y + 1) * T + x + 1;
        const int cv = t[0];
        int o;
        if (type == 4)
        {
            const int k = (sao_band<P>(cv) - bandPos) & 31;
            o = k == 0 ? o0 : k == 1 ? o1 : k == 2 ? o2 : k == 3 ? o3 : 0;
        }
        else
        {
            const int et = sao_edge_type(cv, t[dya * T + dxa], t[-dya * T - dxa]);
            o = et == 0 ? o0 : et == 1 ? o1 : et == 3 ? o2 : et == 4 ? o3 : 0;
        }
        plane[(ptrdiff_t)py * st + px] = (P)clipP<P>(cv + o);
    }
}

// The calls' launches (arguments validated by the callers)
template <typename P>
static int launch_sao_stats_frame(x265cu_ctx* c, const SaoStatsArgs& a, int numCtus)     // CTUs from row a.row0 on
{
    k_sao_stats_frame<P><<<dim3(numCtus, 3), 256, 0, c->stream>>>(a);
    CU_LAUNCH_CHECK(c);
    return 0;
}

// In place (src == plane): the line save, then the apply of every CTU.  Out of place: the apply of the CTU rows
// [a.row0, row1) only, with no line save.
template <typename P>
static int launch_sao_apply_frame(x265cu_ctx* c, SaoApplyArgs a, int row1)
{
    const bool copy = a.src[0] != a.plane[0];
    if (copy)
    {
        k_sao_apply_frame<P><<<dim3(a.cols * (row1 - a.row0), 3), 256, 0, c->stream>>>(a);
        CU_LAUNCH_CHECK(c);
        return 0;
    }
    size_t need = 0, off[3] = { 0, 0, 0 };
    for (int p = 0; p < a.planes; p++)
    {
        const int s = p ? 1 : 0;
        off[p] = need;
        if (a.on[p])
            need += ((size_t)a.rows * 2 * (a.width >> s) + (size_t)a.cols * 2 * (a.height >> s)) * sizeof(P);
        need = (need + 255) & ~(size_t)255;
    }
    if (need)
    {
        if (c->sao_lines_bytes < need)
        {
            if (c->d_sao_lines) { CU_CHECK(cudaStreamSynchronize(c->stream)); cudaFree(c->d_sao_lines); c->d_sao_lines = NULL; c->sao_lines_bytes = 0; }
            CU_CHECK(cudaMalloc(&c->d_sao_lines, need));
            c->sao_lines_bytes = need;
        }
        for (int p = 0; p < a.planes; p++) a.lines[p] = (uint8_t*)c->d_sao_lines + off[p];
        k_sao_save_lines<P><<<dim3(2 * c->sm_count, 3), 256, 0, c->stream>>>(a);
        CU_LAUNCH_CHECK(c);
    }
    if (need || a.units)
    {
        k_sao_apply_frame<P><<<dim3(a.cols * a.rows, 3), 256, 0, c->stream>>>(a);
        CU_LAUNCH_CHECK(c);
    }
    return 0;
}

} // namespace lf
