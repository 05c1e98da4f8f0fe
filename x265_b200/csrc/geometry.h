// x265_b200/csrc/geometry.h -- host-only (no CUDA): the static geometry tables of the frame analyser.
// PU / CU / TU lists of a picture in canonical order (CTU raster; per CTU and reference the CUs 64..8 in raster order, each
// with its 2Nx2N PU, then -- rect -- 2NxN x2, Nx2N x2, then -- amp, CU >= 16 -- 2NxnU, 2NxnD, nLx2N, nRx2N; preset slow has rect
// on and AMP off, slower / veryslow have both: common/param.cpp:478-520).  A CU must lie fully inside the picture
// (analysis.cpp only visits CUs inside it); no partition of a CU that crosses the edge is emitted.  Kept free of CUDA so that tests/test_geometry.py can check it on the CPU
// against the oracle's independent enumeration (oracle/frame_spec.h) at every BASELINE picture size.
#pragma once
#include <stdint.h>
#include <vector>
#include <utility>

struct PuDesc { int32_t offset; int16_t cuX, cuY; int8_t pw, ph; int16_t ref; };   // static per geometry
struct CuDesc { int16_t x, y, size, pad; int64_t coef_off; };
struct TuDesc { int32_t cu; int16_t tx, ty; };                                        // TU origin inside the CU

struct FrameGeometry
{
    std::vector<PuDesc> pus; std::vector<CuDesc> cus; std::vector<TuDesc> tus;
    std::vector<int32_t> cu_jobs;                 // [cu][ref] -> index of the CU's 2Nx2N PU job
    // first PU job / CU / TU of every CTU row (+ one past the end): the lists are in CTU raster order, so a CTU-row
    // range [r0, r1) is one contiguous slice of each list (what a WPP row shard owns, frameencoder.cpp:850-868)
    int ctuRows; std::vector<int> rowJob, rowCu, rowTu;
    // per-size work lists of the residual and intra stages, each launch of one block size reading only its own list: tuBy[k]
    // = the TUs of luma size 8 << k (k = 0..2), cuBy[k] = the CUs of size 8 << k (k = 0..3), absolute indices in list order.
    // rowTuBy[k] / rowCuBy[k] = first entry of every CTU row (+ one past the end), so a CTU-row range is one slice of each.
    std::vector<int32_t> tuBy[3], cuBy[4]; std::vector<int> rowTuBy[3], rowCuBy[4];
    int64_t ncoef;
    // job groups of the shared-memory-window integer search (me_window.cuh): per (CTU, ref) the 64x64 CU's PUs, each 32x32
    // CU's PUs, and per 16x16 cell the PUs of the 16x16 CU and of its four 8x8 CUs.  grpJobs holds absolute job indices,
    // largest PU first inside a group; groups are in CTU raster order (rowGrp = first group of every CTU row + end).
    // Three classes, launched separately (different shared-memory budgets): [0] = CU 64 groups, [1] = CU 32 groups, [2] = 16x16 cells.
    std::vector<int32_t> grpFirst[3], grpCount[3], grpJobs[3]; std::vector<int> rowGrp[3];
    // the jobs of every CTU row sorted by PU shape (largest first; absolute job indices; row r = order[rowJob[r] .. rowJob[r + 1])):
    // the pre-check and sub-pel launches hand out jobs in this order so that all warps run the same code paths together
    std::vector<int32_t> order;
};

// partitions of a CU of `size`: returns the count and fills part[k] = {x, y, w, h} relative to the CU origin
static inline int geometry_cu_parts(int size, int rect, int amp, int part[13][4])
{
    const int h2 = size / 2, q = size / 4;
    int n = 0;
#define GEO_PART(x, y, w, h) do { part[n][0] = (x); part[n][1] = (y); part[n][2] = (w); part[n][3] = (h); n++; } while (0)
    GEO_PART(0, 0, size, size);
    if (rect)
    {
        GEO_PART(0, 0, size, h2); GEO_PART(0, h2, size, h2);
        GEO_PART(0, 0, h2, size); GEO_PART(h2, 0, h2, size);
    }
    if (amp && size >= 16)
    {   // 2NxnU, 2NxnD, nLx2N, nRx2N (AMP is not allowed at the minimum CU size)
        GEO_PART(0, 0, size, q);          GEO_PART(0, q, size, size - q);
        GEO_PART(0, 0, size, size - q);   GEO_PART(0, size - q, size, q);
        GEO_PART(0, 0, q, size);          GEO_PART(q, 0, size - q, size);
        GEO_PART(0, 0, size - q, size);   GEO_PART(size - q, 0, q, size);
    }
#undef GEO_PART
    return n;
}

// ---- residual stages: TU placement per plane ----
#ifdef __CUDACC__
#define GEO_HD __host__ __device__ __forceinline__
#else
#define GEO_HD inline
#endif

// The TU of a plane subsampled by `sub` (0 luma, 1 4:2:0 chroma) for a luma TU (T = min(S, 32)): (T >> sub) square at the
// luma coordinates >> sub.  Its levels start at coef_off >> (2 * sub) + (TU index in the CU) * (T >> sub)^2, so a plane
// holds ncoef >> (2 * sub) levels in the luma TU order.
struct PlaneTu { int x, y, size; int64_t off; };
GEO_HD PlaneTu geometry_plane_tu(const CuDesc& cu, const TuDesc& tu, int sub)
{
    const int S = cu.size, T = S > 32 ? 32 : S, Tp = T >> sub;
    PlaneTu p;
    p.x = (cu.x + tu.tx) >> sub; p.y = (cu.y + tu.ty) >> sub; p.size = Tp;
    p.off = (cu.coef_off >> (2 * sub)) + (int64_t)((tu.ty / T) * (S / T) + tu.tx / T) * Tp * Tp;
    return p;
}
// the 4:2:0 chroma TU of a luma TU
typedef PlaneTu ChromaTu;
GEO_HD ChromaTu geometry_chroma_tu(const CuDesc& cu, const TuDesc& tu) { return geometry_plane_tu(cu, tu, 1); }

// Quant::setChromaQP (quant.cpp:221-244) for 4:2:0: qp is the analyser's quantiser QP (QP_BD_OFFSET included), offset the
// plane's PPS + slice offset (-12..12).  Returns the plane's quantiser QP.
static inline int geometry_chroma_qp(int qp, int offset, int depth)
{
    static const uint8_t chromaScale[58] = {                      // g_chromaScale (constants.cpp:346), entries 0..57
        0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28, 29,
        29, 30, 31, 32, 33, 33, 34, 34, 35, 35, 36, 36, 37, 37, 38, 39, 40, 41, 42, 43, 44, 45, 46, 47, 48, 49, 50, 51 };
    const int bd = 6 * (depth - 8);
    int q = qp - bd + offset;
    q = q < -bd ? -bd : (q > 57 ? 57 : q);
    if (q >= 30) q = chromaScale[q];
    return q + bd;
}

// Chroma pixels (picture-relative, inclusive) that the chroma MC of the TUs [tu0, tu1) can read.  The vector of a CU is its
// 2Nx2N PU's search result (or 0 before any search: the ME output is zeroed at creation).  The search clips with
// k_build_me_jobs' rule, full-pel x in [-(71 + cuX), W + 7 - cuX] and y in [-(71 + cuY), H + 7 - cuY]; y stays inside that
// range in quarter pels, x can leave it by 5 full pels below and 4 above plus the quarter-pel fraction (analyser.cuh, above
// AN_PLANE_X).  The luma quarter-pel vector is the chroma eighth-pel vector; the 4-tap filter reads 1 pixel before and 2
// after the block, and the kernel loads single pixels (no wider over-read).
struct GeoRect { int x0, y0, x1, y1; };
static inline int geo_floor_div(int a, int b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }
static inline GeoRect geometry_chroma_reach(int W, int H, const std::vector<CuDesc>& cus, const std::vector<TuDesc>& tus, int tu0, int tu1)
{
    GeoRect r = { 1 << 30, 1 << 30, -(1 << 30), -(1 << 30) };
    for (int t = tu0; t < tu1; t++)
    {
        const CuDesc& cu = cus[tus[t].cu];
        const ChromaTu c = geometry_chroma_tu(cu, tus[t]);
        const int qxmin = 4 * (-(71 + cu.x) - 5), qxmax = 4 * (W + 7 - cu.x + 4) + 3;
        const int qymin = 4 * (-(71 + cu.y)), qymax = 4 * (H + 7 - cu.y);
        const int x0 = c.x + geo_floor_div(qxmin, 8) - 1, x1 = c.x + c.size - 1 + geo_floor_div(qxmax, 8) + 2;
        const int y0 = c.y + geo_floor_div(qymin, 8) - 1, y1 = c.y + c.size - 1 + geo_floor_div(qymax, 8) + 2;
        if (x0 < r.x0) r.x0 = x0;
        if (y0 < r.y0) r.y0 = y0;
        if (x1 > r.x1) r.x1 = x1;
        if (y1 > r.y1) r.y1 = y1;
    }
    return r;
}

// The reach lies inside a chroma plane allocation of `cstride` elements per row with the picture origin at (mx, my) and
// (H / 2 + 2 * my) rows
static inline bool geometry_chroma_reach_inside(const GeoRect& r, int W, int H, int cstride, int mx, int my)
{
    if (r.x0 > r.x1) return true;                                  // no TU
    return r.x0 >= -mx && r.x1 < cstride - mx && r.y0 >= -my && r.y1 < (H >> 1) + my && W / 2 + mx <= cstride;
}

static inline void geometry_build(int W, int H, int stride, int nref, int rect, int amp, FrameGeometry& g)
{
    // CU list: CTU raster, sizes 64..8, raster inside the CTU; CUs must lie fully inside the picture
    const int ctuW = (W + 63) / 64, ctuH = (H + 63) / 64;
    int64_t coefOff = 0;
    g.ctuRows = ctuH;
    for (int cty = 0; cty < ctuH; cty++)
    {
        g.rowJob.push_back((int)g.pus.size()); g.rowCu.push_back((int)g.cus.size()); g.rowTu.push_back((int)g.tus.size());
        for (int k = 0; k < 3; k++) g.rowGrp[k].push_back((int)g.grpFirst[k].size());
        for (int ctx = 0; ctx < ctuW; ctx++)
        {
            int local[85]; int nl = 0;
            for (int size = 64; size >= 8; size >>= 1)
                for (int cy = 0; cy < 64; cy += size)
                    for (int cx = 0; cx < 64; cx += size, nl++)
                    {
                        const int x = ctx * 64 + cx, y = cty * 64 + cy;
                        local[nl] = -1;
                        if (x + size > W || y + size > H) continue;
                        local[nl] = (int)g.cus.size();
                        CuDesc c; c.x = (int16_t)x; c.y = (int16_t)y; c.size = (int16_t)size; c.pad = 0; c.coef_off = coefOff;
                        coefOff += (int64_t)size * size;
                        const int T = size > 32 ? 32 : size;
                        for (int ty = 0; ty < size; ty += T)
                            for (int tx = 0; tx < size; tx += T)
                            {
                                TuDesc t; t.cu = (int32_t)g.cus.size(); t.tx = (int16_t)tx; t.ty = (int16_t)ty;
                                g.tus.push_back(t);
                            }
                        g.cus.push_back(c);
                    }
            g.cu_jobs.resize(g.cus.size() * nref, -1);
            // PU jobs of this CTU: per ref, per CU (same order), the CU's partitions in geometry_cu_parts order
            for (int r = 0; r < nref; r++)
            {
                int li = 0;
                int jobStart[85], jobCount[85];
                for (int q = 0; q < 85; q++) { jobStart[q] = 0; jobCount[q] = 0; }
                for (int size = 64; size >= 8; size >>= 1)
                    for (int cy = 0; cy < 64; cy += size)
                        for (int cx = 0; cx < 64; cx += size, li++)
                        {
                            if (local[li] < 0) continue;          // CU crosses the picture edge: no partition of it is evaluated
                            int part[13][4];
                            const int np = geometry_cu_parts(size, rect, amp, part);
                            jobStart[li] = (int)g.pus.size(); jobCount[li] = np;
                            for (int k = 0; k < np; k++)
                            {
                                const int x = ctx * 64 + cx + part[k][0], y = cty * 64 + cy + part[k][1], w = part[k][2], h = part[k][3];
                                PuDesc d; d.offset = y * stride + x; d.cuX = (int16_t)(ctx * 64 + cx); d.cuY = (int16_t)(cty * 64 + cy);
                                d.pw = (int8_t)w; d.ph = (int8_t)h; d.ref = (int16_t)r;
                                if (k == 0) g.cu_jobs[(size_t)local[li] * nref + r] = (int32_t)g.pus.size();
                                g.pus.push_back(d);
                            }
                        }
                // groups of this (CTU, ref): CU 64, CUs 32, then the 16x16 cells (CU 16 + its four CUs 8)
                for (int gi = 0; gi < 21; gi++)
                {
                    int members[5], nm = 0;
                    members[nm++] = gi;
                    if (gi >= 5)
                    {
                        const int k = gi - 5, cy16 = k >> 2, cx16 = k & 3;
                        for (int a8 = 0; a8 < 2; a8++)
                            for (int b8 = 0; b8 < 2; b8++) members[nm++] = 21 + (2 * cy16 + a8) * 8 + (2 * cx16 + b8);
                    }
                    const int cl = gi == 0 ? 0 : (gi < 5 ? 1 : 2);
                    std::vector<int32_t>& gj = g.grpJobs[cl];
                    const int first = (int)gj.size();
                    for (int m = 0; m < nm; m++)
                        for (int q = 0; q < jobCount[members[m]]; q++) gj.push_back(jobStart[members[m]] + q);
                    const int count = (int)gj.size() - first;
                    if (!count) continue;
                    // largest PU first (stable insertion sort: groups hold at most 33 jobs)
                    for (int a = first + 1; a < first + count; a++)
                    {
                        const int32_t v = gj[a];
                        const int av = g.pus[v].pw * g.pus[v].ph;
                        int b = a - 1;
                        while (b >= first && g.pus[gj[b]].pw * g.pus[gj[b]].ph < av) { gj[b + 1] = gj[b]; b--; }
                        gj[b + 1] = v;
                    }
                    g.grpFirst[cl].push_back(first); g.grpCount[cl].push_back(count);
                }
            }
        }
    }
    for (int k = 0; k < 3; k++) g.rowGrp[k].push_back((int)g.grpFirst[k].size());
    g.rowJob.push_back((int)g.pus.size()); g.rowCu.push_back((int)g.cus.size()); g.rowTu.push_back((int)g.tus.size());
    g.ncoef = coefOff;
    for (int r = 0; r < ctuH; r++)
    {
        for (int k = 0; k < 3; k++) g.rowTuBy[k].push_back((int)g.tuBy[k].size());
        for (int k = 0; k < 4; k++) g.rowCuBy[k].push_back((int)g.cuBy[k].size());
        for (int t = g.rowTu[r]; t < g.rowTu[r + 1]; t++)
        {
            const int S = g.cus[g.tus[t].cu].size;
            g.tuBy[S >= 32 ? 2 : (S == 16 ? 1 : 0)].push_back(t);
        }
        for (int c = g.rowCu[r]; c < g.rowCu[r + 1]; c++)
        {
            const int S = g.cus[c].size;
            g.cuBy[S == 64 ? 3 : (S == 32 ? 2 : (S == 16 ? 1 : 0))].push_back(c);
        }
    }
    for (int k = 0; k < 3; k++) g.rowTuBy[k].push_back((int)g.tuBy[k].size());
    for (int k = 0; k < 4; k++) g.rowCuBy[k].push_back((int)g.cuBy[k].size());
    // shape-sorted job order per CTU row: counting sort on (w, h) keys, stable (area descending, then width descending)
    g.order.resize(g.pus.size());
    for (int r = 0; r < ctuH; r++)
    {
        const int j0 = g.rowJob[r], j1 = g.rowJob[r + 1];
        // key = (area, w): collect distinct shapes
        std::vector<std::pair<int, int> > shapes;
        for (int j = j0; j < j1; j++)
        {
            const std::pair<int, int> sh(g.pus[j].pw * g.pus[j].ph, g.pus[j].pw);
            bool seen = false;
            for (size_t q = 0; q < shapes.size(); q++) if (shapes[q] == sh) { seen = true; break; }
            if (!seen) shapes.push_back(sh);
        }
        for (size_t a = 1; a < shapes.size(); a++)          // insertion sort, descending
        {
            const std::pair<int, int> v = shapes[a]; size_t b = a;
            while (b > 0 && shapes[b - 1] < v) { shapes[b] = shapes[b - 1]; b--; }
            shapes[b] = v;
        }
        int pos = j0;
        for (size_t q = 0; q < shapes.size(); q++)
            for (int j = j0; j < j1; j++)
                if (g.pus[j].pw * g.pus[j].ph == shapes[q].first && g.pus[j].pw == shapes[q].second) g.order[pos++] = j;
    }
}
