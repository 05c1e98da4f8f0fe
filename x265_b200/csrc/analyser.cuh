// x265_b200/csrc/analyser.cuh -- host side of the frame-level CTU-analysis pipeline: geometry tables,
// device residency of the source / reference planes, and the e2e (host buffers) / resident entry points.
#pragma once
#include "common.cuh"
#include "frame.cuh"
#include "resid.cuh"
#include "bidir.cuh"
#include "part.cuh"
#include "me.cuh"
#include "me_window.cuh"
#include <vector>
#include <climits>
#include <stdlib.h>

struct x265cu_analyser
{
    x265cu_ctx* ctx;
    x265cu_analysis_params p;
    int stride, planeRows, fw, fh;
    size_t planeBytes, orgBytes;        // origin pixel byte offset inside a plane allocation
    int njobs, ncu, ntu; int64_t ncoef;
    // device
    uint8_t* d_fenc; uint8_t* d_refs[16]; uint8_t* d_recon[4];
    void** d_refTable; void** d_reconTable;
    int16_t* d_field; uint16_t* d_mvcost; int mvrange;
    PuDesc* d_pus; CuDesc* d_cus; TuDesc* d_tus; int32_t* d_cu_jobs;
    x265cu_me_job* d_jobs; int32_t* d_me_out; int2* d_me_packed;
    int16_t* d_coef; unsigned long long* d_cu_sse; uint32_t* d_cu_numsig; int32_t* d_cu_ref; uint32_t* d_intra;
    // pinned host staging for the e2e path
    uint8_t* h_fenc; int16_t* h_field;
    cudaEvent_t ev[6]; int ev_valid;      // stage boundaries of the last an_run (ME build+search+pack | BIDIR | residual | intra)
    std::vector<PuDesc> pus; std::vector<CuDesc> cus; std::vector<TuDesc> tus; std::vector<int32_t> cu_jobs;
    // first PU job / CU / TU of every CTU row (+ one past the end): the lists are in CTU raster order, so a CTU-row
    // range [r0, r1) is one contiguous slice of each list (what a WPP row shard owns, frameencoder.cpp:850-868)
    int ctuRows; std::vector<int> rowJob, rowCu, rowTu;
    // per-size TU and CU lists of the residual and intra launches and their CTU-row offsets (geometry.h tuBy / cuBy)
    int32_t* d_tuBy[3]; int32_t* d_cuBy[4]; std::vector<int> rowTuBy[3], rowCuBy[4];
    // 4:2:0 chroma planes for the chroma-SATD term of subpelCompare (x265cu_analyser_enable_chroma): half resolution,
    // stride / 2 elements per row, margins = half the luma margins (picyuv.cpp:87-94)
    int chromaOn, cstride, cRows; size_t cPlaneBytes, cOrgBytes;
    uint8_t* d_fencC[2]; uint8_t* d_refC[16][2];
    void** d_refCbTable; void** d_refCrTable;
    // shared-memory-window integer search (me_window.cuh): group tables (two classes), tensor maps of the reference
    // planes [ref][MEW_NCLS], leftover list.  windowOn = 0 (X265CU_ME_WINDOW=0) keeps the global-memory kernel for all jobs.
    int windowOn; MeGroup* d_groups[3]; int32_t* d_grpJobs[3]; std::vector<int> rowGrp[3];
    int cellJobsFit;                      // no 16x16 cell has more than 32 class-0 PUs (one lane each in k_me_subpel_cell)
    CUtensorMap* d_tmaps; int32_t* d_left;
    int32_t* d_order;                     // jobs of every CTU row sorted by PU shape (geometry.h)
    // quarter-pel phase planes of the sub-pel refinement (MePlanes, me.cuh): d_refs[r] is a block of 16 planes planeBytes
    // apart, slot 0 = the reference plane, slot yf * 4 + xf = phase (xf, yf); tile jobs of their build (hpp / vpp / hvpp
    // phases, the same for every reference); per CTU row, the rectangle its sub-pel launches can read (AnRect below)
    x265cu_interp_job* d_planeJobs[3]; int nPlaneJobs[3];
    std::vector<int4> rowRead;
    // 4:2:0 chroma residual stage (stage bit 3, x265cu_analyser_enable_chroma_residual): quantiser QP of Cb / Cr, levels of
    // each plane (ncoef / 4), recon planes [depthIdx][plane] in the chroma geometry, per-CU [ncu][2] SSE / numSig
    int chromaResOn, qpC[2];
    int16_t* d_coefC[2]; uint8_t* d_reconC[4][2]; void** d_reconCTable;
    unsigned long long* d_cu_sseC; uint32_t* d_cu_numsigC;
    std::vector<GeoRect> rowReachC;       // per CTU row, the chroma pixels its chroma MC can read (geometry_chroma_reach)
    // weighted P-slice references (x265cu_analyser_set_ref_weights): wp = the caller's m_weightPredTable[0][r] row, all zero
    // for an unweighted reference.  A weighted reference gets its own ME block d_wrefs[r] (slot 0 its weighted plane, slots
    // 1..15 that plane's phases) and, for each weighted chroma plane, d_wrefC[r][plane], allocated on first use.  wDirty[r]:
    // the weighted planes of r no longer match its pixels or weights; the next run rebuilds them (an_weights_prepare).  While
    // nWeighted > 0 the search reads d_meRefTable / d_meCbTable / d_meCrTable and the residual stages d_wtab ([16][3]
    // {weighted, w0, offset, shift}); d_wjobs holds the weight_pp band jobs of every (reference, plane).
    x265cu_wp_entry wp[16][3]; int nWeighted, wDirty[16];
    uint8_t* d_wrefs[16]; uint8_t* d_wrefC[16][2];
    void** d_meRefTable; void** d_meCbTable; void** d_meCrTable; int4* d_wtab; x265cu_blk_job* d_wjobs;
    // B slices (x265cu_analyser_set_lists): slots [0, numRefL0) are list 0, the rest list 1 (numRefL1 == 0: a P slice);
    // d_bidir = the BIDIR stage's record of every CU (stage bit 4), allocated by the first set_lists with a list 1
    int numRefL0, numRefL1; x265cu_bidir_cu* d_bidir;
    // the PART stage's record of every CU (stage bit 5), allocated zeroed by the first run with that bit; the same for the
    // PART_B stage (stage bit 6)
    x265cu_part_cu* d_part; x265cu_part_b_cu* d_partB;
};

static const int AN_MARGIN_X = 96, AN_MARGIN_Y = 80;       // picyuv.cpp:87-88 with maxCUSize 64

template <typename T> static T* an_upload(x265cu_ctx* c, const std::vector<T>& v)
{
    T* d = (T*)x265cu_malloc(c, v.size() * sizeof(T) + 16);
    if (d && !v.empty()) cudaMemcpy(d, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice);
    return d;
}

static void an_build_geometry(x265cu_analyser* a)
{
    FrameGeometry g;
    geometry_build(a->p.width, a->p.height, a->stride, a->p.numRefs, a->p.rect, a->p.amp, g);
    a->pus.swap(g.pus); a->cus.swap(g.cus); a->tus.swap(g.tus); a->cu_jobs.swap(g.cu_jobs);
    a->ctuRows = g.ctuRows; a->rowJob.swap(g.rowJob); a->rowCu.swap(g.rowCu); a->rowTu.swap(g.rowTu);
    a->njobs = (int)a->pus.size(); a->ncu = (int)a->cus.size(); a->ntu = (int)a->tus.size(); a->ncoef = g.ncoef;
    a->d_order = an_upload(a->ctx, g.order);
    for (int k = 0; k < 3; k++) { a->d_tuBy[k] = an_upload(a->ctx, g.tuBy[k]); a->rowTuBy[k].swap(g.rowTuBy[k]); }
    for (int k = 0; k < 4; k++) { a->d_cuBy[k] = an_upload(a->ctx, g.cuBy[k]); a->rowCuBy[k].swap(g.rowCuBy[k]); }
    for (int k = 0; k < 3; k++)
    {
        std::vector<MeGroup> grp(g.grpFirst[k].size());
        for (size_t i = 0; i < grp.size(); i++) { grp[i].first = g.grpFirst[k][i]; grp[i].count = g.grpCount[k][i]; }
        a->d_groups[k] = an_upload(a->ctx, grp);
        a->d_grpJobs[k] = an_upload(a->ctx, g.grpJobs[k]);
        a->rowGrp[k].swap(g.rowGrp[k]);
    }
    // class-0 PUs (me_subpel_class: power-of-two sides of at most 16) per cell: at most 9 of the 16x16 CU + 5 per 8x8 CU
    a->cellJobsFit = 1;
    for (size_t i = 0; i < g.grpFirst[2].size(); i++)
    {
        int n = 0;
        for (int q = g.grpFirst[2][i]; q < g.grpFirst[2][i] + g.grpCount[2][i]; q++)
        {
            const int w = a->pus[g.grpJobs[2][q]].pw, h = a->pus[g.grpJobs[2][q]].ph;
            n += !((w & (w - 1)) | (h & (h - 1))) && w <= 16 && h <= 16;
        }
        if (n > 32) a->cellJobsFit = 0;
    }
}

// ---- phase planes: what the sub-pel launches read and what the build writes ----
// Rectangles are picture-relative pixel coordinates of a phase plane, x0..x1 and y0..y1 inclusive.
// READ, per PU: k_build_me_jobs clips the search range to full-pel vectors in [-(71 + cuX), width + 7 - cuX] x
// [-(71 + cuY), height + 7 - cuY] (clipMv, cudata.cpp:1915-1928).  y: me_phase3 keeps every sub-pel candidate inside
// [qminy, qmaxy], its centre is the search winner (in range, or MV 0), so the block's rows are the PU's rows moved by
// [-(71 + cuY), height + 7 - cuY].  x is not range-checked: the HEX search ends up to 3 full pels outside [minx, maxx]
// (DIA 1, STAR and FULL 0, or at MV 0), then the sub-pel rounds move up to 6 quarter pels (2 half-pel + 2 quarter-pel
// iterations at subme 7), so the block's full-pel column lies in [minx - 5, maxx + 4].
// BUILT: columns [-AN_PLANE_X, width + AN_PLANE_X), rows [-AN_PLANE_Y, height + AN_PLANE_Y).  The 8-tap support of a built
// pixel (3 before, 4 after) and the aligned-word over-read of the row filter (up to 8 bytes past it) stay inside the margins.
// The clip does not depend on where the CU is, so the PUs of any CTU row can reach rows -71 .. height + 70: every run
// builds the whole rectangle, whatever rows it analyses.  Pixels outside BUILT stay 0 (zeroed at allocation) and are only
// ever loaded as the unused bytes of an aligned word.
static const int AN_PLANE_X = 80, AN_PLANE_Y = 76, AN_PLANE_TILE = 64;

static int4 an_rect_union(int4 a, int4 b) { return make_int4(min(a.x, b.x), min(a.y, b.y), max(a.z, b.z), max(a.w, b.w)); }

// READ of the PUs of every CTU row, (x0, y0, x1, y1)
static void an_build_read_rects(x265cu_analyser* a)
{
    const int W = a->p.width, H = a->p.height;
    a->rowRead.assign(a->ctuRows, make_int4(INT_MAX, INT_MAX, INT_MIN, INT_MIN));
    for (int r = 0; r < a->ctuRows; r++)
        for (int i = a->rowJob[r]; i < a->rowJob[r + 1]; i++)
        {
            const PuDesc& d = a->pus[i];
            const int y = d.offset / a->stride, x = d.offset - y * a->stride;
            a->rowRead[r] = an_rect_union(a->rowRead[r], make_int4(x - (71 + d.cuX) - 5, y - (71 + d.cuY),
                                                                   x + d.pw - 1 + (W + 7 - d.cuX) + 4, y + d.ph - 1 + (H + 7 - d.cuY)));
        }
}

// BUILT contains READ of the CTU rows [r0, r1), and BUILT's filter support lies inside the plane allocation
static bool an_planes_cover(const x265cu_analyser* a, int r0, int r1)
{
    const int W = a->p.width, H = a->p.height;
    int4 rd = make_int4(INT_MAX, INT_MAX, INT_MIN, INT_MIN);
    for (int r = r0; r < r1; r++) rd = an_rect_union(rd, a->rowRead[r]);
    const bool covers = rd.x >= -AN_PLANE_X && rd.y >= -AN_PLANE_Y && rd.z < W + AN_PLANE_X && rd.w < H + AN_PLANE_Y;
    const int es = a->p.depth == 8 ? 1 : 2;
    const bool inside = -AN_PLANE_X - 3 >= -AN_MARGIN_X && -AN_PLANE_Y - 3 >= -AN_MARGIN_Y &&
                        (W + AN_PLANE_X + 4) * es + 8 <= (a->stride - AN_MARGIN_X) * es && H + AN_PLANE_Y + 4 <= H + AN_MARGIN_Y;
    return covers && inside;
}

// tile jobs of the build over BUILT, relative to a reference's block base: hpp (xf = 1..3), vpp (yf = 1..3), hvpp (both)
static int an_build_plane_jobs(x265cu_analyser* a)
{
    const size_t es = a->p.depth == 8 ? 1 : 2;
    const int64_t ppitch = (int64_t)(a->planeBytes / es), org = (int64_t)(a->orgBytes / es);
    const int X1 = a->p.width + AN_PLANE_X, Y1 = a->p.height + AN_PLANE_Y;
    for (int g = 0; g < 3; g++)
    {
        std::vector<x265cu_interp_job> jobs;
        for (int yf = 0; yf < 4; yf++)
            for (int xf = 0; xf < 4; xf++)
            {
                if ((g == 0 && (!xf || yf)) || (g == 1 && (xf || !yf)) || (g == 2 && (!xf || !yf))) continue;
                for (int y = -AN_PLANE_Y; y < Y1; y += AN_PLANE_TILE)
                    for (int x = -AN_PLANE_X; x < X1; x += AN_PLANE_TILE)
                    {
                        x265cu_interp_job j = {};
                        j.s_off = org + (int64_t)y * a->stride + x;
                        j.d_off = (yf * 4 + xf) * ppitch + j.s_off;
                        j.s_stride = j.d_stride = a->stride;
                        j.w = (int16_t)min(AN_PLANE_TILE, X1 - x); j.h = (int16_t)min(AN_PLANE_TILE, Y1 - y);
                        j.idxX = (int8_t)(g == 1 ? yf : xf); j.idxY = (int8_t)yf;          // the vertical filters take idxX
                        j.ntaps = 8;
                        jobs.push_back(j);
                    }
            }
        a->nPlaneJobs[g] = (int)jobs.size();
        a->d_planeJobs[g] = an_upload(a->ctx, jobs);
        if (!a->d_planeJobs[g]) return -1;
    }
    return 0;
}

// the chroma MC of the CTU rows [r0, r1) reads inside the chroma plane allocations
static bool an_chroma_reach_ok(const x265cu_analyser* a, int r0, int r1)
{
    GeoRect u = { 1 << 30, 1 << 30, -(1 << 30), -(1 << 30) };
    for (int r = r0; r < r1; r++)
    {
        const GeoRect& g = a->rowReachC[r];
        if (g.x0 > g.x1) continue;
        u.x0 = min(u.x0, g.x0); u.y0 = min(u.y0, g.y0); u.x1 = max(u.x1, g.x1); u.y1 = max(u.y1, g.y1);
    }
    return geometry_chroma_reach_inside(u, a->p.width, a->p.height, a->cstride, AN_MARGIN_X / 2, AN_MARGIN_Y / 2);
}

// the chroma reach of every CTU row (built once, on the first stage that needs it)
static void an_build_chroma_reach(x265cu_analyser* a)
{
    if (!a->rowReachC.empty()) return;
    a->rowReachC.resize(a->ctuRows);
    for (int r = 0; r < a->ctuRows; r++)
        a->rowReachC[r] = geometry_chroma_reach(a->p.width, a->p.height, a->cus, a->tus, a->rowTu[r], a->rowTu[r + 1]);
}

// ---- weighted references: MotionReference::init / applyWeight (encoder/reference.cpp:51-185) on the resident planes ----
static bool an_ref_weighted(const x265cu_analyser* a, int r) { return a->wp[r][0].wtPresent != 0; }
// chroma plane c (1 Cb, 2 Cr) of reference r is weighted for the search when the reference is (frameencoder.cpp:550), the
// plane's own wtPresent is set and the search has the chroma-SATD term (numInterpPlanes = 3 at subme > 2, reference.cpp:57)
static bool an_refc_weighted(const x265cu_analyser* a, int r, int c)
{
    return an_ref_weighted(a, r) && a->chromaOn && a->p.subme > 2 && a->wp[r][c].wtPresent;
}

static int an_band_jobs(int h) { return (h + 15) / 16; }

// applyWeight's result once every row is weighted: weight_pp of the picture (w = inputWeight, round = (denom ? 1 << (denom - 1)
// : 0) << (14 - depth), shift = denom + 14 - depth, offset = inputOffset << (depth - 8)), then the borders replicated as its
// extendRowBorder and the above / below copies do.  One weight_pp job per 16-row band, in jobs (device, an_band_jobs(h)).
static int an_weight_plane(x265cu_analyser* a, const uint8_t* src, uint8_t* dst, int stride, int w, int h, int mx, int my,
                           const x265cu_wp_entry& e, x265cu_blk_job* jobs)
{
    const int depth = a->p.depth, corr = 14 - depth, denom = e.log2WeightDenom;
    std::vector<x265cu_blk_job> hj(an_band_jobs(h));
    for (size_t j = 0; j < hj.size(); j++)
    {
        x265cu_blk_job& b = hj[j];
        memset(&b, 0, sizeof(b));
        b.d_off = b.a_off = (int64_t)j * 16 * stride;
        b.d_stride = b.a_stride = b.b_stride = stride;
        b.w = (int16_t)w; b.h = (int16_t)min(16, h - (int)j * 16);
        b.p0 = e.inputWeight; b.p1 = (denom ? 1 << (denom - 1) : 0) << corr; b.p2 = denom + corr; b.p3 = e.inputOffset * (1 << (depth - 8));
    }
    CU_CHECK(cudaMemcpy(jobs, hj.data(), sizeof(x265cu_blk_job) * hj.size(), cudaMemcpyHostToDevice));
    if (launch_blockop(a->ctx, depth, X265CU_WEIGHT_PP, dst, src, NULL, jobs, (int)hj.size())) return -1;
    return x265cu_extend_border(a->ctx, depth, dst, stride, w, h, mx, my);
}

static uint8_t* an_alloc_zeroed(x265cu_ctx* c, size_t bytes)
{
    uint8_t* d = (uint8_t*)x265cu_malloc(c, bytes);
    if (d && cudaMemset(d, 0, bytes) != cudaSuccess) return NULL;
    return d;
}

// Brings the weighted planes, the search's pointer tables, the tensor maps and the residual weight table up to date with the
// references changed since the last run (wDirty).  Nothing runs while no reference has ever been weighted.
static int an_weights_prepare(x265cu_analyser* a)
{
    x265cu_ctx* c = a->ctx;
    const int n = a->p.numRefs, depth = a->p.depth;
    const size_t es = depth == 8 ? 1 : 2;
    bool dirty = false;
    for (int r = 0; r < n; r++) dirty = dirty || a->wDirty[r];
    if (!dirty) return 0;
    CU_CHECK(cudaStreamSynchronize(c->stream));          // no launch still reads the job lists and tables rewritten below
    const int lj = an_band_jobs(a->p.height), cj = an_band_jobs(a->p.height >> 1);
    if (!a->d_wjobs) a->d_wjobs = (x265cu_blk_job*)x265cu_malloc(c, sizeof(x265cu_blk_job) * (size_t)16 * (lj + 2 * cj));
    if (!a->d_meRefTable) a->d_meRefTable = (void**)x265cu_malloc(c, sizeof(void*) * 16);
    if (!a->d_meCbTable) a->d_meCbTable = (void**)x265cu_malloc(c, sizeof(void*) * 16);
    if (!a->d_meCrTable) a->d_meCrTable = (void**)x265cu_malloc(c, sizeof(void*) * 16);
    if (!a->d_wtab) a->d_wtab = (int4*)x265cu_malloc(c, sizeof(int4) * 48);
    if (!a->d_wjobs || !a->d_meRefTable || !a->d_meCbTable || !a->d_meCrTable || !a->d_wtab) return -1;
    void* me[16] = {}; void* mc[2][16] = {}; int4 wt[48] = {};
    for (int r = 0; r < n; r++)
    {
        const bool wl = an_ref_weighted(a, r);
        x265cu_blk_job* jobs = a->d_wjobs + (size_t)r * (lj + 2 * cj);
        if (wl && !a->d_wrefs[r] && !(a->d_wrefs[r] = an_alloc_zeroed(c, 16 * a->planeBytes)))
        {
            x265cu_set_error("analyser: no device memory for a weighted reference and its 15 phase planes", cudaErrorMemoryAllocation, __FILE__, __LINE__);
            return -1;
        }
        if (wl && a->wDirty[r] && an_weight_plane(a, a->d_refs[r] + a->orgBytes, a->d_wrefs[r] + a->orgBytes, a->stride, a->p.width,
                                                  a->p.height, AN_MARGIN_X, AN_MARGIN_Y, a->wp[r][0], jobs)) return -1;
        me[r] = (wl ? a->d_wrefs[r] : a->d_refs[r]) + a->orgBytes;
        for (int k = 0; k < 2 && a->chromaOn; k++)
        {
            const bool wc = an_refc_weighted(a, r, k + 1);
            if (wc && !a->d_wrefC[r][k] && !(a->d_wrefC[r][k] = an_alloc_zeroed(c, a->cPlaneBytes)))
            {
                x265cu_set_error("analyser: no device memory for a weighted chroma reference plane", cudaErrorMemoryAllocation, __FILE__, __LINE__);
                return -1;
            }
            if (wc && a->wDirty[r] && an_weight_plane(a, a->d_refC[r][k] + a->cOrgBytes, a->d_wrefC[r][k] + a->cOrgBytes, a->cstride,
                                                      a->p.width >> 1, a->p.height >> 1, AN_MARGIN_X / 2, AN_MARGIN_Y / 2, a->wp[r][k + 1],
                                                      jobs + lj + k * cj)) return -1;
            mc[k][r] = (wc ? a->d_wrefC[r][k] : a->d_refC[r][k]) + a->cOrgBytes;
        }
        if (a->windowOn && a->wDirty[r])
        {
            CUtensorMap tm[MEW_NCLS];
            if (mew_build_tmaps(wl ? a->d_wrefs[r] : a->d_refs[r], a->stride, a->planeRows, (int)es, tm)) return -1;
            CU_CHECK(cudaMemcpy(a->d_tmaps + (size_t)r * MEW_NCLS, tm, sizeof(tm), cudaMemcpyHostToDevice));
        }
        for (int p = 0; p < 3; p++)
            wt[3 * r + p] = make_int4(wl, a->wp[r][p].inputWeight, a->wp[r][p].inputOffset * (1 << (depth - 8)),
                                      a->wp[r][p].log2WeightDenom + 14 - depth);
        a->wDirty[r] = 0;
    }
    CU_CHECK(cudaMemcpy(a->d_meRefTable, me, sizeof(void*) * 16, cudaMemcpyHostToDevice));
    CU_CHECK(cudaMemcpy(a->d_meCbTable, mc[0], sizeof(void*) * 16, cudaMemcpyHostToDevice));
    CU_CHECK(cudaMemcpy(a->d_meCrTable, mc[1], sizeof(void*) * 16, cudaMemcpyHostToDevice));
    CU_CHECK(cudaMemcpy(a->d_wtab, wt, sizeof(wt), cudaMemcpyHostToDevice));
    return 0;
}

// the pixels of reference idx changed: its weighted planes are rebuilt before the next run
static void an_ref_changed(x265cu_analyser* a, int idx) { if (an_ref_weighted(a, idx)) a->wDirty[idx] = 1; }

// the residual stage of the luma plane or of both 4:2:0 chroma planes over the CUs [cu0, cu0 + ncu) and their TUs, the
// CTU rows [r0, r1)
static int an_residual(x265cu_analyser* a, bool chroma, int cu0, int ncu, int r0, int r1)
{
    x265cu_ctx* c = a->ctx;
    const int npl = chroma ? 2 : 1;
    ResidArgs r = {};
    for (int p = 0; p < npl; p++)
    {
        r.fenc[p] = chroma ? a->d_fencC[p] + a->cOrgBytes : a->d_fenc + a->orgBytes;
        r.refs[p] = chroma ? (p ? a->d_refCrTable : a->d_refCbTable) : a->d_refTable;
        r.coef[p] = chroma ? a->d_coefC[p] : a->d_coef;
        r.qp[p] = chroma ? a->qpC[p] : a->p.qp;
    }
    r.stride = chroma ? a->cstride : a->stride; r.recon = chroma ? a->d_reconCTable : a->d_reconTable;
    r.cus = a->d_cus; r.tus = a->d_tus; r.cu_jobs = a->d_cu_jobs; r.numRefs = a->p.numRefs; r.me_out = a->d_me_out;
    r.cu_sse = chroma ? a->d_cu_sseC : a->d_cu_sse; r.cu_numsig = chroma ? a->d_cu_numsigC : a->d_cu_numsig;
    r.cu_ref = chroma ? NULL : a->d_cu_ref;
    CU_CHECK(cudaMemsetAsync(r.cu_sse + (size_t)npl * cu0, 0, sizeof(unsigned long long) * npl * ncu, c->stream));
    CU_CHECK(cudaMemsetAsync(r.cu_numsig + (size_t)npl * cu0, 0, sizeof(uint32_t) * npl * ncu, c->stream));
    const int32_t* lists[3]; int n[3];
    for (int k = 0; k < 3; k++) { lists[k] = a->d_tuBy[k] + a->rowTuBy[k][r0]; n[k] = a->rowTuBy[k][r1] - a->rowTuBy[k][r0]; }
    const int4* wt = a->nWeighted ? a->d_wtab : nullptr;
    const x265cu_bidir_cu* bd = a->numRefL1 ? a->d_bidir : nullptr;   // a B slice: the BIDIR records of this same run
    return a->p.depth == 8 ? launch_resid<uint8_t>(c, chroma, r, lists, n, wt, bd) : launch_resid<uint16_t>(c, chroma, r, lists, n, wt, bd);
}

// Runs the stages over the CTU rows [r0, r1).  Every list is sliced by pointer offset only: PU jobs, ME results and
// the intra table are indexed by the slice-local index inside the kernels, CU / TU records carry absolute indices.
static int an_run(x265cu_analyser* a, int stages, int r0, int r1)
{
    x265cu_ctx* c = a->ctx;
    const int depth = a->p.depth;
    cudaSetDevice(c->device);
    if (r0 < 0 || r1 > a->ctuRows || r0 >= r1) { x265cu_set_error("analyser: bad CTU row range", cudaErrorInvalidValue, __FILE__, __LINE__); return -1; }
    if ((stages & 8) && !(a->chromaOn && a->chromaResOn))
    {
        x265cu_set_error("analyser: stage bit 3 (chroma residual) needs x265cu_analyser_enable_chroma and _enable_chroma_residual", cudaErrorInvalidValue, __FILE__, __LINE__);
        return -1;
    }
    if ((stages & 8) && !an_chroma_reach_ok(a, r0, r1))
    {
        x265cu_set_error("analyser: the chroma planes do not cover what the chroma residual MC can read", cudaErrorInvalidValue, __FILE__, __LINE__);
        return -1;
    }
    if ((stages & 1) && !an_planes_cover(a, r0, r1))
    {
        x265cu_set_error("analyser: the phase planes do not cover the rows the sub-pel search can read", cudaErrorInvalidValue, __FILE__, __LINE__);
        return -1;
    }
    const char* bad = NULL;
    if ((stages & 16) && !a->numRefL1) bad = "analyser: stage bit 4 (BIDIR) needs a B slice (x265cu_analyser_set_lists with numRefL1 > 0)";
    else if (a->numRefL1 && (stages & 10) && !(stages & 16))
        bad = "analyser: the residual stages of a B slice (bits 1, 3) need stage bit 4 (BIDIR) in the same call";
    else if (a->numRefL1 && a->nWeighted) bad = "analyser: B-slice weights are not applied; clear every reference's weights first";
    // Reach of the BIDIR stage and of the bi residual: every vector they use is an ME result of a CU's 2Nx2N job, which
    // k_build_me_jobs' clip bounds as it bounds the vectors of the uni residual, or zero.  Their luma reads are the 8-tap
    // windows of those vectors on the reference planes, inside what an_planes_cover checks for the sub-pel search (which
    // reads the same vectors' windows); their chroma reads are the 4-tap windows of the CU's chroma block, the union of its
    // TUs' blocks, inside what an_chroma_reach_ok checks for the chroma residual.
    else if ((stages & 16) && !an_planes_cover(a, r0, r1)) bad = "analyser: the reference planes do not cover what the BIDIR stage can read";
    else if ((stages & 16) && a->chromaOn && (an_build_chroma_reach(a), !an_chroma_reach_ok(a, r0, r1)))
        bad = "analyser: the chroma planes do not cover what the BIDIR stage's chroma MC can read";
    // Reach of the PART stage: every vector it uses is the ME result of one of the CU's PU jobs, which k_build_me_jobs' clip
    // bounds relative to the CU origin, the same for every PU of the CU; each PU lies inside its CU.  Its luma reads are the
    // 8-tap windows of the PUs' blocks at those vectors, the windows the sub-pel search reads for the same jobs, inside what
    // an_planes_cover checks per PU; its chroma reads are the 4-tap windows of the PUs' chroma blocks, inside the CU's chroma
    // block (the union of its TUs' blocks) moved by a vector inside the same clip, which an_chroma_reach_ok checks.
    else if ((stages & 32) && a->numRefL1)
        bad = "analyser: stage bit 5 (PART) needs a P slice: a B slice's rect / AMP PUs need the per-PU list choice and bi-prediction";
    else if ((stages & 32) && !an_planes_cover(a, r0, r1)) bad = "analyser: the reference planes do not cover what the PART stage can read";
    else if ((stages & 32) && a->chromaOn && (an_build_chroma_reach(a), !an_chroma_reach_ok(a, r0, r1)))
        bad = "analyser: the chroma planes do not cover what the PART stage's chroma MC can read";
    // Reach of the PART_B stage: every vector it reads is a PU job's ME result, or zero in the bi try's zero pair, and every PU
    // lies inside its CU, so its reads are those of the PART stage (above) or the CU's own blocks at zero, inside what the
    // same two checks check.  Weighted slots never reach it: a B slice is refused while weighted (above).
    else if ((stages & 64) && !a->numRefL1)
        bad = "analyser: stage bit 6 (PART_B) needs a B slice (x265cu_analyser_set_lists with numRefL1 > 0); stage bit 5 is a P slice's";
    else if ((stages & 64) && !an_planes_cover(a, r0, r1)) bad = "analyser: the reference planes do not cover what the PART_B stage can read";
    else if ((stages & 64) && a->chromaOn && (an_build_chroma_reach(a), !an_chroma_reach_ok(a, r0, r1)))
        bad = "analyser: the chroma planes do not cover what the PART_B stage's chroma MC can read";
    if (bad) { x265cu_set_error(bad, cudaErrorInvalidValue, __FILE__, __LINE__); return -1; }
    const int job0 = a->rowJob[r0], nj = a->rowJob[r1] - job0;
    const int cu0 = a->rowCu[r0], ncu = a->rowCu[r1] - cu0;
    const int ntu = a->rowTu[r1] - a->rowTu[r0];
    if (an_weights_prepare(a)) return -1;
    if ((stages & 32) && !a->d_part && !(a->d_part = (x265cu_part_cu*)an_alloc_zeroed(c, sizeof(x265cu_part_cu) * a->ncu)))
    {
        x265cu_set_error("analyser: no device memory for the PART records", cudaErrorMemoryAllocation, __FILE__, __LINE__);
        return -1;
    }
    if ((stages & 64) && !a->d_partB && !(a->d_partB = (x265cu_part_b_cu*)an_alloc_zeroed(c, sizeof(x265cu_part_b_cu) * a->ncu)))
    {
        x265cu_set_error("analyser: no device memory for the PART_B records", cudaErrorMemoryAllocation, __FILE__, __LINE__);
        return -1;
    }
    a->ev_valid = stages;
    CU_CHECK(cudaEventRecord(a->ev[0], c->stream));
    if ((stages & 1) && nj > 0)
    {
        k_build_me_jobs<<<(nj + 255) / 256, 256, 0, c->stream>>>(a->d_pus + job0, nj, a->d_field, a->fw, a->fh, a->p.width, a->p.height,
                                                                 a->stride, a->p.method, a->p.subme, a->p.merange, a->d_jobs + job0);
        CU_LAUNCH_CHECK(c);
        MeChromaArgs ch;
        if (a->chromaOn)
        {
            ch.fencCb = a->d_fencC[0] + a->cOrgBytes; ch.fencCr = a->d_fencC[1] + a->cOrgBytes;
            ch.refCb = (const void* const*)(a->nWeighted ? a->d_meCbTable : a->d_refCbTable);
            ch.refCr = (const void* const*)(a->nWeighted ? a->d_meCrTable : a->d_refCrTable); ch.cstride = a->cstride;
        }
        MeWinLaunch win;
        if (a->windowOn)
        {
            win.tmaps = a->d_tmaps; win.allocX = AN_MARGIN_X; win.allocY = AN_MARGIN_Y;
            win.amp = a->p.amp;
            for (int k = 0; k < 3; k++)
            {
                win.groups[k] = a->d_groups[k] + a->rowGrp[k][r0]; win.ngroups[k] = a->rowGrp[k][r1] - a->rowGrp[k][r0];
                win.grp_jobs[k] = a->d_grpJobs[k];
            }
            win.job0 = job0; win.left_count = c->d_counter + 9; win.left_list = a->d_left;
            win.order = a->d_order + job0;
            // workload[subme].hpel_satd (motion.cpp:48-58) is set from subme 2 on
            win.subpelCells = a->p.subme >= 2 && a->cellJobsFit;
        }
        MePlanes pl;
        pl.nrefs = a->p.numRefs; pl.ppitch = (ptrdiff_t)(a->planeBytes / (depth == 8 ? 1 : 2));
        for (int r = 0; r < a->p.numRefs; r++) pl.blocks[r] = an_ref_weighted(a, r) ? a->d_wrefs[r] : a->d_refs[r];
        for (int g = 0; g < 3; g++) { pl.jobs[g] = a->d_planeJobs[g]; pl.njobs[g] = a->nPlaneJobs[g]; }
        if (launch_me(c, depth, a->d_fenc + a->orgBytes, a->stride, (const void* const*)(a->nWeighted ? a->d_meRefTable : a->d_refTable), a->stride, 0,
                      a->d_mvcost + a->mvrange, a->d_jobs + job0, nj, a->d_me_out + (size_t)job0 * 4, c->d_counter,
                      a->chromaOn ? &ch : NULL, a->windowOn ? &win : NULL, &pl)) return -1;
        CU_CHECK(cudaEventRecord(a->ev[4], c->stream));      // ME search kernel alone ends here
        k_pack_me<<<(nj + 255) / 256, 256, 0, c->stream>>>(a->d_me_out + (size_t)job0 * 4, nj, a->d_me_packed + job0);
        CU_LAUNCH_CHECK(c);
    }
    else if (stages & 1) CU_CHECK(cudaEventRecord(a->ev[4], c->stream));
    CU_CHECK(cudaEventRecord(a->ev[1], c->stream));
    if ((stages & 16) && ncu > 0)
    {
        BidirArgs b;
        b.fenc[0] = a->d_fenc + a->orgBytes; b.refs[0] = a->d_refTable; b.stride = a->stride; b.chroma = a->chromaOn;
        for (int k = 0; k < 2 && a->chromaOn; k++)
        {
            b.fenc[1 + k] = a->d_fencC[k] + a->cOrgBytes; b.refs[1 + k] = k ? a->d_refCrTable : a->d_refCbTable;
        }
        b.cstride = a->cstride;
        b.cus = a->d_cus; b.cu_jobs = a->d_cu_jobs; b.numRefs = a->p.numRefs; b.numRefL0 = a->numRefL0; b.me_out = a->d_me_out;
        b.jobs = a->d_jobs; b.mvc = a->d_mvcost + a->mvrange; b.width = a->p.width; b.height = a->p.height; b.out = a->d_bidir;
        const int32_t* lists[4]; int n[4];
        for (int k = 0; k < 4; k++) { lists[k] = a->d_cuBy[k] + a->rowCuBy[k][r0]; n[k] = a->rowCuBy[k][r1] - a->rowCuBy[k][r0]; }
        if (depth == 8 ? launch_bidir<uint8_t>(c, b, lists, n) : launch_bidir<uint16_t>(c, b, lists, n)) return -1;
    }
    if ((stages & 96) && ncu > 0)
    {
        PartArgs q;
        q.fenc[0] = a->d_fenc + a->orgBytes; q.refs[0] = a->d_refTable; q.stride = a->stride; q.chroma = a->chromaOn;
        for (int k = 0; k < 2 && a->chromaOn; k++)
        {
            q.fenc[1 + k] = a->d_fencC[k] + a->cOrgBytes; q.refs[1 + k] = k ? a->d_refCrTable : a->d_refCbTable;
        }
        q.cstride = a->cstride;
        q.cus = a->d_cus; q.pus = a->d_pus; q.cu_jobs = a->d_cu_jobs; q.numRefs = a->p.numRefs; q.rect = a->p.rect; q.amp = a->p.amp;
        q.me_out = a->d_me_out; q.jobs = a->d_jobs; q.mvc = a->d_mvcost + a->mvrange; q.wt = a->nWeighted ? a->d_wtab : nullptr;
        q.out = a->d_part;
        const int32_t* lists[4]; int n[4];
        for (int k = 0; k < 4; k++) { lists[k] = a->d_cuBy[k] + a->rowCuBy[k][r0]; n[k] = a->rowCuBy[k][r1] - a->rowCuBy[k][r0]; }
        if ((stages & 32) && (depth == 8 ? launch_part<uint8_t>(c, q, lists, n) : launch_part<uint16_t>(c, q, lists, n))) return -1;
        if (stages & 64)
        {
            PartBArgs b;
            b.p = q; b.numRefL0 = a->numRefL0; b.width = a->p.width; b.height = a->p.height;
            b.chromaSatd = a->chromaOn && a->p.subme > 2; b.out = a->d_partB;
            if (depth == 8 ? launch_part_b<uint8_t>(c, b, lists, n) : launch_part_b<uint16_t>(c, b, lists, n)) return -1;
        }
    }
    CU_CHECK(cudaEventRecord(a->ev[5], c->stream));
    if ((stages & 2) && ntu > 0 && an_residual(a, false, cu0, ncu, r0, r1)) return -1;
    CU_CHECK(cudaEventRecord(a->ev[2], c->stream));
    if ((stages & 4) && ncu > 0)
    {
        const int32_t* lists[4]; int n[4];
        for (int k = 0; k < 4; k++) { lists[k] = a->d_cuBy[k] + a->rowCuBy[k][r0]; n[k] = a->rowCuBy[k][r1] - a->rowCuBy[k][r0]; }
        const int e = depth == 8 ? launch_intra<uint8_t>(c, a->d_fenc + a->orgBytes, a->stride, a->d_cus, lists, n, a->d_intra)
                                 : launch_intra<uint16_t>(c, a->d_fenc + a->orgBytes, a->stride, a->d_cus, lists, n, a->d_intra);
        if (e) return -1;
    }
    CU_CHECK(cudaEventRecord(a->ev[3], c->stream));
    if ((stages & 8) && ntu > 0 && an_residual(a, true, cu0, ncu, r0, r1)) return -1;
    return 0;
}

// upload a width x height host image into a margin-extended device plane
static int an_upload_plane(x265cu_analyser* a, uint8_t* d_plane, const void* host, int hostStride)
{
    x265cu_ctx* c = a->ctx;
    const size_t es = a->p.depth == 8 ? 1 : 2;
    cudaSetDevice(c->device);
    CU_CHECK(cudaMemcpy2DAsync(d_plane + a->orgBytes, (size_t)a->stride * es, host, (size_t)hostStride * es,
                               (size_t)a->p.width * es, a->p.height, cudaMemcpyHostToDevice, c->stream));
    return x265cu_extend_border(c, a->p.depth, d_plane + a->orgBytes, a->stride, a->p.width, a->p.height, AN_MARGIN_X, AN_MARGIN_Y);
}

extern "C" {

x265cu_analyser* x265cu_analyser_create(x265cu_ctx* ctx, const x265cu_analysis_params* p)
{
    if (!ctx || p->numRefs < 1 || p->numRefs > 16 || (p->depth != 8 && p->depth != 10)) return NULL;
    // parameters the kernels cannot run as the reference does: refused rather than silently searched differently
    const char* bad = NULL;
    if (p->method != 0 && p->method != 1 && p->method != 3 && p->method != 5)
        bad = "x265cu_analyser_create: search method not 0 (DIA), 1 (HEX), 3 (STAR) or 5 (FULL)";
    else if (p->merange < 0 || p->merange > 127) bad = "x265cu_analyser_create: merange outside 0..127 (the job record holds it in 8 bits)";
    else if (p->subme < 0 || p->subme > 7) bad = "x265cu_analyser_create: subme outside 0..7";
    else if (p->width <= 0 || p->height <= 0 || (p->width & 7) || (p->height & 7))
        bad = "x265cu_analyser_create: width and height not positive multiples of 8";
    // the quantiser's QPs: 0..51 + QP_BD_OFFSET (quant.cpp:224); resid_quant has scales for rem = qp % 6 in 0..5 only
    else if (p->qp < 0 || p->qp > 51 + 6 * (p->depth - 8))
        bad = "x265cu_analyser_create: qp outside 0..51 + 6 * (depth - 8)";
    else if (!isfinite(p->lambda) || p->lambda < 0)
        bad = "x265cu_analyser_create: lambda negative or not finite";
    if (bad) { x265cu_set_error(bad, cudaErrorInvalidValue, __FILE__, __LINE__); return NULL; }
    cudaSetDevice(ctx->device);
    x265cu_analyser* a = new x265cu_analyser();
    a->ctx = ctx; a->p = *p;
    const size_t es = p->depth == 8 ? 1 : 2;
    a->stride = (p->width + 2 * AN_MARGIN_X + 63) / 64 * 64;
    a->planeRows = p->height + 2 * AN_MARGIN_Y;
    a->planeBytes = (size_t)a->stride * a->planeRows * es + 256;
    a->orgBytes = ((size_t)AN_MARGIN_Y * a->stride + AN_MARGIN_X) * es;
    a->fw = (p->width + 15) / 16; a->fh = (p->height + 15) / 16;
    an_build_geometry(a);
    a->d_fenc = (uint8_t*)x265cu_malloc(ctx, a->planeBytes);
    if (a->d_fenc) cudaMemset(a->d_fenc, 0, a->planeBytes);
    void* reft[16]; void* rect[4];
    // every reference is a block of 16 planes: slot 0 the reference, slots 1..15 its phase planes.  The 15 phase planes add
    // 15 x planeBytes per reference: 561 MB at 3840x2160 8-bit with 4 references (bench.py c3), 1.40 GB at 3840x2160 10-bit
    // with 5 (c4), 5.3 GB at 7680x4320 10-bit with 5 (c5)
    for (int r = 0; r < p->numRefs; r++)
    {
        a->d_refs[r] = (uint8_t*)x265cu_malloc(ctx, 16 * a->planeBytes);
        if (!a->d_refs[r])
        {
            x265cu_set_error("x265cu_analyser_create: no device memory for a reference and its 15 phase planes", cudaErrorMemoryAllocation, __FILE__, __LINE__);
            return NULL;
        }
        cudaMemset(a->d_refs[r], 0, 16 * a->planeBytes);
        reft[r] = a->d_refs[r] + a->orgBytes;
    }
    for (int d = 0; d < 4; d++) { a->d_recon[d] = (uint8_t*)x265cu_malloc(ctx, a->planeBytes); rect[d] = a->d_recon[d] + a->orgBytes; cudaMemset(a->d_recon[d], 0, a->planeBytes); }
    a->d_refTable = (void**)x265cu_malloc(ctx, sizeof(void*) * 16);
    a->d_reconTable = (void**)x265cu_malloc(ctx, sizeof(void*) * 4);
    cudaMemcpy(a->d_refTable, reft, sizeof(void*) * p->numRefs, cudaMemcpyHostToDevice);
    cudaMemcpy(a->d_reconTable, rect, sizeof(void*) * 4, cudaMemcpyHostToDevice);
    const size_t fieldBytes = (size_t)p->numRefs * a->fw * a->fh * 2 * sizeof(int16_t);
    a->d_field = (int16_t*)x265cu_malloc(ctx, fieldBytes);
    a->mvrange = 65536;                                   // +-2*BC_MAX_MV like bitcost.h:77
    std::vector<uint16_t> tab(2 * a->mvrange + 1);
    x265cu_mvcost_table(p->lambda, a->mvrange, tab.data());
    a->d_mvcost = an_upload(ctx, tab);
    a->d_pus = an_upload(ctx, a->pus); a->d_cus = an_upload(ctx, a->cus); a->d_tus = an_upload(ctx, a->tus); a->d_cu_jobs = an_upload(ctx, a->cu_jobs);
    a->d_jobs = (x265cu_me_job*)x265cu_malloc(ctx, sizeof(x265cu_me_job) * a->njobs);
    if (a->d_jobs) cudaMemset(a->d_jobs, 0, sizeof(x265cu_me_job) * a->njobs);     // the MVPs a BIDIR run before any search reads
    a->d_me_out = (int32_t*)x265cu_malloc(ctx, sizeof(int32_t) * 4 * a->njobs);
    // a residual stage run before any search reads vector 0 of every CU, which lies inside every plane's reach
    if (a->d_me_out) cudaMemset(a->d_me_out, 0, sizeof(int32_t) * 4 * a->njobs);
    a->d_me_packed = (int2*)x265cu_malloc(ctx, sizeof(int2) * a->njobs);
    // shared-memory-window search: tensor maps over the reference plane allocations (STAR only; the other methods and any
    // group whose window does not fit go through the global-memory kernel)
    {
        const char* e = getenv("X265CU_ME_WINDOW");
        a->windowOn = !(e && e[0] == '0') && p->method == 3;
        a->d_tmaps = NULL;
        a->d_left = (int32_t*)x265cu_malloc(ctx, sizeof(int32_t) * (a->njobs + 1));
        if (a->windowOn)
        {
            std::vector<CUtensorMap> tm((size_t)p->numRefs * MEW_NCLS);
            bool ok = a->d_left != NULL;
            for (int r = 0; r < p->numRefs && ok; r++)
                ok = a->d_refs[r] && mew_build_tmaps(a->d_refs[r], a->stride, a->planeRows, (int)es, &tm[(size_t)r * MEW_NCLS]) == 0;
            if (ok)
            {
                a->d_tmaps = (CUtensorMap*)x265cu_malloc(ctx, sizeof(CUtensorMap) * tm.size());
                ok = a->d_tmaps && cudaMemcpy(a->d_tmaps, tm.data(), sizeof(CUtensorMap) * tm.size(), cudaMemcpyHostToDevice) == cudaSuccess;
            }
            if (!ok) { fprintf(stderr, "x265cu: tensor maps unavailable, integer search stays on the global-memory kernel: %s\n", x265cu_last_error()); a->windowOn = 0; }
        }
    }
    a->d_coef = (int16_t*)x265cu_malloc(ctx, sizeof(int16_t) * a->ncoef);
    a->d_cu_sse = (unsigned long long*)x265cu_malloc(ctx, sizeof(unsigned long long) * a->ncu);
    a->d_cu_numsig = (uint32_t*)x265cu_malloc(ctx, sizeof(uint32_t) * a->ncu);
    a->d_cu_ref = (int32_t*)x265cu_malloc(ctx, sizeof(int32_t) * a->ncu);
    a->d_intra = (uint32_t*)x265cu_malloc(ctx, sizeof(uint32_t) * 36 * a->ncu);
    for (int i = 0; i < 6; i++) cudaEventCreate(&a->ev[i]);
    a->numRefL0 = p->numRefs; a->numRefL1 = 0;
    a->ev_valid = 0;
    a->chromaOn = 0; a->d_refCbTable = a->d_refCrTable = NULL;
    a->d_fencC[0] = a->d_fencC[1] = NULL;
    for (int r = 0; r < 16; r++) a->d_refC[r][0] = a->d_refC[r][1] = NULL;
    a->h_fenc = (uint8_t*)x265cu_host_alloc((size_t)p->width * p->height * es);
    a->h_field = (int16_t*)x265cu_host_alloc(fieldBytes);
    if (!a->d_intra || !a->d_coef || !a->d_me_out || !a->h_fenc || !a->h_field) return NULL;
    an_build_read_rects(a);
    if (an_build_plane_jobs(a)) return NULL;
    if (!an_planes_cover(a, 0, a->ctuRows))
    {
        x265cu_set_error("x265cu_analyser_create: the phase planes do not cover what the sub-pel search can read", cudaErrorInvalidValue, __FILE__, __LINE__);
        return NULL;
    }
    cudaDeviceSynchronize();
    return a;
}

void x265cu_analyser_destroy(x265cu_analyser* a)
{
    if (!a) return;
    x265cu_ctx* c = a->ctx;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    void* bufs[] = { a->d_fenc, a->d_refTable, a->d_reconTable, a->d_field, a->d_mvcost, a->d_pus, a->d_cus, a->d_tus, a->d_cu_jobs, a->d_jobs,
                     a->d_me_out, a->d_me_packed, a->d_coef, a->d_cu_sse, a->d_cu_numsig, a->d_cu_ref, a->d_intra,
                     a->d_groups[0], a->d_groups[1], a->d_groups[2], a->d_grpJobs[0], a->d_grpJobs[1], a->d_grpJobs[2], a->d_tmaps, a->d_left, a->d_order,
                     a->d_tuBy[0], a->d_tuBy[1], a->d_tuBy[2], a->d_cuBy[0], a->d_cuBy[1], a->d_cuBy[2], a->d_cuBy[3],
                     a->d_planeJobs[0], a->d_planeJobs[1], a->d_planeJobs[2] };
    for (void* b : bufs) cudaFree(b);
    for (int r = 0; r < a->p.numRefs; r++) cudaFree(a->d_refs[r]);
    for (int d = 0; d < 4; d++) cudaFree(a->d_recon[d]);
    for (int k = 0; k < 2; k++) { cudaFree(a->d_fencC[k]); for (int r = 0; r < a->p.numRefs; r++) cudaFree(a->d_refC[r][k]); }
    cudaFree(a->d_refCbTable); cudaFree(a->d_refCrTable);
    for (int k = 0; k < 2; k++) { cudaFree(a->d_coefC[k]); for (int d = 0; d < 4; d++) cudaFree(a->d_reconC[d][k]); }
    cudaFree(a->d_reconCTable); cudaFree(a->d_cu_sseC); cudaFree(a->d_cu_numsigC);
    for (int r = 0; r < 16; r++) { cudaFree(a->d_wrefs[r]); cudaFree(a->d_wrefC[r][0]); cudaFree(a->d_wrefC[r][1]); }
    cudaFree(a->d_meRefTable); cudaFree(a->d_meCbTable); cudaFree(a->d_meCrTable); cudaFree(a->d_wtab); cudaFree(a->d_wjobs);
    cudaFree(a->d_bidir); cudaFree(a->d_part); cudaFree(a->d_partB);
    x265cu_host_free(a->h_fenc); x265cu_host_free(a->h_field);
    delete a;
}

int x265cu_analyser_counts(x265cu_analyser* a, int* njobs, int* ncu, int* ntu, int64_t* ncoef, int* stride)
{
    *njobs = a->njobs; *ncu = a->ncu; *ntu = a->ntu; *ncoef = a->ncoef; *stride = a->stride;
    return 0;
}

int x265cu_analyser_set_ref(x265cu_analyser* a, int idx, const void* host_luma, int host_stride)
{
    if (idx < 0 || idx >= a->p.numRefs) return -1;
    an_ref_changed(a, idx);
    if (an_upload_plane(a, a->d_refs[idx], host_luma, host_stride)) return -1;
    return x265cu_sync(a->ctx);
}

int x265cu_analyser_load_inputs(x265cu_analyser* a, const void* fenc_host, int host_stride, const int16_t* field_host)
{
    x265cu_ctx* c = a->ctx;
    const size_t es = a->p.depth == 8 ? 1 : 2;
    // copies are issued straight from the caller's buffers: pass pinned memory (x265cu_host_alloc)
    // for true asynchronous DMA; pageable memory also works (the driver stages it)
    (void)es;
    const size_t fieldBytes = (size_t)a->p.numRefs * a->fw * a->fh * 2 * sizeof(int16_t);
    if (an_upload_plane(a, a->d_fenc, fenc_host, host_stride)) return -1;
    CU_CHECK(cudaMemcpyAsync(a->d_field, field_host, fieldBytes, cudaMemcpyHostToDevice, c->stream));
    return 0;
}

// ---- 4:2:0 chroma for the chroma-SATD term of subpelCompare (MotionEstimate::bChromaSATD, motion.cpp:204-212, 1601-1661) ----
// After enable_chroma() the ME stage runs the chroma instantiations of k_me (x265cu_me_batch_chroma's kernels) on the resident chroma
// planes; the caller uploads the source's Cb / Cr with load_chroma() and every reference's with set_ref_chroma().
static int an_upload_cplane(x265cu_analyser* a, uint8_t* d_plane, const void* host, int hostStride)
{
    x265cu_ctx* c = a->ctx;
    const size_t es = a->p.depth == 8 ? 1 : 2;
    const int cw = a->p.width >> 1, ch = a->p.height >> 1;
    cudaSetDevice(c->device);
    CU_CHECK(cudaMemcpy2DAsync(d_plane + a->cOrgBytes, (size_t)a->cstride * es, host, (size_t)hostStride * es,
                               (size_t)cw * es, ch, cudaMemcpyHostToDevice, c->stream));
    return x265cu_extend_border(c, a->p.depth, d_plane + a->cOrgBytes, a->cstride, cw, ch, AN_MARGIN_X / 2, AN_MARGIN_Y / 2);
}

int x265cu_analyser_enable_chroma(x265cu_analyser* a)
{
    if (a->chromaOn) return 0;
    x265cu_ctx* c = a->ctx;
    cudaSetDevice(c->device);
    const size_t es = a->p.depth == 8 ? 1 : 2;
    a->cstride = a->stride / 2;
    a->cRows = (a->p.height >> 1) + AN_MARGIN_Y;                 // 2 * (AN_MARGIN_Y / 2)
    a->cPlaneBytes = (size_t)a->cstride * a->cRows * es + 256;
    a->cOrgBytes = ((size_t)(AN_MARGIN_Y / 2) * a->cstride + AN_MARGIN_X / 2) * es;
    void* cbt[16]; void* crt[16];
    for (int k = 0; k < 2; k++)
    {
        a->d_fencC[k] = (uint8_t*)x265cu_malloc(c, a->cPlaneBytes);
        if (!a->d_fencC[k]) return -1;
        CU_CHECK(cudaMemset(a->d_fencC[k], 0, a->cPlaneBytes));
        for (int r = 0; r < a->p.numRefs; r++)
        {
            a->d_refC[r][k] = (uint8_t*)x265cu_malloc(c, a->cPlaneBytes);
            if (!a->d_refC[r][k]) return -1;
            CU_CHECK(cudaMemset(a->d_refC[r][k], 0, a->cPlaneBytes));
            (k ? crt : cbt)[r] = a->d_refC[r][k] + a->cOrgBytes;
        }
    }
    a->d_refCbTable = (void**)x265cu_malloc(c, sizeof(void*) * 16);
    a->d_refCrTable = (void**)x265cu_malloc(c, sizeof(void*) * 16);
    if (!a->d_refCbTable || !a->d_refCrTable) return -1;
    CU_CHECK(cudaMemcpy(a->d_refCbTable, cbt, sizeof(void*) * a->p.numRefs, cudaMemcpyHostToDevice));
    CU_CHECK(cudaMemcpy(a->d_refCrTable, crt, sizeof(void*) * a->p.numRefs, cudaMemcpyHostToDevice));
    a->chromaOn = 1;
    for (int r = 0; r < a->p.numRefs; r++) an_ref_changed(a, r);
    return 0;
}

int x265cu_analyser_set_ref_chroma(x265cu_analyser* a, int idx, const void* cb_host, const void* cr_host, int host_stride)
{
    if (!a->chromaOn || idx < 0 || idx >= a->p.numRefs) return -1;
    an_ref_changed(a, idx);
    if (an_upload_cplane(a, a->d_refC[idx][0], cb_host, host_stride) || an_upload_cplane(a, a->d_refC[idx][1], cr_host, host_stride)) return -1;
    return x265cu_sync(a->ctx);
}

int x265cu_analyser_load_chroma(x265cu_analyser* a, const void* cb_host, const void* cr_host, int host_stride)
{
    if (!a->chromaOn) return -1;
    if (an_upload_cplane(a, a->d_fencC[0], cb_host, host_stride) || an_upload_cplane(a, a->d_fencC[1], cr_host, host_stride)) return -1;
    return 0;
}

// ---- 4:2:0 chroma residual chain (stage bit 3, resid.cuh) ----
int x265cu_analyser_enable_chroma_residual(x265cu_analyser* a, int cbQpOffset, int crQpOffset)
{
    const char* bad = NULL;
    if (!a->chromaOn) bad = "x265cu_analyser_enable_chroma_residual: chroma planes not enabled (x265cu_analyser_enable_chroma)";
    // HEVC limits the PPS + slice chroma QP offset to -12..12; x265 checks the same range (param.cpp:1572-1575)
    else if (cbQpOffset < -12 || cbQpOffset > 12 || crQpOffset < -12 || crQpOffset > 12)
        bad = "x265cu_analyser_enable_chroma_residual: chroma QP offset outside -12..12";
    if (bad) { x265cu_set_error(bad, cudaErrorInvalidValue, __FILE__, __LINE__); return -1; }
    x265cu_ctx* c = a->ctx;
    cudaSetDevice(c->device);
    a->qpC[0] = geometry_chroma_qp(a->p.qp, cbQpOffset, a->p.depth);
    a->qpC[1] = geometry_chroma_qp(a->p.qp, crQpOffset, a->p.depth);
    if (a->chromaResOn) return 0;
    an_build_chroma_reach(a);
    if (!an_chroma_reach_ok(a, 0, a->ctuRows))
    {
        x265cu_set_error("x265cu_analyser_enable_chroma_residual: the chroma planes do not cover what the chroma MC can read", cudaErrorInvalidValue, __FILE__, __LINE__);
        return -1;
    }
    void* rect[8];
    for (int k = 0; k < 2; k++)
    {
        a->d_coefC[k] = (int16_t*)x265cu_malloc(c, sizeof(int16_t) * (a->ncoef / 4) + 16);
        if (!a->d_coefC[k]) return -1;
        for (int d = 0; d < 4; d++)
        {
            a->d_reconC[d][k] = (uint8_t*)x265cu_malloc(c, a->cPlaneBytes);
            if (!a->d_reconC[d][k]) return -1;
            CU_CHECK(cudaMemset(a->d_reconC[d][k], 0, a->cPlaneBytes));
            rect[2 * d + k] = a->d_reconC[d][k] + a->cOrgBytes;
        }
    }
    a->d_reconCTable = (void**)x265cu_malloc(c, sizeof(void*) * 8);
    a->d_cu_sseC = (unsigned long long*)x265cu_malloc(c, sizeof(unsigned long long) * 2 * a->ncu);
    a->d_cu_numsigC = (uint32_t*)x265cu_malloc(c, sizeof(uint32_t) * 2 * a->ncu);
    if (!a->d_reconCTable || !a->d_cu_sseC || !a->d_cu_numsigC) return -1;
    CU_CHECK(cudaMemcpy(a->d_reconCTable, rect, sizeof(rect), cudaMemcpyHostToDevice));
    CU_CHECK(cudaMemset(a->d_cu_sseC, 0, sizeof(unsigned long long) * 2 * a->ncu));
    CU_CHECK(cudaMemset(a->d_cu_numsigC, 0, sizeof(uint32_t) * 2 * a->ncu));
    a->chromaResOn = 1;
    return 0;
}

// quantiser QP of Cb and Cr (Quant::setChromaQP, quant.cpp:221-244)
int x265cu_analyser_chroma_qp(x265cu_analyser* a, int* qp2)
{
    if (!a->chromaResOn) return -1;
    qp2[0] = a->qpC[0]; qp2[1] = a->qpC[1];
    return 0;
}

// per-CU [cu][plane] SSE and numSig of the CTU rows [r0, r1) into full-frame sized host arrays (synchronous)
int x265cu_analyser_chroma_results(x265cu_analyser* a, int ctuRow0, int ctuRow1, uint64_t* sse, uint32_t* numsig)
{
    if (!a->chromaResOn || ctuRow0 < 0 || ctuRow1 > a->ctuRows || ctuRow0 > ctuRow1) return -1;
    x265cu_ctx* c = a->ctx;
    cudaSetDevice(c->device);
    const size_t c0 = a->rowCu[ctuRow0], nc = a->rowCu[ctuRow1] - c0;
    if (sse && nc) CU_CHECK(cudaMemcpyAsync(sse + 2 * c0, a->d_cu_sseC + 2 * c0, sizeof(uint64_t) * 2 * nc, cudaMemcpyDeviceToHost, c->stream));
    if (numsig && nc) CU_CHECK(cudaMemcpyAsync(numsig + 2 * c0, a->d_cu_numsigC + 2 * c0, sizeof(uint32_t) * 2 * nc, cudaMemcpyDeviceToHost, c->stream));
    CU_CHECK(cudaStreamSynchronize(c->stream));
    return 0;
}

// what: 0 / 1 the Cb / Cr levels (ncoef / 4 each); 2 + 2 * depthIdx + plane the whole allocation of a chroma recon plane,
// 10 + 2 * ref + plane the whole allocation of a reference's chroma plane (cstride x (height / 2 + 80) elements each);
// 10 + 2 * numRefs + 2 * ref + plane the chroma plane the chroma-SATD term of the search reads for the reference: its weighted
// plane when it has one, else the reference's plane (needs enable_chroma only)
int x265cu_analyser_fetch_chroma(x265cu_analyser* a, int what, void* host)
{
    const int nr = a->p.numRefs;
    if (!a->chromaOn || what < 0 || what >= 10 + 4 * nr || (what < 10 + 2 * nr && !a->chromaResOn)) return -1;
    x265cu_ctx* c = a->ctx;
    const size_t es = a->p.depth == 8 ? 1 : 2, planeBytes = (size_t)a->cstride * a->cRows * es;
    const void* src; size_t bytes;
    if (what < 2) { src = a->d_coefC[what]; bytes = sizeof(int16_t) * (a->ncoef / 4); }
    else if (what < 10) { src = a->d_reconC[(what - 2) >> 1][what & 1]; bytes = planeBytes; }
    else if (what < 10 + 2 * nr) { src = a->d_refC[(what - 10) >> 1][what & 1]; bytes = planeBytes; }
    else
    {
        const int r = (what - 10 - 2 * nr) >> 1, k = what & 1;
        if (an_weights_prepare(a)) return -1;
        src = an_refc_weighted(a, r, k + 1) ? a->d_wrefC[r][k] : a->d_refC[r][k]; bytes = planeBytes;
    }
    cudaSetDevice(c->device);
    CU_CHECK(cudaMemcpyAsync(host, src, bytes, cudaMemcpyDeviceToHost, c->stream));
    CU_CHECK(cudaStreamSynchronize(c->stream));
    return 0;
}

// device address of the origin pixel of chroma recon plane (depthIdx, plane) and its stride in elements
void* x265cu_analyser_recon_plane_chroma(x265cu_analyser* a, int depthIdx, int plane, int* cstride)
{
    if (!a->chromaResOn || depthIdx < 0 || depthIdx >= 4 || plane < 0 || plane > 1) return NULL;
    *cstride = a->cstride;
    return a->d_reconC[depthIdx][plane] + a->cOrgBytes;
}

// promote the chroma rows of CTU rows [ctuRow0, ctuRow1) of recon depth depthIdx (both planes) to reference idx; call
// x265cu_analyser_ref_chroma_updated() once all rows of the new reference are in place
int x265cu_analyser_recon_to_ref_chroma(x265cu_analyser* a, int depthIdx, int idx, int ctuRow0, int ctuRow1)
{
    if (!a->chromaResOn || depthIdx < 0 || depthIdx >= 4 || idx < 0 || idx >= a->p.numRefs || ctuRow0 < 0 || ctuRow1 > a->ctuRows || ctuRow0 >= ctuRow1) return -1;
    const size_t es = a->p.depth == 8 ? 1 : 2;
    const int ch = a->p.height >> 1, y0 = ctuRow0 * 32, y1 = ctuRow1 * 32 < ch ? ctuRow1 * 32 : ch;
    cudaSetDevice(a->ctx->device);
    const size_t off = a->cOrgBytes + (size_t)y0 * a->cstride * es, pitch = (size_t)a->cstride * es;
    an_ref_changed(a, idx);
    for (int k = 0; k < 2; k++)
        CU_CHECK(cudaMemcpy2DAsync(a->d_refC[idx][k] + off, pitch, a->d_reconC[depthIdx][k] + off, pitch, (size_t)(a->p.width >> 1) * es, y1 - y0,
                                   cudaMemcpyDeviceToDevice, a->ctx->stream));
    return 0;
}

// re-extend the borders of reference idx's chroma planes (extendPicBorder with the chroma margins)
int x265cu_analyser_ref_chroma_updated(x265cu_analyser* a, int idx)
{
    if (!a->chromaOn || idx < 0 || idx >= a->p.numRefs) return -1;
    cudaSetDevice(a->ctx->device);
    an_ref_changed(a, idx);
    for (int k = 0; k < 2; k++)
        if (x265cu_extend_border(a->ctx, a->p.depth, a->d_refC[idx][k] + a->cOrgBytes, a->cstride, a->p.width >> 1, a->p.height >> 1,
                                 AN_MARGIN_X / 2, AN_MARGIN_Y / 2)) return -1;
    return 0;
}

// device address of chroma plane `plane` of reference idx at its origin pixel, and the chroma stride in elements
void* x265cu_analyser_ref_plane_chroma(x265cu_analyser* a, int idx, int plane, int* cstride)
{
    if (!a->chromaOn || idx < 0 || idx >= a->p.numRefs || plane < 0 || plane > 1) return NULL;
    *cstride = a->cstride;
    return a->d_refC[idx][plane] + a->cOrgBytes;
}

// device address of source plane `plane` (0 luma, 1 Cb, 2 Cr) at its origin pixel and its stride in elements: the twin of
// ref_plane / ref_plane_chroma for the calls that read the source, e.g. x265cu_sao_stats_frame
void* x265cu_analyser_src_plane(x265cu_analyser* a, int plane, int* stride)
{
    if (plane == 0) { *stride = a->stride; return a->d_fenc + a->orgBytes; }
    if (!a->chromaOn || plane < 0 || plane > 2) return NULL;
    *stride = a->cstride;
    return a->d_fencC[plane - 1] + a->cOrgBytes;
}

int x265cu_analyser_run_resident(x265cu_analyser* a, int stages) { return an_run(a, stages, 0, a->ctuRows); }

// ---- CTU-row shards (the WPP row partition of SURVEY 8(e): frameencoder.cpp:850-868 enables row r once the
// reference rows it needs are reconstructed; a rank owns a set of CTU rows and analyses exactly those) ----
int x265cu_analyser_ctu_rows(x265cu_analyser* a) { return a->ctuRows; }

int x265cu_analyser_row_range(x265cu_analyser* a, int ctuRow0, int ctuRow1, int* job0, int* njobs, int* cu0, int* ncu)
{
    if (ctuRow0 < 0 || ctuRow1 > a->ctuRows || ctuRow0 > ctuRow1) return -1;
    *job0 = a->rowJob[ctuRow0]; *njobs = a->rowJob[ctuRow1] - a->rowJob[ctuRow0];
    *cu0 = a->rowCu[ctuRow0];   *ncu = a->rowCu[ctuRow1] - a->rowCu[ctuRow0];
    return 0;
}

int x265cu_analyser_run_rows(x265cu_analyser* a, int stages, int ctuRow0, int ctuRow1) { return an_run(a, stages, ctuRow0, ctuRow1); }

// `out` arrays are always full-frame sized; a row shard fills only the entries of its own rows.
int x265cu_analyser_analyse_rows(x265cu_analyser* a, const void* fenc_host, int host_stride, const int16_t* field_host, int stages,
                                 int ctuRow0, int ctuRow1, x265cu_analysis_out* out)
{
    x265cu_ctx* c = a->ctx;
    if (x265cu_analyser_load_inputs(a, fenc_host, host_stride, field_host)) return -1;
    if (an_run(a, stages, ctuRow0, ctuRow1)) return -1;
    if (out)
    {
        const size_t j0 = a->rowJob[ctuRow0], nj = a->rowJob[ctuRow1] - j0, c0 = a->rowCu[ctuRow0], nc = a->rowCu[ctuRow1] - c0;
        if (out->me_packed && nj) CU_CHECK(cudaMemcpyAsync(out->me_packed + 2 * j0, a->d_me_packed + j0, sizeof(int2) * nj, cudaMemcpyDeviceToHost, c->stream));
        if (out->cu_sse && nc) CU_CHECK(cudaMemcpyAsync(out->cu_sse + c0, a->d_cu_sse + c0, sizeof(uint64_t) * nc, cudaMemcpyDeviceToHost, c->stream));
        if (out->cu_numsig && nc) CU_CHECK(cudaMemcpyAsync(out->cu_numsig + c0, a->d_cu_numsig + c0, sizeof(uint32_t) * nc, cudaMemcpyDeviceToHost, c->stream));
        if (out->cu_ref && nc) CU_CHECK(cudaMemcpyAsync(out->cu_ref + c0, a->d_cu_ref + c0, sizeof(int32_t) * nc, cudaMemcpyDeviceToHost, c->stream));
        if (out->intra_cost && nc) CU_CHECK(cudaMemcpyAsync(out->intra_cost + 36 * c0, a->d_intra + 36 * c0, sizeof(uint32_t) * 36 * nc, cudaMemcpyDeviceToHost, c->stream));
    }
    CU_CHECK(cudaStreamSynchronize(c->stream));
    return 0;
}

int x265cu_analyser_analyse(x265cu_analyser* a, const void* fenc_host, int host_stride, const int16_t* field_host, int stages,
                            x265cu_analysis_out* out)
{
    return x265cu_analyser_analyse_rows(a, fenc_host, host_stride, field_host, stages, 0, a->ctuRows, out);
}

// per-stage device time of the last run (ms): [0] ME stage (job build + search + pack), [1] residual,
// [2] intra, [3] the ME search kernel alone.  Synchronises the stream.
int x265cu_analyser_stage_ms(x265cu_analyser* a, float* ms)
{
    CU_CHECK(cudaEventSynchronize(a->ev[3]));
    for (int i = 0; i < 3; i++) CU_CHECK(cudaEventElapsedTime(&ms[i], a->ev[i == 1 ? 5 : i], a->ev[i + 1]));   // [1] from after BIDIR
    ms[3] = 0.f;
    if (a->ev_valid & 1) CU_CHECK(cudaEventElapsedTime(&ms[3], a->ev[0], a->ev[4]));
    return 0;
}

// device address of reference plane idx's origin pixel and the plane geometry, so that the owner of the
// reconstructed pixels (e.g. an NCCL broadcast) can write them in place; call x265cu_analyser_ref_updated()
// afterwards to re-extend the borders.
void* x265cu_analyser_ref_plane(x265cu_analyser* a, int idx, int* stride)
{
    if (idx < 0 || idx >= a->p.numRefs) return NULL;
    *stride = a->stride;
    return a->d_refs[idx] + a->orgBytes;
}
int x265cu_analyser_ref_updated(x265cu_analyser* a, int idx)
{
    if (idx < 0 || idx >= a->p.numRefs) return -1;
    cudaSetDevice(a->ctx->device);
    an_ref_changed(a, idx);
    return x265cu_extend_border(a->ctx, a->p.depth, a->d_refs[idx] + a->orgBytes, a->stride, a->p.width, a->p.height, AN_MARGIN_X, AN_MARGIN_Y);
}

// device address of the origin pixel of reconstruction plane `depthIdx` (0..3 = CU size 64, 32, 16, 8): what a row
// shard's owner broadcasts (the producer side of m_reconRowFlag, framefilter.cpp:664)
void* x265cu_analyser_recon_plane(x265cu_analyser* a, int depthIdx, int* stride)
{
    if (depthIdx < 0 || depthIdx >= 4) return NULL;
    *stride = a->stride;
    return a->d_recon[depthIdx] + a->orgBytes;
}
// promote the reconstructed CTU rows [ctuRow0, ctuRow1) of recon plane depthIdx to reference idx (device copy);
// call x265cu_analyser_ref_updated() once all rows of the new reference are in place
int x265cu_analyser_recon_to_ref(x265cu_analyser* a, int depthIdx, int idx, int ctuRow0, int ctuRow1)
{
    if (depthIdx < 0 || depthIdx >= 4 || idx < 0 || idx >= a->p.numRefs || ctuRow0 < 0 || ctuRow1 > a->ctuRows || ctuRow0 >= ctuRow1) return -1;
    const size_t es = a->p.depth == 8 ? 1 : 2;
    const int y0 = ctuRow0 * 64, y1 = ctuRow1 * 64 < a->p.height ? ctuRow1 * 64 : a->p.height;
    cudaSetDevice(a->ctx->device);
    const size_t off = a->orgBytes + (size_t)y0 * a->stride * es, pitch = (size_t)a->stride * es;
    an_ref_changed(a, idx);
    CU_CHECK(cudaMemcpy2DAsync(a->d_refs[idx] + off, pitch, a->d_recon[depthIdx] + off, pitch, (size_t)a->p.width * es, y1 - y0,
                               cudaMemcpyDeviceToDevice, a->ctx->stream));
    return 0;
}

// debugging / parity access to device-resident results
int x265cu_analyser_fetch(x265cu_analyser* a, int what, void* host)
{
    x265cu_ctx* c = a->ctx;
    const size_t es = a->p.depth == 8 ? 1 : 2;
    const void* src = NULL; size_t bytes = 0;
    cudaSetDevice(c->device);
    switch (what)
    {
    case 0: src = a->d_jobs; bytes = sizeof(x265cu_me_job) * a->njobs; break;
    case 1: src = a->d_me_out; bytes = sizeof(int32_t) * 4 * a->njobs; break;
    case 2: src = a->d_coef; bytes = sizeof(int16_t) * a->ncoef; break;
    case 3: case 4: case 5: case 6: src = a->d_recon[what - 3]; bytes = (size_t)a->stride * a->planeRows * es; break;
    case 7: src = a->d_cu_jobs; bytes = sizeof(int32_t) * a->ncu * a->p.numRefs; break;
    case 8: src = a->d_fenc; bytes = (size_t)a->stride * a->planeRows * es; break;
    default:
        // 16 + 16 * ref + phase: the whole allocation of phase plane yf * 4 + xf of what the search reads for reference `ref`
        // (phase 0 = the plane itself): its weighted block when it is weighted, else the reference's
        if (what < 16 || what >= 16 + 16 * a->p.numRefs) return -1;
        {
            const int r = (what - 16) >> 4;
            if (an_weights_prepare(a)) return -1;
            src = (an_ref_weighted(a, r) ? a->d_wrefs[r] : a->d_refs[r]) + (size_t)((what - 16) & 15) * a->planeBytes;
            bytes = (size_t)a->stride * a->planeRows * es;
        }
    }
    CU_CHECK(cudaMemcpyAsync(host, src, bytes, cudaMemcpyDeviceToHost, c->stream));
    CU_CHECK(cudaStreamSynchronize(c->stream));
    return 0;
}

// Weighted prediction of reference idx (list 0 of a P slice): w = m_weightPredTable[0][idx][0..2] (luma, Cb, Cr), NULL or
// w[0].wtPresent == 0 = unweighted.  Refused before any state change: a bad index or entry (x265cu_last_error).
int x265cu_analyser_set_ref_weights(x265cu_analyser* a, int idx, const x265cu_wp_entry* w)
{
    const char* bad = NULL;
    if (idx < 0 || idx >= a->p.numRefs) bad = "x265cu_analyser_set_ref_weights: reference index outside 0..numRefs - 1";
    for (int k = 0; k < 3 && w && !bad; k++)
    {
        if (w[k].wtPresent != 0 && w[k].wtPresent != 1) bad = "x265cu_analyser_set_ref_weights: wtPresent not 0 or 1";
        else if (w[k].log2WeightDenom < 0 || w[k].log2WeightDenom > 7) bad = "x265cu_analyser_set_ref_weights: log2WeightDenom outside 0..7";
        else if (w[k].inputWeight < -128 || w[k].inputWeight > 255) bad = "x265cu_analyser_set_ref_weights: inputWeight outside -128..255";
        else if (w[k].inputOffset < -128 || w[k].inputOffset > 127) bad = "x265cu_analyser_set_ref_weights: inputOffset outside -128..127";
    }
    if (bad) { x265cu_set_error(bad, cudaErrorInvalidValue, __FILE__, __LINE__); return -1; }
    const bool on = w && w[0].wtPresent, was = an_ref_weighted(a, idx);
    if (!on && !was) return 0;
    for (int k = 0; k < 3; k++) a->wp[idx][k] = on ? w[k] : x265cu_wp_entry{};
    a->nWeighted += (int)on - (int)was;
    a->wDirty[idx] = 1;
    return 0;
}

// Lists of a B slice: slots [0, numRefL0) list 0, [numRefL0, numRefs) list 1; numRefL1 == 0 a P slice.  Refused before
// any state change unless numRefL0 >= 1, numRefL1 >= 0 and numRefL0 + numRefL1 == numRefs.
int x265cu_analyser_set_lists(x265cu_analyser* a, int numRefL0, int numRefL1)
{
    if (numRefL0 < 1 || numRefL1 < 0 || numRefL0 + numRefL1 != a->p.numRefs)
    {
        x265cu_set_error("x265cu_analyser_set_lists: needs numRefL0 >= 1, numRefL1 >= 0 and numRefL0 + numRefL1 == numRefs", cudaErrorInvalidValue, __FILE__, __LINE__);
        return -1;
    }
    if (numRefL1 && !a->d_bidir)
    {
        cudaSetDevice(a->ctx->device);
        a->d_bidir = (x265cu_bidir_cu*)an_alloc_zeroed(a->ctx, sizeof(x265cu_bidir_cu) * a->ncu);
        if (!a->d_bidir)
        {
            x265cu_set_error("x265cu_analyser_set_lists: no device memory for the BIDIR records", cudaErrorMemoryAllocation, __FILE__, __LINE__);
            return -1;
        }
    }
    a->numRefL0 = numRefL0; a->numRefL1 = numRefL1;
    return 0;
}

// the BIDIR records of the CTU rows [r0, r1) into a full-frame sized host array (synchronous)
int x265cu_analyser_bidir_results(x265cu_analyser* a, int ctuRow0, int ctuRow1, x265cu_bidir_cu* out)
{
    if (!a->d_bidir || ctuRow0 < 0 || ctuRow1 > a->ctuRows || ctuRow0 > ctuRow1)
    {
        x265cu_set_error("x265cu_analyser_bidir_results: no B slice set, or a bad CTU row range", cudaErrorInvalidValue, __FILE__, __LINE__);
        return -1;
    }
    x265cu_ctx* c = a->ctx;
    cudaSetDevice(c->device);
    const size_t c0 = a->rowCu[ctuRow0], nc = a->rowCu[ctuRow1] - c0;
    if (nc) CU_CHECK(cudaMemcpyAsync(out + c0, a->d_bidir + c0, sizeof(x265cu_bidir_cu) * nc, cudaMemcpyDeviceToHost, c->stream));
    CU_CHECK(cudaStreamSynchronize(c->stream));
    return 0;
}

// the PART records of the CTU rows [r0, r1) into a full-frame sized host array (synchronous)
int x265cu_analyser_part_results(x265cu_analyser* a, int ctuRow0, int ctuRow1, x265cu_part_cu* out)
{
    if (!a->d_part || ctuRow0 < 0 || ctuRow1 > a->ctuRows || ctuRow0 > ctuRow1)
    {
        x265cu_set_error("x265cu_analyser_part_results: no run with stage bit 5 (PART) yet, or a bad CTU row range", cudaErrorInvalidValue, __FILE__, __LINE__);
        return -1;
    }
    x265cu_ctx* c = a->ctx;
    cudaSetDevice(c->device);
    const size_t c0 = a->rowCu[ctuRow0], nc = a->rowCu[ctuRow1] - c0;
    if (nc) CU_CHECK(cudaMemcpyAsync(out + c0, a->d_part + c0, sizeof(x265cu_part_cu) * nc, cudaMemcpyDeviceToHost, c->stream));
    CU_CHECK(cudaStreamSynchronize(c->stream));
    return 0;
}

// the PART_B records of the CTU rows [r0, r1) into a full-frame sized host array (synchronous)
int x265cu_analyser_part_b_results(x265cu_analyser* a, int ctuRow0, int ctuRow1, x265cu_part_b_cu* out)
{
    if (!a->d_partB || ctuRow0 < 0 || ctuRow1 > a->ctuRows || ctuRow0 > ctuRow1)
    {
        x265cu_set_error("x265cu_analyser_part_b_results: no run with stage bit 6 (PART_B) yet, or a bad CTU row range", cudaErrorInvalidValue, __FILE__, __LINE__);
        return -1;
    }
    x265cu_ctx* c = a->ctx;
    cudaSetDevice(c->device);
    const size_t c0 = a->rowCu[ctuRow0], nc = a->rowCu[ctuRow1] - c0;
    if (nc) CU_CHECK(cudaMemcpyAsync(out + c0, a->d_partB + c0, sizeof(x265cu_part_b_cu) * nc, cudaMemcpyDeviceToHost, c->stream));
    CU_CHECK(cudaStreamSynchronize(c->stream));
    return 0;
}

} // extern "C"
