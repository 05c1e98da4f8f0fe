// x265_b200/csrc/me_window.cuh -- integer motion search (phase 2 of the batched motionEstimate, STAR: motion.cpp:362-604,
// 1132-1240) on a SHARED-MEMORY SEARCH WINDOW.
//
// One CTA per job GROUP: the PUs of one CU (64x64 groups, 32x32 groups) or of one 16x16 cell (the 16x16 CU and its four 8x8 CUs)
// against ONE reference.  Their search windows [PU + mvmin, PU + mvmax + size) overlap almost completely, so the CTA
//   1. takes the union rectangle of the group's windows,
//   2. has ONE thread issue TMA tile loads (cp.async.bulk.tensor.2d, box = CLS x 16 rows, mbarrier complete_tx) of that
//      rectangle from the reference plane into shared memory -- row pitch = box width = 16 (mod 32) bytes, so successive rows
//      start 4 banks apart -- while the other threads stage the group's source block,
//   3. lets its warps pull the group's PU jobs (largest first) and run the search entirely out of shared memory:
//      * star bursts: the same (candidate, 16-byte segment) lane mapping as the global-memory core (me_sad_multi_t), but a
//        burst of scattered candidates costs bank conflicts (2-4 wavefronts) instead of one L1 tag lookup per distinct
//        line (up to 32);
//      * raster refinement (60 % of all SADs): a lane owns one grid COLUMN (fixed x, candidates every 5 rows).  It walks down
//        the window once; every window row it loads (funnel-shifted to its byte phase once) is differenced against the
//        source row of EVERY candidate whose block covers that row -- ceil(h / 5) accumulators in a register ring -- and the
//        source rows come from shared memory as warp-wide broadcasts (all lanes are at the same row phase).  Per
//        (candidate, row, 16 bytes): one broadcast LDS.128 + four VABSDIFF4, the reference row is fetched once per
//        ceil(h / 5) candidates.  Costs, ties and the `mvcost(tmv << 3)` quirk of every 4th column are the reference's.
// Groups whose union window does not fit the shared-memory budget, or that are not STAR jobs, are appended to a leftover
// list that the global-memory kernel (k_me<P, 2, -1, false>) drains afterwards: same results, no CPU or library fallback.
#pragma once
#include "common.cuh"
#include "me.cuh"
#include <cuda.h>
#include <type_traits>

#define MEW_BOX_ROWS 16                    // rows per TMA tile
#define MEW_NCLS 5                         // box-width classes
#define MEW_HDR 256                        // bytes of CTA header (mbarrier, counters, window rectangle)
#define MEW_MAX_GROUP 48                   // jobs per group (cell with AMP: 13 + 4 * 5 = 33)

// box widths in BYTES: 16 (mod 32), so that the row pitch skews successive rows by 4 banks
__host__ __device__ __forceinline__ int mew_cls_bytes(int es, int cls)
{
    // 8-bit: 144 176 208 240 256 (256 = the largest box, last resort)      16-bit: 304 336 400 464 512
    return es == 1 ? (cls == 4 ? 256 : 144 + 32 * cls) : (cls == 0 ? 304 : cls == 1 ? 336 : cls == 2 ? 400 : cls == 3 ? 464 : 512);
}

struct MeGroup { int32_t first, count; };  // jobs grp_jobs[first .. first + count), largest PU first

template <typename P>
struct MeWin
{
    uint32_t win; int pitch;               // shared address of the window origin, row pitch in bytes
    int ox, oy;                            // PU origin relative to the window origin (pixels)
    uint32_t fenc; int fpitch;             // shared address of the PU's source block, its row pitch in bytes
    const uint16_t* mvc; int mvpx, mvpy;
    int minx, miny, maxx, maxy;            // full-pel bounds
    int w, h, lane;
    bool pow2; int nw, lgnw, lgwpr, lgsegw;
    const struct MewCell* cell;            // shared 4x4 SAD maps of the 16x16 cell (NULL: this job walks its own raster)
    bool star;                             // this job starts at the cell's common start point: first star round out of the star table
    // only in-range starts: k_me_window hands the others to the global-memory kernel
    static constexpr bool startsOutside = false;
    static constexpr bool hasStarTable = false;
};

// The context of the 16x16-cell kernel: same fields, its own me_raster overload and the star table, so that each kernel
// instantiation carries only the code it can execute (the kernels are instruction-cache bound: the CU 32 / CU 64 kernel has
// no map / star-table code, the cell kernel none of the wide column-walk variants).
template <typename P> struct MeWinCell : MeWin<P> { static constexpr bool hasStarTable = true; };

// 16x16 cell groups: all PUs of the cell (16x16 CU + four 8x8 CUs) that share one raster grid (same mvmin / mvmax: the
// predictor field is 16x16-granular, so inside the picture they all do) get their raster costs from ONE set of SAD maps:
// the SAD of each of the cell's sixteen 4x4 blocks at every grid point, computed once by whichever warps need it
// (tasks = (block row, grid row), lanes = grid columns) and summed per PU (a PU's SAD at a vector is the sum of its 4x4
// blocks' SADs at that vector: exact).  A 16x16 PU then costs 16 loads per grid point instead of 256 pixel differences.
#define MEW_MAP_ROWS 23                    // grid rows (merange 57: (2 * 57) / 5 + 1)
#define MEW_STAR_POINTS 60                 // first star round: levels 0-3 (4 + 3 * 8) and levels 4, 5 (distances 16, 32: 2 * 16)
#define MEW_STAR_BYTES (MEW_STAR_POINTS * 4 * 8)
#define MEW_MAP_BYTES (16 * MEW_MAP_ROWS * 32 * 2 + 2048)          // raster maps + star table
struct MewCell
{
    int on;                                // maps usable for this group
    int minx, miny, maxx, maxy;            // the shared grid (full-pel bounds of the group's first job)
    int ncols, nrows;
    int ox, oy;                            // cell origin relative to the window origin (pixels)
    uint32_t fenc;                         // shared address of the cell's source block (pitch 64 pixels)
    uint32_t map;                          // shared address of the maps: [block row 4][MEW_MAP_ROWS][32] x (4 x u16 prefix sums)
    int next, done;                        // task queue of the map computation
    // first star round shared by the PUs that start at the same point (the pre-checks leave most of a cell's PUs at the
    // rounded MVP): per candidate of StarPatternSearch's levels 0-5 the same 4 x (4 x u16 prefix sums) as the raster maps
    int starOn, sx, sy;                    // table valid; the common start point (full-pel, relative like minx)
    uint32_t star;                         // shared address: [MEW_STAR_POINTS][block row 4] x 8 bytes
    uint32_t zero;                         // shared address of a zero word
    int zeroWord;
};

__device__ __forceinline__ uint32_t lds32(uint32_t a) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ uint2 lds64(uint32_t a) { uint2 v; asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(a)); return v; }
__device__ __forceinline__ uint32_t lds16(uint32_t a) { uint32_t v; asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ void sts16(uint32_t a, uint32_t v) { asm volatile("st.shared.u16 [%0], %1;" :: "r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ void sts64(uint32_t a, uint2 v) { asm volatile("st.shared.v2.u32 [%0], {%1, %2};" :: "r"(a), "r"(v.x), "r"(v.y) : "memory"); }
__device__ __forceinline__ uint4 lds128(uint32_t a) { uint4 v; asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a)); return v; }

// SEGW words of a window row starting at a byte address of any phase: SEGW + 1 aligned LDS.32 + SEGW funnel shifts.
// (The global-memory core reads 8-byte aligned LDG.64 pairs and selects: fewer load instructions matter on the L1 path.  Out
// of shared memory the ALU pipe is the limiter, and a warp-wide LDS.32 is one conflict-free wavefront where an LDS.64 is
// two, so five LDS.32 + four SHF beat three LDS.64 + five SEL + four SHF.)  `a4` = the address rounded down to 4 bytes,
// `sh` = 8 * (address & 3).
template <int SEGW>
__device__ __forceinline__ void mew_load_ref(uint32_t a4, unsigned sh, uint32_t (&r)[SEGW])
{
    uint32_t w[SEGW + 1];
#pragma unroll
    for (int k = 0; k <= SEGW; k++) w[k] = lds32(a4 + 4 * k);
#pragma unroll
    for (int k = 0; k < SEGW; k++) r[k] = __funnelshift_r(w[k], w[k + 1], sh);
}

template <int SEGW>
__device__ __forceinline__ void mew_load_fenc(uint32_t a, uint32_t (&f)[SEGW])
{
    if (SEGW == 4) { const uint4 t = lds128(a); f[0] = t.x; f[1 % SEGW] = t.y; f[2 % SEGW] = t.z; f[3 % SEGW] = t.w; }
    else if (SEGW == 2) { const uint2 t = lds64(a); f[0] = t.x; f[1 % SEGW] = t.y; }
    else f[0] = lds32(a);
}

// ---- full-pel SAD of up to 32 candidates at once out of the window (pow2 PUs): the lane mapping of me_sad_multi_t ----
// `offB` = byte offset of lane i's candidate block from the window origin (lanes >= n ignored).  Result in lane i < n.
template <typename P, int LGSEGW>
__device__ __forceinline__ int mew_sad_multi_t(const MeWin<P>& c, int n, int offB)
{
    constexpr int SEGW = 1 << LGSEGW;
    const int lane = c.lane;
    const int lgn = n <= 1 ? 0 : 32 - __clz(n - 1);
    const int lgnseg = c.lgnw - LGSEGW, lgspr = c.lgwpr - LGSEGW;          // log2 segments per PU / per row
    const int lglpc = min(5 - lgn, lgnseg);
    const int lgcols = min(lglpc, lgspr), lgrows = lglpc - lgcols;         // lanes of a candidate: 2^lgcols across, 2^lgrows down
    const int sub = lane & ((1 << lglpc) - 1);
    const int ob = __shfl_sync(0xffffffffu, offB, min(lane >> lglpc, n - 1));
    const uint32_t cptr = c.win + (uint32_t)ob;                            // my candidate's block origin; any byte phase
    const unsigned sh = (cptr & 3u) * 8u;
    const int subcol = sub & ((1 << lgcols) - 1), subrow = sub >> lgcols;
    uint32_t rrow = (cptr & ~3u) + subrow * c.pitch + subcol * (SEGW * 4);
    uint32_t frow = c.fenc + subrow * c.fpitch + subcol * (SEGW * 4);
    const int rowStepR = c.pitch << lgrows, rowStepF = c.fpitch << lgrows, colStep = (SEGW * 4) << lgcols;
    const int nrows = c.h >> lgrows, ncols = 1 << (lgspr - lgcols);
    int acc = 0;
    for (int jc = 0; jc < ncols; jc++, rrow += colStep, frow += colStep)
    {
        uint32_t rp = rrow, fp = frow;
#pragma unroll 2
        for (int i = 0; i < nrows; i++, rp += rowStepR, fp += rowStepF)
        {
            uint32_t f[SEGW], r[SEGW];
            mew_load_fenc<SEGW>(fp, f);
            mew_load_ref<SEGW>(rp, sh, r);
            acc = sad_words<P, SEGW>(f, r, acc);
        }
    }
    for (int o = 1; o < (1 << lglpc); o <<= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    return __shfl_sync(0xffffffffu, acc, (lane << lglpc) & 31);
}

// SAD of the source block against ONE window position (byte offset from the window origin), generic word walk: the AMP
// sizes (12 / 24 / 48 wide or high).  All lanes get it.
template <typename P>
__device__ __forceinline__ int mew_sad_generic(const MeWin<P>& c, int offB)
{
    const uint32_t cptr = c.win + (uint32_t)offB;
    const unsigned sh = (cptr & 3u) * 8u;
    const uint32_t c4 = cptr & ~3u;
    const int wprg = (c.w * (int)sizeof(P)) >> 2, nwg = wprg * c.h;
    int acc = 0;
    for (int wd = c.lane; wd < nwg; wd += 32)
    {
        const int row = wd / wprg, col = wd - row * wprg;
        const uint32_t a = c4 + row * c.pitch + col * 4;
        acc = sad_word<P>(lds32(c.fenc + row * c.fpitch + col * 4), __funnelshift_r(lds32(a), lds32(a + 4), sh), acc);
    }
    return warp_sum(acc);
}

// Full-pel SAD + mvcost of up to 32 candidate positions at once (the window counterpart of me_eval_points(MeCtx)).
template <typename P>
__device__ __forceinline__ int me_eval_points(const MeWin<P>& c, int n, int px, int py, bool x8)
{
    const int offB = (c.oy + py) * c.pitch + (c.ox + px) * (int)sizeof(P);
    int mysad = 0;
    if (c.pow2)
    {
        if (c.lgsegw == 2)      mysad = mew_sad_multi_t<P, 2>(c, n, offB);
        else if (c.lgsegw == 1) mysad = mew_sad_multi_t<P, 1>(c, n, offB);
        else                    mysad = mew_sad_multi_t<P, 0>(c, n, offB);
    }
    else
    {
        for (int p = 0; p < n; p++)
        {
            const int v = mew_sad_generic(c, __shfl_sync(0xffffffffu, offB, p));
            if (c.lane == p) mysad = v;
        }
    }
    int cost = 0x7fffffff;
    if (c.lane < n) cost = mysad + (x8 ? me_mvcost(c, px * 8, py * 8) : me_mvcost(c, px * 4, py * 4));
    return cost;
}
// ---- raster refinement out of the window (motion.cpp:1171-1201) ---------------------------------------------------
// Grid of step 5 over [minx, maxx] x [miny, maxy] in raster order; the reference's sequential `cost < bcost` chain = the
// minimum with ties to the lowest raster index.  Each lane brings its best (cost, raster index); the grid's winner is the
// warp's minimum cost, then the lowest index among the lanes that reach it.
__device__ __forceinline__ void mew_grid_fold(int best, int bestIdx, int ncols, int minx, int miny, MeStar& s)
{
    const int m = __reduce_min_sync(0xffffffffu, best);
    const int mi = __reduce_min_sync(0xffffffffu, best == m ? bestIdx : 0x7fffffff);
    if (m < s.bcost)
    {
        s.bcost = m;
        const int rj = mi / ncols, ri = mi - rj * ncols;
        s.bx = minx + ri * 5; s.by = miny + rj * 5;
    }
}

// Column walk: lane = grid column; NA = accumulators = ceil(h / 5) (template: 2/4/7/13).  Row policy:
//   NSEG = 0: the row in SEGW-word segments, each loaded once and differenced against every live ring slot whose source row
//             exists (a test per slot and segment);
//   NSEG = 1, 2, 4: PUs whose rows are NSEG aligned 16-byte segments (LGSEGW = 2): the lane's whole reference row is loaded
//             once into registers, then every live candidate (one bound per row) differences its source row against it,
//             NSEG x (broadcast LDS.128 + 4 VABSDIFF4) with no per-segment conditions.
template <typename P, int NA, int LGSEGW, int NSEG>
__device__ __forceinline__ void mew_raster_t(const MeWin<P>& c, MeStar& s)
{
    constexpr int SEGW = 1 << LGSEGW, SEGB = 4 * SEGW, RD = 5;
    const int ncols = (c.maxx - c.minx) / RD + 1, nrows = (c.maxy - c.miny) / RD + 1;
    const int nseg = (c.w * (int)sizeof(P)) / SEGB;
    const int lastRow = (nrows - 1) * RD + c.h - 1;
    const int nblk = nrows + NA - 1;
    int best = 0x7fffffff, bestIdx = 0x7fffffff;
    for (int cbase = 0; cbase < ncols; cbase += 32)
    {
        const int ri = cbase + c.lane;
        const bool act = ri < ncols;
        const int cx = c.minx + (act ? ri : 0) * RD;                 // idle lanes walk column 0 (inside the window), results ignored
        const bool x8 = (ri & 3) == 3;
        const int xc = (int)__ldg(c.mvc + ((x8 ? cx * 8 : cx * 4) - c.mvpx));
        const uint32_t a0 = c.win + (uint32_t)((c.oy + c.miny) * c.pitch + (c.ox + cx) * (int)sizeof(P));
        const unsigned sh = (a0 & 3u) * 8u;
        uint32_t rowaddr = a0 & ~3u;                                 // the pitch is a multiple of 16: the phase never changes
        int acc[NA];
#pragma unroll
        for (int i = 0; i < NA; i++) acc[i] = 0;
        for (int b = 0; b < nblk; b++)
        {
            const int lo = max(0, b - nrows + 1), hi = min(b, NA - 1);     // live ring slots: candidate k = b - i in [0, nrows)
#pragma unroll 1
            for (int t = 0; t < RD; t++, rowaddr += c.pitch)              // a loop, not unrolled: only the ring index i must be static
            {
                if (b * RD + t > lastRow) continue;                        // warp-uniform
                const uint32_t fa = c.fenc + t * c.fpitch;
                if constexpr (NSEG > 0)
                {
                    uint32_t r[4 * NSEG];
                    mew_load_ref<4 * NSEG>(rowaddr, sh, r);
                    // slot i is live iff lo <= i <= hi and its source row 5 i + t exists
                    const int ihi = c.h - 1 - t >= 0 ? min(hi, (c.h - 1 - t) / RD) : -1;
#pragma unroll
                    for (int i = 0; i < NA; i++)
                    {
                        if (i >= lo && i <= ihi)                           // warp-uniform
                        {
#pragma unroll
                            for (int sg = 0; sg < NSEG; sg++)
                            {
                                uint32_t f[4];
                                mew_load_fenc<4>(fa + (RD * i) * c.fpitch + sg * 16, f);     // same address in every lane: broadcast
                                const uint32_t rw[4] = { r[4 * sg], r[4 * sg + 1], r[4 * sg + 2], r[4 * sg + 3] };
                                acc[i] = sad_words<P, 4>(f, rw, acc[i]);
                            }
                        }
                    }
                }
                else
                {
                    for (int sg = 0; sg < nseg; sg++)
                    {
                        uint32_t r[SEGW];
                        mew_load_ref<SEGW>(rowaddr + sg * SEGB, sh, r);
#pragma unroll
                        for (int i = 0; i < NA; i++)
                        {
                            if (i >= lo && i <= hi && RD * i + t < c.h)    // warp-uniform
                            {
                                uint32_t f[SEGW];
                                mew_load_fenc<SEGW>(fa + sg * SEGB + (RD * i) * c.fpitch, f);    // same address in every lane: broadcast
                                acc[i] = sad_words<P, SEGW>(f, r, acc[i]);
                            }
                        }
                    }
                }
            }
            const int k = b - (NA - 1);                                    // the candidate in the last ring slot is complete
            if (k >= 0)
            {
                const int py = c.miny + k * RD;
                const int cost = acc[NA - 1] + (int)(uint16_t)(xc + (int)__ldg(c.mvc + ((x8 ? py * 8 : py * 4) - c.mvpy)));
                const int idx = k * ncols + ri;
                if (act && (cost < best || (cost == best && idx < bestIdx))) { best = cost; bestIdx = idx; }
            }
#pragma unroll
            for (int i = NA - 1; i > 0; i--) acc[i] = acc[i - 1];
            acc[0] = 0;
        }
    }
    mew_grid_fold(best, bestIdx, ncols, c.minx, c.miny, s);
}

template <typename P, int LGSEGW, int NSEG>
__device__ __forceinline__ void mew_raster_na(const MeWin<P>& c, MeStar& s)
{
    if (c.h <= 10)      mew_raster_t<P, 2, LGSEGW, NSEG>(c, s);
    else if (c.h <= 20) mew_raster_t<P, 4, LGSEGW, NSEG>(c, s);
    else if (c.h <= 35) mew_raster_t<P, 7, LGSEGW, NSEG>(c, s);
    else                mew_raster_t<P, 13, LGSEGW, NSEG>(c, s);
}

// One entry of the cell maps and of the star table: the SADs S[bx] of the four 4x4 blocks of a 16-pixel span over four rows
// (window rows from `a4` at byte phase `sh`, row pitch `pitch`; source rows from `fa`, pitch 64 pixels), stored as the 4
// prefix sums over the block columns, P[bx] = S[0] + .. + S[bx], as 4 x u16 in one 8-byte word (4 blocks of 16 ten-bit
// pixels: <= 65472), so that a PU's block-row sum is P[last] - P[first - 1].
template <typename P>
__device__ __forceinline__ uint2 mew_block_row_prefix(uint32_t a4, unsigned sh, int pitch, uint32_t fa)
{
    constexpr int ES = (int)sizeof(P), WB = ES;                    // words per 4-pixel block row
    int acc[4] = { 0, 0, 0, 0 };
#pragma unroll
    for (int r = 0; r < 4; r++)
    {
#pragma unroll
        for (int hw = 0; hw < WB; hw++)                            // 16 bytes of the row per step: 4 (8-bit) / 2 (16-bit) blocks
        {
            uint32_t rr[4], ff[4];
            mew_load_ref<4>(a4 + r * pitch + hw * 16, sh, rr);
            mew_load_fenc<4>(fa + r * 64 * ES + hw * 16, ff);      // same address in every lane of a map task: broadcast
#pragma unroll
            for (int wd = 0; wd < 4; wd++)
            {
                const int bx = (hw * 4 + wd) / WB;                 // block column of this word
                acc[bx] = sad_word<P>(ff[wd], rr[wd], acc[bx]);
            }
        }
    }
    const uint32_t p0 = (uint32_t)acc[0], p1 = p0 + (uint32_t)acc[1], p2 = p1 + (uint32_t)acc[2], p3 = p2 + (uint32_t)acc[3];
    return make_uint2(p0 | (p1 << 16), p2 | (p3 << 16));
}

// One task of the cell maps: grid row k, every grid column (lane = column), the cell's 4 block rows one after the other.
// Stored per (block row, k, column).
template <typename P>
__device__ __forceinline__ void mew_cell_map_task(const MeWin<P>& c, const MewCell& cell, int k)
{
    constexpr int ES = (int)sizeof(P);
    const int col = c.lane;
    const bool act = col < cell.ncols;
    const int gx = cell.minx + (act ? col : 0) * 5, gy = cell.miny + k * 5;
    const uint32_t a0 = c.win + (uint32_t)((cell.oy + gy) * c.pitch + (cell.ox + gx) * ES);
    const unsigned sh = (a0 & 3u) * 8u;
    uint32_t a4 = a0 & ~3u;
    uint32_t fa = cell.fenc;
#pragma unroll 1
    for (int by = 0; by < 4; by++)
    {
        const uint2 v = mew_block_row_prefix<P>(a4, sh, c.pitch, fa);
        if (act) sts64(cell.map + (uint32_t)(((by * MEW_MAP_ROWS + k) * 32 + col) * 8), v);
        a4 += 4 * c.pitch; fa += 4 * 64 * ES;
    }
}

// Scan of one grid column (this lane) over the grid rows: cost(k) = sum of NBY block-row sums + mvcost; returns the minimum
// and its first row.  NBY (block rows of the PU: 1 / 2 / 4, 3 for the 12-row AMP parts) is a template so that the loads of a
// grid point are straight-line code.
template <int NBY>
__device__ __forceinline__ void mew_maps_scan(uint32_t base, int nrows, uint32_t eoff, unsigned esh, uint32_t soff, unsigned ssh, bool hasS, uint32_t zaddr,
                                              int xc, const uint16_t* __restrict__ yp, int ystep, int& best, int& bestRow)
{
    constexpr uint32_t BR = MEW_MAP_ROWS * 32 * 8;                  // bytes between block rows
    // a PU at the cell's left edge subtracts nothing: its "P[-1]" reads a zero word (one code path for both cases)
    uint32_t ae = base + eoff, as = hasS ? base + soff : zaddr;
    const uint32_t sk = hasS ? 32u * 8u : 0u, sb = hasS ? BR : 0u;
    for (int k = 0; k < nrows; k++, ae += 32 * 8, as += sk, yp += ystep)
    {
        int sad = 0;
#pragma unroll
        for (int by = 0; by < NBY; by++)
            sad += (int)((lds32(ae + by * BR) >> esh) & 0xffffu) - (int)((lds32(as + by * sb) >> ssh) & 0xffffu);
        const int cost = sad + (int)(uint16_t)(xc + (int)__ldg(yp));
        if (cost < best) { best = cost; bestRow = k; }              // k ascending: strict '<' keeps the earliest
    }
}

// Raster refinement of one PU out of the cell maps (same result as mew_raster_t: minimum cost, ties to the lowest raster index).
template <typename P>
__device__ __forceinline__ void mew_raster_maps(const MeWin<P>& c, MeStar& s)
{
    MewCell* cell = const_cast<MewCell*>(c.cell);
    const int ntasks = cell->nrows;
    // every warp that needs the maps helps to build them, then waits until all tasks are done
    for (;;)
    {
        int t = 0;
        if (c.lane == 0) t = atomicAdd(&cell->next, 1);
        t = __shfl_sync(0xffffffffu, t, 0);
        if (t >= ntasks) break;
        mew_cell_map_task<P>(c, *cell, t);
        __syncwarp();
        if (c.lane == 0) { __threadfence_block(); atomicAdd(&cell->done, 1); }
    }
    if (c.lane == 0) { while (*(volatile int*)&cell->done < ntasks) __nanosleep(40); }
    __syncwarp();
    __threadfence_block();
    const int ncols = cell->ncols, nrows = cell->nrows;
    const int col = c.lane;
    const bool act = col < ncols;
    const int gx = c.minx + (act ? col : 0) * 5;
    const bool x8 = (col & 3) == 3;
    const int xc = (int)__ldg(c.mvc + ((x8 ? gx * 8 : gx * 4) - c.mvpx));
    const int bx0 = (c.ox - cell->ox) >> 2, by0 = (c.oy - cell->oy) >> 2, nbx = c.w >> 2, nby = c.h >> 2;
    // block-row sum = P[e] - P[bx0 - 1] (nothing to subtract when the PU starts at the cell's left edge); each prefix is the
    // 16-bit half `sh` of the 32-bit word `off` of the entry
    const int e = bx0 + nbx - 1, sx = bx0 - 1;
    const uint32_t eoff = (uint32_t)(e >> 1) * 4u, soff = (uint32_t)(max(sx, 0) >> 1) * 4u;
    const unsigned esh = (unsigned)(e & 1) * 16u, ssh = sx >= 0 ? (unsigned)(sx & 1) * 16u : 0u;
    const uint32_t base = cell->map + (uint32_t)((by0 * MEW_MAP_ROWS * 32 + col) * 8);
    const int ymul = x8 ? 8 : 4;
    const uint16_t* yp = c.mvc - c.mvpy + c.miny * ymul;                 // the vertical mvcost term of grid row k: yp[k * 5 * ymul]
    const int ystep = 5 * ymul;
    int best = 0x7fffffff, bestRow = 0;
    if (nby == 4)      mew_maps_scan<4>(base, nrows, eoff, esh, soff, ssh, sx >= 0, cell->zero, xc, yp, ystep, best, bestRow);
    else if (nby == 2) mew_maps_scan<2>(base, nrows, eoff, esh, soff, ssh, sx >= 0, cell->zero, xc, yp, ystep, best, bestRow);
    else if (nby == 1) mew_maps_scan<1>(base, nrows, eoff, esh, soff, ssh, sx >= 0, cell->zero, xc, yp, ystep, best, bestRow);
    else               mew_maps_scan<3>(base, nrows, eoff, esh, soff, ssh, sx >= 0, cell->zero, xc, yp, ystep, best, bestRow);   // AMP: 12 rows
    if (!act) best = 0x7fffffff;
    mew_grid_fold(best, bestRow * ncols + col, ncols, c.minx, c.miny, s);
}

template <typename P>
__device__ __forceinline__ void me_raster(const MeWin<P>& c, MeStar& s)
{
    // CU 32 / CU 64 groups.  pow2 PUs use the widest aligned segment; AMP widths (12 / 24 / 48) walk 4-byte words
    const int rowB = c.w * (int)sizeof(P);
    if (c.pow2 && c.lgsegw == 2 && rowB == 64)      mew_raster_na<P, 2, 4>(c, s);
    else if (c.pow2 && c.lgsegw == 2 && rowB == 32) mew_raster_na<P, 2, 2>(c, s);
    else if (c.pow2 && c.lgsegw == 2 && rowB == 16) mew_raster_na<P, 2, 1>(c, s);
    else if (c.pow2 && c.lgsegw == 2) mew_raster_na<P, 2, 0>(c, s);
    else if (c.pow2 && c.lgsegw == 1) mew_raster_na<P, 1, 0>(c, s);
    else                              mew_raster_na<P, 0, 0>(c, s);
}
template <typename P>
__device__ __forceinline__ void me_raster(const MeWinCell<P>& c, MeStar& s)
{
    // 16x16 cells: costs out of the shared SAD maps; a PU whose grid differs from the cell's (picture edges) walks its own
    // raster with the generic 4-byte-word variant
    if (c.cell) mew_raster_maps<P>(c, s);
    else        mew_raster_na<P, 0, 0>(c, s);
}

// First star round out of the cell's star table (me.cuh: me_star_pattern): candidate k of level `mylvl` around the common start.
template <typename P>
__device__ __forceinline__ int me_star_lookup(const MeWinCell<P>& c, int mylvl, int k, int px, int py)
{
    const MewCell* cell = c.cell;
    const int idx = mylvl == 0 ? k : mylvl < 4 ? 4 + (mylvl - 1) * 8 + (k & 7) : 28 + (mylvl - 4) * 16 + (k & 15);
    const int bx0 = (c.ox - cell->ox) >> 2, by0 = (c.oy - cell->oy) >> 2, nbx = c.w >> 2, nby = c.h >> 2;
    const int e = bx0 + nbx - 1, sx = bx0 - 1;
    uint32_t a = cell->star + (uint32_t)((idx * 4 + by0) * 8);
    int sad = 0;
    for (int by = 0; by < nby; by++, a += 8)
    {
        const uint2 v = lds64(a);
        sad += (int)(((e >= 2 ? v.y : v.x) >> ((e & 1) * 16)) & 0xffffu);
        if (sx >= 0) sad -= (int)(((sx >= 2 ? v.y : v.x) >> ((sx & 1) * 16)) & 0xffffu);
    }
    return sad + me_mvcost(c, px * 4, py * 4);
}

// Star table of a cell: thread = (candidate, block row); 4 rows of the cell against the window at the candidate's vector.
template <typename P>
__device__ __forceinline__ void mew_cell_star_build(const MewCell& cell, uint32_t win, int pitch, int tid)
{
    constexpr int ES = (int)sizeof(P);
    const int idx = tid >> 2, by = tid & 3;
    if (idx >= MEW_STAR_POINTS) return;
    const int mylvl = idx < 4 ? 0 : idx < 28 ? 1 + ((idx - 4) >> 3) : 4 + ((idx - 28) >> 4);
    const int k = idx < 4 ? idx : idx < 28 ? (idx - 4) & 7 : (idx - 28) & 15;
    int px, py, point, dist;
    me_star_point(mylvl, k, cell.sx, cell.sy, px, py, point, dist);
    if (px < cell.minx || px > cell.maxx || py < cell.miny || py > cell.maxy) return;        // never looked up (out of the search range)
    const uint32_t a0 = win + (uint32_t)((cell.oy + py + 4 * by) * pitch + (cell.ox + px) * ES);
    const uint32_t fa = cell.fenc + (uint32_t)(4 * by * 64 * ES);
    sts64(cell.star + (uint32_t)((idx * 4 + by) * 8), mew_block_row_prefix<P>(a0 & ~3u, (a0 & 3u) * 8u, pitch, fa));
}

// ---- mbarrier / TMA (PTX) -----------------------------------------------------------------------------------------
__device__ __forceinline__ void mew_mbar_init(uint32_t bar, int count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(bar), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mew_mbar_expect_tx(uint32_t bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mew_mbar_wait(uint32_t bar, uint32_t parity)
{
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "MEW_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra MEW_DONE;\n"
        "bra MEW_WAIT;\n"
        "MEW_DONE:\n"
        "}\n" :: "r"(bar), "r"(parity) : "memory");
}
// one TMA tile: box (tensor-map box width x MEW_BOX_ROWS rows) at element coordinates (x, y) of the plane allocation
__device__ __forceinline__ void mew_tma_load_2d(uint32_t dst, const CUtensorMap* tmap, int x, int y, uint32_t bar)
{
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 :: "r"(dst), "l"((uint64_t)tmap), "r"(bar), "r"(x), "r"(y) : "memory");
}

struct MeWinArgs
{
    const CUtensorMap* tmaps;              // [ref][MEW_NCLS] tensor maps over the reference plane ALLOCATIONS (device memory)
    int allocX, allocY;                    // position of the picture origin inside the allocation (margins), pixels
    int smemBytes;                         // dynamic shared memory of the launch (header + source block + window)
    int fencBytes;                         // bytes reserved for the source block (64 x 64 x es for L groups, 16 x 16 x es for cells)
};

// Group header in shared memory
struct MewHdr
{
    unsigned long long mbar;
    int next;                              // job queue of the CTA
    int ok;                                // window fits
    int wx0, wy0, pitch, ntiles, cls;      // window origin (picture coordinates, pixels), pitch in bytes
    int fx0, fy0, fw, fh;                  // source-block bounding box (picture coordinates, pixels)
    int ref;
    MewCell cell;                          // shared SAD maps of a 16x16 cell group (CELL launches)
};

template <typename P, bool CELL>
__global__ void __launch_bounds__(256, 3) k_me_window(const P* __restrict__ fenc, int fstride, MeWinArgs wa,
                                                      const uint16_t* __restrict__ mvcost, const x265cu_me_job* __restrict__ jobs,
                                                      const MeGroup* __restrict__ groups, const int32_t* __restrict__ grp_jobs, int job0,
                                                      MeState* __restrict__ state, int* __restrict__ left_count, int32_t* __restrict__ left_list)
{
    extern __shared__ __align__(128) unsigned char mew_smem[];
    constexpr int ES = (int)sizeof(P);
    MewHdr* hdr = (MewHdr*)mew_smem;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const MeGroup g = groups[blockIdx.x];
    const uint32_t sbase = (uint32_t)__cvta_generic_to_shared(mew_smem);
    const uint32_t s_fenc = sbase + MEW_HDR, s_win = sbase + MEW_HDR + wa.fencBytes;
    const uint32_t s_map = sbase + (uint32_t)(wa.smemBytes - MEW_MAP_BYTES);      // CELL launches: the maps sit at the end

    // ---- 1. union rectangle of the group's search windows and of its source blocks (warp 0) ----
    if (warp == 0)
    {
        int x0 = 0x7fffffff, y0 = 0x7fffffff, x1 = -0x7fffffff, y1 = -0x7fffffff;
        int fx0 = 0x7fffffff, fy0 = 0x7fffffff, fx1 = -0x7fffffff, fy1 = -0x7fffffff;
        int bad = 0, ref = 0;
        int g0minx = 0, g0miny = 0, g0maxx = 0, g0maxy = 0;
        for (int i = lane; i < g.count; i += 32)
        {
            const int jid = grp_jobs[g.first + i] - job0;
            const x265cu_me_job j = jobs[jid];
            const MeState st = state[jid];
            if (i == 0) { g0minx = j.mvmin[0]; g0miny = j.mvmin[1]; g0maxx = j.mvmax[0]; g0maxy = j.mvmax[1]; }
            const int py = j.offset / fstride, px = j.offset - py * fstride;
            x0 = min(x0, px + j.mvmin[0]); x1 = max(x1, px + j.mvmax[0] + j.pw);
            y0 = min(y0, py + j.mvmin[1]); y1 = max(y1, py + j.mvmax[1] + j.ph);
            fx0 = min(fx0, px); fx1 = max(fx1, px + j.pw); fy0 = min(fy0, py); fy1 = max(fy1, py + j.ph);
            bad |= (j.method != 3) | (j.mvmax[0] < j.mvmin[0]) | (j.mvmax[1] < j.mvmin[1]);
            // a star that starts outside its range (MV 0 won the pre-checks) evaluates points outside it, which the window
            // does not stage: the group goes to the global-memory kernel
            bad |= (st.bmx < j.mvmin[0]) | (st.bmx > j.mvmax[0]) | (st.bmy < j.mvmin[1]) | (st.bmy > j.mvmax[1]);
            ref = j.ref;
        }
        x0 = __reduce_min_sync(0xffffffffu, x0); y0 = __reduce_min_sync(0xffffffffu, y0);
        x1 = __reduce_max_sync(0xffffffffu, x1); y1 = __reduce_max_sync(0xffffffffu, y1);
        fx0 = __reduce_min_sync(0xffffffffu, fx0); fy0 = __reduce_min_sync(0xffffffffu, fy0);
        fx1 = __reduce_max_sync(0xffffffffu, fx1); fy1 = __reduce_max_sync(0xffffffffu, fy1);
        bad = __reduce_or_sync(0xffffffffu, (unsigned)bad);
        ref = __shfl_sync(0xffffffffu, ref, 0);
        if (lane == 0)
        {
            // window origin aligned down to 16 bytes (in allocation coordinates); 8 bytes of slack on the right for the
            // 8-byte aligned row loads
            const int ax0 = x0 + wa.allocX;
            const int ax0a = ax0 & ~(16 / ES - 1);
            const int needB = (x1 + wa.allocX - ax0a) * ES + 8;
            int cls = -1;
            for (int k = 0; k < MEW_NCLS; k++) if (cls < 0 && mew_cls_bytes(ES, k) >= needB) cls = k;
            const int rows = y1 - y0, ntiles = (rows + MEW_BOX_ROWS - 1) / MEW_BOX_ROWS;
            // source block: origin aligned down to 16 bytes, pitch = 64 pixels
            const int fx0a = fx0 & ~(16 / ES - 1);
            const int fwB = (fx1 - fx0a) * ES, fhh = fy1 - fy0;
            int ok = !bad && cls >= 0;
            if (ok)
            {
                const int pitch = mew_cls_bytes(ES, cls);
                ok = MEW_HDR + wa.fencBytes + pitch * ntiles * MEW_BOX_ROWS + (CELL ? MEW_MAP_BYTES : 0) <= wa.smemBytes && fwB <= 64 * ES && 64 * ES * fhh <= wa.fencBytes;
                hdr->pitch = pitch;
            }
            hdr->ok = ok; hdr->next = 0; hdr->cls = cls; hdr->ntiles = ntiles;
            hdr->wx0 = ax0a - wa.allocX; hdr->wy0 = y0;
            hdr->fx0 = fx0a; hdr->fy0 = fy0; hdr->fw = fwB; hdr->fh = fhh; hdr->ref = ref;
            // shared SAD maps: a complete 16x16 cell and a grid of at most 32 x MEW_MAP_ROWS points (lane 0 holds job 0's range)
            MewCell& cl = hdr->cell;
            cl.on = 0; cl.starOn = 0; cl.zeroWord = 0;
            cl.zero = sbase + (uint32_t)offsetof(MewHdr, cell) + (uint32_t)offsetof(MewCell, zeroWord);
            if (CELL && ok && fx1 - fx0 == 16 && fy1 - fy0 == 16 && fx0a == fx0)
            {
                const int ncols = (g0maxx - g0minx) / 5 + 1, nrows = (g0maxy - g0miny) / 5 + 1;
                if (ncols <= 32 && nrows <= MEW_MAP_ROWS)
                {
                    cl.on = 1; cl.minx = g0minx; cl.miny = g0miny; cl.maxx = g0maxx; cl.maxy = g0maxy; cl.ncols = ncols; cl.nrows = nrows;
                    cl.ox = fx0 - hdr->wx0; cl.oy = fy0 - y0; cl.fenc = s_fenc; cl.map = s_map; cl.next = 0; cl.done = 0;
                    // common start of the first star round: where the pre-checks left the group's first job (its state)
                    const MeState st0 = state[grp_jobs[g.first] - job0];
                    cl.star = s_map + (uint32_t)(16 * MEW_MAP_ROWS * 32 * 2);
                    cl.sx = st0.bmx; cl.sy = st0.bmy;
                    cl.starOn = st0.bmx >= g0minx && st0.bmx <= g0maxx && st0.bmy >= g0miny && st0.bmy <= g0maxy;
                }
            }
        }
    }
    __syncthreads();
    if (!hdr->ok)
    {   // the global-memory kernel takes these jobs
        if (tid < g.count)
        {
            const int slot = atomicAdd(left_count, 1);
            left_list[slot] = grp_jobs[g.first + tid] - job0;
        }
        for (int i = tid + blockDim.x; i < g.count; i += blockDim.x) left_list[atomicAdd(left_count, 1)] = grp_jobs[g.first + i] - job0;
        return;
    }
    const uint32_t bar = sbase + (uint32_t)offsetof(MewHdr, mbar);
    if (tid == 0) mew_mbar_init(bar, 1);
    __syncthreads();
    const int pitch = hdr->pitch, wx0 = hdr->wx0, wy0 = hdr->wy0;
    // ---- 2. one thread: TMA tile loads of the window; everybody: the source block ----
    if (tid == 0)
    {
        const int nt = hdr->ntiles;
        mew_mbar_expect_tx(bar, (uint32_t)(nt * MEW_BOX_ROWS * pitch));
        const CUtensorMap* tm = wa.tmaps + (size_t)hdr->ref * MEW_NCLS + hdr->cls;
        for (int t = 0; t < nt; t++)
            mew_tma_load_2d(s_win + t * MEW_BOX_ROWS * pitch, tm, wx0 + wa.allocX, wy0 + wa.allocY + t * MEW_BOX_ROWS, bar);
    }
    {
        const int fpitch = 64 * ES, fwB = hdr->fw, fhh = hdr->fh;
        const P* fsrc = fenc + (ptrdiff_t)hdr->fy0 * fstride + hdr->fx0;
        const int chunks = (fwB + 15) >> 4;
        for (int i = tid; i < chunks * fhh; i += blockDim.x)
        {
            const int row = i / chunks, ch = i - row * chunks;
            const uint4 v = __ldg((const uint4*)((const uint8_t*)(fsrc + (ptrdiff_t)row * fstride) + ch * 16));
            *(uint4*)(mew_smem + MEW_HDR + row * fpitch + ch * 16) = v;
        }
    }
    __syncthreads();
    mew_mbar_wait(bar, 0);
    if (CELL && hdr->cell.on && hdr->cell.starOn)
    {   // the first star round of the cell's PUs: one (candidate, block row) per thread, then everybody may look it up
        mew_cell_star_build<P>(hdr->cell, s_win, pitch, tid);
        __syncthreads();
    }

    // ---- 3. the group's jobs, largest first, one warp each ----
    for (;;)
    {
        int slot = 0;
        if (lane == 0) slot = atomicAdd(&hdr->next, 1);
        slot = __shfl_sync(0xffffffffu, slot, 0);
        if (slot >= g.count) break;
        const int jid = grp_jobs[g.first + slot] - job0;
        const x265cu_me_job j = jobs[jid];
        typename std::conditional<CELL, MeWinCell<P>, MeWin<P> >::type c;
        const int py = j.offset / fstride, px = j.offset - py * fstride;
        c.win = s_win; c.pitch = pitch; c.ox = px - wx0; c.oy = py - wy0;
        c.fpitch = 64 * ES; c.fenc = s_fenc + (py - hdr->fy0) * c.fpitch + (px - hdr->fx0) * ES;
        c.mvc = mvcost; c.mvpx = j.qmvp[0]; c.mvpy = j.qmvp[1];
        c.minx = j.mvmin[0]; c.miny = j.mvmin[1]; c.maxx = j.mvmax[0]; c.maxy = j.mvmax[1];
        c.w = j.pw; c.h = j.ph; c.lane = lane;
        me_set_shape<P>(c);                                        // the window's pitch is a multiple of 16 bytes
        c.cell = NULL;
        if (CELL && hdr->cell.on && c.minx == hdr->cell.minx && c.maxx == hdr->cell.maxx && c.miny == hdr->cell.miny && c.maxy == hdr->cell.maxy)
            c.cell = &hdr->cell;
        MeState st = state[jid];
        // merange < 64: the first round's far levels are distances 16 and 32 only (levels 4, 5), what the table holds
        c.star = c.cell != NULL && hdr->cell.starOn && j.merange < 64 && st.bmx == hdr->cell.sx && st.bmy == hdr->cell.sy;
        MeStar s; s.bx = st.bmx; s.by = st.bmy; s.bcost = st.bcost; s.point = 0; s.dist = 0;
        me_star_search(c, s, (int)j.merange);
        if (lane == 0) { st.bmx = s.bx; st.bmy = s.by; st.bcost = s.bcost; state[jid] = st; }
        __syncwarp();
    }
}

// ---- host side: tensor maps ------------------------------------------------------------------------------------------
typedef CUresult (*mew_encode_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// cuTensorMapEncodeTiled through the runtime's driver entry point (libx265cu.so does not link libcuda: it must load on a
// box without a driver for the ABI checks)
static mew_encode_fn mew_encoder()
{
    static mew_encode_fn fn = NULL;
    static bool tried = false;
    if (!tried)
    {
        tried = true;
        void* p = NULL;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = (mew_encode_fn)p;
        else cudaGetLastError();
    }
    return fn;
}

// MEW_NCLS tensor maps (one per box width) over a plane allocation of `stride` x `rows` pixels of `es` bytes
static int mew_build_tmaps(void* base, int stride, int rows, int es, CUtensorMap* out)
{
    mew_encode_fn enc = mew_encoder();
    if (!enc) { x265cu_set_error("cuTensorMapEncodeTiled unavailable", cudaErrorNotSupported, __FILE__, __LINE__); return -1; }
    for (int k = 0; k < MEW_NCLS; k++)
    {
        const cuuint64_t gdim[2] = { (cuuint64_t)stride, (cuuint64_t)rows };
        const cuuint64_t gstr[1] = { (cuuint64_t)stride * es };
        const cuuint32_t box[2] = { (cuuint32_t)(mew_cls_bytes(es, k) / es), MEW_BOX_ROWS };
        const cuuint32_t estr[2] = { 1, 1 };
        const CUresult r = enc(&out[k], es == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_UINT16, 2, base, gdim, gstr, box, estr,
                               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { x265cu_set_error("cuTensorMapEncodeTiled", cudaErrorInvalidValue, __FILE__, __LINE__); return -1; }
    }
    return 0;
}

// shared-memory budgets (bytes) of the three group classes: header + source block + window (+ SAD maps)
static inline int mew_smem_bytes(int es, int cls, int* fencBytes)
{
    if (cls == 0) { *fencBytes = 64 * 64 * es; return MEW_HDR + *fencBytes + (es == 1 ? 240 * 192 : 464 * 192); }    // CU 64 groups
    if (cls == 1) { *fencBytes = 32 * 64 * es; return MEW_HDR + *fencBytes + (es == 1 ? 208 * 160 : 400 * 160); }    // CU 32 groups
    *fencBytes = 16 * 64 * es;
    return MEW_HDR + *fencBytes + (es == 1 ? 208 * 160 : 336 * 144) + MEW_MAP_BYTES;                                  // 16x16 cells (+ SAD maps)
}

template <typename P>
static int launch_me_window(x265cu_ctx* ctx, const void* fenc, int fstride, const uint16_t* mvcost, const x265cu_me_job* jobs,
                            MeState* st, const MeWinLaunch& w)
{
    CU_CHECK(cudaMemsetAsync(w.left_count, 0, sizeof(int), ctx->stream));
    for (int cls = 0; cls < 3; cls++)
    {
        if (w.ngroups[cls] <= 0) continue;
        // one warp per PU of a CU group (5, or 13 with AMP); cells hold 25 (33) PUs that 8 warps pull from a queue
        const int threads = cls == 2 ? 256 : (w.amp ? 256 : 160);
        MeWinArgs a;
        a.tmaps = (const CUtensorMap*)w.tmaps; a.allocX = w.allocX; a.allocY = w.allocY;
        a.smemBytes = mew_smem_bytes((int)sizeof(P), cls, &a.fencBytes);
        const auto kernel = cls == 2 ? k_me_window<P, true> : k_me_window<P, false>;
        CU_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, a.smemBytes));
        kernel<<<w.ngroups[cls], threads, a.smemBytes, ctx->stream>>>((const P*)fenc, fstride, a, mvcost, jobs, (const MeGroup*)w.groups[cls],
                                                                      w.grp_jobs[cls], w.job0, st, w.left_count, w.left_list);
        CU_LAUNCH_CHECK(ctx);
    }
    return 0;
}

// ---- pre-checks of the 16x16 cell groups (phase 1, motion.cpp:771-814) -------------------------------------------------
// Every job of a cell takes its MVP and both candidates from the field block of the cell (k_build_me_jobs), so -- unless a
// picture-edge clamp of mvmin / mvmax moves a clip -- all of them evaluate the same positions: the clipped MVP, its full-pel
// rounding, MV 0 and the candidates.  A PU's SAD is the sum of its 4x4 blocks' SADs, and its chroma SATD is the sum of 4x4
// (chroma width 4) or 8x4 (width 8) tiles, an 8x4 tile being the two un-halved 4x4 Hadamard sums added and halved
// (pixel.cpp:239-297).  The interpolated prediction at a position does not depend on the block.  So one warp per cell
// evaluates each position ONCE over the whole 16x16 cell into a table of 4x4 quantities and folds every job from it, one
// lane per job, exactly as me_phase1 does.  A job whose clipped positions differ from the cell's first job goes to
// `left_list` for the per-PU kernels, and so do all jobs of the CU 64 / CU 32 groups (CELL == false launches).
struct MePreTab
{
    int16_t mid[(16 + 7) * 16];            // hps(rowExt) rows of an hv position (me_subpel_small_t's layout for a 16x16 PU)
    int lum[5][16];                        // luma 4x4 SADs: MVP, its full-pel rounding, MV 0, candidate 0, candidate 1
    int chr[3][8];                         // un-halved chroma 4x4 Hadamard sums [MVP, cand 0, cand 1][Cb tiles 0-3, Cr tiles 0-3]
};

template <typename P, bool CHROMA>
__global__ void __launch_bounds__(256) k_me_precheck_cell(const P* __restrict__ fenc, int fstride, const P* const* __restrict__ refs, int rstride,
                                                          MeChromaArgs ch, const uint16_t* __restrict__ mvcost, const x265cu_me_job* __restrict__ jobs,
                                                          const MeGroup* __restrict__ groups, int ngroups, const int32_t* __restrict__ grp_jobs, int job0,
                                                          int cell, MeState* __restrict__ state, int* __restrict__ left_count, int32_t* __restrict__ left_list)
{
    __shared__ __align__(16) MePreTab tabs[8];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int gi = blockIdx.x * 8 + warp;
    if (gi >= ngroups) return;
    const MeGroup g = groups[gi];
    if (!cell)
    {
        int base = 0;
        if (lane == 0) base = atomicAdd(left_count, g.count);
        base = __shfl_sync(0xffffffffu, base, 0);
        for (int i = lane; i < g.count; i += 32) left_list[base + i] = grp_jobs[g.first + i] - job0;
        return;
    }
    MePreTab& t = tabs[warp];

    // the cell's positions: those of its first job
    const x265cu_me_job j0 = jobs[grp_jobs[g.first] - job0];
    const int qminx = j0.mvmin[0] * 4, qminy = j0.mvmin[1] * 4, qmaxx = j0.mvmax[0] * 4, qmaxy = j0.mvmax[1] * 4;
    const int pmvx = max(min((int)j0.qmvp[0], qmaxx), qminx), pmvy = max(min((int)j0.qmvp[1], qmaxy), qminy);
    const int bmx = (pmvx + 2) >> 2, bmy = (pmvy + 2) >> 2;
    const int c0x = max(min((int)j0.mvc[0], qmaxx), qminx), c0y = max(min((int)j0.mvc[1], qmaxy), qminy);
    const int c1x = max(min((int)j0.mvc[2], qmaxx), qminx), c1y = max(min((int)j0.mvc[3], qmaxy), qminy);
    const int ncand = j0.numCand;
    const bool frac = ((pmvx & 3) | (pmvy & 3)) != 0, nonzero = (pmvx | pmvy) != 0;
    const bool v0 = ncand > 0 && (c0x | c0y) && !(c0x == pmvx && c0y == pmvy);
    const bool v1 = ncand > 1 && (c1x | c1y) && !(c1x == pmvx && c1y == pmvy);
    const int oy0 = j0.offset / fstride, ox0 = j0.offset - oy0 * fstride;
    const int cx = ox0 & ~15, cy = oy0 & ~15;
    const ptrdiff_t coff = (ptrdiff_t)cy * fstride + cx;
    const P* rb = refs[j0.ref] + coff;
    const P* fb = fenc + coff;

    // ---- luma: lane = (8-pixel segment, row) of the cell, as me_subpel_small_t maps a 16x16 PU ----
    const int row = lane & 15, seg = lane >> 4;
#pragma unroll 1
    for (int k = 0; k < 5; k++)
    {
        if ((k == 1 && !frac) || (k == 2 && !nonzero) || (k == 3 && !v0) || (k == 4 && !v1)) continue;
        const int qx = k == 0 ? pmvx : k == 1 ? bmx * 4 : k == 2 ? 0 : k == 3 ? c0x : c1x;
        const int qy = k == 0 ? pmvy : k == 1 ? bmy * 4 : k == 2 ? 0 : k == 3 ? c0y : c1y;
        const int xf = qx & 3, yf = qy & 3;
        const P* r = rb + (qx >> 2) + (ptrdiff_t)(qy >> 2) * rstride;
        if (xf && yf)
        {
            __syncwarp();
            for (int tk = lane; tk < (16 + 7) * 2; tk += 32)
            {
                const int mrow = tk >> 1, sg = tk & 1;
                me_hv_row<P, 8>(r + (ptrdiff_t)(mrow - 3) * rstride + sg * 8, xf, t.mid + mrow * 16 + sg * 8);
            }
            __syncwarp();
        }
        // full-pel rows as aligned words (me_ld_px): here they cost fewer instructions than me_pred_seg's scalar loads
        const P* rr = r + (ptrdiff_t)row * rstride + seg * 8;
        int pr[8];
        if (!(xf | yf)) me_ld_px<P, 8>(rr, pr);
        else me_pred_seg<P, 8, false>(rr, rstride, xf, yf, t.mid + row * 16 + seg * 8, 16, pr);
        int fv[8];
        me_ld_px<P, 8>(fb + (ptrdiff_t)row * fstride + seg * 8, fv);
        int sl = 0, sr = 0;
#pragma unroll
        for (int x = 0; x < 4; x++) { sl += abs(fv[x] - pr[x]); sr += abs(fv[x + 4] - pr[x + 4]); }
#pragma unroll
        for (int o = 1; o <= 2; o <<= 1) { sl += __shfl_xor_sync(0xffffffffu, sl, o); sr += __shfl_xor_sync(0xffffffffu, sr, o); }
        if ((row & 3) == 0) { t.lum[k][(row >> 2) * 4 + seg * 2] = sl; t.lum[k][(row >> 2) * 4 + seg * 2 + 1] = sr; }
    }
    // ---- chroma: lane = (position, plane, 4x4 tile) of the cell's 8x8 chroma block ----
    if (CHROMA && lane < 24)
    {
        const int k = lane >> 3, cr = (lane >> 2) & 1, tt = lane & 3;
        const int qx = k == 0 ? pmvx : k == 1 ? c0x : c1x, qy = k == 0 ? pmvy : k == 1 ? c0y : c1y;
        if (k == 0 || (k == 1 && v0) || (k == 2 && v1))
        {
            const ptrdiff_t o = (ptrdiff_t)(cy >> 1) * ch.cstride + (cx >> 1) + (ptrdiff_t)((tt >> 1) * 4) * ch.cstride + (tt & 1) * 4;
            const P* f = (const P*)(cr ? ch.fencCr : ch.fencCb) + o;
            const P* r = ((const P* const*)(cr ? ch.refCr : ch.refCb))[j0.ref] + o + (qx >> 3) + (ptrdiff_t)(qy >> 3) * ch.cstride;
            t.chr[k][cr * 4 + tt] = me_chroma_had4x4<P>(f, r, ch.cstride, qx & 7, qy & 7);
        }
    }
    __syncwarp();

    // ---- fold: one lane per job (a cell holds up to 33 jobs with AMP) ----
    for (int base = 0; base < g.count; base += 32)
    {
        const int slot = base + lane;
        const bool live = slot < g.count;
        const int jid = live ? grp_jobs[g.first + slot] - job0 : 0;
        const x265cu_me_job j = jobs[jid];
        const int jqminx = j.mvmin[0] * 4, jqminy = j.mvmin[1] * 4, jqmaxx = j.mvmax[0] * 4, jqmaxy = j.mvmax[1] * 4;
        const bool same = j.numCand == ncand && ncand <= 2 &&
                          max(min((int)j.qmvp[0], jqmaxx), jqminx) == pmvx && max(min((int)j.qmvp[1], jqmaxy), jqminy) == pmvy &&
                          (ncand < 1 || (max(min((int)j.mvc[0], jqmaxx), jqminx) == c0x && max(min((int)j.mvc[1], jqmaxy), jqminy) == c0y)) &&
                          (ncand < 2 || (max(min((int)j.mvc[2], jqmaxx), jqminx) == c1x && max(min((int)j.mvc[3], jqmaxy), jqminy) == c1y));
        const unsigned lost = __ballot_sync(0xffffffffu, live && !same);
        if (lost)
        {
            int lb = 0;
            if (lane == 0) lb = atomicAdd(left_count, __popc(lost));
            lb = __shfl_sync(0xffffffffu, lb, 0);
            if ((lost >> lane) & 1u) left_list[lb + __popc(lost & ((1u << lane) - 1u))] = jid;
        }
        if (!live || !same) continue;
        const int py = j.offset / fstride, px = j.offset - py * fstride;
        const int bx0 = (px - cx) >> 2, by0 = (py - cy) >> 2, bw = j.pw >> 2, bh = j.ph >> 2;
        int L[5];
#pragma unroll
        for (int k = 0; k < 5; k++)
        {
            int s = 0;
            for (int by = by0; by < by0 + bh; by++)
                for (int bx = bx0; bx < bx0 + bw; bx++) s += t.lum[k][by * 4 + bx];
            L[k] = s;
        }
        int C[3] = { 0, 0, 0 };
        if (CHROMA && j.subme > 2 && !(j.pw & 7) && !(j.ph & 7))
        {   // chroma block (w/2) x (h/2): 8x4 tiles when its width is 8, else 4x4 tiles; each tile halved on its own
            const int tx0 = (px - cx) >> 3, ty0 = (py - cy) >> 3, th = j.ph >> 3;
#pragma unroll
            for (int k = 0; k < 3; k++)
#pragma unroll
                for (int cr = 0; cr < 2; cr++)
                    for (int ty = ty0; ty < ty0 + th; ty++)
                    {
                        const int* s = &t.chr[k][cr * 4 + ty * 2];
                        C[k] += j.pw == 16 ? (s[0] + s[1]) >> 1 : s[tx0] >> 1;
                    }
        }
        // me_phase1's fold
        const int mvpx = j.qmvp[0], mvpy = j.qmvp[1];
        int bprecost = L[0] + C[0], bcost = bprecost, bestprex = pmvx, bestprey = pmvy, jbmx = bmx, jbmy = bmy;
        if (frac) bcost = L[1] + me_mvcost(mvcost, mvpx, mvpy, bmx * 4, bmy * 4);
        if (nonzero)
        {
            const int cz = L[2] + me_mvcost(mvcost, mvpx, mvpy, 0, 0);
            if (cz < bcost) { bcost = cz; jbmx = 0; jbmy = max(min(0, (int)j.mvmax[1]), (int)j.mvmin[1]); }
        }
        int cbest = 0x7fffffff, cbx = 0, cby = 0;
        if (v0)
        {
            const int cost = L[3] + C[1] + me_mvcost(mvcost, mvpx, mvpy, c0x, c0y);
            cbest = cost; cbx = c0x; cby = c0y;
        }
        if (v1)
        {
            const int cost = L[4] + C[2] + me_mvcost(mvcost, mvpx, mvpy, c1x, c1y);
            if (cost < cbest) { cbest = cost; cbx = c1x; cby = c1y; }
        }
        if (cbest < bprecost) { bprecost = cbest; bestprex = cbx; bestprey = cby; }
        MeState st;
        st.bmx = jbmx; st.bmy = jbmy; st.bcost = bcost; st.bprecost = bprecost; st.bestprex = bestprex; st.bestprey = bestprey;
        state[jid] = st;
    }
}

// ---- sub-pel refinement of the 16x16 cell groups (phase 3, motion.cpp:1440-1558) ---------------------------------------
// What a candidate position yields does not depend on the PU that asks for it: the luma prediction at (qx, qy) is the
// full-pel block of phase plane (qy & 3) * 4 + (qx & 3), the chroma prediction is fixed by the eighth-pel vector, and a PU's
// SATD is the sum of its tiles -- 8x4 tiles (u_left + u_right) >> 1 for luma widths 8 and 16, 4x4 tiles u >> 1 for width 4,
// u the un-halved 4x4 Hadamard sum (pixel.cpp:239-297); chroma as in k_me_precheck_cell.  So one warp runs the me_phase3
// state machine of all small PUs of a cell (me_subpel_class 0: one lane per job, a cell has at most 29 of them) together,
// and every step evaluates each distinct position the jobs ask for ONCE, over only the 8x4 luma units and chroma tiles that
// the asking PUs cover.  Per job only the range test, mvcost and the arg-min remain.  The cell's 12-wide / 12-high AMP
// parts (class 1) stay with the per-PU class-1 launch.  hpel-SATD workloads only (subme >= 2).
#define MEC_NP 40                          // distinct positions per table fill; a step with more is evaluated in chunks
struct MeSubTab
{
    int qx[MEC_NP], qy[MEC_NP];
    int mask[MEC_NP];                      // bits 0-7: 8x4 luma units (tile row * 2 + 8-pixel column); 8-15: chroma tiles (plane * 4 + tile)
    int start[MEC_NP];                     // exclusive prefix over the entries of the unit counts (bits 0-15) and tile counts (16-31)
    int lum[MEC_NP][16];                   // un-halved luma 4x4 Hadamard sums, tile row * 4 + tile column
    int chr[MEC_NP][8];                    // un-halved chroma 4x4 Hadamard sums [Cb tiles 0-3, Cr tiles 0-3]
};

// the entry of item `it` (0 <= it < total) of the 16-bit count field at `sh` of MeSubTab::start: the last entry starting at or
// before it (which has a non-zero count)
__device__ __forceinline__ int mec_find(const MeSubTab& t, int E, int it, int sh)
{
    int lo = 0, hi = E - 1;
    while (lo < hi)
    {
        const int mid = (lo + hi + 1) >> 1;
        if (((t.start[mid] >> sh) & 0xffff) <= it) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// me_phase3's stage machine (hpel-SATD workloads: SATD at the start point, half-pel rounds, quarter-pel rounds) of the jobs
// of one group, one lane per job (`mine`), shared by the per-cell and the per-CU kernels.  Per step the lanes' candidate
// positions are de-duplicated on (qx, qy) into t.qx / t.qy (at most MEC_NP at a time: a step with more is evaluated in
// chunks) and t.mask[e] collects the OR of the askers' coverage `mask`; `eval(E)` evaluates entries 0 .. E - 1 over their
// masks, `dist(e)` returns this lane's distortion at entry e.  Each job starts from `st` as me_phase3 does, tests its own
// qminy / qmaxy, adds its mvcost and folds its candidates in direction order with ties to the earliest (me_argmin).
template <typename Tab, typename Eval, typename Dist>
__device__ __forceinline__ void me_subpel_lanes(Tab& t, int lane, bool mine, const x265cu_me_job& j, int mask, const MeState& st,
                                                const uint16_t* __restrict__ mvcost, int32_t* __restrict__ o, Eval eval, Dist dist)
{
    const unsigned FULL = 0xffffffffu;
    const int qminy = j.mvmin[1] * 4, qmaxy = j.mvmax[1] * 4, mvpx = j.qmvp[0], mvpy = j.qmvp[1];
    const int8_t* wl = c_workload[j.subme];
    int bcost = st.bcost, bx, by;
    if (st.bprecost < bcost) { bx = st.bestprex; by = st.bestprey; bcost = st.bprecost; }
    else { bx = st.bmx * 4; by = st.bmy * 4; }
    bool live = mine && bcost != 0;
    if (mine && !bcost) bcost = me_mvcost(mvcost, mvpx, mvpy, bx, by);
    int stage = 0, it = 0;                                         // hpel SATD: stage 0 = SATD at the start point

    for (;;)
    {
        if (live && stage == 1 && it >= wl[0]) { stage = 3; it = 0; }
        if (live && stage == 3 && it >= wl[2]) live = false;
        if (!__any_sync(FULL, live)) break;
        const bool centre = stage == 0;
        const int dirs = !live ? 0 : centre ? 1 : stage == 1 ? wl[1] : wl[3];
        const int step = stage == 1 ? 2 : 1;
        const int ndir = __reduce_max_sync(FULL, (unsigned)dirs);
        unsigned sl0 = FULL, sl1 = FULL;                           // table entry of candidate i: byte i & 3 of (i < 4 ? sl0 : sl1)
        int best = bcost, bdir = 0;
        for (int i0 = 0; i0 < ndir;)
        {
            // ---- requests of candidates i0 .. i1 - 1, deduplicated on (qx, qy), while the table has room ----
            int E = 0, i1 = i0;
            for (; i1 < ndir; i1++)
            {
                const int d1 = centre ? 0 : i1 + 1;
                const int qx = bx + c_square1[d1][0] * step, qy = by + c_square1[d1][1] * step;
                const bool have = i1 < dirs && (centre || !((qy < qminy) | (qy > qmaxy)));
                const unsigned long long key = have ? ((unsigned long long)(uint32_t)qy << 32) | (uint32_t)qx : 0x8000000080000000ull;
                const unsigned gm = __match_any_sync(FULL, key);
                const int leader = __ffs(gm) - 1;
                const bool lead = have && lane == leader;
                int e = -1;
                if (lead)
                    for (int k = 0; k < E; k++) if (t.qx[k] == qx && t.qy[k] == qy) { e = k; break; }
                const unsigned nb = __ballot_sync(FULL, lead && e < 0);
                if (E + __popc(nb) > MEC_NP) break;                  // warp-uniform; E = 0 always has room
                if (lead && e < 0) { e = E + __popc(nb & ((1u << lane) - 1u)); t.qx[e] = qx; t.qy[e] = qy; t.mask[e] = 0; }
                E += __popc(nb);
                e = __shfl_sync(FULL, e, leader);
                __syncwarp();
                if (have)
                {
                    atomicOr(&t.mask[e], mask);
                    const unsigned sh = 8u * (i1 & 3), v = ((unsigned)e << sh) | ~(0xffu << sh);
                    if (i1 < 4) sl0 &= v; else sl1 &= v;
                }
            }
            __syncwarp();
            eval(E);
            __syncwarp();
            // ---- each job folds its candidates i0 .. i1 - 1 in order (me_argmin: ties to the earliest) ----
            for (int i = i0; i < i1; i++)
            {
                const int e = (int)(((i < 4 ? sl0 : sl1) >> (8 * (i & 3))) & 0xffu);
                if (e == 0xff) continue;
                const int d1 = centre ? 0 : i + 1;
                const int qx = bx + c_square1[d1][0] * step, qy = by + c_square1[d1][1] * step;
                const int cost = dist(e) + me_mvcost(mvcost, mvpx, mvpy, qx, qy);
                if (centre) best = cost;
                else if (cost < best) { best = cost; bdir = d1; }
            }
            __syncwarp();
            i0 = i1;
        }
        // ---- the next stage, as me_phase3 ----
        if (live)
        {
            if (centre) { bcost = best; stage = 1; }
            else if (bdir) { bcost = best; bx += c_square1[bdir][0] * step; by += c_square1[bdir][1] * step; it++; }
            else if (stage == 1) { stage = 3; it = 0; }
            else live = false;
        }
    }
    if (mine) { o[0] = bcost; o[1] = bx; o[2] = by; o[3] = 0; }
}

template <typename P, bool CHROMA>
__global__ void __launch_bounds__(256) k_me_subpel_cell(const P* __restrict__ fenc, int fstride, const P* const* __restrict__ refs, int rstride, ptrdiff_t ppitch,
                                                        MeChromaArgs ch, const uint16_t* __restrict__ mvcost, const x265cu_me_job* __restrict__ jobs,
                                                        const MeGroup* __restrict__ groups, int ngroups, const int32_t* __restrict__ grp_jobs, int job0,
                                                        const MeState* __restrict__ state, int32_t* __restrict__ out)
{
    __shared__ __align__(16) MeSubTab tabs[8];
    const unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int gi = blockIdx.x * 8 + warp;
    if (gi >= ngroups) return;
    const MeGroup g = groups[gi];
    MeSubTab& t = tabs[warp];

    // ---- the cell's class-0 jobs, one per lane, in group order (members lane and lane + 32: a cell holds up to 33 jobs) ----
    int nj;
    {
        int m[2]; bool small[2];
#pragma unroll
        for (int h = 0; h < 2; h++)
        {
            const int i = lane + 32 * h;
            m[h] = i < g.count ? grp_jobs[g.first + i] - job0 : 0;
            small[h] = i < g.count && me_subpel_kernel(jobs[m[h]].pw, jobs[m[h]].ph) == 0;
        }
        const unsigned b0 = __ballot_sync(FULL, small[0]), b1 = __ballot_sync(FULL, small[1]);
        const unsigned lt = (1u << lane) - 1u;
        // the analyser launches this kernel only when every cell has at most 32 of them (an_build_geometry)
        if (small[0]) t.qx[__popc(b0 & lt)] = m[0];
        if (small[1]) t.qx[__popc(b0) + __popc(b1 & lt)] = m[1];
        nj = __popc(b0) + __popc(b1);
    }
    __syncwarp();
    const bool mine = lane < nj;
    const int jid = mine ? t.qx[lane] : grp_jobs[g.first] - job0;
    __syncwarp();
    const x265cu_me_job j = jobs[jid];
    const int py = j.offset / fstride, px = j.offset - py * fstride;
    const int cx = __shfl_sync(FULL, px, 0) & ~15, cy = __shfl_sync(FULL, py, 0) & ~15;
    const ptrdiff_t coff = (ptrdiff_t)cy * fstride + cx;
    const P* rb = refs[j.ref] + coff;                              // every job of a group has the same reference
    const P* fb = fenc + coff;

    // per job: its 4x4 tiles inside the cell, its units and chroma tiles
    const int bx0 = (px - cx) >> 2, by0 = (py - cy) >> 2, bw = j.pw >> 2, bh = j.ph >> 2;
    const bool chromaOn = CHROMA && j.subme > 2 && !(j.pw & 7) && !(j.ph & 7);           // me_set_chroma
    int mask = 0;
    {
        const int segs = (1 << (((bx0 + bw - 1) >> 1) + 1)) - (1 << (bx0 >> 1));
        for (int y = by0; y < by0 + bh; y++) mask |= segs << (2 * y);
        if (chromaOn)
        {
            const int tx0 = bx0 >> 1, ty0 = by0 >> 1, tw = j.pw >> 3, th = j.ph >> 3;
            int cm = 0;
            for (int y = ty0; y < ty0 + th; y++) for (int x = tx0; x < tx0 + tw; x++) cm |= 1 << (y * 2 + x);
            mask |= (cm | (cm << 4)) << 8;
        }
    }

    me_subpel_lanes(t, lane, mine, j, mask, state[jid], mvcost, out + (size_t)jid * 4,
        [&](int E)
        {
            // ---- prefix of the entries' unit and tile counts ----
            int total = 0;
            for (int e0 = 0; e0 < E; e0 += 32)
            {
                const int e = e0 + lane;
                const int m = e < E ? t.mask[e] : 0;
                const int own = __popc(m & 0xff) | (__popc((m >> 8) & 0xff) << 16);
                int v = own;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) { const int n = __shfl_up_sync(FULL, v, o); if (lane >= o) v += n; }
                if (e < E) t.start[e] = total + v - own;
                total += __shfl_sync(FULL, v, 31);
            }
            __syncwarp();
            // ---- luma: 8 units per pass, a unit's 4 rows on 4 consecutive lanes (me_seg_cost's butterflies) ----
            const int nu = total & 0xffff, nt = total >> 16;
            for (int u0 = 0; u0 < nu; u0 += 8)
            {
                const int item = u0 + (lane >> 2), row = lane & 3;
                const bool on = item < nu;
                int e = 0, unit = 0;
                int d[8];
                if (on)
                {
                    e = mec_find(t, E, item, 0);
                    unit = me_nth_set_bit((unsigned)t.mask[e] & 0xffu, item - (t.start[e] & 0xffff));
                    const int qx = t.qx[e], qy = t.qy[e];
                    const int y = (unit >> 1) * 4 + row, x = (unit & 1) * 8;
                    int pr[8], fv[8];
                    me_ld_px<P, 8>(rb + (qx >> 2) + (ptrdiff_t)((qy >> 2) + y) * rstride + x + ((qy & 3) * 4 + (qx & 3)) * ppitch, pr);
                    me_ld_px<P, 8>(fb + (ptrdiff_t)y * fstride + x, fv);
#pragma unroll
                    for (int k = 0; k < 8; k++) d[k] = fv[k] - pr[k];
                }
                else
                {
#pragma unroll
                    for (int k = 0; k < 8; k++) d[k] = 0;
                }
                had4(d[0], d[1], d[2], d[3]); had4(d[4], d[5], d[6], d[7]);
#pragma unroll
                for (int s = 1; s <= 2; s <<= 1)
                {
                    const bool up = (lane & s) != 0;
#pragma unroll
                    for (int k = 0; k < 8; k++)
                    {
                        const int o = __shfl_xor_sync(FULL, d[k], s);
                        d[k] = up ? o - d[k] : o + d[k];
                    }
                }
                int sl = abs(d[0]) + abs(d[1]) + abs(d[2]) + abs(d[3]), sr = abs(d[4]) + abs(d[5]) + abs(d[6]) + abs(d[7]);
#pragma unroll
                for (int s = 1; s <= 2; s <<= 1) { sl += __shfl_xor_sync(FULL, sl, s); sr += __shfl_xor_sync(FULL, sr, s); }
                if (on && row == 0) { int* L = &t.lum[e][(unit >> 1) * 4 + (unit & 1) * 2]; L[0] = sl; L[1] = sr; }
            }
            // ---- chroma: one lane per (position, plane, tile) ----
            if (CHROMA)
                for (int c0 = 0; c0 < nt; c0 += 32)
                {
                    const int item = c0 + lane;
                    if (item < nt)
                    {
                        const int e = mec_find(t, E, item, 16);
                        const int k = me_nth_set_bit(((unsigned)t.mask[e] >> 8) & 0xffu, item - (t.start[e] >> 16));
                        const int cr = k >> 2, tt = k & 3, qx = t.qx[e], qy = t.qy[e];
                        const ptrdiff_t o = (ptrdiff_t)(cy >> 1) * ch.cstride + (cx >> 1) + (ptrdiff_t)((tt >> 1) * 4) * ch.cstride + (tt & 1) * 4;
                        const P* f = (const P*)(cr ? ch.fencCr : ch.fencCb) + o;
                        const P* r = ((const P* const*)(cr ? ch.refCr : ch.refCb))[j.ref] + o + (qx >> 3) + (ptrdiff_t)(qy >> 3) * ch.cstride;
                        t.chr[e][k] = me_chroma_had4x4<P>(f, r, ch.cstride, qx & 7, qy & 7);
                    }
                }
        },
        [&](int e)
        {
            const int* L = t.lum[e];
            int cost = 0;
            for (int y = by0; y < by0 + bh; y++)
            {
                if (bw == 1) cost += L[y * 4 + bx0] >> 1;
                else for (int x = bx0; x < bx0 + bw; x += 2) cost += (L[y * 4 + x] + L[y * 4 + x + 1]) >> 1;
            }
            if (chromaOn)
            {
                const int tx0 = bx0 >> 1, ty0 = by0 >> 1, th = j.ph >> 3;
#pragma unroll
                for (int cr = 0; cr < 2; cr++)
                    for (int y = ty0; y < ty0 + th; y++)
                    {
                        const int* s = &t.chr[e][cr * 4 + y * 2];
                        cost += j.pw == 16 ? (s[0] + s[1]) >> 1 : s[tx0] >> 1;
                    }
            }
            return cost;
        });
}

// ---- sub-pel refinement of the CU 64 / CU 32 groups --------------------------------------------------------------------
// The same sharing one level up.  The five PUs of a CU (2Nx2N, 2 x 2NxN, 2 x Nx2N) cover it three times; on the same
// integer vector they ask for the same half-pel and quarter-pel positions.  One warp runs the stage machine of a CU's PUs
// (me_subpel_lanes, one lane per PU) and evaluates each distinct position once per 32x32 quadrant the askers cover (a CU 32
// is one quadrant): the quadrant's 32 luma 8x4 units are one warp pass, the whole Hadamard in the lane as in
// me_subpel_big, and its 2 x 16 chroma 4x4 tiles are one pass of me_chroma_had4x4.  Every PU side is a multiple of 16, so
// luma is tiled 8x4 and chroma (widths 8 / 16 / 32) 8x4 for all of them: a lane's unit, and a lane pair's chroma tile, is a
// whole tile of every PU that covers it, and a PU's SATD is the sum of the lanes it covers.  Coverage is kept per 16x16
// block of the CU (a 4x4 grid of bits; 2x2 used by a CU 32).  The CUs' AMP parts stay with the per-PU class-1 launch.
struct MeGrpTab
{
    int qx[MEC_NP], qy[MEC_NP];
    int mask[MEC_NP];                      // bits 0-15: 16x16 blocks (row * 4 + column) asked for in luma; 16-31: in chroma
    int dist[MEC_NP][8];                   // per job slot (a CU has five such PUs): luma + chroma SATD at the entry
};

template <typename P, bool CHROMA>
__global__ void __launch_bounds__(256, 2) k_me_subpel_group(const P* __restrict__ fenc, int fstride, const P* const* __restrict__ refs, int rstride, ptrdiff_t ppitch,
                                                            MeChromaArgs ch, const uint16_t* __restrict__ mvcost, const x265cu_me_job* __restrict__ jobs,
                                                            const MeGroup* __restrict__ groups64, int n64, const int32_t* __restrict__ grp_jobs64,
                                                            const MeGroup* __restrict__ groups32, int n32, const int32_t* __restrict__ grp_jobs32, int job0,
                                                            const MeState* __restrict__ state, int32_t* __restrict__ out)
{
    __shared__ __align__(16) MeGrpTab tabs[8];
    const unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    // the CU 64 groups (four times the work) first, so that they do not form the tail of the launch
    const int gi = blockIdx.x * 8 + warp;
    if (gi >= n64 + n32) return;
    const bool big = gi < n64;
    const MeGroup g = big ? groups64[gi] : groups32[gi - n64];
    const int32_t* grp_jobs = big ? grp_jobs64 : grp_jobs32;
    MeGrpTab& t = tabs[warp];

    // ---- the CU's 2Nx2N / 2NxN / Nx2N jobs, one per lane, in group order (a group holds up to 13 jobs with AMP) ----
    int nj;
    {
        const int m = lane < g.count ? grp_jobs[g.first + lane] - job0 : 0;
        const bool take = lane < g.count && me_subpel_kernel(jobs[m].pw, jobs[m].ph) == 1;
        const unsigned b = __ballot_sync(FULL, take);
        if (take) t.qx[__popc(b & ((1u << lane) - 1u))] = m;
        nj = __popc(b);
    }
    __syncwarp();
    const bool mine = lane < nj;
    const int jid = mine ? t.qx[lane] : grp_jobs[g.first] - job0;
    __syncwarp();
    const x265cu_me_job j = jobs[jid];
    const int py = j.offset / fstride, px = j.offset - py * fstride;
    const int edge = big ? 64 : 32;
    const int cx = __shfl_sync(FULL, px, 0) & ~(edge - 1), cy = __shfl_sync(FULL, py, 0) & ~(edge - 1);
    const ptrdiff_t coff = (ptrdiff_t)cy * fstride + cx;
    const P* rb = refs[j.ref] + coff;                              // every job of a group has the same reference
    const P* fb = fenc + coff;
    const ptrdiff_t coffC = CHROMA ? (ptrdiff_t)(cy >> 1) * ch.cstride + (cx >> 1) : 0;

    int mask = 0;
    for (int y = (py - cy) >> 4; y < (py - cy + j.ph) >> 4; y++)
        for (int x = (px - cx) >> 4; x < (px - cx + j.pw) >> 4; x++) mask |= 1 << (y * 4 + x);
    if (CHROMA && j.subme > 2) mask |= mask << 16;                 // me_set_chroma: the sides are multiples of 8
    if (!mine) mask = 0;

    // my 8x4 luma unit of a quadrant: column lane & 3, row lane >> 2; my chroma tile: plane (lane >> 2) & 1, column lane & 3,
    // row lane >> 3 -- so that both lie in the quadrant's 16x16 block ((lane >> 1) & 1, lane >> 4)
    const int ux = lane & 3, uy = lane >> 2, blk = (lane >> 4) * 4 + ((lane >> 1) & 1);
    const int cty = lane >> 3;
    const bool cr = (lane >> 2) & 1;
    const P* fC = (const P*)(cr ? ch.fencCr : ch.fencCb) + coffC;
    const P* rC = CHROMA ? ((const P* const*)(cr ? ch.refCr : ch.refCb))[j.ref] + coffC : nullptr;

    me_subpel_lanes(t, lane, mine, j, mask, state[jid], mvcost, out + (size_t)jid * 4,
        [&](int E)
        {
            for (int e = 0; e < E; e++)
            {
                const int m = t.mask[e], qx = t.qx[e], qy = t.qy[e];
                const P* r0 = rb + (qx >> 2) + (ptrdiff_t)(qy >> 2) * rstride + ((qy & 3) * 4 + (qx & 3)) * ppitch;
                int acc = 0;
                for (int q = 0; q < (big ? 4 : 1); q++)
                {
                    const int X0 = (q & 1) * 2, Y0 = (q >> 1) * 2;         // the quadrant's first 16x16 block
                    if (!((m | (m >> 16)) & (0x33 << (Y0 * 4 + X0)))) continue;
                    const int bit = Y0 * 4 + X0 + blk;
                    int lum = 0, chr = 0;
                    if ((m >> bit) & 1)
                    {   // one 8x4 tile (pixel.cpp:239-261): two 4x4 Hadamards, halved together
                        const int x = X0 * 16 + ux * 8, y = Y0 * 16 + uy * 4;
                        int d[4][8];
#pragma unroll
                        for (int k = 0; k < 4; k++)
                        {
                            int fv[8];
                            me_load_row8<P>(r0 + (ptrdiff_t)(y + k) * rstride + x, d[k]);
                            me_load_row8<P>(fb + (ptrdiff_t)(y + k) * fstride + x, fv);
#pragma unroll
                            for (int i = 0; i < 8; i++) d[k][i] = fv[i] - d[k][i];
                            had4(d[k][0], d[k][1], d[k][2], d[k][3]); had4(d[k][4], d[k][5], d[k][6], d[k][7]);
                        }
#pragma unroll
                        for (int i = 0; i < 8; i++)
                        {
                            had4(d[0][i], d[1][i], d[2][i], d[3][i]);
                            lum += abs(d[0][i]) + abs(d[1][i]) + abs(d[2][i]) + abs(d[3][i]);
                        }
                        lum >>= 1;
                    }
                    if (CHROMA)
                    {
                        if ((m >> (16 + bit)) & 1)
                        {
                            const ptrdiff_t o = (ptrdiff_t)(Y0 * 8 + cty * 4) * ch.cstride + X0 * 8 + ux * 4;
                            chr = me_chroma_had4x4<P>(fC + o, rC + o + (qx >> 3) + (ptrdiff_t)(qy >> 3) * ch.cstride, ch.cstride, qx & 7, qy & 7);
                        }
                        // 8x4 chroma tiles: the two 4x4 sums of a lane pair added and halved, kept by the even lane
                        chr += __shfl_xor_sync(FULL, chr, 1);
                        chr = (lane & 1) ? 0 : chr >> 1;
                    }
                    for (int s = 0; s < nj; s++)
                    {
                        const int jm = __shfl_sync(FULL, mask, s);
                        const int v = __reduce_add_sync(FULL, (((jm >> bit) & 1) ? lum : 0) + (((jm >> (16 + bit)) & 1) ? chr : 0));
                        if (lane == s) acc += v;
                    }
                }
                if (mine) t.dist[e][lane] = acc;
            }
        },
        [&](int e) { return t.dist[e][lane]; });
}

// Sub-pel refinement of the class-0 jobs of a frame slice's 16x16 cells (k_me_subpel_cell), on the phase planes `ppitch`
// elements apart.
template <typename P>
static int launch_me_subpel_cells(x265cu_ctx* ctx, const void* fenc, int fstride, const void* const* refs, int rstride, ptrdiff_t ppitch,
                                  const MeChromaArgs* ch, const uint16_t* mvcost, const x265cu_me_job* jobs, const MeState* st, int32_t* out,
                                  const MeWinLaunch& w)
{
    if (w.ngroups[2] <= 0) return 0;
    const MeChromaArgs none = {};
    const auto kernel = ch ? k_me_subpel_cell<P, true> : k_me_subpel_cell<P, false>;
    kernel<<<(w.ngroups[2] + 7) / 8, 256, 0, ctx->stream>>>((const P*)fenc, fstride, (const P* const*)refs, rstride, ppitch, ch ? *ch : none, mvcost, jobs,
                                                           (const MeGroup*)w.groups[2], w.ngroups[2], w.grp_jobs[2], w.job0, st, out);
    CU_LAUNCH_CHECK(ctx);
    return 0;
}

// Sub-pel refinement of the 2Nx2N / 2NxN / Nx2N jobs of a frame slice's CU 64 and CU 32 groups (k_me_subpel_group)
template <typename P>
static int launch_me_subpel_groups(x265cu_ctx* ctx, const void* fenc, int fstride, const void* const* refs, int rstride, ptrdiff_t ppitch,
                                   const MeChromaArgs* ch, const uint16_t* mvcost, const x265cu_me_job* jobs, const MeState* st, int32_t* out,
                                   const MeWinLaunch& w)
{
    const int n = w.ngroups[0] + w.ngroups[1];
    if (n <= 0) return 0;
    const MeChromaArgs none = {};
    const auto kernel = ch ? k_me_subpel_group<P, true> : k_me_subpel_group<P, false>;
    kernel<<<(n + 7) / 8, 256, 0, ctx->stream>>>((const P*)fenc, fstride, (const P* const*)refs, rstride, ppitch, ch ? *ch : none, mvcost, jobs,
                                                 (const MeGroup*)w.groups[0], w.ngroups[0], w.grp_jobs[0], (const MeGroup*)w.groups[1], w.ngroups[1],
                                                 w.grp_jobs[1], w.job0, st, out);
    CU_LAUNCH_CHECK(ctx);
    return 0;
}

// The jobs of a launch slice that neither of the two kernels above refines (AMP parts), appended to `left_list` in the
// order of `order` (NULL: job order) for the per-PU class-1 launch
__global__ void __launch_bounds__(256) k_me_subpel_rest(const x265cu_me_job* __restrict__ jobs, int n, const int32_t* __restrict__ order, int order0,
                                                        int* __restrict__ left_count, int32_t* __restrict__ left_list)
{
    const int i = blockIdx.x * 256 + threadIdx.x, lane = threadIdx.x & 31;
    const int jid = i >= n ? 0 : order ? order[i] - order0 : i;
    const bool keep = i < n && me_subpel_kernel(jobs[jid].pw, jobs[jid].ph) == 2;
    const unsigned b = __ballot_sync(0xffffffffu, keep);
    int base = 0;
    if (b && lane == 0) base = atomicAdd(left_count, __popc(b));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (keep) left_list[base + __popc(b & ((1u << lane) - 1u))] = jid;
}

static int launch_me_subpel_rest(x265cu_ctx* ctx, const x265cu_me_job* jobs, int n, const int32_t* order, int order0, const MeWinLaunch& w)
{
    CU_CHECK(cudaMemsetAsync(w.left_count, 0, sizeof(int), ctx->stream));
    k_me_subpel_rest<<<(n + 255) / 256, 256, 0, ctx->stream>>>(jobs, n, order, order0, w.left_count, w.left_list);
    CU_LAUNCH_CHECK(ctx);
    return 0;
}

// Pre-checks of a frame slice's groups: cells out of shared tables, every other job (CU 64 / CU 32 groups, cells' jobs with
// other clips) appended to `left_list` (count in *left_count, zeroed here) for the per-PU kernels.
template <typename P>
static int launch_me_precheck_groups(x265cu_ctx* ctx, const void* fenc, int fstride, const void* const* refs, int rstride, const MeChromaArgs* ch,
                                     const uint16_t* mvcost, const x265cu_me_job* jobs, MeState* st, const MeWinLaunch& w, int* left_count, int32_t* left_list)
{
    CU_CHECK(cudaMemsetAsync(left_count, 0, sizeof(int), ctx->stream));
    const MeChromaArgs none = {};
    for (int cls = 0; cls < 3; cls++)
    {
        if (w.ngroups[cls] <= 0) continue;
        const int blocks = (w.ngroups[cls] + 7) / 8;
        const auto kernel = ch ? k_me_precheck_cell<P, true> : k_me_precheck_cell<P, false>;
        kernel<<<blocks, 256, 0, ctx->stream>>>((const P*)fenc, fstride, (const P* const*)refs, rstride, ch ? *ch : none, mvcost, jobs,
                                                (const MeGroup*)w.groups[cls], w.ngroups[cls], w.grp_jobs[cls], w.job0, cls == 2, st, left_count, left_list);
        CU_LAUNCH_CHECK(ctx);
    }
    return 0;
}
