/* oracle/oracle_sao.c -- TEST INFRASTRUCTURE ONLY.
 *
 * Frame-level SAO restated in plain C over whole planes, for one slice per picture:
 *   orc_sao_stats_frame: the count / offsetOrg arrays of SAO::calcSaoStatsCTU (sao.cpp:735-917, with the C bodies
 *                        saoCuStatsBO_c / E0_c .. E3_c, sao.cpp:1762-1925) for every CTU and plane;
 *   orc_sao_apply_frame: generateLumaOffsets / generateChromaOffsets / applyPixelOffsets (sao.cpp:274-732) of every CTU with
 *                        the given per-CTU parameters, then the transquant-bypass restoration (framefilter.cpp:254-298).
 * Both read only the deblocked, not-yet-SAO'd picture: the statistics skip the samples the next CTU row's deblocking still
 * changes, and the apply of a CTU reads its left / top neighbours from copies taken before any SAO (m_tmpL1 / m_tmpU) and
 * its right / bottom neighbours from CTUs that are filtered later.  So apply is a stencil of the deblocked picture.  That
 * claim is pinned to FrameFilter's interleaved order by tests/test_sao_oracle_vs_ref.py (oracle/ref_shim_sao.cpp).
 * Citations are to the reference's source/encoder/sao.cpp unless noted.
 */
#include "oracle.h"
#include <stdlib.h>
#include <string.h>

typedef struct {                 /* x265cu_sao_ctu */
    int8_t  typeIdx;             /* -1 off, 0..3 SAO_EO_0..3, 4 SAO_BO; anything else off */
    uint8_t bandPos;
    int8_t  offset[4];
    uint8_t pad[2];
} orc_sao_ctu;

typedef struct {                 /* x265cu_deblock_unit: only flags bit 2 (tq-bypass) is read here */
    int8_t qp; uint8_t flags, log2CuSize, partSize, tuDepth; int8_t refPic[2]; int16_t mv[2][2];
} orc_unit;

enum { SAO_EO_0, SAO_EO_1, SAO_EO_2, SAO_EO_3, SAO_BO, NUM_TYPES };
#define NUM_CLASS 32
#define PLANE_REC (NUM_TYPES * NUM_CLASS)        /* one SAO::PerClass */
#define CTU_REC (2 * 3 * PLANE_REC)              /* count PerPlane, offsetOrg PerPlane */
#define PIXEL_MAX ((1 << ORC_DEPTH) - 1)
#define BO_SHIFT (ORC_DEPTH - 5)
static const int eoTable[5] = { 1, 2, 0, 3, 4 };                 /* SAO::s_eoTable (:65-72) */

/* decision counters (`counters` of both entry points) */
enum { CNT_STATS_RIGHT, CNT_STATS_BOTTOM, CNT_STATS_INNER, CNT_STATS_TOP, CNT_STATS_LEFT,
       CNT_APPLY_OFF, CNT_APPLY_EO0, CNT_APPLY_EO1, CNT_APPLY_EO2, CNT_APPLY_EO3, CNT_APPLY_BO,
       CNT_BAND_WRAP, CNT_CLIP_LO, CNT_CLIP_HI, CNT_CR_CB_TYPE, CNT_CR_SKIPPED, CNT_BYPASS, CNT_N };

static int sgn(int x) { return (x > 0) - (x < 0); }

/* one CTU of one plane: region rules of calcSaoStatsCTU (:764-916), skipB 4 / skipR 5 with the chroma plane_offset 2 */
static void ctu_stats(const pixel* f, intptr_t fs, const pixel* r, intptr_t rs, int picW, int picH, int lpelx, int tpely, int size,
                      int po, int32_t* count, int32_t* org, int64_t* cnt)
{
    const int rpelx = lpelx + size < picW ? lpelx + size : picW, bpely = tpely + size < picH ? tpely + size : picH;
    const int w = rpelx - lpelx, h = bpely - tpely, right = rpelx == picW, bottom = bpely == picH;
    const int skipB = 4, skipR = 5;
    const int startX = !lpelx, startY = !tpely;
    f += (intptr_t)tpely * fs + lpelx;
    r += (intptr_t)tpely * rs + lpelx;
    cnt[right ? CNT_STATS_RIGHT : bottom ? CNT_STATS_BOTTOM : CNT_STATS_INNER]++;
    if (startY) cnt[CNT_STATS_TOP]++;
    if (startX) cnt[CNT_STATS_LEFT]++;
#define DIFF(x, y) ((int)f[(intptr_t)(y) * fs + (x)] - (int)r[(intptr_t)(y) * rs + (x)])
#define REC(x, y) ((int)r[(intptr_t)(y) * rs + (x)])
#define ADD(type, cls, x, y) do { count[(type) * NUM_CLASS + (cls)]++; org[(type) * NUM_CLASS + (cls)] += DIFF(x, y); } while (0)

    /* SAO_BO (:810-822) */
    int endX = right ? w : w - skipR + po, endY = bottom ? h : h - skipB + po;
    for (int y = 0; y < endY; y++)
        for (int x = 0; x < endX; x++)
            ADD(SAO_BO, REC(x, y) >> BO_SHIFT, x, y);

    /* SAO_EO_0 (:825-837): the row count ignores the picture bottom */
    endX = right ? w - 1 : w - skipR + po;
    endY = h - skipB + po;
    for (int y = 0; y < endY; y++)
        for (int x = startX; x < endX; x++)
            ADD(SAO_EO_0, eoTable[sgn(REC(x, y) - REC(x + 1, y)) + sgn(REC(x, y) - REC(x - 1, y)) + 2], x, y);

    /* SAO_EO_1 (:839-860) */
    endX = right ? w : w - skipR + po;
    endY = bottom ? h - 1 : h - skipB + po;
    for (int y = startY; y < endY; y++)
        for (int x = 0; x < endX; x++)
            ADD(SAO_EO_1, eoTable[sgn(REC(x, y) - REC(x, y + 1)) + sgn(REC(x, y) - REC(x, y - 1)) + 2], x, y);

    /* SAO_EO_2 / SAO_EO_3 (:861-915; bLimitSAO is the caller's, see INTEGRATION.md) */
    endX = right ? w - 1 : w - skipR + po;
    for (int y = startY; y < endY; y++)
        for (int x = startX; x < endX; x++)
        {
            ADD(SAO_EO_2, eoTable[sgn(REC(x, y) - REC(x + 1, y + 1)) + sgn(REC(x, y) - REC(x - 1, y - 1)) + 2], x, y);
            ADD(SAO_EO_3, eoTable[sgn(REC(x, y) - REC(x - 1, y + 1)) + sgn(REC(x, y) - REC(x + 1, y - 1)) + 2], x, y);
        }
#undef ADD
#undef REC
#undef DIFF
}

/* stats: int32 [numCtus][2: count, offsetOrg][3][5][32], every entry written (chroma zero without chroma planes) */
int orc_sao_stats_frame(const pixel* fy, const pixel* fcb, const pixel* fcr, intptr_t fstride, intptr_t fcstride,
                        const pixel* ry, const pixel* rcb, const pixel* rcr, intptr_t stride, intptr_t cstride,
                        int width, int height, int ctuSize, int32_t* stats, int64_t* counters)
{
    int64_t local[CNT_N] = { 0 };
    if ((width & 7) || (height & 7) || width <= 0 || height <= 0 || (ctuSize != 16 && ctuSize != 32 && ctuSize != 64))
        return -1;
    const int cols = (width + ctuSize - 1) / ctuSize, rows = (height + ctuSize - 1) / ctuSize;
    const pixel* fp[3] = { fy, fcb, fcr };
    const pixel* rp[3] = { ry, rcb, rcr };
    memset(stats, 0, sizeof(int32_t) * CTU_REC * (size_t)cols * rows);
    for (int addr = 0; addr < cols * rows; addr++)
        for (int p = 0; p < (fcb ? 3 : 1); p++)
        {
            int32_t* rec = stats + (size_t)addr * CTU_REC;
            const int s = p ? 1 : 0;
            ctu_stats(fp[p], p ? fcstride : fstride, rp[p], p ? cstride : stride, width >> s, height >> s,
                      (addr % cols) * ctuSize >> s, (addr / cols) * ctuSize >> s, ctuSize >> s, p ? 2 : 0,
                      rec + p * PLANE_REC, rec + 3 * PLANE_REC + p * PLANE_REC, local);
        }
    if (counters)
        for (int i = 0; i < CNT_N; i++)
            counters[i] += local[i];
    return 0;
}

/* The offset table of one record (generateLumaOffsets :604-625): BO 32 entries from bandPos (mod 32), EO 5 entries indexed
 * by edgeType through s_eoTable */
static void offsets_of(const orc_sao_ctu* prm, int type, int* table, int64_t* cnt)
{
    memset(table, 0, sizeof(int) * NUM_CLASS);
    if (type == SAO_BO)
    {
        for (int i = 0; i < 4; i++)
        {
            if ((prm->bandPos & 31) + i > 31) cnt[CNT_BAND_WRAP]++;
            table[(prm->bandPos + i) & 31] = prm->offset[i];
        }
    }
    else
    {
        const int off[5] = { 0, prm->offset[0], prm->offset[1], prm->offset[2], prm->offset[3] };
        for (int et = 0; et < 5; et++)
            table[et] = off[eoTable[et]];
    }
}

/* applyPixelOffsets (:274-569) of one CTU as a stencil of the deblocked plane `src` into `dst`: which samples each type
 * changes (BO all; EO_0 not the picture's left / right column; EO_1 not its top / bottom row; EO_2 / EO_3 neither) */
static void ctu_apply(pixel* dst, intptr_t ds, const pixel* src, intptr_t ss, int picW, int picH, int lpelx, int tpely, int size,
                      int type, const int* table, int64_t* cnt)
{
    const int rpelx = lpelx + size < picW ? lpelx + size : picW, bpely = tpely + size < picH ? tpely + size : picH;
    const int w = rpelx - lpelx, h = bpely - tpely;
    const int x0 = type != SAO_BO && type != SAO_EO_1 ? !lpelx : 0, x1 = type != SAO_BO && type != SAO_EO_1 && rpelx == picW ? w - 1 : w;
    const int y0 = type != SAO_BO && type != SAO_EO_0 ? !tpely : 0, y1 = type != SAO_BO && type != SAO_EO_0 && bpely == picH ? h - 1 : h;
    static const int dx[4][2] = { { -1, 1 }, { 0, 0 }, { -1, 1 }, { 1, -1 } }, dy[4][2] = { { 0, 0 }, { -1, 1 }, { -1, 1 }, { -1, 1 } };
    cnt[CNT_APPLY_EO0 + type]++;
    src += (intptr_t)tpely * ss + lpelx;
    dst += (intptr_t)tpely * ds + lpelx;
    for (int y = y0; y < y1; y++)
        for (int x = x0; x < x1; x++)
        {
            const int c = src[(intptr_t)y * ss + x];
            int o;
            if (type == SAO_BO)
                o = table[c >> BO_SHIFT];
            else
            {
                const int a = src[(intptr_t)(y + dy[type][0]) * ss + x + dx[type][0]];
                const int b = src[(intptr_t)(y + dy[type][1]) * ss + x + dx[type][1]];
                o = table[sgn(c - a) + sgn(c - b) + 2];
            }
            int v = c + o;
            if (v < 0) { v = 0; cnt[CNT_CLIP_LO]++; }
            if (v > PIXEL_MAX) { v = PIXEL_MAX; cnt[CNT_CLIP_HI]++; }
            dst[(intptr_t)y * ds + x] = (pixel)v;
        }
}

static int valid_type(int t) { return t >= 0 && t <= SAO_BO; }

/* params: orc_sao_ctu [3][numCtus] (raster order; [1], [2] read only with saoChroma).  Cr is filtered with Cb's type and its
 * own offsets, and only when both types are >= 0 (generateChromaOffsets :704-728).  units: NULL, or the x265cu_deblock_unit
 * map whose bypass units (flags bit 2) get the source samples back afterwards (luma 4x4, chroma 2x2). */
int orc_sao_apply_frame(pixel* y, pixel* cb, pixel* cr, intptr_t stride, intptr_t cstride, int width, int height, int ctuSize,
                        const void* params, int saoLuma, int saoChroma, const void* units,
                        const pixel* fy, const pixel* fcb, const pixel* fcr, intptr_t fstride, intptr_t fcstride, int64_t* counters)
{
    int64_t local[CNT_N] = { 0 };
    if ((width & 7) || (height & 7) || width <= 0 || height <= 0 || (ctuSize != 16 && ctuSize != 32 && ctuSize != 64))
        return -1;
    const int cols = (width + ctuSize - 1) / ctuSize, rows = (height + ctuSize - 1) / ctuSize, n = cols * rows;
    const orc_sao_ctu* prm = (const orc_sao_ctu*)params;
    pixel* planes[3] = { y, cb, cr };
    const intptr_t strides[3] = { stride, cstride, cstride };
    for (int p = 0; p < (cb ? 3 : 1); p++)
    {
        if (!(p ? saoChroma : saoLuma))
            continue;
        const int s = p ? 1 : 0, pw = width >> s, ph = height >> s;
        pixel* src = (pixel*)malloc(sizeof(pixel) * (size_t)pw * ph);       /* the deblocked plane */
        for (int j = 0; j < ph; j++)
            memcpy(src + (size_t)j * pw, planes[p] + (intptr_t)j * strides[p], sizeof(pixel) * pw);
        for (int addr = 0; addr < n; addr++)
        {
            const orc_sao_ctu* own = &prm[p * n + addr];
            int type = own->typeIdx;
            if (p == 2)
            {
                const int tcb = prm[n + addr].typeIdx;
                if (valid_type(type) && !valid_type(tcb)) local[CNT_CR_SKIPPED]++;
                if (valid_type(type) && valid_type(tcb) && tcb != type) local[CNT_CR_CB_TYPE]++;
                type = valid_type(type) ? tcb : -1;
            }
            if (!valid_type(type))
            {
                local[CNT_APPLY_OFF]++;
                continue;
            }
            int table[NUM_CLASS];
            offsets_of(own, type, table, local);
            ctu_apply(planes[p], strides[p], src, pw, pw, ph, (addr % cols) * ctuSize >> s, (addr / cols) * ctuSize >> s,
                      ctuSize >> s, type, table, local);
        }
        free(src);
    }
    if (units)
    {
        const orc_unit* u = (const orc_unit*)units;
        const int upr = width >> 2;
        for (int uy = 0; uy < (height >> 2); uy++)
            for (int ux = 0; ux < upr; ux++)
            {
                if (!(u[uy * upr + ux].flags & 4))
                    continue;
                local[CNT_BYPASS]++;
                for (int j = 0; j < 4; j++)
                    memcpy(y + (intptr_t)(4 * uy + j) * stride + 4 * ux, fy + (intptr_t)(4 * uy + j) * fstride + 4 * ux, 4 * sizeof(pixel));
                if (cb)
                    for (int j = 0; j < 2; j++)
                    {
                        memcpy(cb + (intptr_t)(2 * uy + j) * cstride + 2 * ux, fcb + (intptr_t)(2 * uy + j) * fcstride + 2 * ux, 2 * sizeof(pixel));
                        memcpy(cr + (intptr_t)(2 * uy + j) * cstride + 2 * ux, fcr + (intptr_t)(2 * uy + j) * fcstride + 2 * ux, 2 * sizeof(pixel));
                    }
            }
    }
    if (counters)
        for (int i = 0; i < CNT_N; i++)
            counters[i] += local[i];
    return 0;
}
