/* oracle/oracle_deblock.c -- TEST INFRASTRUCTURE ONLY.
 *
 * Frame-level deblocking restated in plain C over the per-4x4 decision map of x265cu_deblock_frame (include/x265_b200.h):
 * every vertical edge of the picture first, then every horizontal edge of the result, the order Deblock::deblockCTU over
 * FrameFilter's CTU order amounts to (framefilter.cpp:457-516).  Citations are to the reference's source/common/deblock.cpp
 * unless noted.  Pinned to the real Deblock class by tests/test_deblock_oracle_vs_ref.py (oracle/ref_shim.cpp:
 * x265ref_deblock_frame).
 */
#include "oracle.h"
#include <stdlib.h>

typedef struct {                 /* x265cu_deblock_unit */
    int8_t  qp;
    uint8_t flags;               /* bit 0 intra, bit 1 luma cbf, bit 2 tq-bypass */
    uint8_t log2CuSize, partSize, tuDepth;
    int8_t  refPic[2];
    int16_t mv[2][2];
} orc_dbk_unit;

enum { SIZE_2Nx2N, SIZE_2NxN, SIZE_Nx2N, SIZE_NxN, SIZE_2NxnU, SIZE_2NxnD, SIZE_nLx2N, SIZE_nRx2N };
enum { EDGE_VER, EDGE_HOR };
enum { B_SLICE, P_SLICE, I_SLICE };
#define DEFAULT_INTRA_TC_OFFSET 2
#define PIXEL_MAX ((1 << ORC_DEPTH) - 1)

/* Deblock::s_tcTable / s_betaTable (:499-509); g_chromaScale (constants.cpp:346) */
static const uint8_t tcTable[54] = {
    0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 1, 1, 1, 1, 2,
    2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 5, 5, 6, 6, 7, 8, 9, 10, 11, 13, 14, 16, 18, 20, 22, 24 };
static const uint8_t betaTable[52] = {
    0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17,
    18, 20, 22, 24, 26, 28, 30, 32, 34, 36, 38, 40, 42, 44, 46, 48, 50, 52, 54, 56, 58, 60, 62, 64 };
static const uint8_t chromaScale[70] = {
    0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28, 29, 29, 30, 31,
    32, 33, 33, 34, 34, 35, 35, 36, 36, 37, 37, 38, 39, 40, 41, 42, 43, 44, 45, 46, 47, 48, 49, 50, 51,
    51, 51, 51, 51, 51, 51, 51, 51, 51, 51, 51, 51 };

/* decision counters (orc_deblock_frame's `counters`) */
enum { CNT_BS0, CNT_BS1, CNT_BS2, CNT_BETA_SKIP, CNT_STRONG, CNT_NORMAL_BOTH, CNT_NORMAL_ONE, CNT_NORMAL_NEITHER, CNT_CHROMA, CNT_N };

static int clip3(int lo, int hi, int v) { return v < lo ? lo : v > hi ? hi : v; }
static int clipPel(int v) { return clip3(0, PIXEL_MAX, v); }

/* The flag Deblock::deblockCU leaves at the Q unit of an 8-aligned edge at `pos` (x or y, > 0) (:90-93), in its overwrite
 * order: internal PU edge 1 (setEdgefilterPU :150-189), every TU's left / top edge 2 (setEdgefilterTU :135-148), the CU's own
 * edge 2 (bsCuEdge :46-68; 0 only at the picture border, which is never visited here). */
static int edge_flag(const orc_dbk_unit* q, int dir, int pos)
{
    int log2S = q->log2CuSize < 3 ? 3 : q->log2CuSize > 6 ? 6 : q->log2CuSize;
    int S = 1 << log2S, o = pos & (S - 1), flag = 0;
    int tuDepth = q->tuDepth > 3 ? 3 : q->tuDepth, T = S >> tuDepth;
    int half = S >> 1, quarter = S >> 2;
    switch (q->partSize)
    {
    case SIZE_2NxN:  if (dir == EDGE_HOR && o == half) flag = 1; break;
    case SIZE_Nx2N:  if (dir == EDGE_VER && o == half) flag = 1; break;
    case SIZE_NxN:   if (o == half) flag = 1; break;
    case SIZE_2NxnU: if (dir == EDGE_HOR && o == quarter) flag = 1; break;
    case SIZE_nLx2N: if (dir == EDGE_VER && o == quarter) flag = 1; break;
    case SIZE_2NxnD: if (dir == EDGE_HOR && o == S - quarter) flag = 1; break;
    case SIZE_nRx2N: if (dir == EDGE_VER && o == S - quarter) flag = 1; break;
    default: break;
    }
    if ((o & (T - 1)) == 0) flag = 2;
    if (o == 0) flag = 2;
    return flag;
}

static int mvDiff(int a, int b) { return abs(a - b) >= 4; }

/* Deblock::getBoundaryStrength (:191-247); refPic ids play the Frame pointers, < 0 = NULL (zero vector) */
static int boundary_strength(const orc_dbk_unit* P, const orc_dbk_unit* Q, int flag, int sliceType)
{
    if ((P->flags & 1) || (Q->flags & 1))
        return 2;
    if (flag > 1 && ((Q->flags & 2) || (P->flags & 2)))
        return 1;
    int refP0 = P->refPic[0] >= 0 ? P->refPic[0] : -1, refQ0 = Q->refPic[0] >= 0 ? Q->refPic[0] : -1;
    int mvP0x = refP0 >= 0 ? P->mv[0][0] : 0, mvP0y = refP0 >= 0 ? P->mv[0][1] : 0;
    int mvQ0x = refQ0 >= 0 ? Q->mv[0][0] : 0, mvQ0y = refQ0 >= 0 ? Q->mv[0][1] : 0;
    if (sliceType == P_SLICE)
        return (refP0 != refQ0 || mvDiff(mvQ0x, mvP0x) || mvDiff(mvQ0y, mvP0y)) ? 1 : 0;
    int refP1 = P->refPic[1] >= 0 ? P->refPic[1] : -1, refQ1 = Q->refPic[1] >= 0 ? Q->refPic[1] : -1;
    int mvP1x = refP1 >= 0 ? P->mv[1][0] : 0, mvP1y = refP1 >= 0 ? P->mv[1][1] : 0;
    int mvQ1x = refQ1 >= 0 ? Q->mv[1][0] : 0, mvQ1y = refQ1 >= 0 ? Q->mv[1][1] : 0;
    if ((refP0 == refQ0 && refP1 == refQ1) || (refP0 == refQ1 && refP1 == refQ0))
    {
        if (refP0 != refP1)
        {
            if (refP0 == refQ0)
                return (mvDiff(mvQ0x, mvP0x) || mvDiff(mvQ0y, mvP0y) || mvDiff(mvQ1x, mvP1x) || mvDiff(mvQ1y, mvP1y)) ? 1 : 0;
            return (mvDiff(mvQ1x, mvP0x) || mvDiff(mvQ1y, mvP0y) || mvDiff(mvQ0x, mvP1x) || mvDiff(mvQ0y, mvP1y)) ? 1 : 0;
        }
        return ((mvDiff(mvQ0x, mvP0x) || mvDiff(mvQ0y, mvP0y) || mvDiff(mvQ1x, mvP1x) || mvDiff(mvQ1y, mvP1y)) &&
                (mvDiff(mvQ1x, mvP0x) || mvDiff(mvQ1y, mvP0y) || mvDiff(mvQ0x, mvP1x) || mvDiff(mvQ0y, mvP1y))) ? 1 : 0;
    }
    return 1;
}

/* calcDP / calcDQ / useStrongFiltering (:249-268) */
static int calcDP(const pixel* s, intptr_t off) { return abs((int)s[-off * 3] - 2 * s[-off * 2] + s[-off]); }
static int calcDQ(const pixel* s, intptr_t off) { return abs((int)s[0] - 2 * s[off] + s[off * 2]); }
static int useStrong(intptr_t off, int beta, int tc, const pixel* s)
{
    int m4 = (int16_t)s[0], m3 = (int16_t)s[-off], m7 = (int16_t)s[off * 3], m0 = (int16_t)s[-off * 4];
    return (abs(m0 - m3) + abs(m7 - m4) < (beta >> 3)) && (abs(m3 - m4) < ((tc * 5 + 1) >> 1));
}

/* pelFilterLumaStrong_c (loopfilter.cpp:140-160) */
static void filterStrong(pixel* s, intptr_t step, intptr_t off, int tcP, int tcQ)
{
    for (int i = 0; i < 4; i++, s += step)
    {
        int m4 = (int16_t)s[0], m3 = (int16_t)s[-off], m5 = (int16_t)s[off], m2 = (int16_t)s[-off * 2];
        int m6 = (int16_t)s[off * 2], m1 = (int16_t)s[-off * 3], m7 = (int16_t)s[off * 3], m0 = (int16_t)s[-off * 4];
        s[-off * 3] = (pixel)(clip3(-tcP, tcP, ((2 * m0 + 3 * m1 + m2 + m3 + m4 + 4) >> 3) - m1) + m1);
        s[-off * 2] = (pixel)(clip3(-tcP, tcP, ((m1 + m2 + m3 + m4 + 2) >> 2) - m2) + m2);
        s[-off]     = (pixel)(clip3(-tcP, tcP, ((m1 + 2 * m2 + 2 * m3 + 2 * m4 + m5 + 4) >> 3) - m3) + m3);
        s[0]        = (pixel)(clip3(-tcQ, tcQ, ((m2 + 2 * m3 + 2 * m4 + 2 * m5 + m6 + 4) >> 3) - m4) + m4);
        s[off]      = (pixel)(clip3(-tcQ, tcQ, ((m3 + m4 + m5 + m6 + 2) >> 2) - m5) + m5);
        s[off * 2]  = (pixel)(clip3(-tcQ, tcQ, ((m3 + m4 + m5 + 3 * m6 + 2 * m7 + 4) >> 3) - m6) + m6);
    }
}

/* pelFilterLuma (:278-315) */
static void filterNormal(pixel* s, intptr_t step, intptr_t off, int tc, int maskP, int maskQ, int maskP1, int maskQ1)
{
    int thrCut = tc * 10, tc2 = tc >> 1;
    maskP1 &= maskP;
    maskQ1 &= maskQ;
    for (int i = 0; i < 4; i++, s += step)
    {
        int m4 = (int16_t)s[0], m3 = (int16_t)s[-off], m5 = (int16_t)s[off], m2 = (int16_t)s[-off * 2];
        int delta = (9 * (m4 - m3) - 3 * (m5 - m2) + 8) >> 4;
        if (abs(delta) < thrCut)
        {
            delta = clip3(-tc, tc, delta);
            s[-off] = (pixel)clipPel(m3 + (delta & maskP));
            s[0] = (pixel)clipPel(m4 - (delta & maskQ));
            if (maskP1)
            {
                int m1 = (int16_t)s[-off * 3];
                s[-off * 2] = (pixel)clipPel(m2 + clip3(-tc2, tc2, ((((m1 + m3 + 1) >> 1) - m2 + delta) >> 1)));
            }
            if (maskQ1)
            {
                int m6 = (int16_t)s[off * 2];
                s[off] = (pixel)clipPel(m5 + clip3(-tc2, tc2, ((((m6 + m4 + 1) >> 1) - m5 - delta) >> 1)));
            }
        }
    }
}

/* pelFilterChroma_c (loopfilter.cpp:167-181) */
static void filterChroma(pixel* s, intptr_t step, intptr_t off, int tc, int maskP, int maskQ)
{
    for (int i = 0; i < 4; i++, s += step)
    {
        int m4 = (int16_t)s[0], m3 = (int16_t)s[-off], m5 = (int16_t)s[off], m2 = (int16_t)s[-off * 2];
        int delta = clip3(-tc, tc, ((((m4 - m3) * 4) + m2 - m5 + 4) >> 3));
        s[-off] = (pixel)clipPel(m3 + (delta & maskP));
        s[0] = (pixel)clipPel(m4 - (delta & maskQ));
    }
}

/* One direction over the whole picture: for each 8-aligned edge (pos > 0) and each 4-line luma segment along it, the
 * decisions of edgeFilterLuma (:317-415); chroma edges every 16 luma samples, one 4-line chroma segment per 8 luma lines with
 * the BS and QPs of its first luma unit (edgeFilterChroma :417-497, deblockCU :104-113). */
static void deblock_dir(int dir, pixel* luma, intptr_t stride, pixel* cb, pixel* cr, intptr_t cstride, int width, int height,
                        const orc_dbk_unit* units, const int32_t* prm, int64_t* cnt)
{
    const int sliceType = prm[0], betaOffset = prm[1] * 2, tcOffset = prm[2] * 2, bypass = prm[5];
    const int shift = ORC_DEPTH - 8, upr = width >> 2;
    const int edgeLen = dir == EDGE_VER ? width : height, segs = (dir == EDGE_VER ? height : width) >> 2;
    for (int pos = 8; pos < edgeLen; pos += 8)
        for (int a = 0; a < segs; a++)
        {
            const orc_dbk_unit* Q = dir == EDGE_VER ? &units[a * upr + (pos >> 2)] : &units[(pos >> 2) * upr + a];
            const orc_dbk_unit* P = dir == EDGE_VER ? Q - 1 : Q - upr;
            int flag = edge_flag(Q, dir, pos);
            if (!flag)
                continue;
            int bs = boundary_strength(P, Q, flag, sliceType);
            cnt[bs == 0 ? CNT_BS0 : bs == 1 ? CNT_BS1 : CNT_BS2]++;
            if (!bs)
                continue;
            int maskP = -1, maskQ = -1;
            if (bypass)
            {
                maskP = (P->flags & 4) ? 0 : -1;
                maskQ = (Q->flags & 4) ? 0 : -1;
                if (!(maskP | maskQ))
                    continue;
            }
            int qp = (P->qp + Q->qp + 1) >> 1;

            /* luma */
            intptr_t off = dir == EDGE_VER ? 1 : stride, step = dir == EDGE_VER ? stride : 1;
            pixel* src = dir == EDGE_VER ? luma + (intptr_t)(4 * a) * stride + pos : luma + (intptr_t)pos * stride + 4 * a;
            int beta = betaTable[clip3(0, 51, qp + betaOffset)] << shift;
            int dp0 = calcDP(src, off), dq0 = calcDQ(src, off);
            int dp3 = calcDP(src + step * 3, off), dq3 = calcDQ(src + step * 3, off);
            int d0 = dp0 + dq0, d3 = dp3 + dq3;
            if (d0 + d3 >= beta)
                cnt[CNT_BETA_SKIP]++;
            else
            {
                int tc = tcTable[clip3(0, 51 + DEFAULT_INTRA_TC_OFFSET, qp + DEFAULT_INTRA_TC_OFFSET * (bs - 1) + tcOffset)] << shift;
                if (2 * d0 < (beta >> 2) && 2 * d3 < (beta >> 2) && useStrong(off, beta, tc, src) && useStrong(off, beta, tc, src + step * 3))
                {
                    cnt[CNT_STRONG]++;
                    filterStrong(src, step, off, (2 * tc) & maskP, (2 * tc) & maskQ);
                }
                else
                {
                    int side = (beta + (beta >> 1)) >> 3;
                    int maskP1 = dp0 + dp3 < side ? -1 : 0, maskQ1 = dq0 + dq3 < side ? -1 : 0;
                    int n = ((maskP1 & maskP) != 0) + ((maskQ1 & maskQ) != 0);
                    cnt[n == 2 ? CNT_NORMAL_BOTH : n == 1 ? CNT_NORMAL_ONE : CNT_NORMAL_NEITHER]++;
                    filterNormal(src, step, off, tc, maskP, maskQ, maskP1, maskQ1);
                }
            }

            /* chroma 4:2:0 */
            if (!cb || bs < 2 || (pos & 15) || (a & 1))
                continue;
            intptr_t coff = dir == EDGE_VER ? 1 : cstride, cstep = dir == EDGE_VER ? cstride : 1;
            intptr_t org = dir == EDGE_VER ? (intptr_t)(2 * a) * cstride + (pos >> 1) : (intptr_t)(pos >> 1) * cstride + 2 * a;
            for (int c = 0; c < 2; c++)
            {
                int qpc = qp + prm[3 + c];
                if (qpc >= 30)
                    qpc = chromaScale[qpc > 69 ? 69 : qpc];
                int tc = tcTable[clip3(0, 51 + DEFAULT_INTRA_TC_OFFSET, qpc + DEFAULT_INTRA_TC_OFFSET + tcOffset)] << shift;
                filterChroma((c ? cr : cb) + org, cstep, coff, tc, maskP, maskQ);
            }
            cnt[CNT_CHROMA]++;
        }
}

/* params: {sliceType, betaOffsetDiv2, tcOffsetDiv2, cbQpOffset, crQpOffset, transquantBypass} (x265cu_deblock_params);
 * cb = cr = NULL: luma only.  counters (CNT_N, may be NULL) are accumulated. */
int orc_deblock_frame(pixel* luma, intptr_t stride, pixel* cb, pixel* cr, intptr_t cstride, int width, int height,
                      const void* units, const int32_t* params, int64_t* counters)
{
    int64_t local[CNT_N] = { 0 };
    if ((width & 7) || (height & 7) || width <= 0 || height <= 0)
        return -1;
    deblock_dir(EDGE_VER, luma, stride, cb, cr, cstride, width, height, (const orc_dbk_unit*)units, params, local);
    deblock_dir(EDGE_HOR, luma, stride, cb, cr, cstride, width, height, (const orc_dbk_unit*)units, params, local);
    if (counters)
        for (int i = 0; i < CNT_N; i++)
            counters[i] += local[i];
    return 0;
}
