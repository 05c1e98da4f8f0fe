/* oracle/oracle_aq.c -- TEST INFRASTRUCTURE ONLY: LookaheadTLD::calcAdaptiveQuantFrame (encoder/slicetype.cpp:444-694)
 * restated in plain C, the energies (acEnergyCu, :49-84, 256-275) from the pixels and the float decision after them.
 * Pinned to the real function by oracle/ref_shim_aq.cpp (tests/test_aq_oracle_vs_ref.py); the device pass and the
 * library's finish are compared with it.  Reads past the picture take the nearest in-picture sample, as the reference
 * reads PicYuv's replicated padding.  Built by Makefile.aq with -ffp-contract=off and without fast-math. */
#include <math.h>
#include <stdint.h>
#include <string.h>

typedef struct {
    int32_t aqMode, qgSize, weightp, variance, hevcAq, hdr10Opt, aqMotion, reserved;
    double aqStrength;
    const float* quantOffsets;
} OrcAqParams;

static uint32_t px(const void* pl, int depth, int stride, int w, int h, int x, int y)
{
    if (x > w - 1) x = w - 1;
    if (y > h - 1) y = h - 1;
    return depth == 8 ? ((const uint8_t*)pl)[(intptr_t)y * stride + x] : ((const uint16_t*)pl)[(intptr_t)y * stride + x];
}

/* acEnergyVar on var of an n x n block (pixel.cpp:704-720) */
static uint32_t energy_var(const void* pl, int depth, int stride, int w, int h, int x0, int y0, int n, int shift,
                           uint64_t* tot)
{
    uint32_t sum = 0, ssd = 0;
    for (int y = 0; y < n; y++)
        for (int x = 0; x < n; x++)
        {
            uint32_t v = px(pl, depth, stride, w, h, x0 + x, y0 + y);
            sum += v; ssd += v * v;
        }
    tot[0] += sum; tot[1] += ssd;
    return (uint32_t)(ssd - ((uint64_t)sum * sum >> shift));
}

static uint32_t energy_cu(const void* const* pl, int depth, int stride, int cstride, int W, int H, int bx, int by, int qg,
                          uint64_t* tot)
{
    uint32_t e = qg == 8 ? energy_var(pl[0], depth, stride, W, H, bx, by, 8, 6, tot)
                         : energy_var(pl[0], depth, stride, W, H, bx, by, 16, 8, tot);
    if (pl[1])
        for (int c = 1; c < 3; c++)
            e += qg == 8 ? energy_var(pl[c], depth, cstride, W / 2, H / 2, bx >> 1, by >> 1, 4, 4, tot + 2 * c)
                         : energy_var(pl[c], depth, cstride, W / 2, H / 2, bx >> 1, by >> 1, 8, 6, tot + 2 * c);
    return e;
}

/* energies of the ceil(W / L) x ceil(H / L) grid and one pass's plane totals [3][2] (x265cu_aq_energy's outputs) */
void orc_aq_energy(int depth, const void* y, int stride, const void* cb, const void* cr, int cstride, int W, int H, int qg,
                   uint32_t* energy, uint64_t* totals)
{
    const void* pl[3] = { y, cb, cr };
    const int L = qg == 8 ? 8 : 16;
    memset(totals, 0, 6 * sizeof(uint64_t));
    int b = 0;
    for (int by = 0; by < H; by += L)
        for (int bx = 0; bx < W; bx += L)
            energy[b++] = energy_cu(pl, depth, stride, cstride, W, H, bx, by, qg, totals);
}

static const uint8_t* exp2_lut(void)
{
    static uint8_t lut[64];
    static int done;
    if (!done)
    {
        for (int i = 0; i < 64; i++) lut[i] = (uint8_t)floor((exp2(i / 64.0) - 1) * 256 + 0.5);
        done = 1;
    }
    return lut;
}

/* x265_exp2fix8 (common/common.cpp:96-103) */
static int exp2fix8(double x)
{
    int i = (int)(x * (-64.f / 6.f) + 512.5f);
    if (i < 0) return 0;
    if (i > 1023) return 0xffff;
    return (exp2_lut()[i & 63] + 256) << (i >> 6) >> 8;
}

/* The whole function on the pixels.  Arrays are in / out, as the reference's Lowres fields: qpAqOffset (also what
 * qpCuTreeOffset receives), invQscaleFactor and blockVariance blockCount long, invQscaleFactor8x8 w8 * h8. */
void orc_aq(int depth, const void* y, int stride, const void* cb, const void* cr, int cstride, int W, int H,
            const OrcAqParams* p, double* qpAqOffset, int32_t* invq, int32_t* invq8, uint64_t* wp_sum, uint64_t* wp_ssd,
            uint32_t* blockVariance, double* frameVariance)
{
    const void* pl[3] = { y, cb, cr };
    const int qg = p->qgSize, L = qg == 8 ? 8 : 16;
    const int w8 = ((W / 2) + 7) >> 3, h8 = ((H / 2) + 7) >> 3;
    const int blockCount = qg == 8 ? (2 * w8) * (2 * h8) : w8 * h8;
    const float modeOneConst = qg == 8 ? 11.427f : 14.427f, modeTwoConst = qg == 8 ? 8.f : 11.f;
    const float* quantOffsets = p->quantOffsets;
    uint64_t tot[6] = { 0 };
    double cut[blockCount];
    int maxCol = W, maxRow = H;

    if (p->aqMode == 0 || p->aqStrength == 0)
    {
        if (p->aqMode && p->aqStrength == 0)
            for (int i = 0; i < blockCount; i++)
            {
                qpAqOffset[i] = quantOffsets ? quantOffsets[i] : 0;
                invq[i] = quantOffsets ? exp2fix8(qpAqOffset[i]) : 256;
            }
        if (p->weightp)
            for (int by = 0; by < maxRow; by += L)
                for (int bx = 0; bx < maxCol; bx += L)
                    energy_cu(pl, depth, stride, cstride, W, H, bx, by, qg, tot);
    }
    else
    {
        int b = 0;
        double avg_adj_pow2 = 0, avg_adj = 0, qp_adj = 0, bias_strength = 0.f, strength = 0.f;
        if (p->aqMode == 2 || p->aqMode == 3)
        {
            double bit_depth_correction = 1.f / (1 << (2 * (depth - 8)));
            for (int by = 0; by < maxRow; by += L)
                for (int bx = 0; bx < maxCol; bx += L)
                {
                    uint32_t energy = energy_cu(pl, depth, stride, cstride, W, H, bx, by, qg, tot);
                    qp_adj = pow(energy * bit_depth_correction + 1, 0.1);
                    cut[b] = qp_adj;
                    avg_adj += qp_adj;
                    avg_adj_pow2 += qp_adj * qp_adj;
                    b++;
                }
            avg_adj /= blockCount;
            avg_adj_pow2 /= blockCount;
            strength = p->aqStrength * avg_adj;
            avg_adj = avg_adj - 0.5f * (avg_adj_pow2 - modeTwoConst) / avg_adj;
            bias_strength = p->aqStrength;
        }
        else
            strength = p->aqStrength * 1.0397f;
        b = 0;
        for (int by = 0; by < maxRow; by += L)
            for (int bx = 0; bx < maxCol; bx += L)
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
                    uint32_t energy = energy_cu(pl, depth, stride, cstride, W, H, bx, by, qg, tot);
                    qp_adj = strength * (log2(energy > 1 ? energy : 1) - (modeOneConst + 2 * (depth - 8)));
                }
                if (quantOffsets)
                    qp_adj += quantOffsets[b];
                qpAqOffset[b] = qp_adj;
                invq[b] = exp2fix8(qp_adj);
                b++;
            }
    }
    if (qg == 8 && invq8)
        for (int cuY = 0; cuY < h8; cuY++)
            for (int cuX = 0; cuX < w8; cuX++)
                invq8[cuX + cuY * w8] = (invq[cuX * 2 + cuY * w8 * 4] + invq[cuX * 2 + cuY * w8 * 4 + 1] +
                                         invq[cuX * 2 + cuY * w8 * 4 + 2 * w8] + invq[cuX * 2 + cuY * w8 * 4 + 2 * w8 + 1]) / 4;
    if (p->weightp)
    {
        maxCol = ((maxCol + 8) >> 4) << 4;
        maxRow = ((maxRow + 8) >> 4) << 4;
        const int sh = pl[1] ? 1 : 0;                               /* CHROMA_H_SHIFT / V_SHIFT: 4:2:0 or 4:0:0 */
        int width[3] = { maxCol, maxCol >> sh, maxCol >> sh };
        int height[3] = { maxRow, maxRow >> sh, maxRow >> sh };
        for (int i = 0; i < 3; i++)
        {
            uint64_t sum = tot[2 * i], ssd = tot[2 * i + 1];
            tot[2 * i + 1] = ssd - (sum * sum + (width[i] * height[i]) / 2) / (width[i] * height[i]);
        }
    }
    if (p->variance)
    {
        uint64_t b = 0, rowVariance = 0;
        double fv = 0;
        for (int by = 0; by < maxRow; by += L)
        {
            for (int bx = 0; bx < maxCol; bx += L)
            {
                blockVariance[b] = energy_cu(pl, depth, stride, cstride, W, H, bx, by, qg, tot);
                rowVariance += blockVariance[b];
                b++;
            }
            fv += (rowVariance / maxCol);
        }
        fv /= maxRow;
        *frameVariance = fv;
    }
    for (int i = 0; i < 3; i++)
    {
        wp_sum[i] = tot[2 * i];
        wp_ssd[i] = tot[2 * i + 1];
    }
}
