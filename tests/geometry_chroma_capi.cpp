// tests/geometry_chroma_capi.cpp -- CPU-only test shim: exposes the analyser's host-side geometry builder (x265_b200/csrc/
// geometry.h) and its 4:2:0 chroma residual helpers (geometry_chroma_tu / _reach / _qp) to tests/test_geometry_chroma.py.
#include "../x265_b200/csrc/geometry.h"
#include <string.h>

static FrameGeometry g_geo;

extern "C" {

int geo_build(int W, int H, int stride, int nref, int rect, int amp, int64_t* counts /* njobs, ncu, ntu, ctuRows, ncoef */)
{
    g_geo = FrameGeometry();
    geometry_build(W, H, stride, nref, rect, amp, g_geo);
    counts[0] = (int64_t)g_geo.pus.size(); counts[1] = (int64_t)g_geo.cus.size(); counts[2] = (int64_t)g_geo.tus.size();
    counts[3] = g_geo.ctuRows; counts[4] = g_geo.ncoef;
    return 0;
}

/* what: 1 cus (int64 x 4: x, y, size, coef_off), 2 tus (int32 x 3: cu, tx, ty), 6 rowTu (int32, ctuRows + 1) */
int geo_get(int what, void* out)
{
    switch (what)
    {
    case 1: { int64_t* o = (int64_t*)out; for (size_t i = 0; i < g_geo.cus.size(); i++) { const CuDesc& c = g_geo.cus[i];
              o[4 * i] = c.x; o[4 * i + 1] = c.y; o[4 * i + 2] = c.size; o[4 * i + 3] = c.coef_off; } break; }
    case 2: { int32_t* o = (int32_t*)out; for (size_t i = 0; i < g_geo.tus.size(); i++) { const TuDesc& t = g_geo.tus[i];
              o[3 * i] = t.cu; o[3 * i + 1] = t.tx; o[3 * i + 2] = t.ty; } break; }
    case 6: memcpy(out, g_geo.rowTu.data(), sizeof(int) * g_geo.rowTu.size()); break;
    default: return -1;
    }
    return 0;
}

/* every TU's chroma TU: int64 x 4 (x, y, size, first level) */
int geo_chroma_tus(int64_t* out)
{
    for (size_t i = 0; i < g_geo.tus.size(); i++)
    {
        const ChromaTu c = geometry_chroma_tu(g_geo.cus[g_geo.tus[i].cu], g_geo.tus[i]);
        out[4 * i] = c.x; out[4 * i + 1] = c.y; out[4 * i + 2] = c.size; out[4 * i + 3] = c.off;
    }
    return 0;
}

/* reach of the TUs [tu0, tu1) into out (x0, y0, x1, y1); returns geometry_chroma_reach_inside for a plane of cstride elements
 * per row with margins mx, my */
int geo_chroma_reach(int W, int H, int tu0, int tu1, int cstride, int mx, int my, int* out)
{
    const GeoRect r = geometry_chroma_reach(W, H, g_geo.cus, g_geo.tus, tu0, tu1);
    out[0] = r.x0; out[1] = r.y0; out[2] = r.x1; out[3] = r.y1;
    return geometry_chroma_reach_inside(r, W, H, cstride, mx, my) ? 1 : 0;
}

int geo_chroma_qp(int qp, int offset, int depth) { return geometry_chroma_qp(qp, offset, depth); }

} // extern "C"
