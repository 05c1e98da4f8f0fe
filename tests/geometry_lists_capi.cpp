// tests/geometry_lists_capi.cpp -- CPU-only test shim: the per-size TU and CU work lists of the analyser's host-side
// geometry builder (x265_b200/csrc/geometry.h) for tests/test_geometry_lists.py.
#include "../x265_b200/csrc/geometry.h"
#include <string.h>

static FrameGeometry g_geo;

extern "C" {

// counts: ntu, ncu, ctuRows
int geo_build(int W, int H, int stride, int nref, int rect, int amp, int64_t* counts)
{
    g_geo = FrameGeometry();
    geometry_build(W, H, stride, nref, rect, amp, g_geo);
    counts[0] = (int64_t)g_geo.tus.size(); counts[1] = (int64_t)g_geo.cus.size(); counts[2] = g_geo.ctuRows;
    return 0;
}

/* what: 0 CU size of every TU's CU (int32, ntu), 1 CU sizes (int32, ncu), 2 rowTu, 3 rowCu (int32, ctuRows + 1);
 * 10 + k: tuBy[k] (k = 0..2), 20 + k: rowTuBy[k]; 30 + k: cuBy[k] (k = 0..3), 40 + k: rowCuBy[k].  Returns the element
 * count, or -1. */
int geo_get(int what, int32_t* out)
{
    const std::vector<int>* v = NULL;
    if (what == 0) { for (size_t i = 0; i < g_geo.tus.size(); i++) out[i] = g_geo.cus[g_geo.tus[i].cu].size; return (int)g_geo.tus.size(); }
    if (what == 1) { for (size_t i = 0; i < g_geo.cus.size(); i++) out[i] = g_geo.cus[i].size; return (int)g_geo.cus.size(); }
    if (what == 2) v = &g_geo.rowTu;
    else if (what == 3) v = &g_geo.rowCu;
    else if (what >= 10 && what < 13) v = &g_geo.tuBy[what - 10];
    else if (what >= 20 && what < 23) v = &g_geo.rowTuBy[what - 20];
    else if (what >= 30 && what < 34) v = &g_geo.cuBy[what - 30];
    else if (what >= 40 && what < 44) v = &g_geo.rowCuBy[what - 40];
    else return -1;
    if (out) memcpy(out, v->data(), sizeof(int32_t) * v->size());
    return (int)v->size();
}

} // extern "C"
