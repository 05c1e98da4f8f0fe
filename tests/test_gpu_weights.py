"""GPU parity of the lookahead's weighted-prediction analysis (x265cu_lookahead_weights_analyse = LookaheadTLD::weightsAnalyse
+ weightCostLuma, slicetype.cpp:807-961) against the oracle, which tests/test_lookahead_oracle_vs_ref.py pins to the real
class: the decision, the weight parameters and the 4 re-weighted lowres planes (whole padded buffers), 8 and 10 bit.
The device call is host decision logic over launches of kernels the other GPU tests already cover (weight_pp block op,
grid SATD); first run green on the round-1 driver box (GPUTEST_r01.json)."""
import ctypes as C

import numpy as np
import pytest

from common import load_oracle, ptr, P, I, IP, pixel_dtype
from frame_helpers import MARGIN_X, MARGIN_Y
from lookahead_helpers import OracleLookahead
from test_lookahead_oracle_vs_ref import _wp_stats, weights_decision, weights_frames

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cu():
    import x265_b200
    return x265_b200.load()


@pytest.mark.timeout(180)
@pytest.mark.parametrize("depth", [8, 10])
@pytest.mark.parametrize("case", ["same", "fade", "fade2", "bright", "offset", "from_black_dark", "from_black_bright", "to_black", "constant"])
def test_weights_analyse(cu, depth, case):
    O = load_oracle(depth)
    frames = weights_frames(case, depth)
    orc = OracleLookahead(O, frames, depth)
    planes = [orc.fr[f]["planes"] for f in range(2)]                   # whole padded buffers (Lowres::buffer[i])
    rows, stride = planes[0][0].shape
    planesize = rows * stride
    padoffset = MARGIN_Y * stride + MARGIN_X
    lw, lh = orc.w8 * 8, orc.h8 * 8
    intra = np.ascontiguousarray(orc.fr[1]["intraCost"], np.int32)
    stats = np.array(list(_wp_stats(frames[1])) + list(_wp_stats(frames[0])), np.uint64)

    refarr = (P * 4)(*[C.c_void_p(b.ctypes.data) for b in planes[0]])
    worc = np.zeros(4 * planesize, pixel_dtype(depth))
    wp = np.zeros(3, np.int32)
    O.orc_la_weights_analyse.argtypes = [P, P, P, IP, IP, I, I, IP, P, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, P]
    want = O.orc_la_weights_analyse(ptr(planes[1][0]), refarr, ptr(worc), planesize, stride, lw, lh, padoffset, ptr(intra),
                                    int(stats[0]), int(stats[1]), int(stats[2]), int(stats[3]), ptr(wp))
    assert want == weights_decision(case)

    d_fenc = cu.to_device(planes[1][0])
    d_refs = [cu.to_device(p) for p in planes[0]]
    d_w = cu.alloc(4 * planesize * worc.itemsize)
    got = cu.lookahead_weights_analyse(depth, d_fenc, d_refs, d_w, planesize, stride, lw, lh, padoffset, intra, stats)
    assert got[0] == want
    if want:
        assert list(got[1:]) == wp.tolist()
        assert np.array_equal(d_w.download(pixel_dtype(depth)), worc)
    for d in [d_fenc, d_w] + d_refs:
        d.free()
