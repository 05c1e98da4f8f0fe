"""Helpers of the frame analyser's PART stage (stage bit 5: the inter estimate of every partition of a P slice's CUs): the CPU
drivers with it (oracle/frame_part.h, built by oracle/Makefile.part: liboracle_part{8,10}.so over the oracle,
oracle/_ref/libx265ref_part{8,10}.so over the reference), the ctypes view of their drv_part, the workloads of the tests, a run
of the CPU driver with the stage, the stage's invariants, and the store of the reference's results (tests/golden/part_ref.json)
for where oracle/_ref is not built."""
import copy
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

from common import ROOT, P, I, pixel_dtype
from frame_helpers import DrvFrame, Workload, cpu_analyse, pad_plane, pad_plane_c, MVRANGE
from ref_results import digest
from wref_helpers import DrvWref, PLANE_ARGS, search_planes, fade_workload, entry, identity, table, mvcost_tab_for

_libs = {}
PART_NAMES = ("2Nx2N", "2NxN", "Nx2N", "NxN", "2NxnU", "2NxnD", "nLx2N", "nRx2N")   # PartSize order of the record's entries
STAGES = 1 | 2 | 32                        # ME, luma residual (its cu_ref), PART


def load_oracle_part(depth):
    """The oracle with the PART stage (built on first use where build() has not built it)."""
    if ("orc", depth) not in _libs:
        path = os.path.join(ROOT, "oracle", "liboracle_part%d.so" % depth)
        if not os.path.exists(path):
            subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "-f", "Makefile.part", "oracle"],
                                  stdout=subprocess.DEVNULL)
        L = C.CDLL(path)
        L.orc_wref_planes.argtypes = PLANE_ARGS
        _libs[("orc", depth)] = L
    return _libs[("orc", depth)]


def load_ref_part(depth):
    """The reference-from-source library with the PART stage, or None where oracle/_ref is not built."""
    if ("ref", depth) not in _libs:
        path = os.path.join(ROOT, "oracle", "_ref", "libx265ref_part%d.so" % depth)
        L = None
        if os.path.exists(path):
            L = C.CDLL(path)
            L.x265ref_wref_planes.argtypes = PLANE_ARGS
        _libs[("ref", depth)] = L
    return _libs[("ref", depth)]


GOLDEN = os.path.join(ROOT, "tests", "golden", "part_ref.json")
_golden = {}


class PartRefResults:
    """tests/ref_results.RefResults for the PART stage, with its own store: `same(key, ref_fn, value)` asserts that `value`
    equals the reference's result (computed while oracle/_ref is built, else the stored digest).  X265_WRITE_GOLDEN=1 with
    oracle/_ref built stores the reference's digests instead of checking them."""

    def __init__(self, request, depth):
        self.R = load_ref_part(depth)
        self.test = "%s::%s" % (request.node.module.__name__, request.node.name)
        self.write = self.R is not None and os.environ.get("X265_WRITE_GOLDEN") == "1"
        if not _golden:
            _golden.update(json.load(open(GOLDEN)) if os.path.exists(GOLDEN) else {})
        if self.write:
            _golden[self.test] = {}
            request.addfinalizer(_save_golden)
        elif self.test not in _golden:
            pytest.fail("no stored reference results for %s in %s" % (self.test, GOLDEN))
        self.digests = _golden[self.test]

    def same(self, key, ref_fn, value):
        if self.R is None:
            assert digest(value) == self.digests[key], "%s differs from the reference's stored result" % key
            return
        r = ref_fn()
        assert digest(r) == digest(value), key
        if self.write:
            self.digests[key] = digest(r)
        else:
            assert digest(r) == self.digests[key], "the reference's %s differs from %s" % (key, GOLDEN)


def _save_golden():
    with open(GOLDEN, "w") as f:
        json.dump(_golden, f, indent=0, sort_keys=True)
        f.write("\n")


class DrvPart(C.Structure):
    _fields_ = [("w", DrvWref), ("out", P)]


class PartCu(C.Structure):
    """x265cu_part_cu (include/x265_b200.h)."""
    _fields_ = [("cost", C.c_uint32 * 8), ("sa8d", C.c_uint32 * 8), ("ref", (C.c_int8 * 2) * 8), ("mv", ((C.c_int16 * 2) * 2) * 8)]


# ---- workloads ----
KINDS = ("motion", "split", "tie", "fade")
# the weights of the "fade" workloads: slot 0 weighted in luma and chroma, slot 1 weighted in luma only (its Cb entry the
# identity, its Cr entry not present and not the identity: the prediction applies it all the same)
FADE_TABLE = [[entry(46, 5, 14), entry(60, 6, 9), entry(70, 6, -11)], [entry(75, 6, 10), identity(6), entry(50, 6, 7, 0)]]


def _texture(rng, H, W, depth):
    """Noise low-passed by a 3x3 box: detail at every position, smooth enough for the sub-pel filters."""
    n = rng.integers(0, 256, (H + 2, W + 2)).astype(np.int64)
    b = sum(n[dy:dy + H, dx:dx + W] for dy in range(3) for dx in range(3)) // 9
    return b << (depth - 8)


def _split_labels(H, W):
    """Per pixel 0 / 1: the two motions of the "split" content.  Each 64x64 tile is cut once, horizontally or vertically, at
    an offset of 8 to 56 that changes from tile to tile, so that CUs of every size see cuts at their halves and quarters."""
    yy, xx = np.mgrid[0:H, 0:W]
    tile = (yy // 64) * ((W + 63) // 64) + xx // 64
    offs = np.array([16, 32, 48, 8, 24, 40, 56])
    off = offs[tile % 7]
    horiz = (tile // 7 + tile) % 2 == 0
    return np.where(horiz, yy % 64 >= off, xx % 64 >= off).astype(np.int64)


def part_workload(W, H, depth, numRefs, kind, rect=1, amp=0, chroma=True, subme=3, qp=30, seed=265):
    """A P frame for the PART stage (4:2:0 planes throughout).  kind:
      "motion": the synthetic clip (frame_helpers.Workload), predictors against its motion;
      "split":  a textured picture whose two parts (_split_labels) move differently: in reference r one part is the source
                moved by (2, -2) * (r + 1) px, the other by (-4, 4) * (r + 1) px, so that rect and AMP partitions whose PUs
                follow the cut beat 2Nx2N; predictors zero;
      "tie":    the clip with slot 1 holding slot 0's picture and predictors: every PU's jobs on slots 0 and 1 tie;
      "fade":   the clip's frames darkened towards black (wref_helpers.fade_workload), for FADE_TABLE."""
    assert kind in KINDS, kind
    if kind == "fade":
        wl = fade_workload(W, H, depth, numRefs, subme=subme, qp=qp, seed=seed)
        wl.params.update(rect=rect, amp=amp)
        return wl
    wl = Workload(W, H, depth=depth, numRefs=numRefs, subme=subme, rect=rect, amp=amp, qp=qp, seed=seed, chroma=True,
                  field="zero" if kind == "split" else "against")
    if kind == "tie":
        assert numRefs >= 2
        wl.refs[1] = wl.refs[0].copy()
        wl.refC[1] = [c.copy() for c in wl.refC[0]]
        wl.field[1] = wl.field[0]
    elif kind == "split":
        rng = np.random.default_rng(seed)
        M = 32
        base = _texture(rng, H + 2 * M, W + 2 * M, depth)
        basec = [_texture(rng, H // 2 + M, W // 2 + M, depth) for _ in range(2)]
        lab = _split_labels(H, W)
        labc = lab[::2, ::2]
        wl.fenc = pad_plane(base[M:M + H, M:M + W], depth)[0]
        wl.fencC = [pad_plane_c(b[M // 2:M // 2 + H // 2, M // 2:M // 2 + W // 2], depth, wl.stride)[0] for b in basec]
        for r in range(numRefs):
            (ax, ay), (bx, by) = (2 * (r + 1), -2 * (r + 1)), (-4 * (r + 1), 4 * (r + 1))
            # reference pixel (x, y) of a part moved by (vx, vy) is source pixel (x - vx, y - vy)
            a = base[M - ay:M - ay + H, M - ax:M - ax + W]
            b = base[M - by:M - by + H, M - bx:M - bx + W]
            wl.refs[r] = pad_plane(np.where(lab == 1, b, a).astype(pixel_dtype(depth)), depth)[0]
            m = M // 2
            wl.refC[r] = [pad_plane_c(np.where(labc == 1, c[m - by // 2:m - by // 2 + H // 2, m - bx // 2:m - bx // 2 + W // 2],
                                               c[m - ay // 2:m - ay // 2 + H // 2, m - ax // 2:m - ax // 2 + W // 2]).astype(pixel_dtype(depth)),
                                      depth, wl.stride)[0] for c in basec]
        wl.fenc = wl.fenc.astype(pixel_dtype(depth))
    return wl


class _PartEntry:
    """Stands in for a driver entry point in frame_helpers.cpu_analyse: calls the PART one with `pt`."""

    def __init__(self, fn, pt):
        self.fn, self.pt = fn, pt
        fn.argtypes = [C.POINTER(DrvFrame), I, C.POINTER(DrvPart)]
        fn.restype = I

    def __call__(self, frame, stages):
        assert self.fn(frame, stages, C.byref(self.pt)) == 0


class _Lib:
    def __init__(self, name, entry):
        setattr(self, name, entry)


def cpu_analyse_part(lib, prefix, wl, chroma, tab=None, threads=4, max_ctu_rows=0, stages=STAGES):
    """The CPU driver with the PART stage (prefix "orc": the oracle, "x265ref": the reference), chroma planes in the ME and in
    PART iff `chroma`; with a weight table `tab` ([numRefs][3][4], wref_helpers.table) the search reads each weighted slot's
    weighted planes and PART weights its prediction.  Returns frame_helpers.cpu_analyse's result plus "part" (PART_CU
    records)."""
    from x265_b200.lib import PART_CU
    fn_name = "%s_analyse_frame_part" % prefix
    ctus = ((wl.W + 63) // 64) * ((wl.H + 63) // 64)
    out = np.zeros(ctus * 85, PART_CU)
    es = np.dtype(pixel_dtype(wl.depth)).itemsize
    pt = DrvPart()
    pt.out = out.ctypes.data
    sw = copy.copy(wl)
    sw.chroma = chroma
    nr = wl.params["numRefs"]
    for r in range(nr):
        pt.w.refs[r] = wl.refs[r].ctypes.data + wl.org * es
        for k in range(2):
            pt.w.refC[r][k] = wl.refC[r][k].ctypes.data + wl.corg * es
    if tab is not None:
        for r in range(nr):
            for k in range(3):
                for j in range(4):
                    pt.w.wp[r][k][j] = int(tab[r][k][j])
        sw.refs, sw.refC, _ = search_planes(lib, "%s_wref_planes" % prefix, wl, tab)
    res = cpu_analyse(_Lib(fn_name, _PartEntry(getattr(lib, fn_name), pt)), fn_name, sw, mvcost_tab_for(wl), threads=threads,
                      stages=stages, max_ctu_rows=max_ctu_rows)
    res["part"] = out[:res["ncu"]]
    return res


def summary(res):
    """What the PART pin compares: every PART record byte for byte and the ME results it reads."""
    return dict(part=np.frombuffer(res["part"].tobytes(), np.uint8), me=res["me_out"][:, :3])


def check_invariants(res, wl, kind):
    """The stage's invariants on a CPU driver result: each PU's slot is the first arg-min of its jobs' ME costs and its vector
    that job's; the 2Nx2N slot is cu_ref; cost - sa8d is the PUs' summed mvcost; entries not evaluated hold the sentinels.  On
    "split" content every partition the geometry emits is the lowest-cost entry of some CU; on "tie" content slot 1 is never
    taken.  Returns the number of PUs whose slots 0 and 1 tie."""
    p, nr = wl.params, wl.params["numRefs"]
    part, me, cu_jobs, cus = res["part"], res["me_out"], res["cu_jobs"], res["cus"]
    qmvp = res["jobs"]["qmvp"].astype(np.int64)
    tab = mvcost_tab_for(wl).astype(np.int64)
    assert (part["ref"][:, 0, 0] == res["cu_ref"]).all()
    assert (part["cost"][:, 3] == 0xffffffff).all() and (part["ref"][:, 3] == -1).all()
    ties, wins = 0, set()
    for c in range(res["ncu"]):
        S, k = int(cus[c][2]), 0
        for ps in range(8):
            on = ps == 0 or (ps in (1, 2) and p["rect"]) or (ps >= 4 and p["amp"] and S >= 16)
            if not on:
                assert part["cost"][c, ps] == part["sa8d"][c, ps] == 0xffffffff and (part["ref"][c, ps] == -1).all()
                assert (part["mv"][c, ps] == 0).all()
                continue
            npu, mvc = (2 if ps else 1), 0
            for u in range(npu):
                jobs = cu_jobs[c] + k + u
                costs = me[jobs, 0]
                best = int(np.argmin(costs))
                assert part["ref"][c, ps, u] == best, (c, ps, u)
                assert tuple(part["mv"][c, ps, u]) == tuple(me[jobs[best], 1:3]), (c, ps, u)
                ties += nr > 1 and costs[0] == costs[1]
                d = me[jobs[best], 1:3].astype(np.int64) - qmvp[jobs[best]]
                mvc += (tab[MVRANGE + d[0]] + tab[MVRANGE + d[1]]) & 0xffff
            if npu == 1:
                assert part["ref"][c, ps, 1] == -1 and (part["mv"][c, ps, 1] == 0).all()
            assert int(part["cost"][c, ps]) - int(part["sa8d"][c, ps]) == mvc, (c, ps)
            k += npu
        wins.add(int(np.argmin(part["cost"][c])))
    if kind == "split":
        emitted = {0} | ({1, 2} if p["rect"] else set()) | ({4, 5, 6, 7} if p["amp"] else set())
        assert wins == emitted, sorted(wins)
    if kind == "tie":
        assert ties > 0 and not (part["ref"] == 1).any()
    return ties


# (depth, numRefs, (rect, amp), chroma, (W, H), kind): 8 and 10 bit, 1 to 3 references, rect only / rect + AMP / neither, chroma
# on and off, a picture ending in a partial CTU in both directions (328x200)
SIZES = ((200, 136), (328, 200))
CASES = [(8, 1, (1, 0), True, SIZES[0], "motion"),
         (10, 3, (1, 0), False, SIZES[1], "motion"),
         (10, 1, (0, 0), True, SIZES[0], "motion"),
         (8, 2, (0, 0), False, SIZES[1], "split"),
         (8, 2, (1, 1), True, SIZES[1], "split"),
         (10, 3, (1, 1), False, SIZES[1], "split"),
         (10, 1, (1, 0), True, SIZES[1], "split"),
         (8, 2, (1, 0), False, SIZES[0], "tie"),
         (10, 3, (1, 1), True, SIZES[0], "tie"),
         (8, 2, (1, 1), True, SIZES[1], "fade"),
         (10, 2, (1, 0), True, SIZES[0], "fade")]


def case_id(c):
    d, nr, (rect, amp), ch, (W, H), kind = c
    geo = "rect+amp" if amp else ("rect" if rect else "2Nx2N")
    return "%s-%d-%dref-%s-%s-%dx%d" % (kind, d, nr, geo, "chroma" if ch else "luma", W, H)


def case_workload(case):
    """The workload of a case and its weight table (None: no slot weighted)."""
    d, nr, (rect, amp), ch, (W, H), kind = case
    wl = part_workload(W, H, d, nr, kind, rect=rect, amp=amp)
    return wl, (table(FADE_TABLE[:nr]) if kind == "fade" else None)
