"""Helpers of the frame analyser's PART_B stage (stage bit 6: the inter estimate of every partition of a B slice's CUs): the
CPU drivers with it (oracle/frame_part_b.h, built by oracle/Makefile.part_b: liboracle_part_b{8,10}.so over the oracle,
oracle/_ref/libx265ref_part_b{8,10}.so over the reference), the ctypes view of their drv_part_b, the B-frame workloads of the tests, a run of the CPU driver with the
stage, the stage's invariants, and the store of the reference's results (tests/golden/part_b_ref.json) for where oracle/_ref
is not built."""
import copy
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

from common import ROOT, P, I, pixel_dtype
from frame_helpers import DrvFrame, cpu_analyse, pad_plane, pad_plane_c, MVRANGE
from ref_results import digest
from wref_helpers import DrvWref, PLANE_ARGS, mvcost_tab_for
from bidir_helpers import bidir_workload
from part_helpers import _texture, _split_labels

_libs = {}
# decision counters of drv_part_b (frame_part_b.h), per PU
COUNTERS = ("bi", "uni_l0", "uni_l1", "tie_l0", "bi_cu8", "chroma_satd", "avg_pp", "zero_tried", "zero_taken", "zero_out_of_range",
            "zero_skipped")
STAGES = 1 | 64                            # ME, PART_B


def load_oracle_part_b(depth):
    """The oracle with the PART_B stage (built on first use where build() has not built it)."""
    if ("orc", depth) not in _libs:
        path = os.path.join(ROOT, "oracle", "liboracle_part_b%d.so" % depth)
        if not os.path.exists(path):
            subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "-f", "Makefile.part_b", "oracle"],
                                  stdout=subprocess.DEVNULL)
        L = C.CDLL(path)
        L.orc_wref_planes.argtypes = PLANE_ARGS
        _libs[("orc", depth)] = L
    return _libs[("orc", depth)]


def load_ref_part_b(depth):
    """The reference-from-source library with the PART_B stage, or None where oracle/_ref is not built."""
    if ("ref", depth) not in _libs:
        path = os.path.join(ROOT, "oracle", "_ref", "libx265ref_part_b%d.so" % depth)
        L = None
        if os.path.exists(path):
            L = C.CDLL(path)
            L.x265ref_wref_planes.argtypes = PLANE_ARGS
        _libs[("ref", depth)] = L
    return _libs[("ref", depth)]


GOLDEN = os.path.join(ROOT, "tests", "golden", "part_b_ref.json")
_golden = {}


class PartBRefResults:
    """tests/ref_results.RefResults for the PART_B stage, with its own store: `same(key, ref_fn, value)` asserts that `value`
    equals the reference's result (computed while oracle/_ref is built, else the stored digest).  X265_WRITE_GOLDEN=1 with
    oracle/_ref built stores the reference's digests instead of checking them."""

    def __init__(self, request, R):
        self.R = R
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


class DrvPartB(C.Structure):
    _fields_ = [("w", DrvWref), ("numRefL0", I), ("out", P), ("counts", I * len(COUNTERS))]


class PartBCu(C.Structure):
    """x265cu_part_b_cu (include/x265_b200.h)."""
    _fields_ = [("cost", C.c_uint32 * 8), ("sa8d", C.c_uint32 * 8), ("biCost", (C.c_uint32 * 2) * 8), ("interDir", (C.c_int8 * 2) * 8),
                ("ref", ((C.c_int8 * 2) * 2) * 8), ("zero", (C.c_uint8 * 2) * 8), ("mv", (((C.c_int16 * 2) * 2) * 2) * 8)]


# ---- B-frame workloads ----
KINDS = ("occlusion", "average", "cut", "gpb", "static")


def part_b_workload(W, H, depth, n0, n1, kind, rect=1, amp=0, subme=3, qp=22, seed=265):
    """A B frame for the PART_B stage (4:2:0 planes throughout), list 0 in slots [0, n0), list 1 in [n0, n0 + n1).  kind:
      "occlusion": a textured picture cut in two parts per 64x64 tile (part_helpers._split_labels); in list-0 slot r part 0
                   is the source moved by (2, -2) * (r + 1) px and part 1 another texture, in list-1 slot i part 1 is the
                   source moved by (-4, 4) * (i + 1) px and part 0 another texture: the two PUs of a partition that follows
                   a cut match different lists; predictors zero;
      "average":   bidir_helpers' "between" frame with the source replaced by the rounded mean of the first list-0 and the
                   first list-1 picture: the bi-prediction matches it, so bi wins;
      "cut":       bidir_helpers' "cut": list 0 is another scene, so list-1 uni wins;
      "gpb":       bidir_helpers' "tie" (n0 == n1): the same pictures and predictors in both lists, so ties go to list 0;
      "static":    bidir_helpers' "static": the zero pair skipped (both vectors zero), tried and taken, and refused by the
                   range test where the far predictors leave the CU's range."""
    assert kind in KINDS, kind
    base_kind = dict(occlusion="between", average="between", cut="cut", gpb="tie", static="static")[kind]
    wl = bidir_workload(W, H, depth, n0, n1, base_kind, qp=qp, seed=seed)
    wl.params.update(rect=rect, amp=amp, subme=subme)
    dt = pixel_dtype(depth)
    if kind == "average":
        mean = lambda a, b: ((a.astype(np.int64) + b + 1) >> 1).astype(dt)
        wl.fenc = mean(wl.refs[0], wl.refs[n0])
        wl.fencC = [mean(wl.refC[0][k], wl.refC[n0][k]) for k in range(2)]
    elif kind == "occlusion":
        rng = np.random.default_rng(seed)
        M = 32
        src = _texture(rng, H + 2 * M, W + 2 * M, depth)
        other = _texture(rng, H + 2 * M, W + 2 * M, depth)
        srcc = [_texture(rng, H // 2 + M, W // 2 + M, depth) for _ in range(2)]
        otherc = [_texture(rng, H // 2 + M, W // 2 + M, depth) for _ in range(2)]
        lab = _split_labels(H, W)
        labc = lab[::2, ::2]
        m = M // 2
        wl.fenc = pad_plane(src[M:M + H, M:M + W].astype(dt), depth)[0]
        wl.fencC = [pad_plane_c(b[m:m + H // 2, m:m + W // 2].astype(dt), depth, wl.stride)[0] for b in srcc]
        for r in range(n0 + n1):
            part = 0 if r < n0 else 1
            i = r if r < n0 else r - n0
            vx, vy = (2 * (i + 1), -2 * (i + 1)) if part == 0 else (-4 * (i + 1), 4 * (i + 1))
            # reference pixel (x, y) of a part moved by (vx, vy) is source pixel (x - vx, y - vy)
            moved = src[M - vy:M - vy + H, M - vx:M - vx + W]
            wl.refs[r] = pad_plane(np.where(lab == part, moved, other[M:M + H, M:M + W]).astype(dt), depth)[0]
            wl.refC[r] = [pad_plane_c(np.where(labc == part, c[m - vy // 2:m - vy // 2 + H // 2, m - vx // 2:m - vx // 2 + W // 2],
                                               o[m:m + H // 2, m:m + W // 2]).astype(dt), depth, wl.stride)[0]
                          for c, o in zip(srcc, otherc)]
        wl.field = np.zeros_like(wl.field)
    return wl


class _PartBEntry:
    """Stands in for a driver entry point in frame_helpers.cpu_analyse: calls the PART_B one with `pb`."""

    def __init__(self, fn, pb):
        self.fn, self.pb = fn, pb
        fn.argtypes = [C.POINTER(DrvFrame), I, C.POINTER(DrvPartB)]
        fn.restype = I

    def __call__(self, frame, stages):
        assert self.fn(frame, stages, C.byref(self.pb)) == 0


class _Lib:
    def __init__(self, name, entry):
        setattr(self, name, entry)


def cpu_analyse_part_b(lib, prefix, wl, n0, chroma, threads=4, max_ctu_rows=0, stages=STAGES):
    """The CPU driver with the PART_B stage (prefix "orc": the oracle, "x265ref": the reference), list 0 = slots [0, n0),
    chroma planes in the ME and in PART_B iff `chroma`.  Returns frame_helpers.cpu_analyse's result plus "part_b" (PART_B_CU
    records) and "counts" (COUNTERS)."""
    from x265_b200.lib import PART_B_CU
    fn_name = "%s_analyse_frame_part_b" % prefix
    ctus = ((wl.W + 63) // 64) * ((wl.H + 63) // 64)
    out = np.zeros(ctus * 85, PART_B_CU)
    es = np.dtype(pixel_dtype(wl.depth)).itemsize
    pb = DrvPartB()
    pb.out, pb.numRefL0 = out.ctypes.data, n0
    sw = copy.copy(wl)
    sw.chroma = chroma
    for r in range(wl.params["numRefs"]):
        pb.w.refs[r] = wl.refs[r].ctypes.data + wl.org * es
        for k in range(2):
            pb.w.refC[r][k] = wl.refC[r][k].ctypes.data + wl.corg * es
    res = cpu_analyse(_Lib(fn_name, _PartBEntry(getattr(lib, fn_name), pb)), fn_name, sw, mvcost_tab_for(wl), threads=threads,
                      stages=stages, max_ctu_rows=max_ctu_rows)
    res["part_b"] = out[:res["ncu"]]
    res["counts"] = dict(zip(COUNTERS, list(pb.counts)))
    return res


def summary(res):
    """What the PART_B pin compares: every PART_B record byte for byte, the ME results it reads, and the decision counters."""
    return dict(part_b=np.frombuffer(res["part_b"].tobytes(), np.uint8), me=res["me_out"][:, :3],
                counts=np.array([res["counts"][k] for k in COUNTERS], np.int64))


def _emitted(p, S, ps):
    return ps == 0 or (ps in (1, 2) and p["rect"]) or (ps >= 4 and p["amp"] and S >= 16)


def used_pu(res, c, ps, u, k):
    """(slot, vector) the PU's prediction uses when it is uni-directional: its list's slot and that job's ME vector."""
    pb = res["part_b"]
    d = int(pb["interDir"][c, ps, u])
    slot = int(pb["ref"][c, ps, u, d - 1])
    return slot, tuple(res["me_out"][res["cu_jobs"][c, slot] + k, 1:3])


def check_invariants(res, wl, n0):
    """The stage's invariants on a CPU driver result: each PU's per-list slot is the first arg-min of that list's jobs; interDir
    3 only off 2Nx2N and at CU >= 16; bi iff biCost < min(cost0, cost1), else L0 iff cost0 <= cost1; a zero pair has both
    vectors 0 and a PU without it its lists' ME vectors; cost - sa8d is the PUs' mvcost (one vector for a uni PU, two for a
    bi PU); entries not evaluated hold the sentinels."""
    p, nr = wl.params, wl.params["numRefs"]
    pb, me, cu_jobs, cus = res["part_b"], res["me_out"], res["cu_jobs"], res["cus"]
    qmvp = res["jobs"]["qmvp"].astype(np.int64)
    tab = mvcost_tab_for(wl).astype(np.int64)
    mvc = lambda j, v: int((tab[MVRANGE + int(v[0]) - qmvp[j][0]] + tab[MVRANGE + int(v[1]) - qmvp[j][1]]) & 0xffff)
    lists = (range(0, n0), range(n0, nr))
    for c in range(res["ncu"]):
        S, k = int(cus[c][2]), 0
        for ps in range(8):
            if not _emitted(p, S, ps):
                assert pb["cost"][c, ps] == pb["sa8d"][c, ps] == 0xffffffff and (pb["biCost"][c, ps] == 0xffffffff).all()
                assert (pb["interDir"][c, ps] == 0).all() and (pb["ref"][c, ps] == -1).all() and (pb["mv"][c, ps] == 0).all()
                continue
            npu, total = (2 if ps else 1), 0
            for u in range(npu):
                costs, jobs = [], []
                for l in range(2):
                    js = [cu_jobs[c, r] + k + u for r in lists[l]]
                    best = int(np.argmin(me[js, 0]))
                    assert pb["ref"][c, ps, u, l] == lists[l][best], (c, ps, u, l)
                    costs.append(int(me[js[best], 0]))
                    jobs.append(js[best])
                d, bc, z = int(pb["interDir"][c, ps, u]), int(pb["biCost"][c, ps, u]), int(pb["zero"][c, ps, u])
                if ps == 0 or S == 8:
                    assert bc == 0xffffffff and z == 0
                assert (d == 3) == (bc < min(costs)), (c, ps, u)
                if d != 3:
                    assert d == (1 if costs[0] <= costs[1] else 2)
                for l in range(2):
                    v = pb["mv"][c, ps, u, l]
                    assert (v == 0).all() if z else tuple(v) == tuple(me[jobs[l], 1:3]), (c, ps, u, l)
                total += (mvc(jobs[0], pb["mv"][c, ps, u, 0]) + mvc(jobs[1], pb["mv"][c, ps, u, 1]) if d == 3 else
                          mvc(jobs[d - 1], me[jobs[d - 1], 1:3]))
            if npu == 1:
                assert pb["interDir"][c, ps, 1] == 0 and (pb["ref"][c, ps, 1] == -1).all() and pb["biCost"][c, ps, 1] == 0xffffffff
            assert int(pb["cost"][c, ps]) - int(pb["sa8d"][c, ps]) == total, (c, ps)
            k += npu
    assert not ((pb["interDir"][:, 0] == 3).any()), "a 2Nx2N PU went bi"


def check_bidir_2nx2n(res, bd, me):
    """The 2Nx2N entry against the BIDIR record of the same inputs: uniCost, the list slots and the uni winner."""
    pb = res["part_b"]
    assert np.array_equal(pb["cost"][:, 0], bd["uniCost"])
    assert np.array_equal(pb["ref"][:, 0, 0], bd["ref"])
    c0 = me[res["cu_jobs"][np.arange(res["ncu"]), bd["ref"][:, 0]], 0]
    c1 = me[res["cu_jobs"][np.arange(res["ncu"]), bd["ref"][:, 1]], 0]
    assert np.array_equal(pb["interDir"][:, 0, 0], np.where(c0 <= c1, 1, 2))


def check_p_equivalence(res, pres):
    """B/P equivalence: every partition without a bi PU has the cost, sa8d and per-PU used slot and vector of the P PART entry
    of the same inputs analysed as a P slice.  Returns the number of partitions compared."""
    pb, pp, cus = res["part_b"], pres["part"], res["cus"]
    n = 0
    for c in range(res["ncu"]):
        k = 0
        for ps in range(8):
            if pb["cost"][c, ps] == 0xffffffff:
                continue
            npu = 2 if ps else 1
            if not (pb["interDir"][c, ps, :npu] == 3).any():
                assert pb["cost"][c, ps] == pp["cost"][c, ps] and pb["sa8d"][c, ps] == pp["sa8d"][c, ps], (c, ps)
                for u in range(npu):
                    slot, v = used_pu(res, c, ps, u, k + u)
                    assert slot == pp["ref"][c, ps, u] and v == tuple(pp["mv"][c, ps, u]), (c, ps, u)
                n += 1
            k += npu
    return n


# (depth, (n0, n1), (rect, amp), chroma, (W, H), qp, kind); chroma: "off", "s3" (chroma, subme 3: with AMP both bi cost paths)
# or "s2" (chroma, subme 2: pixelavg_pp only)
SIZES = ((200, 136), (328, 200))
CASES = [(8, (1, 1), (1, 1), "s3", SIZES[0], 22, "average"),
         (10, (2, 2), (1, 0), "off", SIZES[1], 37, "average"),
         (8, (1, 3), (0, 0), "s3", SIZES[0], 37, "average"),
         (8, (2, 2), (1, 1), "s3", SIZES[1], 22, "occlusion"),
         (10, (1, 3), (1, 0), "s2", SIZES[0], 37, "occlusion"),
         (8, (1, 3), (1, 1), "off", SIZES[1], 37, "cut"),
         (10, (1, 1), (1, 0), "s3", SIZES[0], 22, "cut"),
         (10, (2, 2), (0, 0), "off", SIZES[1], 22, "cut"),
         (8, (2, 2), (1, 0), "s2", SIZES[0], 37, "gpb"),
         (10, (1, 1), (1, 1), "s3", SIZES[1], 22, "gpb"),
         (8, (1, 1), (1, 1), "s3", SIZES[0], 22, "static"),
         (10, (2, 2), (1, 0), "off", SIZES[1], 37, "static")]


def case_id(c):
    d, (n0, n1), (rect, amp), ch, (W, H), qp, kind = c
    geo = "rect+amp" if amp else ("rect" if rect else "2Nx2N")
    return "%s-%d-%d+%d-%s-%s-%dx%d-qp%d" % (kind, d, n0, n1, geo, ch, W, H, qp)


def case_workload(case):
    """The workload of a case, its numRefL0 and whether chroma is on."""
    d, (n0, n1), (rect, amp), ch, (W, H), qp, kind = case
    wl = part_b_workload(W, H, d, n0, n1, kind, rect=rect, amp=amp, subme=2 if ch == "s2" else 3, qp=qp)
    return wl, n0, ch != "off"
