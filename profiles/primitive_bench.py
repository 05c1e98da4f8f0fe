"""Per-primitive-class throughput of the batched kernels at frame scale (the second half of BASELINE.json's
metric: "per-primitive HBM GB/s vs peak").  Each class runs ONE launch over a 3840x2160 frame's worth of
jobs on device-resident planes; time = CUDA events, median of `reps` after warm-up, L2 flushed between
repetitions; GB/s = ALGORITHMIC bytes per launch (SURVEY 8(d) per-call formulas x jobs) / time.

    python profiles/primitive_bench.py [--reps 7] [--json out.json]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import x265_b200  # noqa: E402
from x265_b200.lib import CMP_JOB, BLK_JOB, INTERP_JOB, INTRA_JOB  # noqa: E402
from frame_helpers import gen_luma, pad_plane, MARGIN_X, MARGIN_Y  # noqa: E402

W, H = 3840, 2160
FRAMES = 24          # one launch covers a lookahead-window-sized batch: 24 stacked 2160p frames (~200 MB per plane)


SINGLE = False       # --single: every primitive runs exactly once (a pass for a profiler)


def timed(lib, flush, fn, reps):
    if SINGLE:
        lib.sync()
        lib.timer_begin()
        fn()
        return lib.timer_end()
    for _ in range(2):
        fn()
    lib.sync()
    ts = []
    for r in range(reps):
        lib.check(lib.L.x265cu_memset(lib.ctx, flush.ptr, r & 255, flush.nbytes))
        lib.sync()
        lib.timer_begin()
        fn()
        ts.append(lib.timer_end())
    return float(np.median(ts))


def grid_jobs(dtype, bw, bh, stride, org, fields):
    xs, ys = np.meshgrid(np.arange(0, W - bw + 1, bw), np.arange(0, H - bh + 1, bh))
    n = xs.size
    j = np.zeros(n, dtype)
    off = (org + ys.ravel() * stride + xs.ravel()).astype(np.int64)
    return j, off, n


def run(lib, depth=8, reps=7, frames=FRAMES, quiet=False, only=None):
    """One launch per primitive class over `frames` stacked 2160p frames of `depth`-bit pixels; returns the table rows."""
    global H
    H = 2160
    es = 1 if depth == 8 else 2
    pdt = np.uint8 if depth == 8 else np.uint16
    peak = 3350.0          # H100 SXM data sheet, HBM3
    try:
        peak = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
    except Exception:
        pass
    flush = lib.alloc(256 << 20)
    if not quiet:
        print("batch = %d stacked 2160p frames per launch, %d-bit" % (frames, depth))
    fa, fb = gen_luma(W, H, 4, bits=depth), gen_luma(W, H, 3, bits=depth)
    a, stride, org = pad_plane(np.tile(fa, (frames, 1)), depth)       # frames stacked vertically
    b, _, _ = pad_plane(np.tile(fb, (frames, 1)), depth)
    H = H * frames
    dA, dB = lib.to_device(a), lib.to_device(b)
    rows = []
    bufs = [flush, dA, dB]

    def want(name):
        return only is None or any(o in name for o in only)

    launch_mark = [lib.launch_count()]

    def add(name, ms, nbytes, note=""):
        gbs = nbytes / (ms / 1000.0) / 1e9
        l0, l1 = launch_mark[0], lib.launch_count()
        launch_mark[0] = l1
        rows.append({"kernel": name, "depth": depth, "ms": ms, "launch0": l0, "launch1": l1, "algorithmic_MB": nbytes / 1e6, "GBps": gbs, "frac_of_measured_peak": gbs / peak, "note": note})
        if not quiet:
            print("%-34s %8.3f ms %9.1f MB %8.1f GB/s  %5.1f%% of %.0f  %s" % (name, ms, nbytes / 1e6, gbs, 100 * gbs / peak, peak, note), flush=True)

    # ---- pixel compare: whole-frame grids of 8x8 / 16x16 / 64x64 blocks, frame n vs frame n-1 (job-list entry point) ----
    for op, (bw, bh) in (("sad", (8, 8)), ("sad", (16, 16)), ("sad", (64, 64)), ("satd", (8, 8)), ("satd", (16, 16)), ("satd", (64, 64)),
                         ("sa8d", (16, 16)), ("sa8d", (64, 64)), ("sse_pp", (16, 16)), ("sse_pp", (64, 64))):
        name = "k_pixelcmp %s %dx%d grid" % (op, bw, bh)
        if not want(name):
            continue
        j, off, n = grid_jobs(CMP_JOB, bw, bh, stride, org, None)
        j["a_off"] = off; j["b_off"] = off + 3 * stride + 5; j["a_stride"] = stride; j["b_stride"] = stride; j["w"] = bw; j["h"] = bh
        dJ = lib.to_device(j); dO = lib.alloc(8 * n)
        ms = timed(lib, flush, lambda: lib.pixelcmp_batch(depth, op, dA, dB, dJ, n, dO), reps)
        add(name, ms, n * (2 * bw * bh * es + 8), "%d jobs" % n)
        dJ.free(); dO.free()
    # ---- same compares through the grid entry point (no job list; lane per 16-byte column) ----
    for op, (bw, bh) in (("sad", (8, 8)), ("sad", (16, 16)), ("sad", (64, 64)), ("satd", (8, 8)), ("satd", (16, 16)), ("satd", (64, 64)),
                         ("sa8d", (8, 8)), ("sa8d", (16, 16)), ("sa8d", (64, 64)), ("sse_pp", (16, 16)), ("sse_pp", (64, 64))):
        name = "k_pixelcmp_grid %s %dx%d" % (op, bw, bh)
        if not want(name):
            continue
        nbx, nby = W // bw, H // bh
        n = nbx * nby
        dO = lib.alloc(8 * n)
        for tag, boff in (("B displaced (+5,+3)", org + 3 * stride + 5), ("B aligned", org + 16 * stride)):
            ms = timed(lib, flush, lambda: lib.pixelcmp_grid(depth, op, dA.ptr + org * es, stride, dB.ptr + boff * es, stride, bw, bh, nbx, nby, dO), reps)
            add(name + (" displaced" if "disp" in tag else " aligned"), ms, n * (2 * bw * bh * es + 8), "%d blocks, %s" % (n, tag))
        dO.free()
    # ---- interpolation: whole frame as 64x64 / 16x16 jobs ----
    dD = lib.alloc(a.nbytes); bufs.append(dD)
    for op, (bw, bh) in (("hvpp", (64, 64)), ("hvpp", (16, 16)), ("hpp", (64, 64)), ("vpp", (64, 64))):
        name = "k_interp luma_%s %dx%d grid" % (op, bw, bh)
        if not want(name):
            continue
        j, off, n = grid_jobs(INTERP_JOB, bw, bh, stride, org, None)
        j["s_off"] = off; j["d_off"] = off; j["s_stride"] = stride; j["d_stride"] = stride; j["w"] = bw; j["h"] = bh
        j["idxX"] = 2; j["idxY"] = 3; j["ntaps"] = 8
        dJ = lib.to_device(j)
        ms = timed(lib, flush, lambda: lib.interp_batch(depth, op, dA, dD, dJ, n), reps)
        halo_w = bw + (7 if op in ("hvpp", "hpp") else 0); halo_h = bh + (7 if op in ("hvpp", "vpp") else 0)
        add(name, ms, n * (halo_w * halo_h + bw * bh) * es, "%d jobs" % n)
        dJ.free()
    # ---- block ops: sub_ps over the frame as 64x64 blocks (pixel,pixel -> int16) ----
    if want("k_blockop sub_ps"):
        dS = lib.alloc(a.size * 2); bufs.append(dS)
        j, off, n = grid_jobs(BLK_JOB, 64, 64, stride, org, None)
        j["d_off"] = off; j["a_off"] = off; j["b_off"] = off; j["d_stride"] = stride; j["a_stride"] = stride; j["b_stride"] = stride; j["w"] = 64; j["h"] = 64
        dJ = lib.to_device(j)
        ms = timed(lib, flush, lambda: lib.blockop_batch(depth, "sub_ps", dS, dA, dB, dJ, n), reps)
        add("k_blockop sub_ps 64x64 grid", ms, n * 64 * 64 * (2 * es + 2), "%d jobs" % n)
        dJ.free()
    # ---- transforms / quant on a frame of residual (contiguous TUs) ----
    pm = (1 << depth)
    r1 = (np.random.default_rng(1).integers(0, pm, W * 2160) - np.random.default_rng(2).integers(0, pm, W * 2160)).astype(np.int16)
    resid = np.tile(r1, max(1, frames // 2))
    dR = lib.to_device(resid); dC = lib.alloc(resid.nbytes); dQ = lib.alloc(resid.nbytes); dDU = lib.alloc(resid.size * 4)
    bufs += [dR, dC, dQ, dDU]
    for N in (4, 8, 16, 32):
        if not want("k_transform"):
            continue
        n = resid.size // (N * N)
        ms = timed(lib, flush, lambda: lib.transform_batch(depth, "dct", N, dR, dC, N, N * N, n), reps)
        add("k_transform dct%d" % N, ms, n * 4 * N * N, "%d TUs" % n)
        ms = timed(lib, flush, lambda: lib.transform_batch(depth, "idct", N, dC, dQ, N, N * N, n), reps)
        add("k_transform idct%d" % N, ms, n * 4 * N * N, "%d TUs" % n)
    if want("k_quant") or want("k_dequant"):
        qc = lib.to_device(np.full(1024, 18396, np.int32)); ns = lib.alloc(4 * (resid.size // 1024)); bufs += [qc, ns]
        n = resid.size // 1024
        ms = timed(lib, flush, lambda: lib.check(lib.L.x265cu_quant_batch(lib.ctx, dC.ptr, qc.ptr, dDU.ptr, dQ.ptr, 19, 85 << 10, 1024, n, 0, ns.ptr)), reps)
        add("k_quant 32x32", ms, n * 1024 * 12 + n * 4, "%d TUs" % n)
        ms = timed(lib, flush, lambda: lib.check(lib.L.x265cu_dequant_normal_batch(lib.ctx, dQ.ptr, dC.ptr, resid.size, 57 << 5, 6)), reps)
        add("k_dequant_normal", ms, resid.size * 4, "")
    # ---- intra: all-angs for every 16x16 block of the frame ----
    if want("k_intra"):
        N = 16
        nblk = (W // N) * (2160 // N) * 2
        nb = np.random.default_rng(3).integers(0, pm, (nblk, 4 * N + 1)).astype(pdt)
        dNB = lib.to_device(nb); dF = lib.alloc(nb.nbytes); dP = lib.alloc(nblk * 33 * N * N * es); bufs += [dNB, dF, dP]
        ms = timed(lib, flush, lambda: lib.check(lib.L.x265cu_intra_filter_batch(lib.ctx, depth, N, dNB.ptr, dF.ptr, 4 * N + 1, nblk)), reps)
        add("k_intra_filter 16", ms, nblk * 2 * (4 * N + 1) * es, "%d blocks" % nblk)
        ms = timed(lib, flush, lambda: lib.check(lib.L.x265cu_intra_allangs_batch(lib.ctx, depth, N, dNB.ptr, dF.ptr, 4 * N + 1, dP.ptr, 1, nblk)), reps)
        add("k_intra_allangs 16", ms, nblk * (2 * (4 * N + 1) + 33 * N * N) * es, "%d blocks" % nblk)
    # ---- lowres init (+ border extension) ----
    if want("k_lowres_init"):
        lw, lh = W // 2, H // 2
        lstride = (lw + 2 * 32 + 31) // 32 * 32
        planes = [lib.alloc(lstride * (lh + 64) * es) for _ in range(4)]; bufs += planes
        lorg = (32 * lstride + 32) * es
        ms = timed(lib, flush, lambda: lib.check(lib.L.x265cu_frame_init_lowres(lib.ctx, depth, dA.ptr + org * es, stride, planes[0].ptr + lorg, planes[1].ptr + lorg,
                                                                                 planes[2].ptr + lorg, planes[3].ptr + lorg, lstride, lw, lh, 32, 32)), reps)
        add("k_lowres_init + extend (2 launches)", ms, 2 * W * H * es, "")
    lib.sync()
    for bf in bufs:
        bf.free()
    H = 2160
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--frames", type=int, default=FRAMES)
    ap.add_argument("--depth", default="8,10")
    ap.add_argument("--only", default=None, help="comma-separated substrings of kernel names")
    ap.add_argument("--json", default=None)
    ap.add_argument("--single", action="store_true", help="run every primitive exactly once (for the ncu dram-bytes pass)")
    args = ap.parse_args()
    global SINGLE
    SINGLE = args.single
    lib = x265_b200.load()
    rows = []
    for d in [int(x) for x in args.depth.split(",")]:
        rows += run(lib, depth=d, reps=args.reps, frames=args.frames, only=args.only.split(",") if args.only else None)
    if args.json:
        json.dump({"rows": rows}, open(args.json, "w"), indent=1)


if __name__ == "__main__":
    main()
