"""Device time of x265cu_deblock_frame (k_deblock_frame, both passes) at bench.py's c3 (3840x2160 8-bit) and c4 (10-bit)
geometries over a map shaped like preset slow's CU mix, with the card's name, power limit and maximum SM clock read in the
same run.  3 warm-up calls, then CUDA events around each of 20 calls (x265cu_timer_begin / _end): median / min / max.  The
achieved rate is over the compulsory bytes, computed here: the picture read and written once per pass (luma + 4:2:0 chroma)
and the decision map read once per pass.  For context, one single-thread host time of the reference's Deblock
(x265ref_deblock_frame from oracle/_ref, when built) over the same map.  Needs a GPU; prints one JSON line per config.

    python profiles/deblock.py [--configs c3,c4] [--reps 20] [--out DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

CONFIGS = {"c3": dict(W=3840, H=2160, depth=8), "c4": dict(W=3840, H=2160, depth=10)}     # bench.py's c3 / c4 geometries


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in q.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:
        return {"error": repr(e)}


def compulsory_bytes(W, H, es):
    """Both passes: the luma and 4:2:0 chroma picture read and written once per pass, the 16-byte map read once per pass."""
    picture = W * H * 3 // 2 * es
    units = (W // 4) * (H // 4) * 16
    return 2 * (2 * picture + units)


def run(cu, name, reps):
    import numpy as np
    import deblock_helpers as D
    from test_gpu_deblock import slow_map, dparams
    from x265_b200.lib import B_SLICE
    c = CONFIGS[name]
    W, H, depth = c["W"], c["H"], c["depth"]
    rng = np.random.default_rng(2160 + depth)
    units = slow_map(rng, W, H, depth, B_SLICE)
    luma, cb, cr = D.make_planes(rng, W, H, depth)
    prm = D.params_array(B_SLICE)
    bufs = [cu.to_device(p) for p in (luma, cb, cr)]
    ubuf = cu.to_device(units)
    p = dparams(prm)

    def call():
        cu.deblock_frame(depth, bufs[0].ptr, W, bufs[1].ptr, bufs[2].ptr, W // 2, W, H, ubuf, p)

    for _ in range(3):
        call()
    cu.sync()
    t = []
    for _ in range(reps):
        cu.timer_begin()
        call()
        t.append(cu.timer_end())
    host = None
    if D.load_ref_deblock(depth) is not None:
        t0 = time.perf_counter()
        D.ref_deblock(depth, luma, cb, cr, units, prm, 64)
        host = (time.perf_counter() - t0) * 1e3
    for b in bufs + [ubuf]:
        b.free()
    es = 1 if depth == 8 else 2
    nbytes = compulsory_bytes(W, H, es)
    med = statistics.median(t)
    return {"config": name, "W": W, "H": H, "depth": depth, "reps": reps, "ms_median": round(med, 4), "ms_min": round(min(t), 4),
            "ms_max": round(max(t), 4), "compulsory_MB": round(nbytes / 1e6, 2), "GBps_median": round(nbytes / med / 1e6, 1),
            "host_reference_single_thread_ms": round(host, 1) if host is not None else "not measured (oracle/_ref absent)"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="c3,c4")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import x265_b200
    cu = x265_b200.load()
    info = card()
    lines = []
    for name in a.configs.split(","):
        r = run(cu, name, a.reps)
        r["card"] = info
        lines.append(json.dumps(r))
        print(lines[-1], flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "deblock.jsonl"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
