"""Device time of x265cu_sao_stats_frame and x265cu_sao_apply_frame at bench.py's c3 (3840x2160 8-bit) and c4 (10-bit)
geometries, CTU 64, 4:2:0, over a deblocked picture and random per-CTU records (every type; no bypass units), with the
card's name, power limit and maximum SM clock read in the same run.  3 warm-up calls, then CUDA events around each of 20
calls (x265cu_timer_begin / _end): median / min / max per call.  The achieved rates are over the compulsory bytes, computed
here: statistics read source and reconstruction once and write the records; apply reads and writes the picture once and
reads the records.  For context, one single-thread host time of the reference's calcSaoStatsCTU and of its apply over the
same picture (x265ref_sao_stats_frame / x265ref_sao_apply_frame from oracle/_ref, when built).  Needs a GPU; prints one
JSON line per config.

    python profiles/sao.py [--configs c3,c4] [--reps 20] [--out DIR]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "profiles")]

from deblock import CONFIGS, card     # noqa: E402  (the same geometries and card query as profiles/deblock.py)

CTU = 64


def compulsory_bytes(W, H, es, n):
    picture = W * H * 3 // 2 * es
    stats = 2 * picture + n * 2 * 3 * 5 * 32 * 4
    apply = 2 * picture + n * 3 * 8
    return stats, apply


def timed(cu, call, reps):
    for _ in range(3):
        call()
    cu.sync()
    t = []
    for _ in range(reps):
        cu.timer_begin()
        call()
        t.append(cu.timer_end())
    return t


def run(cu, name, reps):
    import numpy as np
    import deblock_helpers as D
    import sao_helpers as S
    from x265_b200.lib import B_SLICE, SAO_STATS_PER_CTU
    c = CONFIGS[name]
    W, H, depth = c["W"], c["H"], c["depth"]
    rng = np.random.default_rng(2160 + depth)
    luma, cb, cr = D.make_planes(rng, W, H, depth)
    units = D.make_map(rng, W, H, CTU, depth, B_SLICE)
    rec = list(D.oracle_deblock(depth, luma, cb, cr, units, D.params_array(B_SLICE)))
    fenc = [np.clip(p.astype(np.int32) + rng.integers(-3, 4, p.shape) * (1 << (depth - 8)), 0, (1 << depth) - 1).astype(p.dtype)
            for p in rec]
    params, merge = S.make_params(rng, W, H, CTU, depth)
    n = S.num_ctus(W, H, CTU)
    R = [cu.to_device(p) for p in rec]
    F = [cu.to_device(p) for p in fenc]
    st = cu.alloc(n * SAO_STATS_PER_CTU * 4)
    pb = cu.to_device(params)
    rp, fp = [b.ptr for b in R], [b.ptr for b in F]
    ts = timed(cu, lambda: cu.sao_stats_frame(depth, W, H, CTU, fp, W, W // 2, rp, W, W // 2, st), reps)
    ta = timed(cu, lambda: cu.sao_apply_frame(depth, W, H, CTU, rp, W, W // 2, pb, 1, 1), reps)
    host = {}
    if S.load_ref_sao(depth) is not None:
        t0 = time.perf_counter()
        S.ref_stats(depth, rec, fenc, CTU)
        host["stats"] = (time.perf_counter() - t0) * 1e3
        t0 = time.perf_counter()
        S.ref_apply(depth, rec, CTU, params, merge, 1, 1, None, fenc)
        host["apply"] = (time.perf_counter() - t0) * 1e3
    for b in R + F + [st, pb]:
        b.free()
    es = 1 if depth == 8 else 2
    bs, ba = compulsory_bytes(W, H, es, n)
    out = {"config": name, "W": W, "H": H, "depth": depth, "ctu": CTU, "reps": reps}
    for key, t, nb in (("stats", ts, bs), ("apply", ta, ba)):
        med = statistics.median(t)
        out[key] = {"ms_median": round(med, 4), "ms_min": round(min(t), 4), "ms_max": round(max(t), 4),
                    "compulsory_MB": round(nb / 1e6, 2), "GBps_median": round(nb / med / 1e6, 1),
                    "host_reference_single_thread_ms": round(host[key], 1) if key in host else "not measured (oracle/_ref absent)"}
    return out


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
        with open(os.path.join(a.out, "sao.jsonl"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
