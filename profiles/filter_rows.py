"""Device time of the band calls x265cu_deblock_rows, x265cu_sao_stats_rows and x265cu_sao_apply_rows, and of the three as a
chain per band, for block partitions into 1, 2, 4 and 8 bands, against the frame calls on the same inputs, at bench.py's c3
geometry (3840x2160 8-bit) and at 7680x4320 10-bit (BASELINE configs[4]), CTU 64, over a map shaped like preset slow's CU mix.
The card's name, power limit and maximum SM clock are read in the same run.  3 warm-up calls, then CUDA events around each
of `reps` calls (x265cu_timer_begin / _end); per band count, the median over the reps of each band, then the mean and the
maximum over the bands.  Also the bytes shard.exchange_halos broadcasts per frame against a whole-band exchange of the
pre-deblock picture (shard.exchange_rows) for the same partition.  Needs a GPU; prints one JSON line per config.

    python profiles/filter_rows.py [--configs c3,8k] [--reps 20] [--out DIR]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from deblock import card                      # noqa: E402  (profiles/deblock.py)

CONFIGS = {"c3": dict(W=3840, H=2160, depth=8), "8k": dict(W=7680, H=4320, depth=10)}
BANDS = (1, 2, 4, 8)


def timed(cu, fn, reps):
    for _ in range(3):
        fn()
    cu.sync()
    t = []
    for _ in range(reps):
        cu.timer_begin()
        fn()
        t.append(cu.timer_end())
    return statistics.median(t)


def exchange_bytes(W, H, ctu, world, es):
    """(halo, whole band) bytes broadcast per frame for luma + 4:2:0 chroma, block partition"""
    from x265_b200 import shard
    nrows = (H + ctu - 1) // ctu
    halo = sum(((y1 - y0) * W + 2 * (c1 - c0) * (W // 2)) * es for _, (y0, y1), (c0, c1) in shard.halo_sends(nrows, world, H, ctu))
    band = sum((min(H, r1 * ctu) - r0 * ctu) * W * 3 // 2 * es for g in range(world) for r0, r1 in shard.row_blocks(nrows, g, world))
    return halo, band if world > 1 else 0


def run(cu, name, reps):
    import numpy as np
    import deblock_helpers as D
    import sao_helpers as S
    from test_gpu_deblock import dparams
    from test_gpu_sao import decide
    from x265_b200 import shard
    from x265_b200.lib import B_SLICE, SAO_STATS_PER_CTU
    c = CONFIGS[name]
    W, H, depth, ctu = c["W"], c["H"], c["depth"], 64
    es = 1 if depth == 8 else 2
    rng = np.random.default_rng(2160 + depth)
    units = D.make_map(rng, W, H, ctu, depth, B_SLICE, p_intra=0.1, split={6: 0.85, 5: 0.6, 4: 0.35})
    rec = D.make_planes(rng, W, H, depth)
    fenc = [np.clip(q.astype(np.int32) + rng.integers(-3, 4, q.shape) * (1 << (depth - 8)), 0, (1 << depth) - 1).astype(q.dtype)
            for q in rec]
    R, F, Sc, Ref = ([cu.to_device(q) for q in planes] for planes in (rec, fenc, rec, rec))
    ptr = lambda bufs: tuple(b.ptr for b in bufs)                          # noqa: E731
    ubuf, p = cu.to_device(units), dparams(D.params_array(B_SLICE))
    n, rows = S.num_ctus(W, H, ctu), (H + ctu - 1) // ctu
    sbuf = cu.alloc(n * SAO_STATS_PER_CTU * 4)
    cu.deblock_frame(depth, Sc[0].ptr, W, Sc[1].ptr, Sc[2].ptr, W // 2, W, H, ubuf, p)
    cu.sao_stats_frame(depth, W, H, ctu, ptr(F), W, W // 2, ptr(Sc), W, W // 2, sbuf)
    pbuf = cu.to_device(decide(sbuf.download(np.int32).reshape((n,) + S.STATS_SHAPE), depth))

    def deblock(r0, r1):
        cu.deblock_rows(depth, W, H, ctu, r0, r1, ptr(R), W, W // 2, ptr(Sc), W, W // 2, ubuf, p)

    def stats(r0, r1):
        cu.sao_stats_rows(depth, W, H, ctu, r0, r1, ptr(F), W, W // 2, ptr(Sc), W, W // 2, sbuf)

    def apply(r0, r1):
        cu.sao_apply_rows(depth, W, H, ctu, r0, r1, ptr(Sc), W, W // 2, ptr(Ref), W, W // 2, pbuf, 1, 1)

    def chain(r0, r1):
        deblock(r0, r1)
        stats(r0, r1)
        apply(r0, r1)

    out = {"config": name, "W": W, "H": H, "depth": depth, "ctu": ctu, "reps": reps, "frame_ms": {
        "deblock": round(timed(cu, lambda: cu.deblock_frame(depth, Sc[0].ptr, W, Sc[1].ptr, Sc[2].ptr, W // 2, W, H, ubuf, p), reps), 4),
        "sao_stats": round(timed(cu, lambda: cu.sao_stats_frame(depth, W, H, ctu, ptr(F), W, W // 2, ptr(Sc), W, W // 2, sbuf), reps), 4),
        "sao_apply": round(timed(cu, lambda: cu.sao_apply_frame(depth, W, H, ctu, ptr(Ref), W, W // 2, pbuf, 1, 1), reps), 4)}}
    for nb in BANDS:
        parts = [b for g in range(nb) for b in shard.row_blocks(rows, g, nb)]
        r = {}
        for what, fn in (("deblock", deblock), ("sao_stats", stats), ("sao_apply", apply), ("chain", chain)):
            t = [timed(cu, lambda: fn(r0, r1), reps) for r0, r1 in parts]
            r[what] = {"mean_ms": round(sum(t) / len(t), 4), "max_ms": round(max(t), 4)}
        halo, band = exchange_bytes(W, H, ctu, nb, es)
        r["exchange_MB"] = {"halos": round(halo / 1e6, 3), "whole_bands": round(band / 1e6, 3)}
        out["bands_%d" % nb] = r
    for b in R + F + Sc + Ref + [ubuf, sbuf, pbuf]:
        b.free()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="c3,8k")
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
        with open(os.path.join(a.out, "filter_rows.jsonl"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
