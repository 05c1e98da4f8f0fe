"""Kernel times of the sub-pel phase of the frame analyser: the phase-plane build (k_interp_rows over plane tiles) and the
sub-pel launches (the groups' k_me_subpel_group and k_me_subpel_cell, or k_me<P, 3, 0, ...> without them, and k_me<P, 3, 1, ...>
for what is left), from torch.profiler, at bench.py's c3 and c4 shapes.  Reports the build's
achieved bandwidth against the H100 SXM data-sheet HBM3 figure (3.35 TB/s), counting one plane read and 15 planes
written per reference over the built rectangle (analyser.cuh: AN_PLANE_X / AN_PLANE_Y), with the card's name and power
limit.  Needs a GPU; prints one JSON line per config.

    python profiles/subpel_planes.py [--configs c3,c4] [--steps 3] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

PLANE_X, PLANE_Y = 80, 76                 # the built rectangle's margins around the picture (analyser.cuh)
HBM_PEAK = 3.35e12                        # H100 SXM data sheet, bytes/s
CONFIGS = {                               # bench.py's c3 / c4 (BASELINE.json)
    "c3": dict(W=3840, H=2160, depth=8, numRefs=4, method=3, subme=3, merange=57, rect=1, amp=0, chroma=True, qp=30),
    "c4": dict(W=3840, H=2160, depth=10, numRefs=5, method=3, subme=4, merange=57, rect=1, amp=1, chroma=True, qp=30),
}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in q.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:
        return {"error": repr(e)}


def kernel_ms(prof, steps):
    """ms per step of the build launches and of the sub-pel launches, by kernel name."""
    build, subpel, names = 0.0, {}, {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = getattr(e, "cuda_time_total", 0.0)
        if t <= 0:
            continue
        n = e.key
        if "k_interp_rows" in n:
            build += t
            names[n] = t / 1000.0 / steps
        elif (n.startswith("void k_me<") and ", 3, " in n) or "k_me_subpel_" in n:
            subpel[n] = t / 1000.0 / steps
    return build / 1000.0 / steps, subpel, names


def run(cu, name, steps):
    import torch
    from torch.profiler import profile, ProfilerActivity
    from frame_helpers import Workload, run_analyser
    c = dict(CONFIGS[name])
    W, H = c.pop("W"), c.pop("H")
    wl = Workload(W, H, **c)
    an = run_analyser(cu, wl)                        # also the warm-up of every launch shape
    an.run_rows(0, an.ctu_rows, 7)
    cu.sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            an.run_rows(0, an.ctu_rows, 7)
        cu.sync()
        torch.cuda.synchronize()
    build_ms, subpel, build_kernels = kernel_ms(prof, steps)
    es = 1 if c["depth"] == 8 else 2
    plane = (W + 2 * PLANE_X) * (H + 2 * PLANE_Y) * es
    nbytes = c["numRefs"] * 16 * plane
    an.close()
    return {"config": name, "steps": steps, "build_ms": build_ms, "build_bytes": nbytes,
            "build_GBps": nbytes / (build_ms / 1000.0) / 1e9 if build_ms else None,
            "build_frac_of_datasheet_hbm": nbytes / (build_ms / 1000.0) / HBM_PEAK if build_ms else None,
            "build_kernels_ms": build_kernels, "subpel_kernels_ms": subpel, "subpel_ms": sum(subpel.values()),
            "added_device_bytes": c["numRefs"] * 15 * ((W + 192 + 63) // 64 * 64 * (H + 160) * es + 256)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="c3,c4")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--out", help="also write the results as DIR/subpel_planes.json")
    args = ap.parse_args()
    import x265_b200
    cu = x265_b200.load()
    res = {"card": card(), "results": []}
    for name in args.configs.split(","):
        r = run(cu, name, args.steps)
        res["results"].append(r)
        print(json.dumps(r))
    print(json.dumps({"card": res["card"]}))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "subpel_planes.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
