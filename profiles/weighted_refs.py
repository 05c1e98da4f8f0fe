"""Cost of weighted P-slice references in the frame analyser at bench.py's c3 and c4 shapes, on a fade.  Reports, per config:
  * the weighted-plane build per reference (weight_pp of the luma plane and of both chroma planes, border extension): a
    run_resident(0) right after set_ref_weights on every reference rebuilds them and launches nothing else, timed with CUDA
    events, median of 10;
  * x265cu_analyser_stage_ms of a full run (stages 1 | 2 | 8) with no reference and with every reference weighted: ME stage,
    luma residual, chroma residual (the weighted planes are already built: only the search's and the residuals' own cost),
    median of 10 after warm-up;
  * the extra device memory (cudaMemGetInfo before and after the first weighted run);
  * the card's name and power limit.
Needs a GPU; prints one JSON line per config.

    python profiles/weighted_refs.py [--configs c3,c4] [--reps 10]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

CONFIGS = {                               # bench.py's c3 / c4 (BASELINE.json)
    "c3": dict(W=3840, H=2160, depth=8, numRefs=4, method=3, subme=3, merange=57, qp=30),
    "c4": dict(W=3840, H=2160, depth=10, numRefs=5, method=3, subme=4, merange=57, qp=30),
}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in q.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:
        return {"error": repr(e)}


def free_bytes():
    import torch
    return torch.cuda.mem_get_info()[0]


def run(cu, name, reps):
    from wref_helpers import fade_workload, entry
    from test_gpu_x_weighted_refs import open_analyser, source
    c = CONFIGS[name]
    wl = fade_workload(c["W"], c["H"], c["depth"], c["numRefs"], subme=c["subme"], method=c["method"], merange=c["merange"], qp=c["qp"])
    an = open_analyser(cu, wl)
    an.load_inputs(source(wl), wl.field)
    row = [entry(46, 5, 14), entry(60, 6, 9), entry(70, 6, -11)]

    def stage_ms():
        out = {"me": [], "luma_residual": [], "chroma_residual": []}
        for _ in range(3):
            an.run_resident(11)
        for _ in range(reps):
            cu.timer_begin()
            an.run_resident(11)
            total = cu.timer_end()
            ms = an.stage_ms()
            out["me"].append(ms[0]); out["luma_residual"].append(ms[1])
            out["chroma_residual"].append(total - ms[0] - ms[1] - ms[2])
        return {k: round(statistics.median(v), 4) for k, v in out.items()}
    plain = stage_ms()
    cu.sync()
    free0 = free_bytes()
    build = []
    for i in range(reps + 1):
        for r in range(c["numRefs"]):
            an.set_ref_weights(r, row if i % 2 == 0 else [entry(47, 5, 14), row[1], row[2]])
        cu.timer_begin()
        an.run_resident(0)                 # rebuilds every reference's weighted planes, no stage runs
        t = cu.timer_end()
        if i:
            build.append(t / c["numRefs"])
    cu.sync()
    extra = free0 - free_bytes()
    weighted = stage_ms()
    res = dict(config=name, card=card(), weighted_plane_build_ms_per_ref=round(statistics.median(build), 4),
               stage_ms_unweighted=plain, stage_ms_all_weighted=weighted, extra_device_mib=round(extra / 2**20, 1),
               numRefs=c["numRefs"])
    an.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="c3,c4")
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    import x265_b200
    cu = x265_b200.load()
    for name in a.configs.split(","):
        print(json.dumps(run(cu, name, a.reps)), flush=True)


if __name__ == "__main__":
    main()
