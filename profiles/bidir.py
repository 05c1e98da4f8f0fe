"""Cost of B slices in the frame analyser at bench.py's c3 and c4 shapes, with 2+2 references and chroma on, on a B frame between
its references (tests/bidir_helpers.py "between").  Reports, per config:
  * the BIDIR stage (stage value 16) alone, after a full run has left the ME results resident: run_resident(16) between CUDA
    events, median of 20 after 3 warm-up runs;
  * x265cu_analyser_stage_ms of a full run on the same data as a P slice (set_lists(4, 0), stages 1 | 2 | 8) and as a B slice
    (set_lists(2, 2), stages 1 | 2 | 8 | 16): luma residual [1] (it excludes the BIDIR stage), chroma residual (the run's time
    less the ME, BIDIR, luma residual and intra stages), median of 20 after 3 warm-up runs, and the share of bi-predicted CUs;
  * the card's name and power limit.
Needs a GPU; prints one JSON line per config.

    python profiles/bidir.py [--configs c3,c4] [--reps 20]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

CONFIGS = {                               # bench.py's c3 / c4 shapes (BASELINE.json), with 2 + 2 references
    "c3": dict(W=3840, H=2160, depth=8, qp=30),
    "c4": dict(W=3840, H=2160, depth=10, qp=30),
}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in q.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:
        return {"error": repr(e)}


def run(cu, name, reps):
    from bidir_helpers import bidir_workload
    from test_gpu_x_bidir import open_analyser, source
    c = CONFIGS[name]
    wl = bidir_workload(c["W"], c["H"], c["depth"], 2, 2, "between", qp=c["qp"])
    an = open_analyser(cu, wl, (2, 2), True)
    an.load_inputs(source(wl), wl.field)

    def timed(stages):
        out = {"luma_residual": [], "chroma_residual": [], "total": []}
        for _ in range(3):
            an.run_resident(stages)
        for _ in range(reps):
            cu.timer_begin()
            an.run_resident(stages)
            total = cu.timer_end()
            ms = an.stage_ms()
            out["luma_residual"].append(ms[1]); out["total"].append(total)
            out["chroma_residual"].append(total - ms[0] - ms[1] - ms[2] - (bidir_ms if stages & 16 else 0.0))
        return {k: round(statistics.median(v), 4) for k, v in out.items()}
    an.set_lists(2, 2)
    an.run_resident(1 | 2 | 8 | 16)
    bi_share = float((an.bidir_results()["interDir"] == 3).mean())
    for _ in range(3):
        an.run_resident(16)
    stage = []
    for _ in range(reps):
        cu.timer_begin()
        an.run_resident(16)
        stage.append(cu.timer_end())
    bidir_ms = statistics.median(stage)
    b = timed(1 | 2 | 8 | 16)
    an.set_lists(4, 0)
    p = timed(1 | 2 | 8)
    res = dict(config=name, card=card(), W=c["W"], H=c["H"], depth=c["depth"], lists="2+2", chroma=True, ncu=an.ncu,
               bi_share=round(bi_share, 3), bidir_stage_ms=round(bidir_ms, 4), b_slice=b, p_slice=p)
    an.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="c3,c4")
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    import x265_b200
    cu = x265_b200.load()
    for name in a.configs.split(","):
        print(json.dumps(run(cu, name, a.reps)), flush=True)


if __name__ == "__main__":
    main()
