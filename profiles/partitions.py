"""Cost of the PART stage (stage value 32: the inter estimate of every partition of a P slice's CUs) at bench.py's c3 and c4
shapes, chroma on.  Reports, per config:
  * the PART stage alone, after an ME run has left the results resident: run_resident(32) between CUDA events, median of
    --reps (at least 10) after 3 warm-up runs;
  * for scale, the ME stage of the same run (x265cu_analyser_stage_ms [0]);
  * the share of CUs whose lowest-cost entry is not 2Nx2N;
  * the card's name, power limit and maximum SM clock, read in the same run.
c3: 3840x2160 8-bit, 4 references, rect (3 partitions per CU); c4: 3840x2160 10-bit, 5 references, rect + AMP, subme 4 (7
partitions per CU >= 16).  Needs a GPU; prints one JSON line per config.

    python profiles/partitions.py [--configs c3,c4] [--reps 20]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

CONFIGS = {                               # bench.py's c3 / c4 shapes (BASELINE.json)
    "c3": dict(W=3840, H=2160, depth=8, numRefs=4, amp=0, subme=3, qp=30),
    "c4": dict(W=3840, H=2160, depth=10, numRefs=5, amp=1, subme=4, qp=30),
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
    from frame_helpers import Workload
    from test_gpu_x_partitions import open_analyser, source
    c = CONFIGS[name]
    wl = Workload(c["W"], c["H"], depth=c["depth"], numRefs=c["numRefs"], subme=c["subme"], rect=1, amp=c["amp"], qp=c["qp"],
                  chroma=True)
    an = open_analyser(cu, wl, True)
    an.load_inputs(source(wl), wl.field)
    an.run_resident(1)
    me_ms = an.stage_ms()[0]
    for _ in range(3):
        an.run_resident(32)
    stage = []
    for _ in range(reps):
        cu.timer_begin()
        an.run_resident(32)
        stage.append(cu.timer_end())
    rec = an.part_results()
    not_2nx2n = float((np.argmin(rec["cost"], axis=1) != 0).mean())
    res = dict(config=name, card=card(), W=c["W"], H=c["H"], depth=c["depth"], numRefs=c["numRefs"], rect=1, amp=c["amp"],
               chroma=True, ncu=an.ncu, reps=reps, part_stage_ms=round(statistics.median(stage), 4),
               part_stage_ms_min=round(min(stage), 4), me_stage_ms=round(me_ms, 4), share_not_2Nx2N=round(not_2nx2n, 3))
    an.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="c3,c4")
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    assert a.reps >= 10
    import x265_b200
    cu = x265_b200.load()
    for name in a.configs.split(","):
        print(json.dumps(run(cu, name, a.reps)), flush=True)


if __name__ == "__main__":
    main()
