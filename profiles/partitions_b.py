"""Cost of the PART_B stage (stage value 64: the inter estimate of every partition of a B slice's CUs) at bench.py's c3 and c4
shapes, chroma on, the c3 references split 2+2 into the lists and the c4 ones 3+2.  Reports, per config:
  * the PART_B stage alone, after an ME run has left the results resident: run_resident(64) between CUDA events, median of
    --reps (at least 10) after 3 warm-up runs;
  * for scale, the PART stage (value 32) on the same resident inputs analysed as a P slice (set_lists(numRefs, 0)), timed
    the same way;
  * the share of PUs that go bi, and of CUs whose lowest-cost entry is not 2Nx2N;
  * the card's name, power limit and maximum SM clock, read in the same run.
Needs a GPU; prints one JSON line per config.

    python profiles/partitions_b.py [--configs c3,c4] [--reps 20]
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "profiles")]

from partitions import card                # noqa: E402

CONFIGS = {                               # bench.py's c3 / c4 shapes (BASELINE.json), as B slices
    "c3": dict(W=3840, H=2160, depth=8, numRefs=4, numRefL0=2, amp=0, subme=3, qp=30),
    "c4": dict(W=3840, H=2160, depth=10, numRefs=5, numRefL0=3, amp=1, subme=4, qp=30),
}


def timed(cu, an, stages, reps):
    for _ in range(3):
        an.run_resident(stages)
    ms = []
    for _ in range(reps):
        cu.timer_begin()
        an.run_resident(stages)
        ms.append(cu.timer_end())
    return ms


def run(cu, name, reps):
    from frame_helpers import Workload
    from test_gpu_x_partitions_b import open_analyser, source
    c = CONFIGS[name]
    wl = Workload(c["W"], c["H"], depth=c["depth"], numRefs=c["numRefs"], subme=c["subme"], rect=1, amp=c["amp"], qp=c["qp"],
                  chroma=True)
    an = open_analyser(cu, wl, c["numRefL0"], True)
    an.load_inputs(source(wl), wl.field)
    an.run_resident(1)
    me_ms = an.stage_ms()[0]
    part_b = timed(cu, an, 64, reps)
    rec = an.part_b_results()
    dirs = rec["interDir"]
    share_bi = float((dirs == 3).sum() / (dirs > 0).sum())
    not_2nx2n = float((np.argmin(rec["cost"], axis=1) != 0).mean())
    an.set_lists(c["numRefs"], 0)
    part_p = timed(cu, an, 32, reps)
    res = dict(config=name, card=card(), W=c["W"], H=c["H"], depth=c["depth"], numRefL0=c["numRefL0"],
               numRefL1=c["numRefs"] - c["numRefL0"], rect=1, amp=c["amp"], subme=c["subme"], chroma=True, ncu=an.ncu, reps=reps,
               part_b_stage_ms=round(statistics.median(part_b), 4), part_b_stage_ms_min=round(min(part_b), 4),
               part_p_stage_ms=round(statistics.median(part_p), 4), me_stage_ms=round(me_ms, 4),
               share_pu_bi=round(share_bi, 3), share_not_2Nx2N=round(not_2nx2n, 3))
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
