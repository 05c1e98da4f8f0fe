"""Device time of the frame analyser's per-CU stages at bench.py's c3 and c4 shapes: the luma residual (stage bit 1), the
intra search (bit 2) and the 4:2:0 chroma residual (bit 3).  The residual stages are instantiations of k_cu_residual
(resid.cuh), the intra stage is k_intra_cu (frame.cuh).  ME runs once; then stages 2, 4 and 8 are timed alternately with
CUDA events (x265cu_timer_begin / _end around run_resident), after warm-up.  Reports the median and min-max of each, the
chroma stage's achieved bandwidth from its compulsory bytes (source and reference chroma read once per TU, levels and recon
written), and the card's name and power limit.  Needs a GPU; prints one JSON line per config.

    python profiles/cu_stages.py [--configs c3,c4] [--reps 20] [--out DIR]
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


def compulsory_bytes(an, es):
    """Per run of stage 8: every CU's chroma block of source and reference read once per plane (all CU sizes: 4 x the chroma
    picture), levels (2 bytes) and recon written once per chroma sample of every CU."""
    samples = 2 * (an.ncoef // 4)         # chroma samples over all CUs, both planes
    return samples * (2 * es + 2 + es)


def run(cu, name, reps):
    from frame_helpers import Workload, run_analyser
    c = dict(CONFIGS[name])
    W, H = c.pop("W"), c.pop("H")
    wl = Workload(W, H, **c)
    an = run_analyser(cu, wl)                        # ME + luma stages once: the vectors both residual stages read
    an.enable_chroma_residual(0, 0)
    for stages in (2, 4, 8, 2, 4, 8):                 # warm-up of every launch shape
        an.run_resident(stages)
    cu.sync()
    t = {2: [], 4: [], 8: []}
    for _ in range(reps):
        for stages in (2, 4, 8):
            cu.timer_begin()
            an.run_resident(stages)
            t[stages].append(cu.timer_end())
    es = 1 if c["depth"] == 8 else 2
    nbytes = compulsory_bytes(an, es)
    luma, intra, chroma = statistics.median(t[2]), statistics.median(t[4]), statistics.median(t[8])
    an.close()
    return {"config": name, "reps": reps, "luma_residual_ms": luma, "intra_ms": intra, "chroma_residual_ms": chroma,
            "luma_ms_min_max": [min(t[2]), max(t[2])], "intra_ms_min_max": [min(t[4]), max(t[4])],
            "chroma_ms_min_max": [min(t[8]), max(t[8])],
            "chroma_over_luma": chroma / luma, "chroma_bytes": nbytes, "chroma_GBps": nbytes / (chroma / 1000.0) / 1e9}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="c3,c4")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", help="also write the results as DIR/cu_stages.json")
    args = ap.parse_args()
    import x265_b200
    cu = x265_b200.load()
    res = {"card": card(), "results": []}
    for name in args.configs.split(","):
        r = run(cu, name, args.reps)
        res["results"].append(r)
        print(json.dumps(r))
    print(json.dumps({"card": res["card"]}))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "cu_stages.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
