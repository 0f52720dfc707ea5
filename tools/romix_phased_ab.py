"""A/B of the two two-scratchpad ROMix layers at bench.py's batch: romix_variant 4 (pipelined: layer m fills while
layer m-1 mixes) against 5 (phased: both labels of a slot fill, then both mix), alternated in one process.

Prints one JSON line per timed call (labels/s from the call's device time) and a summary line with the card, its power
limit and the clocks sampled over the whole run.  Run on the GPU box from the repository root:
    python tools/romix_phased_ab.py [--rounds 3] [--batch 2162688]
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import bench  # noqa: E402  (ClockSampler, batch and N of the flagship workload)
from __graft_entry__ import load_package  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=bench.DEFAULT_BATCH)
    args = ap.parse_args()
    b2 = load_package()
    n = bench.N_SCRYPT
    commitment = b2.commitment(bytes(32), bytes(32))
    keep = b2.get_option("romix_variant")
    start = 0
    rates = {4: [], 5: []}
    sampler = bench.ClockSampler(0)
    try:
        for v in (4, 5):                       # warm-up: module load, scratch and layer buffers of each variant
            b2.set_option("romix_variant", v)
            b2.labels_range(commitment, n, start, args.batch, discard=True)
            start += args.batch
        sampler.start()
        for r in range(args.rounds):
            for v in (4, 5):
                b2.set_option("romix_variant", v)
                b2.labels_range(commitment, n, start, args.batch, discard=True)
                start += args.batch
                rate = args.batch / (b2.last_call_ms() / 1e3)
                rates[v].append(rate)
                print(json.dumps({"romix_variant": v, "round": r, "call_ms": b2.last_call_ms(), "labels_per_s": rate}), flush=True)
        clocks = sampler.stop()
    finally:
        b2.set_option("romix_variant", keep)
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    summary = {v: {"min": min(x), "max": max(x), "spread": (max(x) - min(x)) / min(x)} for v, x in rates.items()}
    print(json.dumps({"card": q, "batch": args.batch, "N": n, "wave_slots": b2.wave_slots(n), "clocks": clocks,
                      "pipelined": summary[4], "phased": summary[5],
                      "phased_over_pipelined_worst_case": summary[5]["min"] / summary[4]["max"]}), flush=True)


if __name__ == "__main__":
    main()
