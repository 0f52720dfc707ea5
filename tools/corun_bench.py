"""Verification latency while a POST initialisation runs on the same GPU, and what the verification load costs the
initialisation.

One thread runs labels_range calls of --batch labels at scrypt-N --n (what a setup session issues per
ComputeBatchSize batch); another submits verify_batch calls of 1, 37 and 1000 proofs (K2 = 37 random indices each, the
pow check skipped) at a fixed rate.  Three phases per batch size:

  init alone   : per-call duration (what a verify call waits today at worst) and labels/s
  verify alone : p50 / p99 latency per batch size
  together     : the same latencies while init runs, init labels/s under that load, rider counters of the library

Only public entry points are used, so --lib points the same script at another build of the library (e.g. one of the
parent commit) for a before/after comparison.  The card name and power limit are printed with the numbers.

    python tools/corun_bench.py [--lib path/to/libb200post.so] [--n 8192] [--batch 1048576 16777216] [--calls 3]
"""
from __future__ import annotations

import argparse
import importlib
import json
import re
import subprocess
import sys
import threading
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
        return {"card": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001
        return {"card": "unknown", "power_limit": f"unknown ({e})"}


def rider_counters(pkg) -> dict:
    text = pkg.metrics_text()
    got = {}
    for key in ("b200post_engine_rider_calls_total", "b200post_engine_rider_labels_total"):
        m = re.search(rf"^{key} (\d+)$", text, re.M)
        got[key] = int(m.group(1)) if m else None   # None: a library without riders
    return got


def make_batches(vf, n: int, sizes, seed: int = 1):
    rng = np.random.default_rng(seed)
    num_labels, k2 = 4 * 2**32, 37
    bits = vf.bits_per_index(num_labels)
    params = vf.VerifyParams(k1=2**31, k2=k2, scrypt_n=n)
    out = {}
    for p in sizes:
        proofs, metas = [], []
        for _ in range(p):
            node, atx, ch = (bytes(rng.integers(0, 256, 32, dtype=np.uint8)) for _ in range(3))
            ix = [int(x) for x in rng.integers(0, num_labels, k2)]
            proofs.append(vf.Proof(int(rng.integers(0, 288)), vf.pack_indices(ix, bits), 0))
            metas.append(vf.ProofMetadata(node, atx, ch, 4, 2**32))
        out[p] = (proofs, metas, params)
    return out


def pct(xs, q):
    return float(np.percentile(np.array(xs), q)) if xs else None


def verify_loop(vf, batches, interval: float, stop: threading.Event, lat: dict, min_rounds: int = 0):
    """Submit the batch sizes round-robin, one call every `interval` s, until `stop` (and at least min_rounds rounds)."""
    rounds = 0
    nxt = time.perf_counter()
    while not stop.is_set() or rounds < min_rounds:
        for p, (proofs, metas, params) in batches.items():
            now = time.perf_counter()
            if nxt > now:
                time.sleep(nxt - now)
            t0 = time.perf_counter()
            vf.verify_batch(proofs, metas, params, pow="skip")
            lat[p].append(time.perf_counter() - t0)
            nxt = max(nxt + interval, time.perf_counter())
            if stop.is_set() and rounds + 1 >= min_rounds:
                break
        rounds += 1


def init_calls(pkg, n: int, batch: int, calls: int, start_at: int = 0):
    commitment = pkg.commitment(bytes(32), bytes(range(32)))
    durs = []
    t0 = time.perf_counter()
    for k in range(calls):
        c0 = time.perf_counter()
        pkg.labels_range(commitment, n, start_at + k * batch, batch, discard=True)
        durs.append(time.perf_counter() - c0)
    return durs, calls * batch / (time.perf_counter() - t0)


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--lib", help="libb200post.so to load instead of the package's own")
    ap.add_argument("--n", type=int, default=8192)
    ap.add_argument("--batch", type=int, nargs="+", default=[1 << 20, 1 << 24])
    ap.add_argument("--calls", type=int, default=3, help="init calls per phase (per batch size)")
    ap.add_argument("--proofs", type=int, nargs="+", default=[1, 37, 1000])
    ap.add_argument("--interval", type=float, default=0.25, help="seconds between verify submissions")
    ap.add_argument("--label", default="", help="name of this build in the output")
    args = ap.parse_args()

    pkg = importlib.import_module("go-spacemesh_b200")
    if args.lib:
        pkg.LIB_PATH = Path(args.lib).resolve()
    vf = importlib.import_module("go-spacemesh_b200.verify")
    head = dict(card(), tool="corun_bench", build=args.label or str(pkg.LIB_PATH), n=args.n)
    print(json.dumps(head), flush=True)
    batches = make_batches(vf, args.n, args.proofs)
    # warm-up: engine scratch, verifier tables, low-latency and layered kernels
    init_calls(pkg, args.n, 1 << 16, 1)
    for proofs, metas, params in batches.values():
        vf.verify_batch(proofs, metas, params, pow="skip")

    lat_alone = {p: [] for p in args.proofs}
    stop = threading.Event()
    stop.set()
    verify_loop(vf, batches, args.interval, stop, lat_alone, min_rounds=8)
    res_verify = {str(p): {"p50_ms": 1e3 * pct(v, 50), "p99_ms": 1e3 * pct(v, 99), "calls": len(v)} for p, v in lat_alone.items()}
    print(json.dumps(dict(head, phase="verify_alone", latency=res_verify)), flush=True)

    for batch in args.batch:
        durs, rate = init_calls(pkg, args.n, batch, args.calls)
        print(json.dumps(dict(head, phase="init_alone", batch=batch, call_s=[round(d, 4) for d in durs], labels_per_s=round(rate))),
              flush=True)
        before = rider_counters(pkg)
        lat = {p: [] for p in args.proofs}
        stop = threading.Event()
        th = threading.Thread(target=verify_loop, args=(vf, batches, args.interval, stop, lat))
        th.start()
        try:
            durs, rate = init_calls(pkg, args.n, batch, args.calls, start_at=args.calls * batch)
        finally:
            stop.set()
            th.join()
        after = rider_counters(pkg)
        riders = {k: (after[k] - before[k]) if after[k] is not None else None for k in after}
        res = {str(p): {"p50_ms": 1e3 * pct(v, 50) if v else None, "p99_ms": 1e3 * pct(v, 99) if v else None, "calls": len(v)}
               for p, v in lat.items()}
        print(json.dumps(dict(head, phase="together", batch=batch, call_s=[round(d, 4) for d in durs], labels_per_s=round(rate),
                              latency=res, riders=riders)), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
