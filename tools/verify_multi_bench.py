"""One verify batch on one device against the same batch split over a list of devices (b200post_verify_batch against
b200post_verify_batch_multi).

The batch is bench.py's verify workload: --proofs proofs x K2 = 37 indices at N = 8192, half of them valid proofs of
small POSTs initialised and proven on device 0, half with one index bumped.  Both calls are warmed up at full size,
then timed alternately, best of --repeat each, without the k2pow check.  --providers defaults to "0,0": on a one-GPU
box the repeated device measures the cost of splitting the batch over host threads, not scaling.  Both must give the
same statuses.  Prints one JSON line with the card name and power limit read in the same run.
Usage: python tools/verify_multi_bench.py [--proofs 10000] [--providers 0,0] [--repeat 5]
"""
from __future__ import annotations

import argparse
import importlib
import json
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

import bench  # noqa: E402  (its verify workload and proof generator)
from tools.prove_multi_bench import power_limit_w  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--proofs", type=int, default=10000)
    ap.add_argument("--providers", default="0,0")
    ap.add_argument("--repeat", type=int, default=5)
    a = ap.parse_args()
    b2 = importlib.import_module("go-spacemesh_b200")
    vf = importlib.import_module("go-spacemesh_b200.verify")
    pr = importlib.import_module("go-spacemesh_b200.prove")
    provs = b2.providers()
    if not provs:
        raise SystemExit("no CUDA device")
    multi = [int(x) for x in a.providers.split(",")]
    labels_per_id, k1, k2 = 4096, 96, 37
    bits = vf.bits_per_index(labels_per_id)
    base = bench._valid_proofs(b2, vf, pr, 0, 48, k2, labels_per_id, k1)
    proofs, metas = [], []
    for i in range(a.proofs):
        p, m = base[i % len(base)]
        if i % 2:
            idx = vf.unpack_indices(p.indices, bits, k2)
            idx[(i // 2) % k2] = (idx[(i // 2) % k2] + 1) % labels_per_id
            p = vf.Proof(p.nonce, vf.pack_indices(idx, bits), p.pow)
        proofs.append(p)
        metas.append(m)
    batch = vf.PreparedBatch(proofs, metas, vf.VerifyParams(k1=k1, k2=k2, scrypt_n=bench.N_SCRYPT))
    runs = {"one": lambda: batch.run(0, "skip"), "multi": lambda: batch.run_multi(multi, "skip")}
    results = {name: run() for name, run in runs.items() for _ in range(2)}   # warm-up
    best = {name: float("inf") for name in runs}
    for _ in range(a.repeat):
        for name, run in runs.items():
            t0 = time.perf_counter()
            results[name] = run()
            best[name] = min(best[name], time.perf_counter() - t0)
    print(json.dumps({"tool": "verify_multi_bench", "gpu": provs[0]["model"], "power_limit_w": power_limit_w(),
                      "proofs": a.proofs, "k2": k2, "providers": multi, "repeat": a.repeat,
                      "one_device_s": best["one"], "multi_s": best["multi"],
                      "one_device_proofs_per_s": a.proofs / best["one"], "multi_proofs_per_s": a.proofs / best["multi"],
                      "same_statuses": results["one"] == results["multi"]}))


if __name__ == "__main__":
    main()
