"""Several identities proving on one box: M single calls (b200post_generate_proof_checked, one after another) against
one b200post_generate_proofs call over the same M POSTs.

Initialises M = 4 N = 8192 POSTs of different identities in a temporary directory, LabelsPerUnit = 2^20 and NumUnits
alternating 1 and 4 (2^20 and 2^22 labels; the k2pow difficulty is the mainnet PowDifficulty divided by NumUnits), then
for each nonce count (16 and 288 by default) alternates the two ways, --repeat times each, with the builtin k2pow at
the mainnet PowDifficulty:
* k2pow alone, nonce window 0: M b200post_k2pow_search_group_range calls against one b200post_k2pow_search_jobs call
  over the same groups: wall time, device time, VM batches and hashes (b200post_randomx_last_timing); same pows;
* whole proofs with max_windows = all: M b200post_generate_proof_checked calls against one generate_proofs call:
  wall time; every item must equal its single call.
Best of the repeats by proving wall time.  The POST files were just written, so the scans read them from the page
cache: cold storage is not measured, nor is more than one GPU.  One JSON line with the card name and power limit read
in the same run.
Usage: python tools/prove_many_bench.py [--repeat 2] [--nonces 16,288]
"""
from __future__ import annotations

import argparse
import importlib
import json
import shutil
import subprocess
import sys
import tempfile
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

LPU, UNITS = 1 << 20, (1, 4, 1, 4)


def power_limit_w() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=2)
    ap.add_argument("--nonces", default="16,288")
    a = ap.parse_args()
    b2 = importlib.import_module("go-spacemesh_b200")
    su = importlib.import_module("go-spacemesh_b200.setup")
    pr = importlib.import_module("go-spacemesh_b200.prove")
    k2 = importlib.import_module("go-spacemesh_b200.k2pow")
    provs = b2.providers()
    if not provs:
        raise SystemExit("no CUDA device")
    cfg = su.PostConfig(labels_per_unit=LPU, max_num_units=4, k1=26, k2=37, k3=37)
    root = Path(tempfile.mkdtemp(prefix="prove_many_bench_"))
    try:
        items = []
        for i, units in enumerate(UNITS):
            d = root / f"id{i}"
            mgr = su.PostSetupManager(cfg)
            mgr.prepare_initializer(su.PostSetupOpts(data_dir=str(d), num_units=units, max_file_size=16 * LPU, provider_id=0,
                                                     scrypt_n=8192), bytes([i + 1]) * 32, bytes(range(33, 65)))
            mgr.start_session()
            items.append((str(d), bytes([100 + i]) * 32))
        k2.prepare()                                  # dataset build (once per key and device) outside the timings
        c = pr._c_cfg(cfg)
        scaled = [k2.scale_difficulty(bytes(c.pow_difficulty), u) for u in UNITS]
        nodes = [bytes([i + 1]) * 32 for i in range(len(UNITS))]
        runs = {}
        for nonces in [int(x) for x in a.nonces.split(",")]:
            groups = nonces // 16
            best = {}
            for _ in range(a.repeat):
                # k2pow alone, window 0: M group searches one after another, then one job search over all their groups
                t0, ms, batches, hashes, pows = time.perf_counter(), 0.0, 0, 0, []
                for (d, ch), node, diff in zip(items, nodes, scaled):
                    pows += k2.search_group_range(ch[:8], node, diff, 0, groups)[0]
                    t = k2.last_timing()
                    ms += t["total_ms"]; batches += t["vm_launches"] // 8; hashes += t["hashes"]
                single = {"wall_s": time.perf_counter() - t0, "device_s": ms / 1e3, "batches": batches, "hashes": hashes}
                t0 = time.perf_counter()
                jp, _ = k2.search_jobs([(node, ch[:8], g, diff) for (d, ch), node, diff in zip(items, nodes, scaled)
                                        for g in range(groups)])
                t = k2.last_timing()
                many = {"wall_s": time.perf_counter() - t0, "device_s": t["total_ms"] / 1e3, "batches": t["vm_launches"] // 8,
                        "hashes": t["hashes"]}
                if jp != pows:
                    raise SystemExit(f"the job search differs from the group searches at {nonces} nonces")
                # whole proofs over every window until one has a proof (a post-service's behaviour): M calls, one call
                t0 = time.perf_counter()
                alone = [pr.generate_proof_checked(d, ch, cfg, nonces=nonces, max_windows="all") for d, ch in items]
                single["prove_wall_s"] = time.perf_counter() - t0
                t0 = time.perf_counter()
                rc, got = pr.generate_proofs(items, cfg, nonces=nonces, max_windows="all")
                many["prove_wall_s"] = time.perf_counter() - t0
                if rc != b2.OK or [(g.proof, g.meta, g.labels_scanned, g.check) for g in got] != [tuple(x) for x in alone]:
                    raise SystemExit(f"generate_proofs differs from the single calls at {nonces} nonces")
                for k, r in (("single_calls", single), ("one_call", many)):
                    if k not in best or r["prove_wall_s"] < best[k]["prove_wall_s"]:
                        best[k] = r
            runs[f"nonces_{nonces}"] = {k: {kk: round(vv, 3) if isinstance(vv, float) else vv for kk, vv in v.items()}
                                        for k, v in best.items()}
            runs[f"nonces_{nonces}"]["prove_speedup"] = round(best["single_calls"]["prove_wall_s"] / best["one_call"]["prove_wall_s"], 3)
            runs[f"nonces_{nonces}"]["k2pow_speedup"] = round(best["single_calls"]["wall_s"] / best["one_call"]["wall_s"], 3)
        out = {"card": provs[0]["model"], "power_limit_w": power_limit_w(), "identities": len(UNITS), "num_units": list(UNITS),
               "labels_per_unit": LPU, "scrypt_n": 8192, "k1": 26, "k2": 37, "pow": "builtin, mainnet PowDifficulty",
               "checked": True, "scan_source": "page cache", "gpus": 1, **runs}
        print(json.dumps(out))
    finally:
        shutil.rmtree(root, ignore_errors=True)


if __name__ == "__main__":
    main()
