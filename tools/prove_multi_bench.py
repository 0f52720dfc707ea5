"""Proving on one device against proving on a list of devices (b200post_generate_proof against
b200post_generate_proof_multi), phase by phase.

Initialises an N = 8192 POST of 2^22 labels (64 MiB, four files) in a temporary directory, with NumUnits = --units (the
k2pow difficulty is the mainnet PowDifficulty divided by NumUnits, so --units sets the k2pow work), then for device 0
alone and for --providers (default "0,0": on a one-GPU box the repeated device measures the cost of sharding, not
scaling):
* k2pow: the builtin search of every nonce group (b200post_k2pow_search_groups[_multi]), hashes done and seconds;
* scan: the proving scan alone (generate_proof with the pows just found handed back through the pow hook, mainnet
  K1 = 26, K2 = 37), labels scanned and seconds, best of --repeat.  The files were just written, so the scan reads
  them from the page cache.
Both lists must give the same proof.  Prints one JSON line with the card name and power limit read in the same run.
Usage: python tools/prove_multi_bench.py [--units 1] [--nonces 288] [--providers 0,0] [--repeat 3]
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

LABELS = 1 << 22


def power_limit_w() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--units", type=int, default=1)
    ap.add_argument("--nonces", type=int, default=288)
    ap.add_argument("--providers", default="0,0")
    ap.add_argument("--repeat", type=int, default=3)
    a = ap.parse_args()
    b2 = importlib.import_module("go-spacemesh_b200")
    su = importlib.import_module("go-spacemesh_b200.setup")
    pr = importlib.import_module("go-spacemesh_b200.prove")
    k2 = importlib.import_module("go-spacemesh_b200.k2pow")
    provs = b2.providers()
    if not provs:
        raise SystemExit("no CUDA device")
    multi = [int(x) for x in a.providers.split(",")]
    if LABELS % a.units:
        raise SystemExit("--units must divide 2^22")
    node, atx, challenge = bytes(range(1, 33)), bytes(range(33, 65)), bytes(range(65, 97))
    cfg = su.PostConfig(labels_per_unit=LABELS // a.units, max_num_units=max(a.units, 1), k1=26, k2=37, k3=37)
    d = Path(tempfile.mkdtemp(prefix="prove_multi_bench_"))
    try:
        mgr = su.PostSetupManager(cfg)
        mgr.prepare_initializer(su.PostSetupOpts(data_dir=str(d), num_units=a.units, max_file_size=16 * (LABELS // 4),
                                                 provider_id=0, scrypt_n=8192), node, atx)
        mgr.start_session()
        md = su.load_metadata(str(d))
        # the library's default PowDifficulty (mainnet), scaled by NumUnits exactly as the prover scales it
        c = pr._c_cfg(cfg)
        scaled = k2.scale_difficulty(bytes(c.pow_difficulty), md["num_units"])
        groups = a.nonces // 16
        k2.prepare()                                  # dataset build (once per key and device) outside the timings
        runs, proofs = {}, []
        for name, plist in (("one_device", [0]), ("list", multi)):
            t0 = time.perf_counter()
            pows, hashes = k2.search_groups(challenge[:8], md["node_id"], scaled, groups, providers=plist)
            t_pow = time.perf_counter() - t0

            def hook(ctx, g, ch8, diff, nid, out, pows=pows):
                out[0] = pows[g]
                return 0
            t_scan, scanned, proof = float("inf"), 0, None
            for _ in range(a.repeat):
                t0 = time.perf_counter()
                proof, _, scanned = pr.generate_proof(str(d), challenge, cfg, nonces=a.nonces, pow=hook, providers=plist)
                t_scan = min(t_scan, time.perf_counter() - t0)
            proofs.append((pows, proof))
            runs[name] = {"providers": plist, "k2pow_s": round(t_pow, 2), "hashes_done": hashes,
                          "k2pow_hashes_per_s": round(hashes / t_pow, 1), "scan_s": round(t_scan, 4),
                          "labels_scanned": scanned, "scan_labels_per_s": round(scanned / t_scan, 1)}
        if proofs[0] != proofs[1]:
            raise SystemExit("the device list gave another proof than device 0")
        out = {"card": provs[0]["model"], "power_limit_w": power_limit_w(), "gpus_in_box": len(provs), "scrypt_n": 8192,
               "labels": LABELS, "num_units": a.units, "nonces": a.nonces, "k1": 26, "k2": 37, "scan_source": "page cache",
               "pow_difficulty_scaled": scaled.hex(), **runs,
               "k2pow_speedup": round(runs["one_device"]["k2pow_s"] / runs["list"]["k2pow_s"], 3),
               "scan_speedup": round(runs["one_device"]["scan_s"] / runs["list"]["scan_s"], 3)}
        print(json.dumps(out))
    finally:
        shutil.rmtree(d, ignore_errors=True)


if __name__ == "__main__":
    main()
