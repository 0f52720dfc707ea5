"""Throughput of checking stored POST data against initialising it, on one GPU.

Initialises an N = 8192 POST of 2^22 labels (4 files of 2^20) in a temporary directory, then times a full check
(fraction 100) and a 1 % check of the same data.  Besides the setup session (which also writes files, saves metadata
and cross-checks labels on the CPU) the engine alone computes the same range (labels to host memory, VRF scan on), the
like-for-like baseline of a full check.  Prints one JSON line with labels/s for each, the card and its power limit.
Usage: python tools/verify_pos_bench.py [--labels-log2 22] [--repeat 2]
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


def power_limit_w() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--labels-log2", type=int, default=22)
    ap.add_argument("--repeat", type=int, default=2)
    a = ap.parse_args()
    b2 = importlib.import_module("go-spacemesh_b200")
    su = importlib.import_module("go-spacemesh_b200.setup")
    provs = b2.providers()
    if not provs:
        raise SystemExit("no CUDA device")
    total = 1 << a.labels_log2
    per_file = min(total, 1 << 20)
    node, atx = bytes(range(32)), bytes(range(1, 33))
    # warm-up: scratch for a full layer is allocated outside the timed regions
    wave = b2.wave_slots(8192)
    b2.labels_range(b2.commitment(node, atx), 8192, 1 << 40, 4 * wave)
    d = Path(tempfile.mkdtemp(prefix="verify_pos_bench_"))
    try:
        mgr = su.PostSetupManager(su.PostConfig(labels_per_unit=total, max_num_units=1))
        mgr.prepare_initializer(su.PostSetupOpts(data_dir=str(d), num_units=1, max_file_size=16 * per_file, provider_id=0,
                                                 scrypt_n=8192), node, atx)
        t0 = time.perf_counter()
        mgr.start_session()
        t_init = time.perf_counter() - t0
        c, diff = b2.commitment(node, atx), b2.vrf_difficulty(total)
        t_engine = float("inf")
        for _ in range(a.repeat):
            t0 = time.perf_counter()
            b2.labels_range(c, 8192, 0, total, vrf_difficulty_=diff)
            t_engine = min(t_engine, time.perf_counter() - t0)
        timings = {}
        for name, fraction in (("full", 100.0), ("sample_1pct", 1.0)):
            best, checked = float("inf"), 0
            for _ in range(a.repeat):
                t0 = time.perf_counter()
                r = su.verify_pos(str(d), fraction=fraction, seed=1)
                el = time.perf_counter() - t0
                if r.code != b2.OK:
                    raise SystemExit(f"{name}: verify_pos returned {r.code} on clean data")
                best, checked = min(best, el), r.labels_checked
            timings[name] = (best, checked)
        out = {
            "card": provs[0]["model"], "power_limit_w": power_limit_w(), "scrypt_n": 8192, "labels": total,
            "init_labels_per_s": round(total / t_init, 1), "init_s": round(t_init, 3),
            "engine_range_labels_per_s": round(total / t_engine, 1), "engine_range_s": round(t_engine, 3),
            "full_check_labels_per_s": round(timings["full"][1] / timings["full"][0], 1), "full_check_s": round(timings["full"][0], 3),
            "sample_1pct_labels_per_s": round(timings["sample_1pct"][1] / timings["sample_1pct"][0], 1),
            "sample_1pct_s": round(timings["sample_1pct"][0], 3), "sample_1pct_labels": timings["sample_1pct"][1],
        }
        out["full_check_vs_init"] = round(out["full_check_labels_per_s"] / out["init_labels_per_s"], 4)
        out["full_check_vs_engine_range"] = round(out["full_check_labels_per_s"] / out["engine_range_labels_per_s"], 4)
        print(json.dumps(out))
    finally:
        shutil.rmtree(d, ignore_errors=True)


if __name__ == "__main__":
    main()
