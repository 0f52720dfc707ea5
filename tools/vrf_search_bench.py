"""Throughput of finding the VRF nonce from stored labels (b200post_search_vrf_nonce) against the full check of the
same data (verify_pos at fraction 100, which recomputes every label), on one GPU.

Initialises an N = 8192 POST of 2^22 labels (4 files of 2^20) in a temporary directory, for an identity whose nonce
lies inside the POST (so that no past-the-end search, which runs at label-engine speed, enters the stored scan's
time), then times both calls on it, the search also at smaller chunk sizes.
The files were just written, so both read them from the page cache: the search's rate here is "from page cache"; the
disk-bound rate is not measured (the page cache is not dropped).  A separate run under torch.profiler (CUDA activity)
gives the K8 kernel time and the H2D copy time per chunk.  Prints one JSON line with labels/s and GB/s of stored bytes,
the card and its power limit.
Usage: python tools/vrf_search_bench.py [--labels-log2 22] [--repeat 3] [--no-profile]
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


def profile_search(su, d: str, total: int) -> dict:
    """Device time per chunk of the two K8 kernels and of the H2D copies, from a torch.profiler trace of one search."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        su.search_vrf_nonce(d)
        torch.cuda.synchronize()
    k_us = {"stored_min_kernel": 0.0, "stored_tie_kernel": 0.0}
    h2d_us, h2d_n = 0.0, 0
    runtime_ms: dict[str, float] = {}
    for ev in prof.events():
        name = ev.name or ""
        dev_us = ev.time_range.elapsed_us()   # device events carry their own device interval
        for k in k_us:
            if k in name:
                k_us[k] += dev_us
        if "HtoD" in name or "Memcpy HtoD" in name:
            if dev_us > 100:   # the chunk copies, not the 4-byte counters
                h2d_us += dev_us
                h2d_n += 1
        elif name.startswith("cuda") and dev_us > 1000:   # host-side runtime calls that take > 1 ms (allocation, waits)
            runtime_ms[name] = round(runtime_ms.get(name, 0.0) + dev_us / 1000, 2)
    chunks = max(1, (total + (1 << 22) - 1) >> 22)
    out = {"chunks": chunks, "h2d_copies": h2d_n, "runtime_calls_over_1ms": runtime_ms}
    for k, v in k_us.items():
        out[k + "_us_per_chunk"] = round(v / chunks, 1)
    out["h2d_us_per_chunk"] = round(h2d_us / max(1, h2d_n), 1)
    out["kernel_share_of_h2d"] = round(sum(k_us.values()) / chunks / out["h2d_us_per_chunk"], 4) if h2d_n else None
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--labels-log2", type=int, default=22)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--no-profile", action="store_true")
    a = ap.parse_args()
    b2 = importlib.import_module("go-spacemesh_b200")
    su = importlib.import_module("go-spacemesh_b200.setup")
    provs = b2.providers()
    if not provs:
        raise SystemExit("no CUDA device")
    total = 1 << a.labels_log2
    per_file = max(1, total // 4)
    atx = bytes(range(1, 33))
    d = Path(tempfile.mkdtemp(prefix="vrf_search_bench_"))
    try:
        for seed in range(16):
            node = bytes([seed]) + bytes(range(1, 32))
            shutil.rmtree(d, ignore_errors=True)
            mgr = su.PostSetupManager(su.PostConfig(labels_per_unit=total, max_num_units=1))
            mgr.prepare_initializer(su.PostSetupOpts(data_dir=str(d), num_units=1, max_file_size=16 * per_file, provider_id=0,
                                                     scrypt_n=8192), node, atx)
            t0 = time.perf_counter()
            mgr.start_session()
            t_init = time.perf_counter() - t0
            want = su.load_metadata(str(d))
            if want["nonce"] < total:
                break
        else:
            raise SystemExit("no identity with its nonce inside the POST in 16 tries")
        su.search_vrf_nonce(str(d))   # warm-up: pinned staging, module load
        t_search = float("inf")
        for _ in range(a.repeat):
            t0 = time.perf_counter()
            got = su.search_vrf_nonce(str(d))
            t_search = min(t_search, time.perf_counter() - t0)
            if got != (want["nonce"], want["nonce_value"]):
                raise SystemExit(f"search_vrf_nonce gave {got[0]}, the init recorded {want['nonce']}")
        by_chunk = {}
        for log2 in (20, 18):
            best = float("inf")
            for _ in range(a.repeat):
                t0 = time.perf_counter()
                su.search_vrf_nonce(str(d), chunk_labels=1 << log2)
                best = min(best, time.perf_counter() - t0)
            by_chunk[f"2^{log2}"] = round(total / best, 1)
        t_full = float("inf")
        for _ in range(a.repeat):
            t0 = time.perf_counter()
            r = su.verify_pos(str(d), fraction=100.0, seed=1)
            t_full = min(t_full, time.perf_counter() - t0)
            if r.code != b2.OK or not r.argmin_ok:
                raise SystemExit(f"verify_pos returned {r.code} on clean data")
        out = {
            "card": provs[0]["model"], "power_limit_w": power_limit_w(), "scrypt_n": 8192, "labels": total, "files": 4,
            "init_labels_per_s": round(total / t_init, 1),
            "search_labels_per_s": round(total / t_search, 1), "search_s": round(t_search, 4),
            "search_stored_gb_per_s": round(16 * total / t_search / 1e9, 2), "search_source": "page cache",
            "search_labels_per_s_by_chunk": by_chunk, "nonce_seed": seed,
            "full_check_labels_per_s": round(total / t_full, 1), "full_check_s": round(t_full, 3),
        }
        out["search_vs_full_check"] = round(t_full / t_search, 1)
        if not a.no_profile:
            out["profile"] = profile_search(su, str(d), total)
        print(json.dumps(out))
    finally:
        shutil.rmtree(d, ignore_errors=True)


if __name__ == "__main__":
    main()
