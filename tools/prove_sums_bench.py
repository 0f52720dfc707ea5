"""What proving over checksummed data costs (b200post_generate_proof_sums against b200post_generate_proof_checked) on
one device.

Initialises an N = 8192 POST of 2^25 labels (512 MiB, eight files) with block checksums in a temporary directory, then,
with 288 nonces, K1 = 26, K2 = 37 and pow SKIP (so that the scan is what is timed; both calls stop at the same label,
the decision point of the proof, or read every label when no nonce reaches K2):
* checked and sums calls on clean data alternately, best of --repeat each, in --runs runs (their spread is the noise);
* the device time of the digest launch (label_range_digests_kernel) per 64 MiB chunk, from one sums call under
  torch.profiler (CUDA activities) in a run of its own;
* the cost per healed block: one label in each of the first 4 blocks rewritten, the sums call's best time over clean
  data's.
The files were just written, so the scan reads them from the page cache.  Prints one JSON line with the card name and
power limit read in the same run.
Usage: python tools/prove_sums_bench.py [--repeat 3] [--runs 3]
"""
from __future__ import annotations

import argparse
import importlib
import json
import shutil
import sys
import tempfile
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

from tools.prove_multi_bench import power_limit_w  # noqa: E402

LABELS, FILES, NONCES, K1, K2, N = 1 << 25, 8, 288, 26, 37, 8192


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    b2 = importlib.import_module("go-spacemesh_b200")
    su = importlib.import_module("go-spacemesh_b200.setup")
    pr = importlib.import_module("go-spacemesh_b200.prove")
    provs = b2.providers()
    if not provs:
        raise SystemExit("no CUDA device")
    node, atx, challenge = bytes(range(1, 33)), bytes(range(33, 65)), bytes(range(65, 97))
    cfg = su.PostConfig(labels_per_unit=LABELS, max_num_units=1, k1=K1, k2=K2, k3=K2)
    per_file = LABELS // FILES
    d = Path(tempfile.mkdtemp(prefix="prove_sums_bench_"))

    def timed(call):
        """-> (seconds, the call's report: ProveCheck or SumsReport)"""
        t0 = time.perf_counter()
        try:
            rep = call(str(d), challenge, cfg, nonces=NONCES, pow="skip")[-1]
        except b2.B200PostError as e:
            if e.code != b2.ERR_INVALID_PROOF:
                raise
            rep = getattr(e, "sums", None)
        return time.perf_counter() - t0, rep

    try:
        t0 = time.perf_counter()
        mgr = su.PostSetupManager(cfg)
        mgr.prepare_initializer(su.PostSetupOpts(data_dir=str(d), num_units=1, max_file_size=16 * per_file, provider_id=0,
                                                 scrypt_n=N), node, atx)
        mgr.request_checksums()
        mgr.start_session()
        init_s = time.perf_counter() - t0
        timed(pr.generate_proof_checked)   # warm-up: engines, pinned staging, the page cache
        timed(pr.generate_proof_sums)
        runs = []
        for _ in range(a.runs):
            best = {"checked": float("inf"), "sums": float("inf")}
            for _ in range(a.repeat):
                best["checked"] = min(best["checked"], timed(pr.generate_proof_checked)[0])
                t, rep = timed(pr.generate_proof_sums)
                best["sums"] = min(best["sums"], t)
            runs.append({k: round(v, 4) for k, v in best.items()} | {"overhead_pct": round(100 * (best["sums"] / best["checked"] - 1), 2)})
        assert rep.blocks_checked > 0 and rep.labels_verified == rep.blocks_checked << 16 and rep.bad_blocks == 0, rep

        # the digest kernel's device time, in a run of its own under the profiler
        import torch
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.init()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            timed(pr.generate_proof_sums)
            torch.cuda.synchronize()
        dig = [ev for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA and "label_range_digests_kernel" in ev.name]
        dig_us = [ev.device_time for ev in dig] if dig and hasattr(dig[0], "device_time") else [ev.cuda_time for ev in dig]
        scan = [ev for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA and "prove_scan_kernel" in ev.name]
        scan_us = [ev.device_time for ev in scan] if scan and hasattr(scan[0], "device_time") else [ev.cuda_time for ev in scan]

        # four damaged blocks, one label each, at the start of the data (every scan reads them)
        with open(d / "postdata_0.bin", "r+b") as fh:
            for b in range(4):
                fh.seek(16 * (b << 16) + 16 * 7)
                fh.write(bytes(16))
        heal = float("inf")
        for _ in range(a.repeat):
            t, rep4 = timed(pr.generate_proof_sums)
            heal = min(heal, t)
        assert rep4.bad_blocks == 4 and rep4.healed_blocks == 4 and rep4.blocks_checked == rep.blocks_checked, rep4
        clean_best = min(r["sums"] for r in runs)
        out = {"card": provs[0]["model"], "power_limit_w": power_limit_w(), "scrypt_n": N, "labels": LABELS, "files": FILES,
               "nonces": NONCES, "k1": K1, "k2": K2, "pow": "skip", "scan_source": "page cache", "init_s": round(init_s, 1),
               "runs": runs, "blocks_checked": rep.blocks_checked,
               "digest_kernel": {"launches": len(dig_us), "mean_us_per_64MiB_chunk": round(sum(dig_us) / max(len(dig_us), 1), 1),
                                 "max_us": round(max(dig_us, default=0), 1), "total_ms": round(sum(dig_us) / 1e3, 2)},
               "scan_kernel_total_ms": round(sum(scan_us) / 1e3, 2),
               "healed_4_blocks_s": round(heal, 4), "heal_cost_ms_per_block": round(1e3 * (heal - clean_best) / 4, 1)}
        print(json.dumps(out))
    finally:
        shutil.rmtree(d, ignore_errors=True)


if __name__ == "__main__":
    main()
