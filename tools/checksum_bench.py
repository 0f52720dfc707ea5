"""Block checksums (postdata_<N>.sum) on one GPU: what they cost at init and what the check and repair take.

On a POST of 2^22 labels at N = 8192 in four files, with its files in the page cache, this times
  - init without and with the checksum request (alternated, best of --repeat each): the overhead of hashing every batch;
  - check_sums (b200postcli -checkSums): labels/s and GB/s of reading and hashing the covered labels;
  - verify_pos at fraction 100 (b200postcli -verify -fraction 100) on the same data, the check it replaces;
  - check_sums with repair of 4 planted bad blocks (the scan plus recomputing, writing and re-reading 4 MiB).
Two scale points beside the N = 8192 POST, since 64 MiB is small next to the fixed cost of a call (pinned buffers,
the first read): check_sums on a 2^25-label (512 MiB) POST initialised at N = 2, and label_block_digests on 1 GiB of
labels already in (pageable) host memory.
It prints one JSON object, with the card's name and power limit, and writes it to --out when given.  Needs a GPU.

    python tools/checksum_bench.py [--labels 4194304] [--repeat 2] [--out FILE.json]
"""
from __future__ import annotations

import argparse
import importlib
import json
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

NODE, ATX = bytes(range(1, 33)), bytes(range(33, 65))
B = 1 << 16


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, _, limit = q.stdout.strip().splitlines()[0].partition(",") if q.returncode == 0 and q.stdout.strip() else ("unknown", "", "unknown")
    return {"gpu": name.strip(), "power_limit": limit.strip()}


def init(su, d: Path, labels: int, per_file: int, sums: bool, n: int = 8192) -> float:
    mgr = su.PostSetupManager(su.PostConfig(labels_per_unit=labels, max_num_units=1))
    mgr.prepare_initializer(su.PostSetupOpts(data_dir=str(d), num_units=1, max_file_size=16 * per_file, provider_id=0,
                                             scrypt_n=n, compute_batch_size=1 << 20), NODE, ATX)
    if sums:
        mgr.request_checksums()
    t = time.perf_counter()
    mgr.start_session()
    dt = time.perf_counter() - t
    assert mgr.status().state == su.STATE_COMPLETE
    return dt


def best_check(su, d: Path, labels: int, repeat: int = 3) -> float:
    for p in d.glob("postdata_*.bin"):   # page-cache the files
        p.read_bytes()
    best = None
    for _ in range(repeat):
        t = time.perf_counter()
        r = su.check_sums(str(d))
        dt = time.perf_counter() - t
        assert r.code == su.OK and r.labels_checked == labels
        best = dt if best is None else min(best, dt)
    return best


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--labels", type=int, default=1 << 22)
    ap.add_argument("--repeat", type=int, default=2)
    ap.add_argument("--out")
    a = ap.parse_args()
    b2 = importlib.import_module("go-spacemesh_b200")
    su = importlib.import_module("go-spacemesh_b200.setup")
    if not b2.providers():
        raise SystemExit("checksum_bench: no CUDA device (there is no CPU path)")
    per_file = a.labels // 4
    res = {"labels": a.labels, "scrypt_n": 8192, "files": 4, **card()}
    with tempfile.TemporaryDirectory() as tmp:
        root = Path(tmp)
        # warm the engine at N = 8192 (module load, scratch) outside the timed runs
        init(su, root / "warm", 1 << 16, 1 << 16, False)
        plain, summed = [], []
        for k in range(a.repeat):
            plain.append(init(su, root / f"plain{k}", a.labels, per_file, False))
            summed.append(init(su, root / f"sums{k}", a.labels, per_file, True))
        res["init_s"], res["init_checksums_s"] = min(plain), min(summed)
        res["init_overhead_pct"] = 100.0 * (min(summed) - min(plain)) / min(plain)
        d = root / f"sums{a.repeat - 1}"
        best = best_check(su, d, a.labels)
        res["check_s"] = best
        res["check_labels_per_s"] = a.labels / best
        res["check_GB_per_s"] = a.labels * 16 / best / 1e9
        t = time.perf_counter()
        v = su.verify_pos(str(d), fraction=100)
        res["verify_full_s"] = time.perf_counter() - t
        assert v.code == su.OK
        res["verify_full_labels_per_s"] = a.labels / res["verify_full_s"]
        for blk in (0, 5, 17, 63):   # four planted bad blocks
            f, off = divmod(blk * B, per_file)
            p = d / f"postdata_{f}.bin"
            with open(p, "r+b") as fh:
                fh.seek(off * 16 + 3)
                c = fh.read(1)
                fh.seek(off * 16 + 3)
                fh.write(bytes([c[0] ^ 0x20]))
        t = time.perf_counter()
        r = su.check_sums(str(d), repair=True)
        res["repair_4_blocks_s"] = time.perf_counter() - t
        assert r.code == su.OK and r.repaired_blocks == 4, r
        assert su.check_sums(str(d)).code == su.OK
        # scale points: a 512 MiB POST (N = 2, so that it is quick to make), and hashing 1 GiB already in host memory
        big = 1 << 25
        init(su, root / "big", big, big // 4, True, n=2)
        t = best_check(su, root / "big", big)
        res["check_512MiB_s"], res["check_512MiB_GB_per_s"] = t, big * 16 / t / 1e9
        buf = np.random.default_rng(0).integers(0, 256, 1 << 30, dtype=np.uint8)
        su.label_block_digests(buf[: 16 * B])
        best = None
        for _ in range(3):
            t = time.perf_counter()
            su.label_block_digests(buf)
            dt = time.perf_counter() - t
            best = dt if best is None else min(best, dt)
        res["hash_1GiB_host_s"], res["hash_1GiB_host_GB_per_s"] = best, (1 << 30) / best / 1e9
    line = json.dumps(res)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
