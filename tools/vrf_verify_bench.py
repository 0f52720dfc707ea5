"""Throughput of VRF-nonce checks at N = 8192 on one GPU: one call per check (b200post_verify_vrf_nonce) against one
batch (b200post_verify_vrf_nonces) at several sizes, and a mixed verifier load of proofs and VRF checks.

- per call: b200post_verify_vrf_nonce over 200 checks, one after another;
- batch: b200post_verify_vrf_nonces at 200, 4096, 10 000 and wave_slots(8192) + 1 checks (best of --repeat, after one
  warm-up call per size); the 200-check batch must give the per-call verdicts;
- mixed: 64 threads on one verifier handle (pow SKIP), each submitting K3 = 1 SUBSET proofs (K2 = 37, 4 units of 2^32
  labels) and VRF checks in equal numbers; and the same proofs alone, for comparison.
Prints one JSON line with checks/s and proofs/s, the card and its power limit.
Usage: python tools/vrf_verify_bench.py [--repeat 2] [--per-thread 24]
"""
from __future__ import annotations

import argparse
import importlib
import json
import subprocess
import sys
import threading
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

N = 8192


def power_limit_w() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def checks(b2, rng, count):
    """Checks as a syncing node sees them: distinct identities, 4 units of 2^32 labels, nonces anywhere in the POST."""
    ids = rng.integers(0, 256, (count, 64), dtype=np.uint8)
    nonces = rng.integers(0, 4 * 2**32, count, dtype=np.uint64)
    return [b2.vrf_check(bytes(ids[i, :32]), bytes(ids[i, 32:]), int(nonces[i]), 4, 2**32, N) for i in range(count)]


def mixed(vf, b2, rng, threads, per_thread, with_vrf):
    k2, num_labels = 37, 4 * 2**32
    bits = vf.bits_per_index(num_labels)
    params = vf.VerifyParams(k1=26, k2=k2, scrypt_n=N)
    work = []
    for _ in range(threads * per_thread):
        ident = bytes(rng.integers(0, 256, 96, dtype=np.uint8))
        proof = vf.Proof(int(rng.integers(0, 288)), vf.pack_indices([int(x) for x in rng.integers(0, num_labels, k2)], bits), 0)
        meta = vf.ProofMetadata(ident[:32], ident[32:64], ident[64:], 4, 2**32)
        work.append((proof, meta, int(rng.integers(0, num_labels))))
    v = vf.PostVerifier(pow="skip")
    errors = []

    def caller(t):
        try:
            for j in range(per_thread):
                proof, meta, nonce = work[t * per_thread + j]
                try:
                    v.verify(proof, meta, params, mode=vf.MODE_SUBSET, k3=1, seed=b"local-peer")
                except vf.ErrInvalidIndex:
                    pass
                if with_vrf:
                    v.verify_vrf_nonce(meta.node_id, meta.commitment_atx_id, nonce, 4, 2**32, N)
        except Exception as e:  # noqa: BLE001
            errors.append(repr(e))

    th = [threading.Thread(target=caller, args=(t,)) for t in range(threads)]
    t0 = time.perf_counter()
    for t in th: t.start()
    for t in th: t.join()
    el = time.perf_counter() - t0
    batches, proofs = v.stats()
    v.close()
    if errors:
        raise SystemExit(f"mixed load failed: {errors[:3]}")
    calls = threads * per_thread
    out = {"proofs": calls, "proofs_per_s": round(calls / el, 1), "batches": batches, "s": round(el, 3)}
    if with_vrf:
        out.update(checks=calls, checks_per_s=round(calls / el, 1))
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=2)
    ap.add_argument("--per-thread", type=int, default=24)
    a = ap.parse_args()
    b2 = importlib.import_module("go-spacemesh_b200")
    vf = importlib.import_module("go-spacemesh_b200.verify")
    provs = b2.providers()
    if not provs:
        raise SystemExit("no CUDA device")
    rng = np.random.default_rng(2026)
    wave = b2.wave_slots(N)

    per_call = checks(b2, rng, 200)
    b2.verify_vrf_nonce(per_call[0].nonce, bytes(per_call[0].node_id), bytes(per_call[0].commitment_atx_id), 4, 2**32, N)   # warm-up
    t0 = time.perf_counter()
    single = [b2.verify_vrf_nonce(c.nonce, bytes(c.node_id), bytes(c.commitment_atx_id), 4, 2**32, N) for c in per_call]
    t_single = time.perf_counter() - t0
    if [g[1] for g in b2.verify_vrf_nonces(per_call)] != single:
        raise SystemExit("the batch and the per-call verdicts differ")

    batch = {}
    for count in (200, 4096, 10000, wave + 1):
        cs = per_call if count == 200 else checks(b2, rng, count)
        b2.verify_vrf_nonces(cs)   # warm-up: scratch and judge buffers at this size
        best = float("inf")
        for _ in range(a.repeat):
            t0 = time.perf_counter()
            got = b2.verify_vrf_nonces(cs)
            best = min(best, time.perf_counter() - t0)
        if any(g[0] != b2.OK for g in got):
            raise SystemExit(f"batch of {count} returned errors")
        batch[str(count)] = {"checks_per_s": round(count / best, 1), "s": round(best, 4)}

    mixed(vf, b2, rng, 8, 2, True)   # warm-up of the verifier path
    out = {
        "card": provs[0]["model"], "power_limit_w": power_limit_w(), "scrypt_n": N, "wave_slots": wave,
        "per_call_checks_per_s": round(len(per_call) / t_single, 1), "per_call_ms": round(1000 * t_single / len(per_call), 2),
        "batch": batch,
        "mixed_64_threads": mixed(vf, b2, rng, 64, a.per_thread, True),
        "proofs_only_64_threads": mixed(vf, b2, rng, 64, a.per_thread, False),
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
