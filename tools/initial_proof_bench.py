"""What producing the initial proof during initialisation costs, and what it saves.

On one device, N = 8192, 2^22 labels (64 MiB) in four files, 288 nonces, K1 = 26, K2 = 37, best of --repeat, the cases
alternating:
* (a) a setup session;
* (b) the same session with the initial proof requested, pow SKIP: (b) - (a) as a share of (a) is what the in-session
  scan costs;
* (c) b200post_generate_proof over the files just written, pow SKIP: the read the request removes.  The files are in
  the page cache, so this is a lower bound on the time of that read from disk;
* (d) once, with pow BUILTIN at the mainnet difficulty: the session's time, (d) - (b) as the pow step's time, and the
  label layer's slot count read while the session runs (after its first batch) next to (a)'s.
Prints one JSON line with the card name and power limit read in the same run.
Usage: python tools/initial_proof_bench.py [--repeat 3]
"""
from __future__ import annotations

import argparse
import importlib
import json
import shutil
import sys
import tempfile
import threading
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

from tools.prove_multi_bench import power_limit_w  # noqa: E402

LABELS, NONCES, K1, K2, N = 1 << 22, 288, 26, 37, 8192


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=3)
    a = ap.parse_args()
    b2 = importlib.import_module("go-spacemesh_b200")
    su = importlib.import_module("go-spacemesh_b200.setup")
    pr = importlib.import_module("go-spacemesh_b200.prove")
    provs = b2.providers()
    if not provs:
        raise SystemExit("no CUDA device")
    node, atx = bytes(range(1, 33)), bytes(range(33, 65))
    cfg = su.PostConfig(labels_per_unit=LABELS, max_num_units=1, k1=K1, k2=K2, k3=K2)   # the mainnet pow difficulty
    per_file = LABELS // 4
    d = Path(tempfile.mkdtemp(prefix="initial_proof_bench_"))

    def session(pow_=None, watch=False):
        mgr = su.PostSetupManager(cfg)
        mgr.prepare_initializer(su.PostSetupOpts(data_dir=str(d), num_units=1, max_file_size=16 * per_file, provider_id=0,
                                                 scrypt_n=N), node, atx)
        if pow_ is not None:
            mgr.request_initial_proof(nonces=NONCES, pow=pow_)
        slots = []

        def read_slots():   # the layer's size once the first batch is written (it re-evaluates free HBM)
            while mgr.status().num_labels_written == 0:
                time.sleep(0.001)
            slots.append(b2.wave_slots(N))

        t = threading.Thread(target=read_slots) if watch else None
        if t:
            t.start()
        t0 = time.perf_counter()
        mgr.start_session()
        el = time.perf_counter() - t0
        if t:
            t.join()
        proof = mgr.initial_proof()[0] if pow_ is not None else None
        return mgr, el, proof, slots[0] if slots else None

    try:
        best = {"a": float("inf"), "b": float("inf"), "c": float("inf")}
        proof_b = proof_c = None
        for _ in range(a.repeat):
            for case in ("a", "b"):
                mgr, el, proof, _ = session("skip" if case == "b" else None)
                best[case] = min(best[case], el)
                if case == "b":
                    proof_b = proof
                    t0 = time.perf_counter()
                    proof_c, _, scanned = pr.generate_proof(str(d), bytes(32), cfg, nonces=NONCES, pow="skip")
                    best["c"] = min(best["c"], time.perf_counter() - t0)
                mgr.reset()
        if (proof_b.nonce, proof_b.indices, proof_b.pow) != (proof_c.nonce, proof_c.indices, proof_c.pow):
            raise SystemExit("the session's initial proof differs from generate_proof over its files")
        mgr, _, _, slots_a = session(None, watch=True)
        mgr.reset()
        mgr, el_d, proof_d, slots_d = session("builtin", watch=True)
        mgr.reset()
        out = {"card": provs[0]["model"], "power_limit_w": power_limit_w(), "scrypt_n": N, "labels": LABELS, "files": 4,
               "nonces": NONCES, "k1": K1, "k2": K2, "repeat": a.repeat,
               "a_session_s": round(best["a"], 3), "b_session_with_proof_s": round(best["b"], 3),
               "b_minus_a_share": round((best["b"] - best["a"]) / best["a"], 4),
               "c_generate_proof_page_cache_s": round(best["c"], 4), "c_labels_scanned": scanned,
               "d_builtin_session_s": round(el_d, 3), "d_pow_step_s_approx": round(el_d - best["b"], 3),
               "slots_without_request": slots_a, "slots_with_builtin_request": slots_d, "proof_nonce": proof_b.nonce}
        print(json.dumps(out))
    finally:
        shutil.rmtree(d, ignore_errors=True)


if __name__ == "__main__":
    main()
