"""What scanning several nonce windows per read of the POST costs and saves (b200post_prove_opts.windows_per_pass) when
the first window holds no proof.

Initialises the POST of prove_multi_bench.py in a temporary directory: N = 8192, 2^22 labels (64 MiB) in four files,
then, with 16 nonces (go-spacemesh's default), K1 = 26, K2 = 37 and max_windows = all:
* a challenge whose window 0 holds no proof (the first of a seeded sequence for which generate_proof with one window
  says "no proof found"), separately for pow SKIP and for BUILTIN at the library's default (mainnet) difficulty;
* windows_per_pass 1, 2, 4 and 8: passes over the data (b200post_prove_passes_total), labels scanned, the time of the
  whole call, and for BUILTIN the time the pows of the groups that call searched take on their own
  (b200post_k2pow_search_group_range over the same groups, run right after).
The files were just written, so every pass reads them from the page cache: the time a pass saves on cold storage
(one full read of the data) is not measured here.  Prints one JSON line with the card name and power limit.
Usage: python tools/prove_windows_bench.py [--per-pass 1,2,4,8]
"""
from __future__ import annotations

import argparse
import importlib
import json
import re
import shutil
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

from tools.prove_multi_bench import power_limit_w  # noqa: E402

LABELS, NONCES, K1, K2 = 1 << 22, 16, 26, 37


def _passes(b2) -> int:
    return int(re.search(r"^b200post_prove_passes_total (\S+)$", b2.metrics_text(), re.M).group(1))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--per-pass", default="1,2,4,8")
    a = ap.parse_args()
    b2 = importlib.import_module("go-spacemesh_b200")
    su = importlib.import_module("go-spacemesh_b200.setup")
    pr = importlib.import_module("go-spacemesh_b200.prove")
    k2 = importlib.import_module("go-spacemesh_b200.k2pow")
    provs = b2.providers()
    if not provs:
        raise SystemExit("no CUDA device")
    node, atx = bytes(range(1, 33)), bytes(range(33, 65))
    cfg = su.PostConfig(labels_per_unit=LABELS, max_num_units=1, k1=K1, k2=K2, k3=K2)
    d = Path(tempfile.mkdtemp(prefix="prove_windows_bench_"))
    try:
        mgr = su.PostSetupManager(cfg)
        mgr.prepare_initializer(su.PostSetupOpts(data_dir=str(d), num_units=1, max_file_size=16 * (LABELS // 4), provider_id=0,
                                                 scrypt_n=8192), node, atx)
        mgr.start_session()
        scaled = k2.scale_difficulty(bytes(pr._c_cfg(cfg).pow_difficulty), 1)
        k2.prepare()                                  # dataset build (once per key and device) outside the timings
        out = {"card": provs[0]["model"], "power_limit_w": power_limit_w(), "scrypt_n": 8192, "labels": LABELS, "nonces": NONCES,
               "k1": K1, "k2": K2, "scan_source": "page cache", "pow_difficulty_scaled": scaled.hex()}
        for pow_ in ("skip", "builtin"):
            rng = np.random.default_rng(17)
            for _ in range(32):                       # P(window 0 has no proof) = 0.674 at these K1, K2, nonces
                challenge = rng.bytes(32)
                try:
                    pr.generate_proof(str(d), challenge, cfg, nonces=NONCES, pow=pow_)
                except b2.B200PostError as e:
                    if "no proof found" in str(e):
                        break
                    raise
            else:
                raise SystemExit("no challenge without a proof in window 0")
            runs, proofs = {}, []
            for m in (int(x) for x in a.per_pass.split(",")):
                before = _passes(b2)
                t0 = time.perf_counter()
                proof, _, scanned = pr.generate_proof(str(d), challenge, cfg, nonces=NONCES, pow=pow_, max_windows="all",
                                                      windows_per_pass=m)
                total = time.perf_counter() - t0
                passes = _passes(b2) - before
                groups = passes * m * NONCES // 16
                run = {"passes": passes, "labels_scanned": scanned, "groups_searched": groups, "total_s": round(total, 3),
                       "window": proof.nonce // NONCES}
                if pow_ == "builtin":
                    t0 = time.perf_counter()
                    k2.search_group_range(challenge[:8], node, scaled, 0, groups)
                    run["pow_s"] = round(time.perf_counter() - t0, 3)
                runs[f"per_pass_{m}"] = run
                proofs.append(proof)
            if any(p != proofs[0] for p in proofs):
                raise SystemExit("windows_per_pass changed the proof")
            out[pow_] = {"challenge": challenge.hex(), **runs}
        print(json.dumps(out))
    finally:
        shutil.rmtree(d, ignore_errors=True)


if __name__ == "__main__":
    main()
