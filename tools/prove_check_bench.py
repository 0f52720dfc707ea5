"""What the checked proof costs over the unchecked one (b200post_generate_proof_checked against
b200post_generate_proof_multi) on one device.

Initialises the POST of prove_multi_bench.py in a temporary directory: N = 8192, 2^22 labels (64 MiB) in four files,
then, with 288 nonces, K1 = 26, K2 = 37 and pow SKIP (the scan and the decision alone):
* unchecked and checked scans alternately, best of --repeat each, with labels scanned, labels rechecked and rounds;
* one checked run after K2 forged hits of one nonce were written at the lowest indices (the recheck drops them all and
  the scan goes on to the real winner).
The files were just written, so the scan reads them from the page cache.  Prints one JSON line with the card name and
power limit read in the same run.
Usage: python tools/prove_check_bench.py [--repeat 3]
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

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

from tools.prove_multi_bench import power_limit_w  # noqa: E402

LABELS, NONCES, K1, K2 = 1 << 22, 288, 26, 37


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=3)
    a = ap.parse_args()
    b2 = importlib.import_module("go-spacemesh_b200")
    su = importlib.import_module("go-spacemesh_b200.setup")
    pr = importlib.import_module("go-spacemesh_b200.prove")
    from oracle import pyoracle as orc
    provs = b2.providers()
    if not provs:
        raise SystemExit("no CUDA device")
    node, atx, challenge = bytes(range(1, 33)), bytes(range(33, 65)), bytes(range(65, 97))
    cfg = su.PostConfig(labels_per_unit=LABELS, max_num_units=1, k1=K1, k2=K2, k3=K2)
    per_file = LABELS // 4
    d = Path(tempfile.mkdtemp(prefix="prove_check_bench_"))
    try:
        mgr = su.PostSetupManager(cfg)
        mgr.prepare_initializer(su.PostSetupOpts(data_dir=str(d), num_units=1, max_file_size=16 * per_file, provider_id=0,
                                                 scrypt_n=8192), node, atx)
        mgr.start_session()
        best = {"unchecked": float("inf"), "checked": float("inf")}
        proofs, info = {}, {}
        for _ in range(a.repeat):
            t0 = time.perf_counter()
            proofs["unchecked"], _, scanned = pr.generate_proof(str(d), challenge, cfg, nonces=NONCES, pow="skip")
            best["unchecked"] = min(best["unchecked"], time.perf_counter() - t0)
            t0 = time.perf_counter()
            proofs["checked"], _, scanned_c, rep = pr.generate_proof_checked(str(d), challenge, cfg, nonces=NONCES, pow="skip")
            best["checked"] = min(best["checked"], time.perf_counter() - t0)
            info = {"labels_scanned": scanned, "labels_scanned_checked": scanned_c, "labels_rechecked": rep.labels_rechecked,
                    "rounds": rep.rounds, "damaged": rep.damaged}
        if proofs["unchecked"] != proofs["checked"]:
            raise SystemExit("the checked proof differs from the unchecked one on clean data")
        # forged winner: K2 random blocks that pass one nonce, at labels 0 .. K2-1
        # (the pass rate is K1 / 2^22, so 2^23 blocks give each nonce of group 0 about 52 passing ones)
        blocks = np.random.default_rng(3).integers(0, 256, (1 << 23, 16), dtype=np.uint8)
        hits = orc.np_prove_hits(blocks, challenge, 16, [0], K1, len(blocks), LABELS)
        nonce = next(n for n, h in hits.items() if len(h) >= K2)
        with open(d / "postdata_0.bin", "r+b") as f:
            f.write(blocks[hits[nonce][:K2]].tobytes())
        t0 = time.perf_counter()
        forged_proof, _, scanned_f, rep_f = pr.generate_proof_checked(str(d), challenge, cfg, nonces=NONCES, pow="skip")
        t_forged = time.perf_counter() - t0
        out = {"card": provs[0]["model"], "power_limit_w": power_limit_w(), "scrypt_n": 8192, "labels": LABELS,
               "nonces": NONCES, "k1": K1, "k2": K2, "pow": "skip", "scan_source": "page cache",
               "unchecked_s": round(best["unchecked"], 4), "checked_s": round(best["checked"], 4),
               "check_cost_ms": round(1e3 * (best["checked"] - best["unchecked"]), 1), **info,
               "forged": {"nonce": nonce, "s": round(t_forged, 4), "labels_scanned": scanned_f,
                          "labels_rechecked": rep_f.labels_rechecked, "rounds": rep_f.rounds, "damaged": rep_f.damaged,
                          "proof_nonce": forged_proof.nonce, "proof_verified": rep_f.proof_verified}}
        print(json.dumps(out))
    finally:
        shutil.rmtree(d, ignore_errors=True)


if __name__ == "__main__":
    main()
