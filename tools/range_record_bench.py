"""What range records cost a range session, and what the merge saves.

On one device, N = 8192, 2^22 labels (64 MiB) in four files, initialised as two ranges (files 0-1, 2-3), 288 nonces,
K1 = 26, K2 = 37, best of --repeat, the cases alternating per range:
* (a) the range session without a record;
* (b) with a VRF-only record;
* (c) with a record and the proof scan, pow SKIP: (b) - (a) and (c) - (a), as shares of (a), are what a record costs;
* (d) b200post_merge_range_records over the merged directory (pow SKIP records), against
* (e) b200post_search_vrf_nonce + b200post_generate_proof over the same files, which the merge replaces.  The files are
  in the page cache, so (e) is a lower bound on the time of those two reads from disk; from cold storage it is larger;
* (f) once, one range with the proof and pow BUILTIN at the mainnet difficulty: (f) - (c) is the pow step each machine
  pays for its range (every machine finds all groups' pows; at 1 SU here).
Prints one JSON line with the card name and power limit read in the same run.
Usage: python tools/range_record_bench.py [--repeat 3]
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

LABELS, NONCES, K1, K2, N = 1 << 22, 288, 26, 37, 8192
RANGES = ((0, 1), (2, 3))


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
    root = Path(tempfile.mkdtemp(prefix="range_record_bench_"))

    def session(d, files, record):
        """One range session into d (emptied first); record: None, {} (VRF only) or request kwargs.  Its time."""
        shutil.rmtree(d, ignore_errors=True)
        mgr = su.PostSetupManager(cfg)
        mgr.prepare_files(su.PostSetupOpts(data_dir=str(d), num_units=1, max_file_size=16 * per_file, provider_id=0, scrypt_n=N),
                          node, atx, *files)
        if record is not None:
            mgr.request_range_record(**record)
        t0 = time.perf_counter()
        mgr.start_session()
        return time.perf_counter() - t0

    def gather(dst, parts):
        shutil.rmtree(dst, ignore_errors=True)
        dst.mkdir()
        for p in parts:
            for f in list(p.glob("postdata_*.bin")) + list(p.glob("range_*.rec")):
                shutil.copy(f, dst / f.name)
        shutil.copy(parts[0] / "postdata_metadata.json", dst / "postdata_metadata.json")
        return dst

    cases = {"a": None, "b": {}, "c": {"initial_proof": True, "nonces": NONCES, "pow": "skip"}}
    try:
        best = {f"{c}{i}": float("inf") for c in cases for i in range(len(RANGES))}
        best.update(d=float("inf"), e=float("inf"))
        for _ in range(a.repeat):
            for i, files in enumerate(RANGES):
                for c, rec in cases.items():
                    best[f"{c}{i}"] = min(best[f"{c}{i}"], session(root / f"{c}{i}", files, rec))
            merged = gather(root / "m", [root / "c0", root / "c1"])
            t0 = time.perf_counter()
            r = su.merge_range_records(str(merged), cfg)
            best["d"] = min(best["d"], time.perf_counter() - t0)
            if r.proof_rc != 0:
                raise SystemExit(f"the merge gave no proof: {r.proof_reason}")
            plain = gather(root / "p", [root / "a0", root / "a1"])
            t0 = time.perf_counter()
            nonce, _ = su.search_vrf_nonce(str(plain))
            proof_e = pr.generate_proof(str(plain), bytes(32), cfg, nonces=NONCES, pow="skip")[0]
            best["e"] = min(best["e"], time.perf_counter() - t0)
            if (nonce, proof_e.nonce, proof_e.indices) != (r.nonce, r.proof.nonce, r.proof.indices):
                raise SystemExit("the merge differs from search_vrf_nonce + generate_proof")
        el_f = session(root / "f", RANGES[0], {"initial_proof": True, "nonces": NONCES, "pow": "builtin"})
        sa, sb, sc = (sum(best[f"{c}{i}"] for i in range(len(RANGES))) for c in "abc")
        out = {"card": provs[0]["model"], "power_limit_w": power_limit_w(), "scrypt_n": N, "labels": LABELS, "files": 4,
               "ranges": len(RANGES), "nonces": NONCES, "k1": K1, "k2": K2, "repeat": a.repeat,
               "a_ranges_no_record_s": round(sa, 3), "b_ranges_vrf_record_s": round(sb, 3), "c_ranges_record_proof_s": round(sc, 3),
               "b_minus_a_share": round((sb - sa) / sa, 4), "c_minus_a_share": round((sc - sa) / sa, 4),
               "per_range_s": {k: round(v, 3) for k, v in best.items() if k[0] in "abc"},
               "d_merge_s": round(best["d"], 4), "e_search_plus_prove_page_cache_s": round(best["e"], 4),
               "f_builtin_range_session_s": round(el_f, 3), "f_pow_step_s_approx": round(el_f - best["c0"], 3),
               "nonce": r.nonce, "proof_nonce": r.proof.nonce}
        print(json.dumps(out))
    finally:
        shutil.rmtree(root, ignore_errors=True)


if __name__ == "__main__":
    main()
