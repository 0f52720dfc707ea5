"""Generates tests/golden/*.json — committed golden vectors for the POST label path.

Every expected value here is produced by the numpy / hashlib / `blake3`-wheel restatement in oracle/pyoracle.py
(py_*), not by oracle/post_oracle.c nor by the CUDA kernels, so the files pin both.  That restatement is itself
pinned against REAL data: checkpoint_vrf.json below.
Inputs mirror the reference's own deterministic test inputs where it has any:
  * checkpoint/checkpointdata.json — 42 identities (publicKey, commitmentAtx, vrfNonce, numUnits) of a
    LabelsPerUnit = 1024, scrypt N = 8192 network: each vrfNonce is the arg-min label index of that identity's
    POST, so label32(nonce) must be of the order of 2^256/numLabels (>= 13 leading zero bits; a wrong label
    function gives ~1).  checkpoint_vrf.json records the identities and their label32 values;
  * activation/validation_test.go:35-36 — nodeID = 32 zero bytes, commitment ATX = 32 zero bytes,
    LabelsPerUnit = 128 (:48), default scrypt N = 8192;
  * activation/post_test.go:354-357 — Scrypt.N = 2, 1024 labels (BASELINE.json configs[0]).

Run:  GO_SPACEMESH_DIR=<go-spacemesh checkout> python oracle/gen_golden.py        (~2 min; the fixture is read from there)
"""
import hashlib
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import pyoracle as o  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def sha(b: bytes) -> str:
    return hashlib.sha256(b).hexdigest()


def main():
    os.makedirs(OUT, exist_ok=True)
    rng = np.random.default_rng(1)   # SURVEY.md §8d cfg1: nodeID, atx from default_rng(1)
    node_id = bytes(rng.integers(0, 256, 32, dtype=np.uint8))
    atx = bytes(rng.integers(0, 256, 32, dtype=np.uint8))
    zero = bytes(32)

    # ---- RFC 7914 §12 scrypt vectors + §11 PBKDF2 vectors (public KATs)
    kats = {
        "scrypt": [
            dict(P="", S="", N=16, r=1, p=1, dkLen=64,
                 out="77d6576238657b203b19ca42c18a0497f16b4844e3074ae8dfdffa3fede21442fcd0069ded0948f8326a753a0fc81f17e8d3e0fb2e0d3628cf35e20c38d18906"),
            dict(P="password", S="NaCl", N=1024, r=8, p=16, dkLen=64,
                 out="fdbabe1c9d3472007856e7190d01e9fe7c6ad7cbc8237830e77376634b3731622eaf30d92e22a3886ff109279d9830dac727afb94a83ee6d8360cbdfa2cc0640"),
            dict(P="pleaseletmein", S="SodiumChloride", N=16384, r=8, p=1, dkLen=64,
                 out="7023bdcb3afd7348461c06cd81fd38ebfda8fbba904f8e3ea9b543f6545da1f2d5432955613f0fcf62d49705242a9af9e61e85dc0d651e40dfcf017b45575887"),
        ],
        "pbkdf2_sha256": [
            dict(P="passwd", S="salt", c=1, dkLen=64,
                 out="55ac046e56e3089fec1691c22544b605f94185216dde0465e68b9d57c20dacbc49ca9cccf179b645991664b39d77ef317c71b845b1e30bd509112041d3a19783"),
            dict(P="Password", S="NaCl", c=80000, dkLen=64,
                 out="4ddcd8f60b98be21830cee5ef22701f9641a4418d04c0414aeff08876b34ab56a1d425a1225833549adb841b51c9b3176a272bdebba1d078478f62b397f33c8d"),
        ],
        "aes128": [dict(key="000102030405060708090a0b0c0d0e0f", pt="00112233445566778899aabbccddeeff",
                        ct="69c4e0d86a7b0430d8cdb78070b4c55a")],   # FIPS-197 Appendix C.1
    }
    # check the KAT table itself against OpenSSL before committing it
    for v in kats["scrypt"]:
        assert hashlib.scrypt(v["P"].encode(), salt=v["S"].encode(), n=v["N"], r=v["r"], p=v["p"], dklen=v["dkLen"],
                              maxmem=1 << 30).hex() == v["out"]
    for v in kats["pbkdf2_sha256"]:
        assert hashlib.pbkdf2_hmac("sha256", v["P"].encode(), v["S"].encode(), v["c"], v["dkLen"]).hex() == v["out"]
    json.dump(kats, open(os.path.join(OUT, "kat_primitives.json"), "w"), indent=1)

    # ---- real identities from the reference's checkpoint fixture: the pin of the label function
    import base64
    ref = os.path.join(os.environ.get("GO_SPACEMESH_DIR", ""), "checkpoint", "checkpointdata.json")
    if os.path.exists(ref):
        seen = {}
        for a in json.load(open(ref))["data"]["atxs"]:
            seen[(a["publicKey"], a["commitmentAtx"], a["vrfNonce"], a["numUnits"])] = 1
        ids = list(seen)
        comms = [o.py_commitment(base64.b64decode(pk), base64.b64decode(ca)) for pk, ca, _, _ in ids]
        l32 = o.py_label32_batch(comms, [nonce for _, _, nonce, _ in ids], 8192)
        rows = []
        for (pk, ca, nonce, units), c, lab in zip(ids, comms, l32):
            num_labels = units * 1024
            ratio = int.from_bytes(lab, "big") * num_labels / 2**256      # ~Exp(1) for an arg-min
            assert ratio < 8, "label function does not reproduce the fixture's VRF nonces"
            # the whole POST of the identity, every label, with the C oracle (1.9 M labels over the 42 identities, ~4 min):
            # the recorded nonce must be the index of the smallest label32
            _, found, idx, best = o.c_labels_range(c, 8192, 0, num_labels, b"\xff" * 32, threads=os.cpu_count())
            assert found and idx == nonce and best == lab, "VRF nonce is not the arg-min of the POST"
            rows.append(dict(node_id=base64.b64decode(pk).hex(), commitment_atx=base64.b64decode(ca).hex(), commitment=c.hex(),
                             vrf_nonce=nonce, num_units=units, labels_per_unit=1024, N=8192, label32=lab.hex(),
                             label32_times_num_labels_over_2p256=round(ratio, 4), vrf_nonce_is_argmin_of_whole_post=True))
        json.dump(dict(note="identities from the reference's checkpoint/checkpointdata.json (snapshot-1152); label32 by "
                            "oracle/pyoracle.py py_label32_batch; vrf_nonce_is_argmin_of_whole_post = the C oracle recomputed "
                            "every label of the identity's POST (num_units x 1024) and the recorded nonce is the index of the "
                            "smallest label32",
                       items=rows), open(os.path.join(OUT, "checkpoint_vrf.json"), "w"), indent=1)
        print("checkpoint_vrf.json:", len(rows), "identities,", sum(r["label32_times_num_labels_over_2p256"] < 1 for r in rows),
              "below 2^256/numLabels")

    # ---- label vectors
    cases = []

    def add(name, nid, atx_, n, start, count, num_labels_for_vrf=None, full=True):
        c = o.py_commitment(nid, atx_)
        labels = o.py_labels_range(c, n, start, count)
        case = dict(name=name, node_id=nid.hex(), commitment_atx=atx_.hex(), commitment=c.hex(), N=n, start=start,
                    count=count, labels_sha256=sha(labels))
        if full:
            case["labels_hex"] = labels.hex()
        if num_labels_for_vrf:
            d = o.py_vrf_difficulty(num_labels_for_vrf)
            idx, l32 = o.py_vrf_scan(c, n, start, count, d)
            case.update(vrf_num_labels=num_labels_for_vrf, vrf_difficulty=d.hex(), vrf_index=idx,
                        vrf_label32=l32.hex() if l32 else None)
        cases.append(case)

    # cfg1 (BASELINE.json configs[0]): 1024 labels, N = 2
    add("cfg1_n2_1024", node_id, atx, 2, 0, 1024, num_labels_for_vrf=1024, full=True)
    # validation_test.go inputs: zero ids, N = 8192, LabelsPerUnit = 128 -> numLabels = 128 * units
    add("zero_ids_n8192_first128", zero, zero, 8192, 0, 128, num_labels_for_vrf=128, full=True)
    add("zero_ids_n2_first4", zero, zero, 2, 0, 4, full=True)
    # 64-bit salt: a range that crosses 2^32, and the top of the index space
    add("cross_2p32_n8192", node_id, atx, 8192, 2**32 - 8, 16, full=True)
    add("cross_2p32_n2", node_id, atx, 2, 2**32 - 300, 600, num_labels_for_vrf=2**20, full=False)
    add("top_of_u64_n16", node_id, atx, 16, 2**64 - 32, 32, full=True)
    # intermediate N values
    for n in (4, 64, 1024):
        add(f"n{n}_ragged_77", node_id, atx, n, 1000003, 77, num_labels_for_vrf=64, full=True)
    json.dump(dict(note="generated by oracle/gen_golden.py with the numpy scrypt-jane restatement (oracle/pyoracle.py py_*) + blake3 wheel", cases=cases),
              open(os.path.join(OUT, "labels.json"), "w"), indent=1)

    # ---- gather vectors (verify path): distinct commitments, scattered indices in [0, 2^34)
    rng3 = np.random.default_rng(3)   # SURVEY.md §8d cfg3 seed
    items = []
    for k in range(48):
        nid = bytes(rng3.integers(0, 256, 32, dtype=np.uint8)); a = bytes(rng3.integers(0, 256, 32, dtype=np.uint8))
        idx = int(rng3.integers(0, 2**34))
        n = 8192 if k < 24 else 2
        c = o.py_commitment(nid, a)
        items.append(dict(node_id=nid.hex(), commitment_atx=a.hex(), commitment=c.hex(), index=idx, N=n))
    for n in (8192, 2):
        sel = [it for it in items if it["N"] == n]
        for it, lab in zip(sel, o.py_label32_batch([bytes.fromhex(it["commitment"]) for it in sel], [it["index"] for it in sel], n)):
            it["label32"] = lab.hex()
    json.dump(dict(items=items), open(os.path.join(OUT, "gather.json"), "w"), indent=1)

    # ---- VRF difficulty table
    json.dump({str(n): o.py_vrf_difficulty(n).hex() for n in (2, 3, 128, 1024, 2**20, 2**34, 2**37, 2**64 - 1)},
              open(os.path.join(OUT, "vrf_difficulty.json"), "w"), indent=1)
    print("golden written to", OUT)


if __name__ == "__main__":
    main()
