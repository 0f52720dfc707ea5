"""Windowed proving restated for the tests, on the oracle's primitives (py_cipher_key, AES-128-ECB over every label at
once): window w of n nonces is the nonces [w*n, (w+1)*n), groups w*n/16 ..; the proof comes from the lowest window in
which some nonce reaches K2 hits, under the prover's selection rule inside it (include/b200post_prove.h)."""
import numpy as np


def window_hits(orc, labels, challenge: bytes, first: int, nonces: int, pows, k1: int, k2: int, num_labels: int) -> dict:
    """{absolute nonce: its first (up to) k2 positions in `labels`} for the nonces [first, first + nonces); pows[g] is the
    pow of group first // 16 + g.  orc.np_prove_hits for any first nonce."""
    labels = np.ascontiguousarray(labels, dtype=np.uint8).reshape(-1, 16)
    diff = orc.py_proving_difficulty(k1, num_labels)
    msb, lsb = diff >> 56, diff & ((1 << 56) - 1)
    out = {}
    for g in range(nonces // 16):
        group = first // 16 + g
        ct = orc._np_aes128_ecb(orc.py_cipher_key(challenge, group, int(pows[g])), labels)
        rows, cols = np.nonzero(ct <= msb)
        keep = ct[rows, cols] != msb
        for b in np.unique(cols[~keep]):
            sel = np.flatnonzero((cols == b) & ~keep)
            lz = orc._np_aes128_ecb(orc.py_cipher_key(challenge, group, int(pows[g]), 16 * group + int(b)), labels[rows[sel]])
            low56 = lz[:, :8].copy().view("<u8")[:, 0] & np.uint64((1 << 56) - 1)
            keep[sel[low56 < np.uint64(lsb)]] = True
        rows, cols = rows[keep], cols[keep]
        for b in range(16):
            out[16 * group + b] = rows[cols == b][:k2]
    return out


def pick(hits: dict, k2: int, usable=None):
    """The selection rule over {nonce: positions}: (nonce, [indices]) or None.  usable: a bool mask of usable positions."""
    best = None
    for n in sorted(hits):
        h = [int(i) for i in hits[n] if usable is None or usable[i]][:k2]
        if len(h) == k2 and (best is None or h[-1] < best[1][-1]):
            best = (n, h)
    return best


def windowed_proof(orc, labels, challenge: bytes, nonces: int, pow_of_group, k1: int, k2: int, num_labels: int,
                   max_windows: int, usable=None, k2_hits: int | None = None):
    """Sequential windows 0 .. max_windows - 1: (window, nonce, indices) of the first that has a proof, or None.
    pow_of_group(g) -> the pow of group g.  With `usable`, hits are looked for among more positions (k2_hits) so that
    K2 usable ones can be found past damaged ones."""
    for w in range(max_windows):
        pows = [pow_of_group(w * nonces // 16 + g) for g in range(nonces // 16)]
        hits = window_hits(orc, labels, challenge, w * nonces, nonces, pows, k1, k2_hits or k2, num_labels)
        best = pick(hits, k2, usable)
        if best:
            return (w, *best)
    return None


def pass_model(hits_by_nonce: dict, n_labels: int, chunk: int, first_window: int, nonces: int, windows: int, k2: int):
    """One pass of the prover over windows [first_window, first_window + windows) on one device, chunk by chunk: it stops
    once a nonce of the pass's lowest window has K2 hits or every nonce of the pass has, and the lowest window with a
    winner gives the proof.  hits_by_nonce: every hit position of every nonce.  -> (proof or None, labels scanned)."""
    lo, hi = first_window * nonces, (first_window + windows) * nonces
    scanned = 0
    while scanned < n_labels:
        scanned = min(n_labels, scanned + chunk)
        seen = {n: [i for i in hits_by_nonce[n] if i < scanned][:k2] for n in range(lo, hi)}
        if any(len(seen[n]) == k2 for n in range(lo, lo + nonces)) or all(len(v) == k2 for v in seen.values()):
            break
    seen = {n: [i for i in hits_by_nonce[n] if i < scanned][:k2] for n in range(lo, hi)}
    for w in range(windows):
        best = pick({n: seen[n] for n in range((first_window + w) * nonces, (first_window + w + 1) * nonces)}, k2)
        if best:
            return best, scanned
    return None, scanned
