"""Search for the label-function conventions that make the real VRF nonces of the reference's checkpoint fixture
(checkpoint/checkpointdata.json: 42 identities of a LabelsPerUnit=1024 network) valid.  A VRF nonce is the index
of a label whose 32-byte scrypt output is below 2^256/numLabels, so the right function shows >= 15 leading zero
bits for every identity; a wrong one shows ~1.  Reads the fixture from the go-spacemesh checkout at $GO_SPACEMESH_DIR."""
import base64, hashlib, hmac, json, struct, sys
import numpy as np
import blake3

M32 = np.uint32(0xffffffff)

def rotl(x, k):
    return ((x << np.uint32(k)) | (x >> np.uint32(32 - k)))

def salsa8(B):       # B: (n,16) uint32
    x = [B[:, i].copy() for i in range(16)]
    def qr(a, b, c, d):
        x[b] ^= rotl(x[a] + x[d], 7); x[c] ^= rotl(x[b] + x[a], 9); x[d] ^= rotl(x[c] + x[b], 13); x[a] ^= rotl(x[d] + x[c], 18)
    for _ in range(4):
        qr(0, 4, 8, 12); qr(5, 9, 13, 1); qr(10, 14, 2, 6); qr(15, 3, 7, 11)
        qr(0, 1, 2, 3); qr(5, 6, 7, 4); qr(10, 11, 8, 9); qr(15, 12, 13, 14)
    return B + np.stack(x, axis=1)

def chacha8(B):
    x = [B[:, i].copy() for i in range(16)]
    def qr(a, b, c, d):
        x[a] += x[b]; x[d] = rotl(x[d] ^ x[a], 16)
        x[c] += x[d]; x[b] = rotl(x[b] ^ x[c], 12)
        x[a] += x[b]; x[d] = rotl(x[d] ^ x[a], 8)
        x[c] += x[d]; x[b] = rotl(x[b] ^ x[c], 7)
    for _ in range(4):
        qr(0, 4, 8, 12); qr(1, 5, 9, 13); qr(2, 6, 10, 14); qr(3, 7, 11, 15)
        qr(0, 5, 10, 15); qr(1, 6, 11, 12); qr(2, 7, 8, 13); qr(3, 4, 9, 14)
    return B + np.stack(x, axis=1)

def blockmix(B, core):       # r = 1: B (n,32)
    X = B[:, 16:] ^ B[:, :16]
    Y0 = core(X)
    Y1 = core(Y0 ^ B[:, 16:])
    return np.concatenate([Y0, Y1], axis=1)

def romix(B, N, core):
    n = B.shape[0]
    V = np.empty((N, n, 32), dtype=np.uint32)
    X = B
    for i in range(N):
        V[i] = X
        X = blockmix(X, core)
    rows = np.arange(n)
    for i in range(N):
        j = X[:, 16] & np.uint32(N - 1)
        X = blockmix(X ^ V[j, rows], core)
    return X

# ---- Keccak-512 with the original 0x01 padding (scrypt-jane's SCRYPT_KECCAK512)
RC = [0x0000000000000001, 0x0000000000008082, 0x800000000000808A, 0x8000000080008000, 0x000000000000808B, 0x0000000080000001,
      0x8000000080008081, 0x8000000000008009, 0x000000000000008A, 0x0000000000000088, 0x0000000080008009, 0x000000008000000A,
      0x000000008000808B, 0x800000000000008B, 0x8000000000008089, 0x8000000000008003, 0x8000000000008002, 0x8000000000000080,
      0x000000000000800A, 0x800000008000000A, 0x8000000080008081, 0x8000000000008080, 0x0000000080000001, 0x8000000080008008]
ROT = [[0, 36, 3, 41, 18], [1, 44, 10, 45, 2], [62, 6, 43, 15, 61], [28, 55, 25, 21, 56], [27, 20, 39, 8, 14]]
M64 = (1 << 64) - 1
def keccak_f(A):
    for rc in RC:
        C = [A[x][0] ^ A[x][1] ^ A[x][2] ^ A[x][3] ^ A[x][4] for x in range(5)]
        D = [C[(x - 1) % 5] ^ (((C[(x + 1) % 5] << 1) | (C[(x + 1) % 5] >> 63)) & M64) for x in range(5)]
        A = [[A[x][y] ^ D[x] for y in range(5)] for x in range(5)]
        Bm = [[0] * 5 for _ in range(5)]
        for x in range(5):
            for y in range(5):
                r = ROT[x][y]; v = A[x][y]
                Bm[y][(2 * x + 3 * y) % 5] = ((v << r) | (v >> (64 - r))) & M64 if r else v
        A = [[Bm[x][y] ^ ((~Bm[(x + 1) % 5][y]) & Bm[(x + 2) % 5][y]) for y in range(5)] for x in range(5)]
        A[0][0] ^= rc
    return A
def keccak512(data, pad=0x01):
    rate = 72
    m = bytearray(data); m.append(pad); m.extend(b"\0" * ((-len(m)) % rate)); m[-1] |= 0x80
    A = [[0] * 5 for _ in range(5)]
    for off in range(0, len(m), rate):
        for i in range(rate // 8):
            A[i % 5][i // 5] ^= int.from_bytes(m[off + 8 * i: off + 8 * i + 8], "little")
        A = keccak_f(A)
    out = b"".join(A[i % 5][i // 5].to_bytes(8, "little") for i in range(8))
    return out
assert keccak512(b"", 0x06) == hashlib.sha3_512(b"").digest()

HASHES = {"sha256": (lambda d: hashlib.sha256(d).digest(), 64), "keccak512": (keccak512, 72),
          "sha512": (lambda d: hashlib.sha512(d).digest(), 128)}
def hmac_(hname, key, msg):
    h, bs = HASHES[hname]
    if len(key) > bs: key = h(key)
    key = key.ljust(bs, b"\0")
    return h(bytes(k ^ 0x5c for k in key) + h(bytes(k ^ 0x36 for k in key) + msg))
def pbkdf2_1(hname, pw, salt, dklen):
    out = b""; i = 1
    while len(out) < dklen:
        out += hmac_(hname, pw, salt + struct.pack(">I", i)); i += 1
    return out[:dklen]
assert pbkdf2_1("sha256", b"pw", b"salt", 40) == hashlib.pbkdf2_hmac("sha256", b"pw", b"salt", 1, 40)

def scrypt_batch(pws, salts, N, core, hname, dklen=32):
    B = np.stack([np.frombuffer(pbkdf2_1(hname, p, s, 128), dtype="<u4") for p, s in zip(pws, salts)]).astype(np.uint32)
    X = romix(B, N, core)
    return [pbkdf2_1(hname, p, X[i].astype("<u4").tobytes(), dklen) for i, p in enumerate(pws)]

def lz(b):
    return len(b) * 8 - int.from_bytes(b, "big").bit_length()

if __name__ == "__main__":
    np.seterr(over="ignore")
    assert scrypt_batch([b"pw"], [b"salt"], 16, salsa8, "sha256") == [hashlib.scrypt(b"pw", salt=b"salt", n=16, r=1, p=1, dklen=32)]
    import os
    d = json.load(open(os.path.join(os.environ["GO_SPACEMESH_DIR"], "checkpoint", "checkpointdata.json")))
    ids = {}
    for a in d["data"]["atxs"]:
        ids[(a["publicKey"], a["commitmentAtx"], a["vrfNonce"], a["numUnits"])] = a
    ids = list(ids)[: int(sys.argv[2]) if len(sys.argv) > 2 else 8]
    N = int(sys.argv[1]) if len(sys.argv) > 1 else 8192
    LAYOUTS = {"c;i": lambda c, i, z: (c, i), "c|i|z;": lambda c, i, z: (c + i + z, b""), "c|i;": lambda c, i, z: (c + i, b""),
               "c|i;z": lambda c, i, z: (c + i, z), "c;i|z": lambda c, i, z: (c, i + z), "c;z|i": lambda c, i, z: (c, z + i),
               "c|z|i;": lambda c, i, z: (c + z + i, b""), "c|i|z;z": lambda c, i, z: (c + i + z, z), "c;z": None}
    del LAYOUTS["c;z"]
    for cname, cf in (("b3(node|catx)", lambda n, c: blake3.blake3(n + c).digest()), ("b3(catx|node)", lambda n, c: blake3.blake3(c + n).digest())):
        for lname, lf in LAYOUTS.items():
            pairs = [lf(cf(base64.b64decode(pk), base64.b64decode(ca)), struct.pack("<Q", nonce), bytes(32)) for (pk, ca, nonce, _) in ids]
            pws = [p for p, _ in pairs]; salts = [s for _, s in pairs]
            for core_name, core in (("chacha8", chacha8), ("salsa8", salsa8)):
                for hname in ("keccak512", "sha256"):
                    if core_name == "salsa8" and hname == "sha256":
                        continue     # covered by the hashlib scan
                    outs = scrypt_batch(pws, salts, N, core, hname)
                    for interp, f in (("be", lambda o: lz(o)), ("le", lambda o: lz(o[::-1])), ("be16", lambda o: lz(o[:16])), ("le16", lambda o: lz(o[:16][::-1]))):
                        v = [f(o) for o in outs]
                        print(N, cname, lname, core_name, hname, interp, v, "MATCH" if min(v) >= 8 else "", flush=True)
