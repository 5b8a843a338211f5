"""The RFC 6979 signer (ibft_sign_batch_rfc6979, verify_core.cuh ecdsa_sign_rfc6979): its big-integer reference and its rows,
shared by the emulation test (test_emul_sign_rfc6979.py) and the GPU test (test_gpu_sign_rfc6979.py).

`rfc6979_candidate` and `sign_libsecp` restate libsecp256k1's default signer over oracle/secp256k1.py's point arithmetic.
`want(ds, zs)` is sign_libsecp for every row (65 zero bytes where it returns None), with the C oracle's k G standing in for the
big-integer point_mul so that 10^5 rows take seconds."""
from __future__ import annotations

import hashlib
import hmac
import json
import os
import random

import sign_edges as S
from oracle import coracle as co
from oracle import secp256k1 as ec

N = ec.N
M = 1 << 256
ZERO_SIG = bytes(65)
EDGE_KEYS = S.KEYS                                  # 1, 2, n-2, n-1, lambda, n-lambda, (n-1)/2, (n+1)/2, 2^128
EDGE_DIGESTS = S.DIGESTS                            # 0, 1, n-1, n, n+1, p, 2^255, 2^256-1
REFUSED_KEYS = [0, N, N + 1, M - 1]


def rfc6979_candidate(d: int, digest: bytes, c: int) -> int:
    """Nonce candidate c (c = 0, 1, ...) of libsecp256k1's nonce_function_rfc6979 with attempt counter c: the (c+1)-th output
    of the RFC 6979 §3.2 DRBG seeded with the raw 32-byte key and the digest reduced mod n, before any range check."""
    x = d.to_bytes(32, "big")
    h1 = (int.from_bytes(digest, "big") % N).to_bytes(32, "big")
    V = b"\x01" * 32
    K = b"\x00" * 32
    K = hmac.new(K, V + b"\x00" + x + h1, hashlib.sha256).digest()
    V = hmac.new(K, V, hashlib.sha256).digest()
    K = hmac.new(K, V + b"\x01" + x + h1, hashlib.sha256).digest()
    V = hmac.new(K, V, hashlib.sha256).digest()
    for i in range(c + 1):
        if i:
            K = hmac.new(K, V + b"\x00", hashlib.sha256).digest()
            V = hmac.new(K, V, hashlib.sha256).digest()
        V = hmac.new(K, V, hashlib.sha256).digest()
    return int.from_bytes(V, "big")


def sign_libsecp(d: int, digest: bytes, max_candidates: int = 4, base_mul=None) -> bytes | None:
    """R||S||V as libsecp256k1's secp256k1_ecdsa_sign_recoverable (go-ethereum's crypto.Sign) signs with its default nonce, or
    None where ibft_sign_batch_rfc6979 returns 65 zero bytes: a key outside [1, n), R.x >= n (libsecp256k1's recovery id 2 or
    3), or no signature from the first `max_candidates` candidates (a candidate outside [1, n) or one that gives s = 0 moves on
    to the next).  base_mul(k) -> (x, y) of k G for k in [1, n); default the big-integer point_mul."""
    if not 1 <= d < N:
        return None
    z = int.from_bytes(digest, "big") % N
    for c in range(max_candidates):
        k = rfc6979_candidate(d, digest, c)
        if not 1 <= k < N:
            continue
        R = base_mul(k) if base_mul is not None else ec.point_mul(k, ec.G)
        if R[0] >= N:
            return None
        r = R[0]
        s = pow(k, -1, N) * (z + r * d) % N
        if s == 0:
            continue
        v = R[1] & 1
        if s > N // 2:
            s, v = N - s, v ^ 1
        return r.to_bytes(32, "big") + s.to_bytes(32, "big") + bytes([v])
    return None


def c_base_mul(k: int):
    xy = co.pubkey_from_scalar(k)
    return int.from_bytes(xy[:32], "big"), int.from_bytes(xy[32:], "big")


def want_one(d: int, z: bytes) -> bytes:
    return sign_libsecp(d, z, base_mul=c_base_mul) or ZERO_SIG


def want(ds, zs) -> list[bytes]:
    return [want_one(d, z) for d, z in zip(ds, zs)]


def edge_rows():
    """every edge key with every edge digest, then the refused keys with a few digests"""
    rows = [(d, z.to_bytes(32, "big")) for d in EDGE_KEYS for z in EDGE_DIGESTS]
    rows += [(d, z.to_bytes(32, "big")) for d in REFUSED_KEYS for z in (0, 1, N + 1, M - 1)]
    return rows


def random_rows(n: int, seed: int):
    """n rows of random keys in [1, n) and random 32-byte digests; every 97th row takes a key or digest from the edge families
    (keys 0, n and above n, digests n, n + 1 and 2^256 - 1) so that a large batch mixes refusals and reductions in"""
    rnd = random.Random(seed)
    ds = [rnd.randrange(1, N) for _ in range(n)]
    zs = [rnd.randbytes(32) for _ in range(n)]
    special_keys = [0, N, N + 1, N + rnd.randrange(1, M - N), M - 1]
    special_digests = [N, N + 1, N + rnd.randrange(1, M - N), M - 1]
    for j, i in enumerate(range(3, n, 97)):
        if j % 2 == 0:
            ds[i] = special_keys[(j // 2) % len(special_keys)]
        else:
            zs[i] = special_digests[(j // 2) % len(special_digests)].to_bytes(32, "big")
    return ds, zs


def golden_vectors():
    """the five published secp256k1 RFC 6979 vectors of tests/golden/third_party_recover.json"""
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "third_party_recover.json")) as f:
        return json.load(f)["sign_rfc6979"]
