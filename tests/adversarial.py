"""Crafted signatures that drive the group law into its exceptional cases (P + P, P - P, a running sum at infinity) and the
Booth digits onto their window edges -- shared by the emulation tests (test_emul.py) and the GPU tests
(test_gpu_adversarial.py).  Random signatures reach these cases with probability ~2^-128; an attacker needs one line.

Expected keys and addresses come from the big-int oracle (oracle/secp256k1.py); test_emul.py cross-checks them once against
the C oracle.

Recover vectors: pick the point R and the scalars u1, u2, then r = R.x, s = u2 r, z = -u1 r (mod n), v = parity(R.y).  Recovery
computes u1 G + u2 R with exactly these scalars (u1 = -z/r, u2 = s/r), so the vector decides which points meet in the adders.
Known-key vectors: pick the key Q and u1 = z/s, u2 = r/s of the verification u1 G + u2 Q = R, then solve for (r, s, z)."""
from __future__ import annotations

import functools
import random
from dataclasses import dataclass

import numpy as np

from arith_edges import fold4_signature_targets
from oracle import secp256k1 as ec

N = ec.N
LAM = 0x5363AD4CC05C30E0A5261C028812645A122E22EA20816678DF02967C1B23BD72
ALL80 = int.from_bytes(b"\x80" * 16, "big")


@dataclass(frozen=True)
class Vector:
    tag: str
    sig: bytes        # 65 bytes R || S || V
    digest: bytes     # 32 bytes, used as z (IBFT_KIND_DIGEST)
    key: tuple | None  # the key recovery yields (affine), None = invalid signature or the point at infinity
    u: tuple = (0, 0)  # (u1, u2) the vector was built for

    @property
    def addr(self) -> bytes | None:
        return None if self.key is None else ec.pubkey_to_address(self.key)


def mul(k, pt=ec.G):
    return ec.point_mul(k, pt)


def recover_vector(tag: str, R, u1: int, u2: int, z_override: bytes | None = None) -> Vector:
    """signature (r, s, z, v) whose recovery computes u1 G + u2 R"""
    r = R[0]
    s = u2 * r % N
    z = (-u1 * r) % N
    digest = z_override if z_override is not None else z.to_bytes(32, "big")
    sig = r.to_bytes(32, "big") + s.to_bytes(32, "big") + bytes([R[1] & 1])
    key = ec.recover_pubkey(int.from_bytes(digest, "big"), r, s, sig[64])
    return Vector(tag, sig, digest, key, (u1 % N, u2 % N))


def high_s_twin(v: Vector) -> Vector:
    """(r, n - s, v ^ 1): the same key (s R = (-s)(-R))"""
    s = int.from_bytes(v.sig[32:64], "big")
    sig = v.sig[:32] + ((N - s) % N).to_bytes(32, "big") + bytes([v.sig[64] ^ 1])
    key = ec.recover_pubkey(int.from_bytes(v.digest, "big"), int.from_bytes(sig[:32], "big"), (N - s) % N, sig[64])
    return Vector(v.tag + "/high-s", sig, v.digest, key, v.u)


# (u1, u2) pairs of test_ecmult: partial sums of the windowed walk collide with table entries when R is a small multiple of G
ECMULT_PAIRS = [(0, 0), (1, 0), (0, 1), (2, 0), (0, 2), (N - 1, 0), (0, N - 1), (1, N - 1), (5, 7), (N - 1, N - 1), (LAM, 0), (0, LAM),
                (N - LAM, LAM), (1, 1), (2, N - 1), (N - 2, 1), (8, 1), (8, N - 1), (3, 5), (LAM, 1), (1, LAM), (7, 1), (16, N - 2)]
WALK_POINTS = [1, N - 1, LAM, N - LAM, 2, N - 2, 8, N - 8]        # R = c G: G, -G, lambda G, -lambda G, 2G, -2G, 8G, -8G
# GLV half-scalars whose 4-bit and 8-bit Booth digits sit on the window edges
HALVES = [0, 1, -1, 7, -7, 8, -8, 9, -9, 127, -127, 128, -128, 129, -129, 2**127, 2**128 - 1, ALL80, -ALL80]
FINAL_ADD_POINTS = [1, 2, 3, N - 1, LAM, 0xC0FFEE]                  # R = c G with u1 = +-c u2: the split pipelines' final add
FINAL_ADD_U2 = [1, 5, 0x1234567890ABCDEF1234567890ABCDEF, N - 3]


@functools.lru_cache(maxsize=None)
def recover_vectors() -> tuple[Vector, ...]:
    out = []
    for c in WALK_POINTS:
        R = mul(c)
        if R[0] >= N:
            continue
        for u1, u2 in ECMULT_PAIRS:
            out.append(recover_vector(f"walk c={c:#x} u=({u1:#x},{u2:#x})", R, u1, u2))
    L = len(HALVES)
    for base in (12345, 1):
        R = mul(base)
        for j in range(L):
            k1, k2, g1, g2 = HALVES[j], HALVES[(3 * j + 1) % L], HALVES[(5 * j + 2) % L], HALVES[(7 * j + 3) % L]
            out.append(recover_vector(f"booth R={base} j={j}", R, g1 + g2 * LAM, k1 + k2 * LAM))
            h = HALVES[j]
            out.append(recover_vector(f"booth-diag R={base} h={h:#x}", R, h - h * LAM, h + h * LAM))
    for c in FINAL_ADD_POINTS:
        R = mul(c)
        if R[0] >= N:
            continue
        for u2 in FINAL_ADD_U2:
            out.append(recover_vector(f"final-add dbl c={c:#x} u2={u2:#x}", R, c * u2, u2))   # u2 R + u1 G = P + P
            out.append(recover_vector(f"final-add inf c={c:#x} u2={u2:#x}", R, -c * u2, u2))  # P - P: Q = infinity, verdict 0
    R = mul(12345)
    for u2 in (1, 7, LAM, 0xDEADBEEF):
        out.append(recover_vector(f"u1=0 z=0 u2={u2:#x}", R, 0, u2))
        out.append(recover_vector(f"u1=0 z=n u2={u2:#x}", R, 0, u2, z_override=N.to_bytes(32, "big")))  # digest >= n, reduces to 0
    # the mod-n products s r^-1 (u2) and z r^-1 (u1) carry into sc_reduce512's fold 4 (tests/arith_edges.py)
    # (the 512-bit product must exceed about 0.62 * 2^512, so r^-1 has to be large: R = c G for the first such c)
    rnd = random.Random(0xF014)
    fold4 = [c for c in range(2, 200) if pow(mul(c)[0], -1, N) > 7 * N // 8][:5]
    for c in fold4:
        R = mul(c)
        t_u2, t_u1 = fold4_signature_targets(rnd, R[0], 2)
        out.append(recover_vector(f"fold4 u2 c={c:#x}", R, rnd.randrange(1, N), t_u2))
        out.append(recover_vector(f"fold4 u1 c={c:#x}", R, -t_u1, rnd.randrange(1, N)))
    twins = [high_s_twin(v) for v in out if 0 < int.from_bytes(v.sig[32:64], "big") < N]
    return tuple(out + twins)


# ------------------------------------------------------------------------------------------------------ known keys
KNOWN_KEYS = [1, N - 1, LAM, N - LAM, 2, 0xC0FFEE]   # Q = G, -G, lambda G, -lambda G, 2G: the key stream meets the generator's
KNOWN_HALVES = [0, 1, -1, 127, 128, -128, 129, 255, 256, 0x8000, ALL80, -ALL80, 2**127, 2**128 - 1, -(2**127) - 5, 0x7F80 << 64]


@dataclass(frozen=True)
class KnownVector:
    key_index: int    # index into KNOWN_KEYS of the signing key
    sig: bytes
    digest: bytes


def _craft_known(u1, u2, Q):
    R = ec.point_add(mul(u1) if u1 else ec.INF, mul(u2, Q))
    if R == ec.INF or R[0] >= N or R[0] == 0:
        return None
    r = R[0]
    s = r * pow(u2, -1, N) % N
    z = u1 * s % N
    if s == 0:
        return None
    return r.to_bytes(32, "big") + s.to_bytes(32, "big") + bytes([R[1] & 1]), z.to_bytes(32, "big")


@functools.lru_cache(maxsize=None)
def known_vectors() -> tuple[KnownVector, ...]:
    """Valid signatures of the KNOWN_KEYS built for constructed (u1, u2): Booth digits on the window edges, u1 = 0 (no generator
    term), and u1 = u2 (with Q = +-G / +-lambda G the two streams add the same or opposite points)."""
    out = []
    L = len(KNOWN_HALVES)
    for i, d in enumerate(KNOWN_KEYS):
        Q = mul(d)
        for j in range(L):
            k1, k2 = KNOWN_HALVES[j], KNOWN_HALVES[(j * 5 + i) % L]
            g1, g2 = KNOWN_HALVES[(j * 3 + 1) % L], KNOWN_HALVES[(j * 7 + i + 2) % L]
            u2 = (k1 + k2 * LAM) % N
            u1 = (g1 + g2 * LAM) % N
            if j % 4 == 0:
                u1 = u2
            if j % 4 == 1:
                u1 = 0
            if u2 == 0:
                continue
            c = _craft_known(u1, u2, Q)
            if c is not None:
                out.append(KnownVector(i, c[0], c[1]))
    return tuple(out)


@functools.lru_cache(maxsize=None)
def known_cancelling() -> tuple[KnownVector, ...]:
    """Signatures with z = -r d (Q = d G): the verification's u1 G and u2 Q cancel, its final add gives the point at infinity
    -- never an accept.  (Recovery yields some other key: verdict 0 for the claimed validator.)"""
    out = []
    for i, d in enumerate(KNOWN_KEYS):
        R = mul(777 + i)
        s = 0x1234567890ABCDEF1234567890ABCDEF + i
        z = (-R[0] * d) % N
        out.append(KnownVector(i, R[0].to_bytes(32, "big") + s.to_bytes(32, "big") + bytes([R[1] & 1]), z.to_bytes(32, "big")))
    return tuple(out)


def known_key(i: int):
    return mul(KNOWN_KEYS[i])


def known_addr(i: int) -> bytes:
    return ec.pubkey_to_address(known_key(i))


def misattributed(v: KnownVector) -> tuple[bytes, int]:
    """(signature, claimed validator): a valid signature of key i presented as validator i + 1"""
    return v.sig, (v.key_index + 1) % len(KNOWN_KEYS)


def flipped(v: KnownVector) -> bytes:
    """the signature with the other recovery id: recovery yields another key"""
    return v.sig[:64] + bytes([v.sig[64] ^ 1])


# ------------------------------------------------------------------------------------------------------ item arrays
def recover_items(vectors, group: int = 0) -> np.ndarray:
    """IBFT_KIND_DIGEST items claiming the recovered address (zero address when there is none)"""
    import workloads as wl
    return np.concatenate([wl.make_item(v.sig, v.addr or bytes(20), 0, v.digest, group) for v in vectors])


def expected_bits(vectors) -> np.ndarray:
    """verdict of every recover vector (0/1), membership aside"""
    return np.array([v.key is not None for v in vectors], dtype=bool)
