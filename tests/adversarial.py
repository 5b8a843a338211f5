"""Crafted signatures that drive the group law into its exceptional cases (P + P, P - P, a running sum at infinity) and the
Booth digits onto their window edges -- shared by the emulation tests (test_emul.py) and the GPU tests
(test_gpu_adversarial.py).  Random signatures reach these cases with probability ~2^-128; an attacker needs one line.

Expected keys and addresses come from the big-int oracle (oracle/secp256k1.py); test_emul.py cross-checks them once against
the C oracle.

Recover vectors: pick the point R and the scalars u1, u2, then r = R.x, s = u2 r, z = -u1 r (mod n), v = parity(R.y).  Recovery
computes u1 G + u2 R with exactly these scalars (u1 = -z/r, u2 = s/r), so the vector decides which points meet in the adders.
Known-key vectors: pick the key Q and u1 = z/s, u2 = r/s of the verification u1 G + u2 Q = R, then solve for (r, s, z).
Coordinate-edge vectors (below): keys and nonce points chosen by their coordinates, and x = r + n forgeries."""
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
    claim: bytes | None = None  # the signer the item names; None = the recovered address (the zero address when there is none)

    @property
    def addr(self) -> bytes | None:
        return None if self.key is None else ec.pubkey_to_address(self.key)

    @property
    def signer(self) -> bytes:
        return self.claim if self.claim is not None else (self.addr or bytes(20))

    @property
    def verdict(self) -> bool:
        return self.key is not None and self.addr == self.signer


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
    return Vector(v.tag + "/high-s", sig, v.digest, key, v.u, v.claim)


# ------------------------------------------------------------------------------------------------ coordinate edges
# Every point above is c G for a chosen c: its coordinates are effectively random.  These families put the coordinates where the
# field's weak reduction shows -- a value v < 2^256 - p has a second 256-bit form v + p, and fe_mul / fe_sqr may return either, so
# a key is only right if it is normalised before it is hashed, stored, tabled or compared -- and the nonce point's abscissa into
# (n, p), where "x == r" and "x mod n == r" part.  None of them needs a discrete log: a key is made from its coordinates, and a
# signature for it as R = a G + b Q (r = R.x, s = r / b, z = a r / b); or the nonce point is chosen and the key follows from it.
P = ec.P
WEAK = 2**256 - P                       # 0x1000003D1: below it a field element has two 256-bit forms
BETA = 0x7AE96A2B657C07106E64479EAC3434E99CF0497512F58995C1396C28719501EE  # a cube root of unity mod p: (x, y) -> (beta x, y)
SMALL_X = [1, 2, 3, 4, 6]               # the smallest abscissas (0 and 5 are none, 7 gives a non-residue)
WEAK_X = [0x1000003BE, 0x1000003BF, 0x1000003C1]  # abscissas just below 2^256 - p
NEAR_P_X = [P - 3, P - 4]
TINY_Y = [1, 6, 11]
NONCE_R = [1, 2, 3, 4, 6, 8, 0x1000003BE, N - 2, N - 3]
# (z, s) of the nonce-edge signatures; None = seeded random.  With r = 1, u2 = s and u1 = -z; z = 0 leaves the generator out.
NONCE_ZS = [(z, s) for z in (None, 0, N, 2**256 - 1) for s in (None, 1, N - 1)]


def _cube_root(a: int) -> int:
    """the cube root of a cubic residue mod p: p = 1 (mod 3) and 3 does not divide (p - 1) / 3, so 3 is invertible mod (p - 1) / 3"""
    x = pow(a, pow(3, -1, (P - 1) // 3), P)
    assert pow(x, 3, P) == a % P
    return x


def _point(x: int, y: int):
    assert ec.on_curve((x, y)), (hex(x), hex(y))
    return (x, y)


@functools.lru_cache(maxsize=None)
def tiny_y_points() -> tuple:
    """(x, y) with y in TINY_Y or p - y: the three abscissas x, beta x, beta^2 x of each"""
    out = []
    for y in TINY_Y:
        x = _cube_root(y * y - 7)
        for k in range(3):
            for yy in (y, P - y):
                out.append(_point(x * pow(BETA, k, P) % P, yy))
    return tuple(out)


@functools.lru_cache(maxsize=None)
def key_edge_points() -> tuple:
    """(tag, Q): keys whose coordinates sit at the field's edges, both parities where the abscissa is given"""
    out = []
    for fam, xs in (("small-x", SMALL_X), ("weak-x", WEAK_X), ("near-p-x", NEAR_P_X)):
        for x in xs:
            for odd in (0, 1):
                out.append((f"key-edge {fam} x={x:#x} odd={odd}", ec.lift_x(x, odd)))
    out += [(f"key-edge tiny-y x={Q[0]:#x} y={Q[1]:#x}", Q) for Q in tiny_y_points()]
    return tuple(out)


def signature_for(tag: str, Q, rnd: random.Random) -> Vector:
    """a valid signature of Q without its private key: R = a G + b Q, r = R.x, s = r / b, z = a r / b (u1 = -a / b, u2 = 1 / b)"""
    while True:
        a, b = rnd.randrange(1, N), rnd.randrange(1, N)
        R = ec.point_add(mul(a), mul(b, Q))
        if R is not None and R[0] < N:
            binv = pow(b, -1, N)
            v = recover_vector(tag, R, -a * binv, binv)
            assert v.key == Q, tag
            return v


def r_plus_n_forgery(tag: str, x: int, odd: int, rnd: random.Random) -> tuple[Vector, tuple]:
    """(vector, Q): a nonce point R with abscissa x in (n, p), r = x - n, and the key Q = r^-1 (s R - z G).  Plain ECDSA, which
    compares x mod n with r, accepts (r, s, z) for Q; recovery lifts x = r and yields another key or none, so the item, which
    names addr(Q), must get verdict 0."""
    R = ec.lift_x(x, odd)
    r = x - N
    assert R is not None and N < x < P and 1 < r
    s, z = rnd.randrange(1, N), rnd.randrange(1, N)
    Q = mul(pow(r, -1, N), ec.point_add(mul(s, R), ec.point_neg(mul(z))))
    assert Q is not None and ec.verify(z, r, s, Q)
    sig = r.to_bytes(32, "big") + s.to_bytes(32, "big") + bytes([odd])
    key = ec.recover_pubkey(z, r, s, odd)
    assert key != Q
    rinv = pow(r, -1, N)
    return Vector(tag, sig, z.to_bytes(32, "big"), key, (-z * rinv % N, s * rinv % N), ec.pubkey_to_address(Q)), Q


def _abscissas_above_n(count: int, lifts: bool) -> list[int]:
    """the first `count` abscissas x > n + 1 whose x - n is (lifts) / is not an abscissa itself"""
    out, x = [], N + 2
    while len(out) < count:
        if ec.lift_x(x, 0) is not None and (ec.lift_x(x - N, 0) is not None) == lifts:
            out.append(x)
        x += 1
    return out


@functools.lru_cache(maxsize=None)
def r_plus_n_forgeries() -> tuple[tuple[Vector, tuple], ...]:
    """half with x - n an abscissa (recovery yields another key), half without (recovery fails)"""
    rnd = random.Random(0x5EED)
    xs = _abscissas_above_n(6, True) + _abscissas_above_n(6, False)
    return tuple(r_plus_n_forgery(f"r+n forgery x=n+{x - N} lifts={ec.lift_x(x - N, 0) is not None}", x, k & 1, rnd)
                 for k, x in enumerate(xs))


@functools.lru_cache(maxsize=None)
def coordinate_edge_vectors() -> tuple[Vector, ...]:
    rnd = random.Random(0xED6E)
    keyed = [signature_for(tag, Q, rnd) for tag, Q in key_edge_points()]
    forged = [v for v, _ in r_plus_n_forgeries()]
    out = keyed + forged + [high_s_twin(v) for v in keyed + forged]
    # nonce points at the edges, both recovery ids; r = 1 takes every (z, s), the others three each
    rs = NONCE_R + [x for x, _ in tiny_y_points()[::2] if x < N]
    for i, r in enumerate(rs):
        for odd in (0, 1):
            R = ec.lift_x(r, odd)
            combos = NONCE_ZS if r == 1 else [NONCE_ZS[(3 * (2 * i + odd) + t) % len(NONCE_ZS)] for t in (0, 5, 7)]
            for z, s in combos:
                z = rnd.randrange(1, N) if z is None else z
                s = rnd.randrange(1, N) if s is None else s
                rinv = pow(r, -1, N)
                out.append(recover_vector(f"nonce-edge r={r:#x} odd={odd} z={z:#x} s={s:#x}", R, -z * rinv, s * rinv,
                                          z_override=z.to_bytes(32, "big")))
    # r an abscissa in (n, p): out of range, no key
    for x in _abscissas_above_n(2, True) + _abscissas_above_n(1, False) + NEAR_P_X:
        for odd in (0, 1):
            sig = x.to_bytes(32, "big") + rnd.randrange(1, N).to_bytes(32, "big") + bytes([odd])
            out.append(Vector(f"r-out-of-range x={x:#x} odd={odd}", sig, rnd.randbytes(32), None))
    return tuple(out)


def check_coordinate_edges() -> None:
    """every coordinate-edge family is present and holds its coordinate claim"""
    keys = dict(key_edge_points())
    fam = lambda p: [Q for t, Q in keys.items() if t.startswith("key-edge " + p)]
    assert len(fam("small-x")) == 10 and all(Q[0] in SMALL_X for Q in fam("small-x"))
    assert len(fam("weak-x")) == 6 and all(Q[0] < WEAK and Q[0] + P < 2**256 for Q in fam("weak-x"))
    assert len(fam("near-p-x")) == 4 and all(P - 5 < Q[0] < P for Q in fam("near-p-x"))
    assert len(fam("tiny-y")) == 18 and all(min(Q[1], P - Q[1]) in TINY_Y for Q in fam("tiny-y"))
    assert {Q[1] & 1 for Q in keys.values()} == {0, 1} and len(set(keys.values())) == len(keys)
    assert ec.lift_x(0, 0) is None and ec.lift_x(5, 0) is None and ec.lift_x(7, 0) is None
    vecs = coordinate_edge_vectors()
    tags = [v.tag for v in vecs]
    for t in ("key-edge small-x", "key-edge weak-x", "key-edge near-p-x", "key-edge tiny-y", "nonce-edge", "r-out-of-range",
              "r+n forgery"):
        assert sum(x.startswith(t) for x in tags) >= 4, t
    for v in vecs:
        r = int.from_bytes(v.sig[:32], "big")
        if v.tag.startswith("key-edge"):
            assert v.verdict and v.key == keys[v.tag.split("/")[0]], v.tag
        if v.tag.startswith("nonce-edge"):
            assert r in NONCE_R or any(r == x for x, _ in tiny_y_points()), v.tag
        if v.tag.startswith("r-out-of-range"):
            assert N < r < P and ec.lift_x(r, 0) is not None and v.key is None, v.tag
    nonce = {(int.from_bytes(v.sig[:32], "big"), v.sig[64]) for v in vecs if v.tag.startswith("nonce-edge")}
    assert all((r, odd) in nonce for r in NONCE_R for odd in (0, 1))
    assert sum(t.startswith("nonce-edge r=0x1 ") for t in tags) == 2 * len(NONCE_ZS)
    forged = r_plus_n_forgeries()
    lifts = [v.key is not None for v, _ in forged]
    assert 4 <= sum(lifts) <= len(forged) - 4
    for v, Q in forged:
        r, s, z = int.from_bytes(v.sig[:32], "big"), int.from_bytes(v.sig[32:64], "big"), int.from_bytes(v.digest, "big")
        assert ec.verify(z, r, s, Q) and ec.recover_pubkey(z, r, s, v.sig[64]) != Q and not v.verdict
        assert N < ec.point_add(mul(z * pow(s, -1, N)), mul(r * pow(s, -1, N), Q))[0] < P


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
    return tuple(out + twins) + coordinate_edge_vectors()


# ------------------------------------------------------------------------------------------------------ known keys
KNOWN_KEYS = [1, N - 1, LAM, N - LAM, 2, 0xC0FFEE]   # Q = G, -G, lambda G, -lambda G, 2G: the key stream meets the generator's
KNOWN_HALVES = [0, 1, -1, 127, 128, -128, 129, 255, 256, 0x8000, ALL80, -ALL80, 2**127, 2**128 - 1, -(2**127) - 5, 0x7F80 << 64]


KNOWN_EDGE_HALVES = 4                  # known-key vectors per coordinate-edge or forgery key (the first j of the loop below)


@dataclass(frozen=True)
class KnownVector:
    key_index: int    # index into known_points() of the signing key
    sig: bytes
    digest: bytes


@functools.lru_cache(maxsize=None)
def known_points() -> tuple:
    """the known-key set: the KNOWN_KEYS multiples, the coordinate-edge keys, and the keys of the x = r + n forgeries"""
    return tuple([mul(d) for d in KNOWN_KEYS] + [Q for _, Q in key_edge_points()] + [Q for _, Q in r_plus_n_forgeries()])


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
    """Valid signatures of the known points built for constructed (u1, u2): Booth digits on the window edges, u1 = 0 (no generator
    term), and u1 = u2 (with Q = +-G / +-lambda G the two streams add the same or opposite points).  The KNOWN_KEYS multiples take
    every j, the other points the first KNOWN_EDGE_HALVES (u1 = u2, u1 = 0 and two of neither)."""
    out = []
    L = len(KNOWN_HALVES)
    for i, Q in enumerate(known_points()):
        for j in range(L if i < len(KNOWN_KEYS) else KNOWN_EDGE_HALVES):
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


@functools.lru_cache(maxsize=None)
def known_r_plus_n() -> tuple[KnownVector, ...]:
    """The x = r + n forgeries and their high-s twins, each presented as its key Q: plain ECDSA accepts them for Q, so a known-key
    pass that compared x mod n with r would accept them; recovery yields another key or none (verdict 0), so the known-key pass
    must reject each and hand it back once."""
    first = len(KNOWN_KEYS) + len(key_edge_points())
    out = []
    for k, (v, Q) in enumerate(r_plus_n_forgeries()):
        assert known_points()[first + k] == Q
        for sig in (v.sig, high_s_twin(v).sig):
            out.append(KnownVector(first + k, sig, v.digest))
    return tuple(out)


def known_key(i: int):
    return known_points()[i]


@functools.lru_cache(maxsize=None)
def known_addr(i: int) -> bytes:
    return ec.pubkey_to_address(known_key(i))


def misattributed(v: KnownVector) -> tuple[bytes, int]:
    """(signature, claimed validator): a valid signature of key i presented as validator i + 1"""
    return v.sig, (v.key_index + 1) % len(known_points())


def flipped(v: KnownVector) -> bytes:
    """the signature with the other recovery id: recovery yields another key"""
    return v.sig[:64] + bytes([v.sig[64] ^ 1])


# ------------------------------------------------------------------------------------------------------ item arrays
def recover_items(vectors, group: int = 0) -> np.ndarray:
    """IBFT_KIND_DIGEST items naming the vector's signer (the recovered address unless it claims another; zero when there is none)"""
    import workloads as wl
    return np.concatenate([wl.make_item(v.sig, v.signer, 0, v.digest, group) for v in vectors])


def in_range(sig: bytes) -> bool:
    """0 < r, s < n and v in {0, 1}: the signature reaches the curve arithmetic"""
    r, s = int.from_bytes(sig[:32], "big"), int.from_bytes(sig[32:64], "big")
    return 0 < r < N and 0 < s < N and sig[64] <= 1


def expected_bits(vectors) -> np.ndarray:
    """verdict of every recover vector (0/1), membership aside"""
    return np.array([v.verdict for v in vectors], dtype=bool)
