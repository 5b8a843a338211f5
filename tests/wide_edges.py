"""Crafted u1 values for the wide generator comb (secp_ec.cuh ecmult_gen_wide, window w = 22, 12 positions) and recover vectors
that make the recovery compute u1 G + u2 R for them (IBFT_KIND_DIGEST items, z = -u1 r mod n over the abscissa r of a real nonce
point R = k G).  Shared by the host-emulation test and the device test."""
from __future__ import annotations

import random

import adversarial as A
from oracle import secp256k1 as ec

N = ec.N
W = 22
POSITIONS = 12
TOP_BITS = 256 - W * (POSITIONS - 1)  # 14: the top digit of a scalar below n is at most 2^14


def u1_values() -> list[tuple[str, int]]:
    out = [("u1=0", 0), ("u1=1", 1), ("u1=n-1 (top digit 2^14)", N - 1), ("u1=n-2", N - 2)]
    windows = ((1 << (W - 1)) - 1, 1 << (W - 1), (1 << (W - 1)) + 1, (1 << W) - 1)
    for j in range(POSITIONS):
        for v in windows:
            out.append((f"window {v:#x} at position {j}", (v << (W * j)) % N))
        out.append((f"top-fitting window at position {j}", ((1 << TOP_BITS) - 1) << (W * j)))
    for v in windows:
        out.append((f"window {v:#x} at every position", sum(v << (W * j) for j in range(POSITIONS)) % N))
    # a Booth carry that ripples from position 0 through every window: 2^242 - 1 = -1 + 2^242 (digits -1, 0, ..., 0, 1)
    out.append(("carry through all 12 windows", (1 << (W * (POSITIONS - 1))) - 1))
    for j in range(1, POSITIONS):
        out.append((f"carry into position {j}", (1 << (W * j)) - 1))
    # alternating maximal positive and negative digits
    out.append(("alternating digits", sum(((1 << (W - 1)) if j & 1 else (1 << W) - 1) << (W * j) for j in range(POSITIONS - 1)) % N))
    return out


def booth_digits(u1: int) -> list[int]:
    """the signed digits ecmult_gen_wide takes from u1 (booth_digit of secp_scalar.cuh): sum d_j 2^(w j) = u1"""
    out = []
    for j in range(POSITIONS):
        lo = W * j - 1
        field = (u1 << 1) & ((2 << W) - 1) if lo < 0 else (u1 >> lo) & ((2 << W) - 1)
        out.append(((field + 1) >> 1) - (((field >> W) & 1) << W))
    return out


def nonce_points(count: int, seed: int) -> list[tuple]:
    """R = k G for random k, with R.x < n (a real signature's nonce point)"""
    rnd = random.Random(seed)
    out = []
    while len(out) < count:
        R = A.mul(rnd.randrange(1, N))
        if R[0] < N:
            out.append(R)
    return out


def vectors(seed: int = 2201, points: int = 2) -> list[A.Vector]:
    """every crafted u1 against `points` nonce points, each with a random u2 and its high-s twin"""
    rnd = random.Random(seed)
    out = []
    for R in nonce_points(points, seed):
        for tag, u1 in u1_values():
            v = A.recover_vector(f"wide {tag} R.x={R[0]:#x}", R, u1, rnd.randrange(1, N))
            out += [v, A.high_s_twin(v)]
    return out
