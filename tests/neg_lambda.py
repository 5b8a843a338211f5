"""Recover vectors whose lambda stream (the second GLV half of u2) adds a NEGATED table entry in every window it adds in: the
mixed addition folds the sign of -Q into r = -S2 - Y1 instead of negating Q's y (secp_ec.cuh jac_add_affine, neg_q).

u2 = k1 + h lambda with h's Booth digits all negative (h = 0x99..9, 0xDD..D: digits -6 / -2 below a top +1), or u2 = k1 - h lambda
with h's digits all positive (h = 0x11..1, 0x77..7: the half is negative, so every digit's addition is negated).  h has 31 hex
digits (one 32-digit 0x11..1): the GLV split gives such a half back as it is, where a 128-bit 0x99..9 comes back as a different
decomposition.  0x77..7 leaves the top windows empty, so with k1 = 0 its first addition meets the accumulator at infinity with a
negated entry.  Built like tests/adversarial.py's vectors (recover_vector), expected keys from the big-int oracle."""
import random

import adversarial as A

LAM = A.LAM
NWIN = 33
# (h, sign of the half in u2): every non-zero Booth digit of the half's magnitude times the half's sign is negative
HALVES = [(int("9" * 31, 16), 1), (int("D" * 31, 16), 1), (int("1" * 31, 16), -1), (int("7" * 31, 16), -1), (int("1" * 32, 16), -1)]


def vectors():
    rnd = random.Random(0x1A3B)
    out = []
    for base in (12345, 1, 0xC0FFEE):
        R = A.mul(base)
        for h, sign in HALVES:
            for k1 in (0, 1, 0x1234567, 2**127 + 3, rnd.getrandbits(120)):
                u2 = (k1 + sign * h * LAM) % A.N
                for u1 in (rnd.randrange(1, A.N), 0):
                    out.append(A.recover_vector(f"neg-lambda R={base} h={h:#x}{'+' if sign > 0 else '-'} k1={k1:#x} u1={u1:#x}",
                                                R, u1, u2))
    return tuple(out)


def negated_windows(digits_le, kneg):
    """windows of one half (its IBFT_DBG_SC_DIGITS record) whose addition adds a negated entry, and the non-zero ones"""
    d = [int.from_bytes(bytes([b]), "little", signed=True) for b in digits_le[32:32 + NWIN]]
    nz = [j for j in range(NWIN) if d[j]]
    return [j for j in nz if (d[j] < 0) != kneg], nz
