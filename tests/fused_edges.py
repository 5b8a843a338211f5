"""Operands at the carry and borrow edges of the fused linear combinations of secp_fe.cuh (fe_mul3, fe_sub_shl, fe_sub_sub_dbl,
fe_dbl_sub_sub, fe_sub_signed), shared by the host-emulation and the device tests.

Each operation builds the exact integer X of its expression as eight limbs and a small signed top word t (X = v + t 2^256), then
folds once: v + t (2^32 + 977) + e, whose carry leaves a second top t2 in {-1, 0, 1} that a two-limb fold removes.  The cases
below are constructed so that every operation reaches every value of t its operands allow, each with and without that second
fold, besides the plain edge values (0, 1, p - 1, p, p + 1, 2^256 - 1, ...)."""
import itertools
import random

P = 2**256 - 2**32 - 977
C = 2**32 + 977
M256 = 2**256

# selector of IBFT_DBG_FE_FUSED -> (name, operand count, exact value)
OPS = {
    0: ("3a", 1, lambda a, b, c: 3 * a),
    1: ("a - 2b", 2, lambda a, b, c: a - 2 * b),
    2: ("a - 8b", 2, lambda a, b, c: a - 8 * b),
    3: ("a - b - 2c", 3, lambda a, b, c: a - b - 2 * c),
    4: ("2 (a - b - c)", 3, lambda a, b, c: 2 * (a - b - c)),
    5: ("a - b", 2, lambda a, b, c: a - b),
    6: ("-a - b", 2, lambda a, b, c: -a - b),
}
# the range of t each operation's operands allow
TOPS = {0: range(0, 3), 1: range(-2, 1), 2: range(-8, 1), 3: range(-3, 1), 4: range(-4, 2), 5: range(-1, 1), 6: range(-2, 0)}

EDGE = [0, 1, 2, 977, C - 1, C, C + 1, P - 2, P - 1, P, P + 1, P + 2, 2**255 - 1, 2**255, M256 - 2, M256 - 1,
        M256 - C - 1, M256 - C, 2**32 - 1, 2**64 - 1, 2**224]


def model(sel, a, b, c):
    """(t, e, t2) of the device routine: the top word it folds, the extra addend of the fold and the second top"""
    if sel == 6:  # ~a - b = -a - 1 - b, and the fold adds the 1
        y, e = -a - 1 - b, 1
    else:
        y, e = OPS[sel][2](a, b, c), 0
    t = y >> 256
    v = y - t * M256
    return t, e, (v + t * C + e) >> 256


def _solve_a(sel, x, b, c):
    """the first operand giving the exact value x with the others fixed, or None"""
    if sel == 0:
        return x // 3 if x % 3 == 0 else None
    if sel in (1, 2):
        return x + (2 if sel == 1 else 8) * b
    if sel == 3:
        return x + b + 2 * c
    if sel == 4:
        return x // 2 + b + c if x % 2 == 0 else None
    if sel == 5:
        return x + b
    return -x - b  # sel == 6


def cases(seed: int = 11):
    """[(sel, a, b, c)]: the edge grid of every operation, then constructed values at each top t with and without a second fold"""
    rnd = random.Random(seed)
    out = []
    for sel, (_, n, _) in OPS.items():
        grid = EDGE if n > 1 else EDGE + [M256 // 3 + d for d in range(-2, 3)] + [2 * M256 // 3 + d for d in range(-2, 3)]
        pick = rnd.sample(EDGE, 6)
        for a, b in itertools.product(grid, EDGE if n > 1 else [0]):
            out.append((sel, a, b, pick[(a + b) % len(pick)] if n > 2 else 0))
        # exact values t 2^256 + v with v at the edges where the first fold wraps (t2 != 0) and where it just does not
        for t in TOPS[sel]:
            for v in (0, 1, 2, 977, C, 2**35, 8 * C, M256 - 9 * C, M256 - 2**36, M256 - C - 2, M256 - 2, M256 - 1):
                x = t * M256 + v
                for _ in range(40):
                    b = (rnd.choice(EDGE) if rnd.random() < 0.3 else rnd.getrandbits(256)) if n > 1 else 0
                    c = (rnd.choice(EDGE) if rnd.random() < 0.3 else rnd.getrandbits(256)) if n > 2 else 0
                    for dx in (0, 1, -1, 2, -2, 3):  # 3a and 2 (...) need a divisible value: move v by a little
                        a = _solve_a(sel, x + dx, b, c)
                        if a is not None and 0 <= a < M256 and OPS[sel][2](a, b, c) == x + dx:
                            out.append((sel, a, b, c))
                            break
                    else:
                        continue
                    break
    return out


def coverage(cs):
    """{sel: set of (t, t2)} the cases reach"""
    cov = {sel: set() for sel in OPS}
    for sel, a, b, c in cs:
        t, _, t2 = model(sel, a, b, c)
        cov[sel].add((t, t2))
    return cov


def c_operand(sel, c):
    """the 64-byte third operand of IBFT_DBG_FE_FUSED: c (32 bytes, big-endian), the selector in the last byte"""
    return c.to_bytes(32, "big") + bytes(31) + bytes([sel])


def check(results, cs):
    """mismatch descriptions of raw results (32-byte big-endian) against the big-integer value of each case"""
    bad = []
    for (sel, a, b, c), r in zip(cs, results):
        got = int.from_bytes(r[:32], "big")
        want = OPS[sel][2](a, b, c) % P
        if got % P != want:  # any representative below 2^256 is what the kernels chain on
            bad.append(f"{OPS[sel][0]}: a={a:#x} b={b:#x} c={c:#x}: got {got:#x}, want {want:#x} mod p")
    return bad


def required_coverage():
    """every top t of every operation, with the second fold that its sign makes possible (t2 = 1 above 0, -1 below)"""
    return {sel: {(t, 0) for t in tops} | {(t, 1 if t > 0 else -1) for t in tops if t} for sel, tops in TOPS.items()}
