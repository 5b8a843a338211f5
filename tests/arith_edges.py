"""Operands at the reduction and rounding edges of the hand-written arithmetic (secp_fe.cuh, secp_scalar.cuh, secp_modinv.cuh),
shared by the emulation test (test_emul_arith_edges.py) and the GPU test (test_gpu_arith_edges.py).  Random 256-bit operands
reach most of these branches with probability about 2^-120; each generator below is built to reach one, and `coverage` counts,
on a value-level model of the routine, how often the sweep takes each branch.

The sweep is a list of cases (op, a, b).  `expected` gives the exact output of each op from Python big integers: for the raw
field ops that is the routine's weakly reduced value (the model of its folds), not merely the residue, so a slip in a carry that
leaves the residue right but the limbs wrong still shows.  `check_sweep(run)` runs every case through `run(op, a, b, stride)`
(a batch of operands in, a list of output byte strings back) and lists the disagreements."""
from __future__ import annotations

import functools
import json
import os
import random
from collections import Counter
from dataclasses import dataclass

from oracle import secp256k1 as ec

P, N = ec.P, ec.N
M = 1 << 256
C = M - P           # 2^32 + 977: 2^256 = C (mod p)
NC = M - N          # 2^256 - n, 129 bits: 2^256 = NC (mod n)
LAM = 0x5363AD4CC05C30E0A5261C028812645A122E22EA20816678DF02967C1B23BD72
# GLV constants of secp_scalar.cuh glv_split: g_i ~ 2^384 * (coordinates of (1, 0) in the lattice basis), basis (a1, b1), (a2, b2)
G1 = 0x3086D221A7D46BCDE86C90E49284EB153DAA8A1471E8CA7FE893209A45DBB031
G2 = 0xE4437ED6010E88286F547FA90ABFE4C4221208AC9DF506C61571B4AE8AC47F71
A1 = 0x3086D221A7D46BCDE86C90E49284EB15
MB1 = 0xE4437ED6010E88286F547FA90ABFE4C3  # -b1
A2 = 0x114CA50F7A8E2F3F657C1108D9D44CFD8
B2 = A1
WR, WG, NWIN_R, NWIN_G = 4, 8, 33, 17     # Booth windows of ecmult_streams (R) and ecmult_gen_comb (G), digits per half


# ------------------------------------------------------------------------------------------------------------ models
def fe_add_model(a, b):
    """raw fe_add and whether the second fold carried (the 'second wrap')"""
    s = a + b
    r1 = s % M + (s >> 256) * C
    return r1 % M + (r1 >> 256) * C, (r1 >> 256) != 0


def fe_sub_model(a, b):
    """raw fe_sub and whether the second correction borrowed"""
    d = a - b
    if d < 0:
        d += M - C
        if d < 0:
            return d + M - C, True
    return d, False


def fe_reduce512_model(R):
    """raw fe_reduce512 of a 512-bit product, and whether its last fold (k = 1) carried"""
    L, H = R % M, R >> 256
    S = L + H * 977 + (H << 32)
    T = S % M + (S >> 256) * C
    k = T >> 256
    return T % M + k * C, k != 0


def fe_mul_model(a, b):
    return fe_reduce512_model(a * b)[0]


def fe_sqrn_model(a, k):
    for _ in range(k):
        a = fe_mul_model(a, a)
    return a


def sc_reduce512_stages(R):
    """(a2 >> 256, a3 >> 256) of sc_reduce512: the third fold's multiplier and whether it carried into fold 4"""
    L, H = R % M, R >> 256
    a1 = L + H * NC
    a2 = a1 % M + (a1 >> 256) * NC
    a3 = a2 % M + (a2 >> 256) * NC
    return a2 >> 256, a3 >> 256


def glv_model(k):
    """the exact restatement of glv_split: c_i = (k g_i + 2^383) >> 384, k1 = k - c1 a1 - c2 a2, k2 = c1 (-b1) - c2 b2"""
    c1 = (k * G1 + (1 << 383)) >> 384
    c2 = (k * G2 + (1 << 383)) >> 384
    return k - c1 * A1 - c2 * A2, c1 * MB1 - c2 * B2


def rounding_offset(k, g):
    """k g / 2^384 minus the nearest half-integer, as a fraction of 1: the distance of c's rounding from its boundary"""
    frac = (k * g) % (1 << 384)
    return (frac - (1 << 383)) / float(1 << 384)


def booth_digits(x, w, count):
    """the signed digits booth_digit<w> reads from a non-negative x: d_j = bits[wj .. wj+w-1] + bit[wj-1] - 2^w bit[wj+w-1]"""
    out = []
    for j in range(count):
        field = ((x << 1) >> (w * j)) & ((2 << w) - 1)
        out.append(((field + 1) >> 1) - (((field >> w) & 1) << w))
    return out


def safegcd_model(x, m):
    """(30-divstep batches, sign of the final f) of secp_modinv.cuh modinv30_var(x) modulo m: the same steps on whole
    integers -- every decision of divsteps_30_var reads low bits only, which agree.  eta = -delta, starting at -1."""
    f, g, eta = m, x, -1
    for it in range(1, 41):
        i = 30
        while True:
            zeros = i if g % (1 << i) == 0 else min((g & -g).bit_length() - 1, i)
            g >>= zeros
            eta -= zeros
            i -= zeros
            if i == 0:
                break
            if eta < 0:
                eta, f, g = -eta, g, -f
            limit = min(eta + 1, i, 8)
            w = (-g * pow(f, -1, 256)) % (1 << limit)
            g += f * w
        if g == 0:
            return it, (1 if f > 0 else -1)
    raise AssertionError("more than 40 batches")


def is_residue(c):
    return pow(c % P, (P - 1) // 2, P) in (0, 1)


def sqrt_inv_model(c, V):
    """y, w of fe_sqrt_inv modulo p: u = (c V^4)^((p-3)/4), y = c V^2 u, w = u V"""
    u = pow(c * pow(V, 4, P) % P, (P - 3) // 4, P)
    return c * V * V * u % P, u * V % P


# ------------------------------------------------------------------------------------------------------------ generators
LIMBS = [0, 1, 977, 2**31 - 1, 2**31, 2**31 + 1, 2**32 - 2, 2**32 - 1]


def from_limbs(ls):
    return sum(x << (32 * i) for i, x in enumerate(ls))


def field_limb_patterns(rnd, count=400):
    """limbs from LIMBS (or random), and all-ones runs broken by a single 0 or 1 limb"""
    out = []
    for _ in range(count):
        out.append(from_limbs([rnd.choice(LIMBS) if rnd.random() < 0.85 else rnd.getrandbits(32) for _ in range(8)]))
    ones = [2**32 - 1] * 8
    for pos in range(8):
        for brk in (0, 1):
            ls = list(ones)
            ls[pos] = brk
            out.append(from_limbs(ls))
            ls[0] = rnd.choice(LIMBS)  # and with the lowest limb taken from the edges
            out.append(from_limbs(ls))
    for lo in range(8):  # runs of all-ones limbs lo..7 over an edge-valued bottom
        out.append(from_limbs([rnd.choice(LIMBS) for _ in range(lo)] + [2**32 - 1] * (8 - lo)))
    return out


NONCANON_T = [0, 1, 2, 976, 977, 978, 2**31, 2**32 - 1, 2**32, 2**32 + 976]


def noncanonical():
    """p + t and 2^256 - 1 - t: the weakly reduced values in [p, 2^256), and the same offsets down from the top"""
    return sorted({P + t for t in NONCANON_T} | {M - 1 - t for t in NONCANON_T})


def sc_fold4_pairs(rnd, count):
    """(a, b, a2[8]) with a, b in [1, n) whose product carries out of sc_reduce512's third fold.  a2 = a b (mod n) and
    a2 < 2^256 + NC^2 takes one of a few values t + j n; a target t within a2[8] NC below a multiple of 2^256, b = t / a."""
    out = []
    while len(out) < count:
        a = rnd.randrange(1, N)
        h = rnd.randrange(1, SC_FOLD4_MAX_A2 + 1)
        t = (h * M + M - 1 - rnd.randrange(h * NC)) % N
        b = t * pow(a, -1, N) % N
        a2h, carry = sc_reduce512_stages(a * b)
        if carry:
            out.append((a, b, a2h))
    return out


# a3 carries only when a2 % 2^256 >= 2^256 - a2[8] NC; with a2 < 2^256 + NC^2 < 3 * 2^256 - 2 NC that needs a2[8] = 1
SC_FOLD4_MAX_A2 = max(h for h in (1, 2, 3) if h * M + M - h * NC <= M - 1 + NC * NC)


def sc_add_pairs(rnd):
    """(a, b) in [0, n)^2: sums over 2^256, in [n, 2^256), equal to n - 1 and to n, and random"""
    out = [(N - 1, N - 1), (N - 1, 1), (N - 1, 0), (0, 0), (1, N - 2), (NC, N - NC), (NC - 1, N - NC), (NC, N - NC - 1), (M - N, N - 1)]
    for _ in range(40):
        s = rnd.randrange(M, 2 * N - 1)          # overflows 2^256
        a = rnd.randrange(s - N + 1, N)
        out.append((a, s - a))
        s = rnd.randrange(N, M)                  # in [n, 2^256): no carry, still >= n
        a = rnd.randrange(s - N + 1, N)
        out.append((a, s - a))
        a = rnd.randrange(N)                     # = n - 1 and = n
        out.append((a, N - 1 - a))
        a = rnd.randrange(1, N)
        out.append((a, N - a))
        out.append((rnd.randrange(N), rnd.randrange(N)))
    return out


def sc_reduce_once_inputs(rnd):
    return [0, 1, N - 1, N, N + 1, M - 1, M - 2, NC, N + NC - 1] + [rnd.randrange(N, M) for _ in range(20)] + [rnd.randrange(N) for _ in range(10)]


def sc_neg_inputs(rnd):
    return [0, 1, 2, N - 1, N - 2, (N - 1) // 2, (N + 1) // 2, NC] + [rnd.randrange(N) for _ in range(10)]


def glv_boundary_scalars(rnd, per_side=24):
    """k in [0, n) with k g_i / 2^384 within 2^-16 of a half-integer, below and above it, for g1 and g2"""
    out = []
    for g in (G1, G2):
        span = (1 << 367) // g + 1   # k steps that move k g / 2^384 by less than 2^-17
        for _ in range(per_side):
            while True:
                m = rnd.randrange(1, (N * g) >> 384)
                k0 = ((2 * m + 1) << 383) // g   # k0 g / 2^384 just below m + 1/2, k0 + 1 just above
                lo, hi = k0 - rnd.randrange(span), k0 + 1 + rnd.randrange(span)
                if 0 <= lo and hi < N:
                    out += [lo, hi, k0, k0 + 1]
                    break
    return out


def glv_corner_scalars(rnd, per_corner=6):
    """k whose halves sit near the corners +-(v1 +- v2)/2 of the rounding domain, v1 = (a1, b1), v2 = (a2, b2): both roundings
    near 1/2 at once, where |k1| and |k2| are largest"""
    b1 = -MB1
    out = []
    for s1 in (1, -1):
        for s2 in (1, -1):
            x, y = s1 * (A1 + s2 * A2), s1 * (b1 + s2 * B2)  # 2 (corner)
            for _ in range(per_corner):
                k1 = (x + rnd.randrange(-3, 4)) // 2 + rnd.randrange(-(1 << 20), 1 << 20)
                k2 = (y + rnd.randrange(-3, 4)) // 2 + rnd.randrange(-(1 << 20), 1 << 20)
                out.append((k1 + k2 * LAM) % N)
    return out


def sqrt_inv_cases(rnd):
    """(c, V): c a residue, a non-residue, 7 (r = 0: 0^3 + 7, not a residue) and non-canonical; V over the edges"""
    cs = [7, 7 + P, 1, P + 1, 4]
    while len(cs) < 9:
        x = rnd.randrange(1, P)
        cs.append(x * x % P)
    while len(cs) < 13:
        x = rnd.randrange(1, P)
        if not is_residue(x):
            cs.append(x)
    cs.append(P + next(x for x in range(2, 100) if not is_residue(x)))  # a non-residue given non-canonically
    Vs = [1, P - 1, P, P + 1, M - 1, P + 977, M - 2**32, rnd.randrange(P, M), rnd.randrange(1, P)]
    return [(c, V) for c in cs for V in Vs]


@functools.lru_cache(maxsize=None)
def safegcd_edges():
    """inputs of the most 30-divstep batches and inputs that end with f = -1 (tests/golden/safegcd_edges.json, found by
    tests/golden/make_safegcd_edges.py with safegcd_model over random candidates)"""
    with open(os.path.join(os.path.dirname(__file__), "golden", "safegcd_edges.json")) as f:
        return json.load(f)


# ------------------------------------------------------------------------------------------------------------ the sweep
@dataclass(frozen=True)
class Case:
    op: str
    a: int
    b: int = 0


FE_OPS = ("FE_MUL_RAW", "FE_SQR_RAW", "FE_ADD_RAW", "FE_SUB_RAW", "FE_NORMALIZE", "FE_EQUAL")


@functools.lru_cache(maxsize=None)
def sweep_cases() -> tuple[Case, ...]:
    rnd = random.Random(0xA817)
    cases = []
    nc = noncanonical()
    edge = nc + [0, 1, 2, 977, C, C - 1, P - 1, P - 2, 2**255, 2**128 - 1, 2**224 - 1, 2**32 - 1]
    pats = field_limb_patterns(rnd)
    vals = edge + pats
    pairs = [(x, y) for x in nc for y in nc]                                # every pair of non-canonical values
    pairs += [(x, y) for x in edge for y in edge]
    pairs += [(rnd.choice(vals), rnd.choice(vals)) for _ in range(3000)]
    pairs += [(x, P - 1 - x + t) for x in pats[:200] for t in (0, rnd.choice(NONCANON_T)) if P - 1 - x + t >= 0]  # sums at p
    pairs += [(t, P + t) for t in NONCANON_T] + [(P + t, t) for t in NONCANON_T]  # equal residues, one side raw
    for x, y in pairs:
        for op in ("FE_MUL_RAW", "FE_ADD_RAW", "FE_SUB_RAW", "FE_EQUAL"):
            cases.append(Case(op, x, y))
    for x in vals:
        cases.append(Case("FE_SQR_RAW", x))
        cases.append(Case("FE_NORMALIZE", x))
    for x in edge + pats[:40]:
        for k in (0, 1, 2, 3, 5, 22, 44, 88, 223, 255):
            cases.append(Case("FE_SQRN", x, k))
    for c, V in sqrt_inv_cases(rnd):
        cases.append(Case("FE_SQRT_INV", c, V))
    # scalars
    for a, b, _ in sc_fold4_pairs(rnd, 60):
        cases += [Case("SC_MUL", a, b), Case("SC_MUL", b, a)]
    cases += [Case("SC_MUL", x, y) for x in (M - 1, M - 2, N - 1, N, 2**255) for y in (M - 1, N - 1, NC, 2**255)]
    cases += [Case("SC_ADD", a, b) for a, b in sc_add_pairs(rnd)]
    cases += [Case("SC_REDUCE_ONCE", a) for a in sc_reduce_once_inputs(rnd)]
    cases += [Case("SC_NEG", a) for a in sc_neg_inputs(rnd)]
    ks = [0, 1, 2, N - 1, N - 2, LAM, N - LAM, (N + 1) // 2, N // 2, 2**128, 2**128 - 1, 2**255]
    ks += glv_boundary_scalars(rnd) + glv_corner_scalars(rnd) + [rnd.randrange(N) for _ in range(300)]
    cases += [Case("SC_DIGITS", k) for k in ks]
    # safegcd
    sg = safegcd_edges()
    for name, op in (("p", "FE_INV"), ("n", "SC_INV")):
        for x in sg[name]["most_batches"] + sg[name]["f_negative"]:
            cases.append(Case(op, int(x, 16)))
    return tuple(cases)


STRIDE = {"FE_SQRT_INV": 64, "SC_DIGITS": 256}


def expected(case: Case):
    """exact output of an op (for FE_SQRT_INV and the two inversions: the residue)"""
    op, a, b = case.op, case.a, case.b
    if op == "FE_MUL_RAW":
        return fe_mul_model(a, b)
    if op == "FE_SQR_RAW":
        return fe_mul_model(a, a)
    if op == "FE_ADD_RAW":
        return fe_add_model(a, b)[0]
    if op == "FE_SUB_RAW":
        return fe_sub_model(a, b)[0]
    if op == "FE_NORMALIZE":
        return a % P
    if op == "FE_EQUAL":
        return int((a - b) % P == 0)
    if op == "FE_SQRN":
        return fe_sqrn_model(a, b)
    if op == "FE_SQRT_INV":
        return sqrt_inv_model(a, b)
    if op == "FE_INV":
        return pow(a, -1, P) if a % P else 0
    if op == "SC_INV":
        return pow(a, -1, N) if a % N else 0
    if op == "SC_MUL":
        return a * b % N
    if op == "SC_ADD":
        return (a + b) % N
    if op == "SC_NEG":
        return -a % N
    if op == "SC_REDUCE_ONCE":
        return a % N
    if op == "SC_DIGITS":
        return glv_model(a)
    raise KeyError(op)


def decode_digits(o: bytes):
    """SC_DIGITS output -> [(magnitude, negative, 4-bit digits, 8-bit digits)] for both halves"""
    halves = []
    for h in range(2):
        q = o[128 * h: 128 * (h + 1)]
        d4 = [int.from_bytes(q[32 + j: 33 + j], "little", signed=True) for j in range(NWIN_R)]
        d8 = [int.from_bytes(q[72 + 2 * j: 74 + 2 * j], "little", signed=True) for j in range(NWIN_G)]
        halves.append((int.from_bytes(q[:24], "little"), bool(q[24]), d4, d8))
    return halves


def mismatch(case: Case, o: bytes) -> str | None:
    """None when the op's output `o` is right, else what is wrong"""
    want = expected(case)
    if case.op == "FE_EQUAL":
        got = o[0]
    elif case.op == "FE_SQRT_INV":
        y, w = int.from_bytes(o[:32], "big"), int.from_bytes(o[32:64], "big")
        got = (y % P, w % P)
    elif case.op in ("FE_INV", "SC_INV"):
        got = int.from_bytes(o[:32], "big")
    elif case.op == "SC_DIGITS":
        halves = decode_digits(o)
        got = tuple((-m if neg else m) for m, neg, _, _ in halves)
        if got != want:
            return f"GLV halves {got} != {want}"
        for m, _, d4, d8 in halves:
            for w, ds in ((WR, d4), (WG, d8)):
                if sum(d << (w * j) for j, d in enumerate(ds)) != m or max(abs(d) for d in ds) > 1 << (w - 1):
                    return f"{w}-bit Booth digits {ds} do not recompose |k| = {m:#x}"
                if ds != booth_digits(m, w, len(ds)):
                    return f"{w}-bit Booth digits {ds} != {booth_digits(m, w, len(ds))}"
        return None
    else:
        got = int.from_bytes(o[:32], "big")
    return None if got == want else f"got {got!r} want {want!r}"


def check_sweep(run, cases=None, limit=20) -> list[str]:
    """run every case through run(op, a_list, b_list, stride) -> list of outputs; returns the disagreements (at most `limit`)"""
    cases = sweep_cases() if cases is None else cases
    by_op: dict[str, list[Case]] = {}
    for c in cases:
        by_op.setdefault(c.op, []).append(c)
    bad = []
    for op, cs in by_op.items():
        outs = run(op, [c.a for c in cs], [c.b for c in cs], STRIDE.get(op, 32))
        for c, o in zip(cs, outs):
            m = mismatch(c, o)
            if m:
                bad.append(f"{op}({c.a:#x}, {c.b:#x}): {m}")
                if len(bad) >= limit:
                    return bad
    return bad


# ------------------------------------------------------------------------------------------------------------ coverage
def coverage(cases=None) -> Counter:
    """how often the sweep takes each named branch, on the models above"""
    cases = sweep_cases() if cases is None else cases
    hit = Counter()
    for c in cases:
        a, b = c.a, c.b
        if c.op == "FE_ADD_RAW":
            r, wrap2 = fe_add_model(a, b)
            hit["fe_add: second wrap"] += wrap2
            hit["fe_add: result in [p, 2^256)"] += r >= P
        elif c.op == "FE_SUB_RAW":
            r, borrow2 = fe_sub_model(a, b)
            hit["fe_sub: second borrow"] += borrow2
            hit["fe_sub: result in [p, 2^256)"] += r >= P
        elif c.op == "FE_MUL_RAW":
            hit["fe_reduce512: last fold carries (mul)"] += fe_reduce512_model(a * b)[1]
            hit["fe_mul: result in [p, 2^256)"] += fe_mul_model(a, b) >= P
        elif c.op == "FE_SQR_RAW":
            hit["fe_reduce512: last fold carries (sqr)"] += fe_reduce512_model(a * a)[1]
        elif c.op == "FE_NORMALIZE":
            hit["fe_normalize: input in [p, 2^256)"] += a >= P
        elif c.op == "FE_EQUAL":
            hit["fe_equal: fe_sub leaves exactly p"] += fe_sub_model(a, b)[0] == P
            hit["fe_equal: equal residues"] += (a - b) % P == 0
        elif c.op == "FE_SQRN":
            hit["fe_sqrn: k >= 88 from a non-canonical start"] += b >= 88 and a >= P
        elif c.op == "FE_SQRT_INV":
            if a % P == 7:
                hit["fe_sqrt_inv: c = 7"] += 1
            hit["fe_sqrt_inv: c a residue" if is_residue(a) else "fe_sqrt_inv: c a non-residue"] += 1
            hit[f"fe_sqrt_inv: V = {SQRT_V_NAMES.get(b, 'other')}"] += 1
            hit["fe_sqrt_inv: V in [p, 2^256)"] += b >= P
        elif c.op == "SC_MUL":
            a2h, carry = sc_reduce512_stages(a * b)
            if carry:
                hit[f"sc_reduce512: fold 4 (a2[8] = {a2h})"] += 1
            hit["sc_reduce512: a2[8] = 2"] += a2h == 2
        elif c.op == "SC_ADD":
            s = a + b
            hit["sc_add: sum >= 2^256"] += s >= M
            hit["sc_add: sum in [n, 2^256)"] += N <= s < M
            hit["sc_add: sum = n - 1"] += s == N - 1
            hit["sc_add: sum = n"] += s == N
        elif c.op == "SC_REDUCE_ONCE":
            for v, name in ((N - 1, "n - 1"), (N, "n"), (N + 1, "n + 1"), (M - 1, "2^256 - 1")):
                hit[f"sc_reduce_once: {name}"] += a == v
        elif c.op == "SC_NEG":
            hit["sc_neg: 0"] += a == 0
        elif c.op == "SC_DIGITS":
            for i, g in enumerate((G1, G2), 1):
                off = rounding_offset(a, g)
                if abs(off) < 2.0**-16:
                    hit[f"glv: c{i} within 2^-16 {'below' if off < 0 else 'above'} its rounding boundary"] += 1
            if abs(rounding_offset(a, G1)) < 2.0**-8 and abs(rounding_offset(a, G2)) < 2.0**-8:
                hit["glv: corner (both roundings within 2^-8 of 1/2)"] += 1
        elif c.op in ("FE_INV", "SC_INV"):
            m = P if c.op == "FE_INV" else N
            batches, sign = safegcd_model(a, m)
            tag = "p" if m == P else "n"
            hit[f"safegcd mod {tag}: {batches} batches"] += 1
            hit[f"safegcd mod {tag}: ends with f = -1"] += sign < 0
    return hit


SQRT_V_NAMES = {1: "1", P - 1: "p - 1", P: "p", P + 1: "p + 1", M - 1: "2^256 - 1"}


def required() -> dict[str, int]:
    """named condition -> how many cases of the sweep must reach it"""
    req = {
        "fe_add: second wrap": 20, "fe_add: result in [p, 2^256)": 20, "fe_sub: second borrow": 20, "fe_sub: result in [p, 2^256)": 20,
        "fe_reduce512: last fold carries (mul)": 20, "fe_reduce512: last fold carries (sqr)": 5, "fe_mul: result in [p, 2^256)": 1,
        "fe_normalize: input in [p, 2^256)": 20, "fe_equal: fe_sub leaves exactly p": 10, "fe_equal: equal residues": 20,
        "fe_sqrn: k >= 88 from a non-canonical start": 20,
        "fe_sqrt_inv: c = 7": 9, "fe_sqrt_inv: c a residue": 40, "fe_sqrt_inv: c a non-residue": 40, "fe_sqrt_inv: V in [p, 2^256)": 40,
        "sc_reduce512: a2[8] = 2": 1,
        "sc_add: sum >= 2^256": 40, "sc_add: sum in [n, 2^256)": 40, "sc_add: sum = n - 1": 40, "sc_add: sum = n": 40,
        "sc_reduce_once: n - 1": 1, "sc_reduce_once: n": 1, "sc_reduce_once: n + 1": 1, "sc_reduce_once: 2^256 - 1": 1, "sc_neg: 0": 1,
        "glv: corner (both roundings within 2^-8 of 1/2)": 12,
    }
    for name in SQRT_V_NAMES.values():
        req[f"fe_sqrt_inv: V = {name}"] = 13
    for h in range(1, SC_FOLD4_MAX_A2 + 1):
        req[f"sc_reduce512: fold 4 (a2[8] = {h})"] = 50
    for i in (1, 2):
        for side in ("below", "above"):
            req[f"glv: c{i} within 2^-16 {side} its rounding boundary"] = 24
    sg = safegcd_edges()
    for tag in ("p", "n"):
        req[f"safegcd mod {tag}: {sg[tag]['batches']} batches"] = 1
        req[f"safegcd mod {tag}: ends with f = -1"] = 8
    return req


# ------------------------------------------------------------------------------------------------------------ signatures
def fold4_signature_targets(rnd, r, count):
    """t in [1, n) such that the product t r * r^-1 -- the sc_mul(s, r^-1) of u2 = s/r with s = t r, or sc_mul(z, r^-1) of
    u1 = -z/r with z = t r -- carries into sc_reduce512's fold 4"""
    rinv = pow(r, -1, N)
    out = []
    for _ in range(100000):
        if len(out) == count:
            return out
        t = (M + M - 1 - rnd.randrange(NC)) % N
        x = t * r % N
        if x and sc_reduce512_stages(x * rinv)[1]:
            out.append(t)
    raise ValueError("r^-1 too small: the product never reaches fold 4")


def check_chains(run, lanes=64, steps=3000, seed=5) -> list[str]:
    """raw field ops chained from non-canonical starts, the way the kernels chain them: every step applies one of fe_mul, fe_sqr,
    fe_add, fe_sub to each lane's previous RAW result and an edge or random operand, with no normalisation in between.  At the
    end every lane's raw limbs must equal the model's, and its residue the plain modular result."""
    rnd = random.Random(seed)
    nc = noncanonical()
    got = [rnd.choice(nc) for _ in range(lanes)]
    model, residue = list(got), [x % P for x in got]
    for _ in range(steps):
        op = rnd.choice(("FE_MUL_RAW", "FE_SQR_RAW", "FE_ADD_RAW", "FE_SUB_RAW"))
        ys = [rnd.choice(nc) if rnd.random() < 0.5 else rnd.getrandbits(256) for _ in range(lanes)]
        got = [int.from_bytes(o[:32], "big") for o in run(op, got, ys, 32)]
        model = [expected(Case(op, x, y)) for x, y in zip(model, ys)]
        f = {"FE_MUL_RAW": lambda x, y: x * y, "FE_SQR_RAW": lambda x, y: x * x, "FE_ADD_RAW": lambda x, y: x + y,
             "FE_SUB_RAW": lambda x, y: x - y}[op]
        residue = [f(x, y) % P for x, y in zip(residue, ys)]
    return [f"lane {i}: raw {g:#x}, model {m:#x}, residue {r:#x}" for i, (g, m, r) in enumerate(zip(got, model, residue))
            if g != m or g % P != r]
