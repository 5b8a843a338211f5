"""Device primitives (the PTX carry-chain code paths) against the oracle, through the C ABI's ibft_debug_op."""
import random

import pytest

from oracle import coracle as co
from oracle import secp256k1 as ec

pytestmark = pytest.mark.gpu
P, N = ec.P, ec.N
LAM = 0x5363AD4CC05C30E0A5261C028812645A122E22EA20816678DF02967C1B23BD72
EDGE = [0, 1, 2, P - 1, P, P + 1, 2**256 - 1, 2**255, N, N - 1, 2**32, 2**32 + 977, 2**256 - 2**32 - 978, (1 << 224) - 1,
        2**256 - 2**32, 0xFFFFFFFF, (2**256 - 1) ^ 0xFFFFFFFF, int("ffffffff00000000" * 4, 16), int("00000000ffffffff" * 4, 16)]


def ints(bs):
    return [int.from_bytes(b, "big") for b in bs]


def test_fe_ops(engine):
    rnd = random.Random(21)
    a = EDGE + [rnd.getrandbits(256) for _ in range(3000)]
    b = [rnd.choice(EDGE) if i % 5 == 0 else rnd.getrandbits(256) for i in range(len(a))]
    # every edge x edge pair
    for x in EDGE:
        for y in EDGE:
            a.append(x)
            b.append(y)
    assert ints(engine.debug_op("FE_MUL", a, b)) == [x * y % P for x, y in zip(a, b)]
    assert ints(engine.debug_op("FE_SQR", a)) == [x * x % P for x in a]
    assert ints(engine.debug_op("FE_ADD", a, b)) == [(x + y) % P for x, y in zip(a, b)]
    assert ints(engine.debug_op("FE_SUB", a, b)) == [(x - y) % P for x, y in zip(a, b)]


def test_fe_inv_sqrt(engine):
    rnd = random.Random(22)
    a = EDGE + [rnd.getrandbits(256) for _ in range(500)]
    assert ints(engine.debug_op("FE_INV", a)) == [pow(x % P, -1, P) if x % P else 0 for x in a]
    assert ints(engine.debug_op("FE_SQRT", a)) == [pow(x % P, (P + 1) // 4, P) for x in a]


def test_scalar_ops(engine):
    rnd = random.Random(23)
    a = EDGE + [rnd.getrandbits(256) for _ in range(1000)]
    b = [rnd.choice(EDGE) if i % 5 == 0 else rnd.getrandbits(256) for i in range(len(a))]
    assert ints(engine.debug_op("SC_MUL", a, b)) == [x * y % N for x, y in zip(a, b)]
    a = a[:300]
    assert ints(engine.debug_op("SC_INV", a)) == [pow(x % N, -1, N) if x % N else 0 for x in a]


def test_glv(engine):
    rnd = random.Random(24)
    ks = [0, 1, 2, N - 1, N - 2, LAM, N - LAM, (N + 1) // 2, N // 2, 2**128, 2**128 - 1, 2**255] + [rnd.getrandbits(256) % N for _ in range(4000)]
    for k, o in zip(ks, engine.debug_op("GLV", ks, out_stride=64)):
        k1 = int.from_bytes(o[0:20], "little") * (-1 if o[20] else 1)
        k2 = int.from_bytes(o[24:44], "little") * (-1 if o[44] else 1)
        assert (k1 + k2 * LAM) % N == k and abs(k1) < 2**129 and abs(k2) < 2**129


def test_ecmult(engine):
    rnd = random.Random(25)
    G = ec.G
    pts, a, b = [], [], []
    base = [ec.point_mul(12345, G), G, ec.point_neg(G), ec.point_mul(2, G), ec.point_mul(LAM, G), ec.point_mul(N - LAM, G),
            ec.point_mul(8, G), ec.point_mul(N - 8, G)]
    special = [(0, 0), (1, 0), (0, 1), (2, 0), (0, 2), (N - 1, 0), (0, N - 1), (1, N - 1), (5, 7), (N - 1, N - 1), (LAM, 0), (0, LAM),
               (N - LAM, LAM), (1, 1), (2, N - 1), (N - 2, 1), (8, 1), (8, N - 1), (3, 5), (LAM, 1), (1, LAM), (7, 1), (16, N - 2)]
    for p in base:
        for x, y in special + [(rnd.getrandbits(256) % N, rnd.getrandbits(256) % N) for _ in range(6)]:
            pts.append(p)
            a.append(x)
            b.append(y)
    out = engine.debug_op("ECMULT", a, b, [p[0].to_bytes(32, "big") + p[1].to_bytes(32, "big") for p in pts], out_stride=64)
    for p, x, y, o in zip(pts, a, b, out):
        want = co.ecmult2(x, y, p[0].to_bytes(32, "big") + p[1].to_bytes(32, "big"))
        assert o == (want or bytes(64)), (x, y)


def test_combined_generator_table_entries(engine):
    """Entries of the device-built generator comb tables against the oracle's scalar multiplication, at EVERY comb position p
    (position 0 = the combined table d1*G + d2*lambda*G of the window loop; positions 1..16 feed the split kernels' u1*G and the
    known-key walk): entry (d1, d2) of position p = (d1 + d2*lambda) * 2^(wc*p) * G, edge digits and random ones."""
    wc, n = engine.combined_table_info()
    if wc == 0:
        pytest.skip("library built without a combined generator table")
    half, d2n = 1 << (wc - 1), (1 << wc) + 1
    assert n == (half + 1) * d2n
    positions = -(-132 // wc)  # comb positions covering the 132 window bits
    rnd = random.Random(26)
    edges = [(d1, d2) for d1 in (0, 1, 2, half - 1, half) for d2 in (-half, -half + 1, -1, 0, 1, half - 1, half)]
    for p in range(positions):
        picks = edges + [(rnd.randint(0, half), rnd.randint(-half, half)) for _ in range(50)]
        for d1, d2 in picks:
            e = engine.combined_table_entries(p * n + d1 * d2n + d2 + half, 1)[0]
            if (d1, d2) == (0, 0):
                assert not e.any(), p                                     # infinity: zeros, never looked up
                continue
            x = sum(int(e[i]) << (32 * i) for i in range(8))
            y = sum(int(e[8 + i]) << (32 * i) for i in range(8))
            want = co.ecmult2((d1 + d2 * LAM) * (1 << (wc * p)) % N, 0, None)
            assert (x.to_bytes(32, "big") + y.to_bytes(32, "big")) == want, (p, d1, d2)
    with pytest.raises(Exception):
        engine.combined_table_entries(positions * n - 1, 2)             # one past the last position
