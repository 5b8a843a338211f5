"""The arithmetic edge sweep of tests/arith_edges.py through the host emulation (the portable path of the very csrc headers),
one operand set per emul_debug_op call, and the coverage of that sweep on the value-level models."""
import ctypes
import random

import adversarial as A
import arith_edges as AE
from oracle import secp256k1 as ec

OPS = {"FE_INV": 3, "SC_INV": 6, "SC_MUL": 5}
OPS.update({k: 11 + i for i, k in enumerate(("FE_MUL_RAW", "FE_SQR_RAW", "FE_ADD_RAW", "FE_SUB_RAW", "FE_NORMALIZE", "FE_EQUAL", "FE_SQRN",
                                             "FE_SQRT_INV", "SC_ADD", "SC_NEG", "SC_REDUCE_ONCE", "SC_DIGITS"))})


def emul_runner(E):
    def run(op, a, b, stride):
        out = (ctypes.c_uint8 * stride)()
        res = []
        for x, y in zip(a, b):
            rc = E.emul_debug_op(OPS[op], x.to_bytes(32, "big"), y.to_bytes(32, "big"), None, out)
            assert rc == 0, op
            res.append(bytes(out))
        return res
    return run


def test_ids_match_the_python_binding():
    """the op ids of include/ibft_verify.h as the emulation and engine.DBG know them"""
    from importlib import import_module
    assert {k: import_module("go-ibft_b200.engine").DBG[k] for k in OPS} == OPS


def test_sweeps_cover_the_boundaries():
    """every named branch is taken by the sweep, as often as stated (value-level models of the routines)"""
    cov = AE.coverage()
    low = {k: (cov.get(k, 0), n) for k, n in AE.required().items() if cov.get(k, 0) < n}
    assert not low, low
    assert AE.SC_FOLD4_MAX_A2 == 1
    sg = AE.safegcd_edges()
    assert sg["candidates"] >= 100_000
    for tag, m in (("p", AE.P), ("n", AE.N)):
        assert all(AE.safegcd_model(int(x, 16), m)[0] == sg[tag]["batches"] for x in sg[tag]["most_batches"])
        assert all(AE.safegcd_model(int(x, 16), m)[1] == -1 for x in sg[tag]["f_negative"])


def test_fold4_signatures_in_recover_vectors():
    """at least 4 signatures drive u2 = s r^-1 and 4 drive u1 = -z r^-1 through sc_reduce512's fold 4; they are valid"""
    u1 = u2 = 0
    for v in A.recover_vectors():
        r, s, z = (int.from_bytes(x, "big") for x in (v.sig[:32], v.sig[32:64], v.digest))
        rinv = pow(r, -1, AE.N)
        u2 += AE.sc_reduce512_stages(s * rinv)[1]
        u1 += AE.sc_reduce512_stages(z % AE.N * rinv)[1]
        if "fold4" in v.tag:
            assert v.key is not None, v.tag
    assert u2 >= 4 and u1 >= 4, (u1, u2)


def test_models_restate_the_contracts():
    """the raw models are weakly reduced representatives of the exact results"""
    rnd = random.Random(1)
    for c in AE.sweep_cases()[::7]:
        if c.op in ("FE_MUL_RAW", "FE_SQR_RAW", "FE_ADD_RAW", "FE_SUB_RAW", "FE_SQRN"):
            want = {"FE_MUL_RAW": lambda: c.a * c.b, "FE_SQR_RAW": lambda: c.a * c.a, "FE_ADD_RAW": lambda: c.a + c.b,
                    "FE_SUB_RAW": lambda: c.a - c.b, "FE_SQRN": lambda: pow(c.a, 1 << c.b, AE.P)}[c.op]()
            got = AE.expected(c)
            assert 0 <= got < AE.M and got % AE.P == want % AE.P, c
    for _ in range(200):
        k = rnd.randrange(AE.N)
        k1, k2 = AE.glv_model(k)
        assert (k1 + k2 * AE.LAM - k) % AE.N == 0 and max(abs(k1), abs(k2)) < 2**129
        for w, cnt in ((4, 33), (8, 17)):
            assert sum(d << (w * j) for j, d in enumerate(AE.booth_digits(abs(k1), w, cnt))) == abs(k1)
    for c, V in AE.sqrt_inv_cases(rnd):
        y, w = AE.sqrt_inv_model(c, V)
        if AE.is_residue(c) and V % AE.P:
            assert y * y % AE.P == c % AE.P and w * y * V % AE.P == 1
    assert ec.P == AE.P


def test_arith_edge_sweep(emul):
    bad = AE.check_sweep(emul_runner(emul))
    assert not bad, "\n".join(bad)


def test_chained_raw_sequences(emul):
    bad = AE.check_chains(emul_runner(emul), lanes=16, steps=1500)
    assert not bad, "\n".join(bad)
