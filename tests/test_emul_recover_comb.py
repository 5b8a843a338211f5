"""The one-thread recovery without field inversions (verify_core.cuh, recover_key for exec_serial) on the host emulation.

k_recover walks u2 R on the isomorphic curve over an inversion-free table, adds u1 G by the per-position comb and takes y and
1 / Z from one exponentiation in the final addition.  tests/emul/recover_comb.cpp runs that composition on the host (the plain
emulation's emul_verify_item runs the table-inversion one): every crafted vector of tests/adversarial.py, non-abscissa r with
both recovery ids, random and corrupted signatures against the C oracle, the config-2 fixture against the other composition,
the branch counters of the final addition's rare cases, and the operation counts tools/fma_budget.py charges."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

from oracle import coracle as co
from oracle import secp256k1 as ec
from oracle.keccak import keccak256

import adversarial as A

HERE = os.path.dirname(os.path.abspath(__file__))
EMUL = os.path.join(HERE, "emul")
P, N = ec.P, ec.N
REC = dict(DBL=0, NEG=1, B_INF=2, NONRES=3)  # IBFT_BR_REC_* of secp_fe.cuh, in emul_rec_branch_counts order
OPS = ["mul_body", "sqr_body", "mul_call", "sqr_call", "sqrn_call", "sqrn_iter", "dbl_front", "fe_inv", "sc_inv", "inv_iter",
       "win", "win_dbl", "win_add", "comb_add", "rec_final"]  # IBFT_OP_* of secp_fe.cuh


@pytest.fixture(scope="module")
def comb(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_comb") / "libibft_recover_comb.so")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-fPIC", "-std=c++17", "-Wall", "-Wextra", "-Wno-unknown-pragmas",
                           '-DEMUL_DIR="%s"' % EMUL, "-shared", "-o", so, os.path.join(EMUL, "recover_comb.cpp"), "-lpthread"])
    return ctypes.CDLL(so)


def run(E, fn, item, arena=None):
    a = arena if arena is not None else np.zeros(1, np.uint8)
    out = (ctypes.c_uint8 * 20)()
    rc = getattr(E, fn)(item.ctypes.data_as(ctypes.c_void_p), a.ctypes.data_as(ctypes.c_void_p),
                        ctypes.c_size_t(len(a) if arena is not None else 0), out)
    return rc, bytes(out)


def rec_counts(E):
    c = (ctypes.c_ulonglong * 4)()
    assert E.emul_rec_branch_counts(c) == 4
    return list(c)


def non_abscissas(count, seed):
    """r < n with r^3 + 7 a non-residue mod p: no point of the curve has this abscissa"""
    rnd = random.Random(seed)
    out = []
    while len(out) < count:
        r = rnd.randrange(1, N)
        if pow((r ** 3 + 7) % P, (P - 1) // 2, P) == P - 1:
            out.append(r)
    return out


def test_crafted_vectors_and_every_rare_branch(comb):
    """every crafted vector gives the oracle's verdict and address; A = B, A = -B (the "final-add" vectors), u1 = 0 (z = 0 and
    z = n) and a non-residue r^3 + 7 (both recovery ids) each reach their branch of the final addition"""
    import workloads as wl
    comb.emul_branch_reset()
    vecs = A.recover_vectors()
    for v in vecs:
        assert run(comb, "emul_verify_item_comb", A.recover_items([v])) == (int(v.key is not None), v.addr or bytes(20)), v.tag
    c = rec_counts(comb)
    assert c[REC["DBL"]] >= 1 and c[REC["NEG"]] >= 1 and c[REC["B_INF"]] >= 8, c
    assert c[REC["NONRES"]] == 0, c
    rnd = random.Random(11)
    for r in non_abscissas(6, 12):
        for v in (0, 1):
            sig = r.to_bytes(32, "big") + rnd.randrange(1, N).to_bytes(32, "big") + bytes([v])
            dig = rnd.randbytes(32)
            assert co.ecrecover_address(dig, sig) is None
            assert run(comb, "emul_verify_item_comb", wl.make_item(sig, bytes(20), 0, dig)) == (0, bytes(20))
    assert rec_counts(comb)[REC["NONRES"]] == 12


def test_random_and_corrupted_signatures_both_parities(comb):
    import workloads as wl
    rnd = random.Random(13)
    parities = set()
    for i in range(40):
        d = rnd.randrange(1, N)
        dig = keccak256(bytes([i, 7]))
        sig = wl.sign(d, dig, low_s=bool(i & 1))
        parities.add(sig[64])
        addr = co.ecrecover_address(dig, sig)
        assert run(comb, "emul_verify_item_comb", wl.make_item(sig, addr, 0, dig)) == (1, addr)
        bad = bytearray(sig)
        bad[rnd.randrange(64)] ^= 1 << rnd.randrange(8)
        exp = co.ecrecover_address(dig, bytes(bad))
        assert run(comb, "emul_verify_item_comb", wl.make_item(bytes(bad), addr, 0, dig)) == (int(exp == addr), exp or bytes(20))
    assert parities == {0, 1}


def test_config2_slice_matches_table_inversion_composition(comb, emul):
    d = np.load(os.path.join(HERE, "golden", "config2.npz"))
    items = np.ascontiguousarray(d["items"]).view(co.ITEM_DTYPE).reshape(-1)
    arena = np.ascontiguousarray(d["arena"])
    for i in range(0, len(items), 11):
        assert run(comb, "emul_verify_item_comb", items[i:i + 1], arena) == run(emul, "emul_verify_item", items[i:i + 1], arena), i


def test_operation_counts_without_field_inversion(comb):
    """per recovery: 33 windows of the R streams only, one doubling in the table, at most 17 comb additions, one final step,
    one scalar inversion and no field inversion (what tools/fma_budget.py charges)"""
    d = np.load(os.path.join(HERE, "golden", "config3.npz"))
    items = np.ascontiguousarray(d["items"]).view(co.ITEM_DTYPE).reshape(-1)
    arena = np.ascontiguousarray(d["arena"])
    comb.emul_op_reset()
    ok = [run(comb, "emul_verify_item_comb", items[i:i + 1], arena)[0] for i in range(30)]
    c = (ctypes.c_ulonglong * 32)()
    n = comb.emul_op_counts_all(c)
    ops = dict(zip(OPS, list(c)[:n]))
    assert n == len(OPS)
    rec = ops["rec_final"]
    assert rec >= sum(1 for r in ok if r == 1) and ops["win"] == 33 * rec
    assert ops["fe_inv"] == 0 and ops["sc_inv"] == rec
    assert rec <= ops["comb_add"] <= 17 * rec
    assert ops["win_add"] <= 66 * rec
    assert ops["dbl_front"] == ops["win_dbl"] + rec  # 2 R of the table; no P + P on these items
    assert ops["sqr_body"] == ops["sqr_call"] + ops["sqrn_iter"] + 3 * ops["dbl_front"]
    assert ops["mul_body"] == ops["mul_call"]
