"""The one-thread recovery with u1 G from the wide generator comb (secp_ec.cuh ecmult_gen_wide) on the host emulation.

tests/emul/recover_wide.cpp runs recover_key's composition with the comb entries m 2^(22 p) G computed on demand: crafted u1
values (zero, one, n - 1, the window values around 2^21 and 2^22 - 1 at every position, Booth carries through every window, the
top digit at its maximum) against the big-integer oracle, every crafted recover vector of tests/adversarial.py, the config-2
fixture against the table-inversion composition, and what tools/fma_budget.py charges for the comb."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from oracle import coracle as co
from oracle import secp256k1 as ec

import adversarial as A
import wide_edges as WE

HERE = os.path.dirname(os.path.abspath(__file__))
EMUL = os.path.join(HERE, "emul")
N = ec.N
REC_B_INF = 2  # IBFT_BR_REC_B_INF in emul_rec_branch_counts order
OPS = ["mul_body", "sqr_body", "mul_call", "sqr_call", "sqrn_call", "sqrn_iter", "dbl_front", "fe_inv", "sc_inv", "inv_iter",
       "win", "win_dbl", "win_add", "comb_add", "rec_final"]  # IBFT_OP_* of secp_fe.cuh


@pytest.fixture(scope="module")
def wide(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_wide") / "libibft_recover_wide.so")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-fPIC", "-std=c++17", "-Wall", "-Wextra", "-Wno-unknown-pragmas",
                           '-DEMUL_DIR="%s"' % EMUL, "-shared", "-o", so, os.path.join(EMUL, "recover_wide.cpp"), "-lpthread"])
    lib = ctypes.CDLL(so)
    lib.emul_wide_reads.restype = ctypes.c_ulonglong
    return lib


def run(E, item, arena=None):
    a = arena if arena is not None else np.zeros(1, np.uint8)
    out = (ctypes.c_uint8 * 20)()
    rc = E.emul_verify_item_wide(item.ctypes.data_as(ctypes.c_void_p), a.ctypes.data_as(ctypes.c_void_p),
                                 ctypes.c_size_t(len(a) if arena is not None else 0), out)
    return rc, bytes(out)


def test_shape(wide):
    s = (ctypes.c_uint32 * 4)()
    wide.emul_wide_shape(s)
    assert list(s) == [WE.W, WE.POSITIONS, 1 << (WE.W - 1), (1 << WE.TOP_BITS) + 1]


def test_digits_of_crafted_u1(wide):
    """the digits the device takes from u1 sum back to u1, stay within +-2^21, and the top one is never negative nor above 2^14"""
    out = (ctypes.c_int32 * WE.POSITIONS)()
    tops = set()
    for tag, u1 in WE.u1_values():
        wide.emul_wide_digits((ctypes.c_uint32 * 8)(*[(u1 >> (32 * i)) & 0xFFFFFFFF for i in range(8)]), out)
        d = list(out)
        assert d == WE.booth_digits(u1), tag
        assert sum(x << (WE.W * j) for j, x in enumerate(d)) == u1, tag
        assert all(abs(x) <= 1 << (WE.W - 1) for x in d) and 0 <= d[-1] <= 1 << WE.TOP_BITS, tag
        tops.add(d[-1])
    assert 1 << WE.TOP_BITS in tops                                     # n - 1
    assert WE.booth_digits((1 << 242) - 1) == [-1] + [0] * 10 + [1]     # the carry ripples through every window


@pytest.mark.parametrize("pos,m", [(0, 1), (0, 2), (0, 1 << 21), (5, 12345), (10, (1 << 21) - 1), (10, 1 << 21), (11, 1),
                                   (11, 1 << 14), (11, (1 << 14) + 1)])
def test_entries_against_oracle(wide, pos, m):
    e = (ctypes.c_uint32 * 16)()
    wide.emul_wide_entry(pos, m, e)
    x, y = ec.point_mul(m * (1 << (WE.W * pos)) % N, ec.G)
    words = list(e)
    assert sum(w << (32 * i) for i, w in enumerate(words[:8])) == x
    assert sum(w << (32 * i) for i, w in enumerate(words[8:])) == y


def test_crafted_u1_against_oracle(wide):
    """every crafted u1 on two nonce points, both s forms: the oracle's verdict and address; u1 = 0 takes the B = infinity branch,
    and each recovery reads one entry per non-zero digit"""
    wide.emul_branch_reset()
    wide.emul_wide_reads()
    vecs = WE.vectors()
    reads = 0
    for v in vecs:
        assert run(wide, A.recover_items([v])) == (int(v.verdict), v.addr or bytes(20)), v.tag
        reads += sum(d != 0 for d in WE.booth_digits(v.u[0]))
    assert all(v.verdict for v in vecs)
    assert wide.emul_wide_reads() == reads
    c = (ctypes.c_ulonglong * 4)()
    wide.emul_rec_branch_counts(c)
    assert c[REC_B_INF] == sum(1 for v in vecs if v.u[0] == 0) >= 4


def test_adversarial_recover_vectors(wide):
    for v in A.recover_vectors():
        assert run(wide, A.recover_items([v])) == (int(v.verdict), v.addr or bytes(20)), v.tag


def test_config2_slice_matches_table_inversion_composition(wide, emul):
    d = np.load(os.path.join(HERE, "golden", "config2.npz"))
    items = np.ascontiguousarray(d["items"]).view(co.ITEM_DTYPE).reshape(-1)
    arena = np.ascontiguousarray(d["arena"])
    out = (ctypes.c_uint8 * 20)()
    for i in range(0, len(items), 13):
        it = items[i:i + 1]
        rc = emul.emul_verify_item(it.ctypes.data_as(ctypes.c_void_p), arena.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(len(arena)), out)
        assert run(wide, it, arena) == (rc, bytes(out)), i


def test_operation_counts(wide):
    """per recovery: at most 12 comb additions (17 with the per-position comb), the rest as before"""
    d = np.load(os.path.join(HERE, "golden", "config3.npz"))
    items = np.ascontiguousarray(d["items"])
    arena = np.ascontiguousarray(d["arena"])
    wide.emul_op_reset()
    ok = [run(wide, items[i:i + 1], arena)[0] for i in range(30)]
    c = (ctypes.c_ulonglong * 32)()
    n = wide.emul_op_counts_all(c)
    ops = dict(zip(OPS, list(c)[:n]))
    rec = ops["rec_final"]
    assert rec >= sum(1 for r in ok if r == 1) and ops["win"] == 33 * rec
    assert ops["fe_inv"] == 0 and ops["sc_inv"] == rec
    assert 11 * rec <= ops["comb_add"] <= 12 * rec
