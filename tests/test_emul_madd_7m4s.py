"""The opt-in 7M + 4S mixed addition (-DIBFT_MADD_7M4S, madd-2007-bl) and the emulation's operation counters.

The product build keeps the 8M + 3S addition (faster on an H100, DESIGN.md §3.1); the 7M + 4S formula stays in the tree as a
measured alternative, so its results are checked here on the host emulation built with the flag: the crafted exceptional-case
vectors on the one-thread and split pipelines (the split chain uses the addition's Z3 / Z1 ratio, 2H in this formula) and a
slice of the config-2 fixture.  Also the operation counters of the emulation (tests/emul/opcount.cpp) that tools/fma_budget.py
reads."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from oracle import coracle as co

import adversarial as A

HERE = os.path.dirname(os.path.abspath(__file__))
EMUL = os.path.join(HERE, "emul")


@pytest.fixture(scope="module")
def emul_7m4s(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_7m4s") / "libibft_emul_7m4s.so")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-fPIC", "-std=c++17", "-Wall", "-Wextra", "-Wno-unknown-pragmas",
                           "-DIBFT_MADD_7M4S", '-DEMUL_DIR="%s"' % EMUL, "-shared", "-o", so, os.path.join(EMUL, "emul.cpp"),
                           "-lpthread"])
    return ctypes.CDLL(so)


def run(E, fn, item, arena=None):
    a = arena if arena is not None else np.zeros(1, np.uint8)
    out = (ctypes.c_uint8 * 20)()
    rc = getattr(E, fn)(item.ctypes.data_as(ctypes.c_void_p), a.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(len(a) if arena is not None else 0), out)
    return rc, bytes(out)


@pytest.mark.parametrize("fn", ["emul_verify_item", "emul_verify_item_split"])
def test_crafted_vectors_with_7m4s_addition(emul_7m4s, fn):
    emul_7m4s.emul_branch_reset()
    for v in A.recover_vectors():
        assert run(emul_7m4s, fn, A.recover_items([v])) == (int(v.key is not None), v.addr or bytes(20)), v.tag
    c = (ctypes.c_ulonglong * 12)()
    emul_7m4s.emul_branch_counts(c)
    assert c[0] >= 1 and c[1] >= 1 and c[2] >= 1, list(c)  # P + P, P - P, accumulator at infinity


def test_config2_slice_with_7m4s_addition(emul_7m4s, emul):
    d = np.load(os.path.join(HERE, "golden", "config2.npz"))
    items = np.ascontiguousarray(d["items"]).view(co.ITEM_DTYPE).reshape(-1)
    arena = np.ascontiguousarray(d["arena"])
    for i in range(0, len(items), 7):
        for fn in ("emul_verify_item", "emul_verify_item_split"):
            assert run(emul_7m4s, fn, items[i:i + 1], arena) == run(emul, fn, items[i:i + 1], arena), (fn, i)


@pytest.fixture(scope="module")
def emul_opcount(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_opcount") / "libibft_opcount.so")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-fPIC", "-std=c++17", '-DEMUL_DIR="%s"' % EMUL, "-shared", "-o", so,
                           os.path.join(EMUL, "opcount.cpp"), "-lpthread"])
    return ctypes.CDLL(so)


def test_operation_counters(emul_opcount):
    """IBFT_OPCOUNT (read by tools/fma_budget.py): one recovery runs 33 windows, one doubling front per doubling, and every
    product is a multiplier or a squarer body"""
    d = np.load(os.path.join(HERE, "golden", "config2.npz"))
    items = np.ascontiguousarray(d["items"]).view(co.ITEM_DTYPE).reshape(-1)
    arena = np.ascontiguousarray(d["arena"])
    run(emul_opcount, "emul_verify_item", items[0:1], arena)
    emul_opcount.emul_op_reset()
    ok = [run(emul_opcount, "emul_verify_item", items[i:i + 1], arena)[0] for i in range(0, 40)]
    c = (ctypes.c_ulonglong * 32)()
    n = emul_opcount.emul_op_counts(c)
    ops = dict(zip(["mul_body", "sqr_body", "mul_call", "sqr_call", "sqrn_call", "sqrn_iter", "dbl_front", "fe_inv", "sc_inv",
                    "inv_iter", "win", "win_dbl", "win_add"], list(c)[:n]))
    assert n == 13 and ops["win"] % 33 == 0 and ops["win"] // 33 >= sum(1 for r in ok if r == 1)
    # doublings: the window loop's, four per table {1..8} R, and a P + P now and then
    assert ops["dbl_front"] >= ops["win_dbl"] + 4 * (ops["win"] // 33)
    assert ops["sqr_body"] == ops["sqr_call"] + ops["sqrn_iter"] + 3 * ops["dbl_front"]
    assert ops["mul_body"] == ops["mul_call"]
