"""The fused linear combinations of the group law (secp_fe.cuh) on the host emulation -- the portable branch the device's PTX
branch mirrors -- against big integers, at the carry and borrow edges of tests/fused_edges.py."""
import ctypes
import os
import subprocess

import pytest

import fused_edges as FE

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def emul_fused(tmp_path_factory):
    emul = os.path.join(HERE, "emul")
    so = str(tmp_path_factory.mktemp("emul_fused") / "libibft_fused.so")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-fPIC", "-std=c++17", "-Wall", "-Wextra", "-Wno-unknown-pragmas",
                           '-DEMUL_DIR="%s"' % emul, "-shared", "-o", so, os.path.join(emul, "fused_driver.cpp"), "-lpthread"])
    lib = ctypes.CDLL(so)
    lib.emul_fe_fused.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_char_p]
    return lib


def test_cases_reach_every_top_and_second_fold():
    cov = FE.coverage(FE.cases())
    for sel, need in FE.required_coverage().items():
        assert need <= cov[sel], (FE.OPS[sel][0], sorted(need - cov[sel]))


def test_fused_ops_match_big_integers(emul_fused):
    cs = FE.cases()
    res = []
    for sel, a, b, c in cs:
        out = ctypes.create_string_buffer(32)
        assert emul_fused.emul_fe_fused(a.to_bytes(32, "big"), b.to_bytes(32, "big"), FE.c_operand(sel, c), out) == 0
        res.append(out.raw)
    bad = FE.check(res, cs)
    assert not bad, "\n".join(bad[:20])


def test_unknown_selector_is_refused(emul_fused):
    out = ctypes.create_string_buffer(32)
    assert emul_fused.emul_fe_fused(bytes(32), bytes(32), FE.c_operand(7, 0), out) == -1
