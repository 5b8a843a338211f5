"""The negated-lambda-digit vectors of tests/neg_lambda.py on the host emulation: the GLV split and Booth digits put a negated
entry into every non-zero window of the lambda stream, and both one-thread compositions -- u1 G by the wide comb and by the
per-position comb -- recover the oracle's address (zero when there is none)."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import adversarial as A
import neg_lambda as NL

EMUL = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul")


def build(tmp_path_factory, src):
    so = str(tmp_path_factory.mktemp("emul_neg_lambda") / (src + ".so"))
    subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-fPIC", "-std=c++17", "-Wall", "-Wextra", "-Wno-unknown-pragmas",
                           '-DEMUL_DIR="%s"' % EMUL, "-shared", "-o", so, os.path.join(EMUL, src), "-lpthread"])
    return ctypes.CDLL(so)


@pytest.fixture(scope="module", params=[("recover_wide.cpp", "emul_verify_item_wide"), ("recover_comb.cpp", "emul_verify_item_comb")])
def composition(request, tmp_path_factory):
    src, fn = request.param
    return getattr(build(tmp_path_factory, src), fn)


def test_every_lambda_window_is_negated(emul):
    for v in NL.vectors():
        u2 = v.u[1] % A.N
        out = (ctypes.c_uint8 * 256)()
        assert emul.emul_debug_op(22, u2.to_bytes(32, "big"), bytes(32), None, out) == 0  # IBFT_DBG_SC_DIGITS
        rec = bytes(out)[128:256]  # the second half: the lambda stream
        neg, nz = NL.negated_windows(rec, rec[24] == 1)
        # every non-zero window but the top +1 digit of 0x99..9 and 0xDD..D
        assert len(neg) >= 31 and neg == [j for j in nz if j < nz[-1] or j in neg], (v.tag, nz, neg)
        assert len(nz) - len(neg) <= 1 and (len(neg) == len(nz) or nz[-1] not in neg), (v.tag, nz, neg)


def test_vectors_recover_on_both_compositions(composition):
    zero = np.zeros(1, np.uint8)
    for v in NL.vectors():
        item = A.recover_items([v])
        out = (ctypes.c_uint8 * 20)()
        rc = composition(item.ctypes.data_as(ctypes.c_void_p), zero.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(0), out)
        assert (rc, bytes(out)) == (int(v.verdict), v.addr or bytes(20)), v.tag
