"""The RFC 6979 signer (ibft_sign_batch_rfc6979) through the host emulation of the very csrc headers: SHA-256 at every padding
edge, the DRBG's nonce candidates and the signer against the big-integer reference of rfc6979_rows.py, and that reference
against the published vectors and OpenSSL's deterministic ECDSA."""
import ctypes
import hashlib
import os
import random
import subprocess

import pytest

import rfc6979_rows as R
from oracle import secp256k1 as ec

N = ec.N
EMUL = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul")


@pytest.fixture(scope="module")
def emul_rfc(tmp_path_factory):
    """tests/emul/sign_rfc6979.cpp: the host emulation with the RFC 6979 signer's entry points"""
    so = str(tmp_path_factory.mktemp("emul_rfc6979") / "libibft_sign_rfc6979.so")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-fPIC", "-std=c++17", "-Wall", "-Wextra", "-Wno-unknown-pragmas",
                           '-DEMUL_DIR="%s"' % EMUL, "-shared", "-o", so, os.path.join(EMUL, "sign_rfc6979.cpp"), "-lpthread"])
    return ctypes.CDLL(so)


def _candidate(E, d: int, z: bytes, c: int) -> int:
    out = (ctypes.c_uint8 * 32)()
    E.emul_rfc6979_candidate(d.to_bytes(32, "big"), z, ctypes.c_uint32(c), out)
    return int.from_bytes(bytes(out), "big")


def _sign(E, d: int, z: bytes) -> bytes:
    out = (ctypes.c_uint8 * 65)()
    ok = E.emul_sign_rfc6979(d.to_bytes(32, "big"), z, out)
    assert ok in (0, 1)
    assert ok or bytes(out) == R.ZERO_SIG, "a refused row must leave 65 zero bytes"
    return bytes(out)


def test_sha256_every_length(emul_rfc):
    """0-200 bytes: the one- and two-block padding edges (55/56, 63/64, 119/120 bytes) and three-block messages"""
    rnd = random.Random(256)
    out = (ctypes.c_uint8 * 32)()
    for n in range(201):
        m = rnd.randbytes(n)
        emul_rfc.emul_sha256(m, ctypes.c_uint32(n), out)
        assert bytes(out) == hashlib.sha256(m).digest(), n


def test_candidates_random_pairs(emul_rfc):
    rnd = random.Random(6979)
    for _ in range(2000):
        d, z = rnd.getrandbits(256), rnd.randbytes(32)
        for c in range(4):
            assert _candidate(emul_rfc, d, z, c) == R.rfc6979_candidate(d, z, c), (hex(d), z.hex(), c)


def test_candidates_at_the_edges(emul_rfc):
    """the signer's key and digest edges, and the debug op's shared body (IBFT_DBG_RFC6979: candidate in the last byte of c)"""
    rows = R.edge_rows()
    assert len(rows) >= 80
    out = (ctypes.c_uint8 * 32)()
    for d, z in rows:
        for c in range(4):
            want = R.rfc6979_candidate(d, z, c)
            assert _candidate(emul_rfc, d, z, c) == want, (hex(d), z.hex(), c)
            assert emul_rfc.emul_debug_rfc6979(d.to_bytes(32, "big"), z, c.to_bytes(64, "big"), out) == 0
            assert int.from_bytes(bytes(out), "big") == want


def test_candidate_zero_is_the_published_nonce(emul_rfc):
    for v in R.golden_vectors():
        d, z = int(v["privkey"], 16), bytes.fromhex(v["digest"])
        assert "%064x" % _candidate(emul_rfc, d, z, 0) == v["k"], v["message"]
        assert "%064x" % R.rfc6979_candidate(d, z, 0) == v["k"]
        assert R.rfc6979_candidate(d, z, 0) == ec.rfc6979_k(d, z)


def test_signer_matches_reference_at_the_edges(emul_rfc):
    rows = R.edge_rows()
    for d, z in rows:
        assert _sign(emul_rfc, d, z) == (R.sign_libsecp(d, z) or R.ZERO_SIG), (hex(d), z.hex())


def test_refused_keys(emul_rfc):
    """a key of 0 or >= n is refused whatever the digest (ibft_sign_batch would sign with d mod n)"""
    for d in R.REFUSED_KEYS:
        for z in (bytes(32), b"\x01" * 32, bytes.fromhex(R.golden_vectors()[0]["digest"])):
            assert _sign(emul_rfc, d, z) == R.ZERO_SIG, hex(d)
            assert R.sign_libsecp(d, z) is None


def test_digest_reduced_mod_n(emul_rfc):
    """z and z + n seed the DRBG with the same bytes and sign identically"""
    rnd = random.Random(5)
    for z in [0, 1, 5, (1 << 256) - 1 - N] + [rnd.randrange((1 << 256) - N) for _ in range(20)]:
        d = rnd.randrange(1, N)
        a, b = z.to_bytes(32, "big"), (z + N).to_bytes(32, "big")
        assert _sign(emul_rfc, d, a) == _sign(emul_rfc, d, b) != R.ZERO_SIG
        assert _sign(emul_rfc, d, a) == R.sign_libsecp(d, a)


def test_fast_rows_equal_the_big_integer_reference():
    """the C oracle's k G that the GPU tests use for bulk rows gives sign_libsecp's own bytes"""
    ds, zs = R.random_rows(300, seed=11)
    assert R.want(ds, zs) == [R.sign_libsecp(d, z) or R.ZERO_SIG for d, z in zip(ds, zs)]


# ---- the reference
def test_reference_signs_the_published_vectors():
    for v in R.golden_vectors():
        d, z = int(v["privkey"], 16), bytes.fromhex(v["digest"])
        sig = R.sign_libsecp(d, z)
        assert (sig[:32].hex(), sig[32:64].hex(), sig[64]) == (v["r"], v["s"], v["v"]), v["message"]
        assert sig == ec.sign(d, z)


def test_reference_matches_openssl_deterministic_ecdsa():
    """OpenSSL's RFC 6979 ECDSA over the prehashed digest: the same r, and the same s once normalised to the low half"""
    cec = pytest.importorskip("cryptography.hazmat.primitives.asymmetric.ec")
    from cryptography.hazmat.primitives import hashes
    from cryptography.hazmat.primitives.asymmetric import utils
    try:
        algo = cec.ECDSA(utils.Prehashed(hashes.SHA256()), deterministic_signing=True)
    except TypeError:
        pytest.skip("this cryptography has no deterministic ECDSA")
    rnd = random.Random(200)
    for _ in range(200):
        d, z = rnd.randrange(1, N), rnd.randbytes(32)
        r, s = utils.decode_dss_signature(cec.derive_private_key(d, cec.SECP256K1()).sign(z, algo))
        sig = R.sign_libsecp(d, z)
        assert int.from_bytes(sig[:32], "big") == r
        assert int.from_bytes(sig[32:64], "big") == min(s, N - s)
