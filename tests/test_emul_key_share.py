"""The check a device of a multi-device engine makes before it adopts a key another device learned: key_matches_address of the
csrc headers (the body k_adopt_peer_keys runs, through the host emulation tests/emul/key_share_driver.cpp) against the
big-integer oracle.  A key may enter a registry entry only when both coordinates are fully reduced, the point is on the curve
and its address is the entry's address."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import adversarial as A
import workloads as wl
from oracle import coracle as co
from oracle import secp256k1 as ec

HERE = os.path.dirname(os.path.abspath(__file__))
P = ec.P
CONFIG3_SAMPLE = 48


def raw_address(x: int, y: int) -> bytes:
    return co.keccak256(x.to_bytes(32, "big") + y.to_bytes(32, "big"))[12:]


def oracle_accepts(x: int, y: int, addr: bytes) -> bool:
    return x < P and y < P and (y * y - x * x * x - 7) % P == 0 and raw_address(x, y) == addr


def key_check_cases():
    """(tag, x, y, addr20): the accepts and refusals the check is specified by.  x and y may be >= p (they are 256-bit values)."""
    d = np.load(os.path.join(HERE, "golden", "config3.npz"))
    addrs = [bytes(a) for a in d["addrs"]]
    config3 = [(int(i), ec.privkey_to_pubkey(wl.privkey(2, int(i)))) for i in np.linspace(0, len(addrs) - 1, CONFIG3_SAMPLE).astype(int)]
    edge = list(A.known_points())
    cases = []
    for i, Q in config3:
        assert ec.pubkey_to_address(Q) == addrs[i]
        cases.append((f"config3 key {i}", Q[0], Q[1], addrs[i]))
    for k, Q in enumerate(edge):
        cases.append((f"edge key {k}", Q[0], Q[1], ec.pubkey_to_address(Q)))
    for j, (tag, x, y, a) in enumerate(list(cases)):
        bit = (j * 13) % 160
        flipped = bytearray(a)
        flipped[bit // 8] ^= 1 << (bit % 8)
        cases.append((f"{tag}, address bit {bit} flipped", x, y, bytes(flipped)))
        cases.append((f"{tag}, y + 1 (off the curve)", x, (y + 1) % P, a))
        other = cases[(j + 1) % len(config3 + edge)]
        cases.append((f"{tag}, address of {other[0]}", x, y, other[3]))
        if x + P < 1 << 256:
            cases.append((f"{tag}, x + p", x + P, y, a))
        if y + P < 1 << 256:
            cases.append((f"{tag}, y + p", x, y + P, a))
    cases.append(("(0, 0)", 0, 0, raw_address(0, 0)))
    cases.append(("(0, 0), zero address", 0, 0, bytes(20)))
    cases.append(("(p, 0)", P, 0, raw_address(0, 0)))
    return cases


@pytest.fixture(scope="module")
def emul_key_share(tmp_path_factory):
    emul = os.path.join(HERE, "emul")
    so = str(tmp_path_factory.mktemp("emul_key_share") / "libibft_key_share.so")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-fPIC", "-std=c++17", "-Wall", "-Wextra", "-Wno-unknown-pragmas",
                           '-DEMUL_DIR="%s"' % emul, "-shared", "-o", so, os.path.join(emul, "key_share_driver.cpp"), "-lpthread"])
    lib = ctypes.CDLL(so)
    lib.emul_key_matches_address.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_char_p]
    return lib


def test_cases_cover_every_kind():
    cases = key_check_cases()
    tags = " | ".join(t for t, *_ in cases)
    for kind in ("config3 key", "edge key", "flipped", "off the curve", "address of", "x + p", "y + p", "(0, 0)"):
        assert kind in tags, kind
    accepts = [oracle_accepts(x, y, a) for _, x, y, a in cases]
    # every key with its own address is accepted, every altered one refused
    for (tag, *_), ok in zip(cases, accepts):
        assert ok == (tag.startswith(("config3 key", "edge key")) and "," not in tag), tag
    # the unreduced forms exist for keys of both coordinate families (small x, small y)
    assert sum("x + p" in t for t, *_ in cases) >= 6 and sum("y + p" in t for t, *_ in cases) >= 6


def test_key_matches_address_against_oracle(emul_key_share):
    for tag, x, y, a in key_check_cases():
        got = emul_key_share.emul_key_matches_address(x.to_bytes(32, "big"), y.to_bytes(32, "big"), a)
        assert got == int(oracle_accepts(x, y, a)), tag
