"""Key sharing between engines of separate processes: the export selection and the adoption decision of k_key_export /
k_key_adopt (key_share.cuh, through the host emulation tests/emul/key_share_sync_driver.cpp) against a big-integer model.

The model: an export takes the entries whose key is known (LEARNED, READY, EVICTED) and not yet exported or adopted, in
ascending entry order, at most IBFT_KEY_SHARE_RECORDS; the rest go at the next export.  An adoption finds a record's entry by
its address in the resident tables, drops it when no table lists the address, refuses a key that is not reduced, not on the
curve or not the address's key, and writes a valid key into an unknown entry, which is then never exported."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import adversarial as A
import workloads as wl
from oracle import secp256k1 as ec
from test_emul_key_share import oracle_accepts

HERE = os.path.dirname(os.path.abspath(__file__))
P = ec.P
C = 1024
REC = 21
WORDS = 21568
UNKNOWN, LEARNED, READY, BUILDING, EVICTED = 0, 1, 2, 3, 4
DROP, REFUSE, KNOWN, ADOPT = 0, 1, 2, 3
N_KEYS = 24


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    emul = os.path.join(HERE, "emul")
    so = str(tmp_path_factory.mktemp("emul_key_share_sync") / "libibft_key_share_sync.so")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-fPIC", "-std=c++17", "-Wall", "-Wextra", "-Wno-unknown-pragmas",
                           '-DEMUL_DIR="%s"' % emul, "-shared", "-o", so, os.path.join(emul, "key_share_sync_driver.cpp"), "-lpthread"])
    lib = ctypes.CDLL(so)
    p = ctypes.c_void_p
    lib.emul_key_share_export.restype = ctypes.c_uint32
    lib.emul_key_share_export.argtypes = [p, p, p, p, ctypes.c_uint32, p]
    lib.emul_key_share_adopt.argtypes = [p, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, p, p, p, ctypes.c_uint32, p, p, p, p, p, p]
    return lib


def ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def words_of(v: int) -> list[int]:
    return [(v >> (32 * i)) & 0xFFFFFFFF for i in range(8)]


@pytest.fixture(scope="module")
def keys():
    """N_KEYS real validators: (address, (x, y))"""
    d = np.load(os.path.join(HERE, "golden", "config3.npz"))
    out = []
    for i in range(N_KEYS):
        Q = ec.privkey_to_pubkey(wl.privkey(2, i))
        a = bytes(d["addrs"][i])
        assert ec.pubkey_to_address(Q) == a
        out.append((a, Q))
    return out


class Registry:
    """one engine's registry as the kernels see it, plus its resident tables (slot -> {address: entry})"""

    def __init__(self, n):
        self.state = np.zeros(n, np.uint32)
        self.shared = np.zeros(n, np.uint32)
        self.xy = np.zeros((n, 16), np.uint32)
        self.addr = np.zeros((n, 20), np.uint8)
        self.tables = []

    def put(self, r, a: bytes, Q=None, state=LEARNED):
        self.addr[r] = np.frombuffer(a, np.uint8)
        if Q is not None:
            self.xy[r] = words_of(Q[0]) + words_of(Q[1])
        self.state[r] = state if Q is not None else UNKNOWN

    def export(self, lib):
        want = [r for r in range(len(self.state)) if self.state[r] in (LEARNED, READY, EVICTED) and not self.shared[r]][:C]
        block = np.full(WORDS, 0xA5A5A5A5, np.uint32)
        n = lib.emul_key_share_export(ptr(self.state), ptr(self.shared), ptr(self.xy), ptr(self.addr), len(self.state), ptr(block))
        assert n == block[0] == len(want)
        for i, r in enumerate(want):
            rec = block[1 + REC * i: 1 + REC * (i + 1)]
            assert rec[:5].tobytes() == self.addr[r].tobytes()     # little-endian words: the bytes in order
            assert np.array_equal(rec[5:], self.xy[r])
            assert self.shared[r] == 1
        return block, want

    def adopt(self, lib, blocks, self_part):
        """run the emulation and the model on the same registry; returns the decisions and counts"""
        model_state, model_shared = self.state.copy(), self.shared.copy()
        model_xy = self.xy.copy()
        n_slots = len(self.tables)
        stride = max([len(t) for t in self.tables] + [1])
        tab_addr = np.zeros((max(n_slots, 1), stride, 20), np.uint8)
        tab_ref = np.zeros((max(n_slots, 1), stride), np.uint32)
        tab_n = np.zeros(max(n_slots, 1), np.uint32)
        for s, t in enumerate(self.tables):
            for j, a in enumerate(sorted(t)):
                tab_addr[s, j] = np.frombuffer(a, np.uint8)
                tab_ref[s, j] = t[a]
            tab_n[s] = len(t)
        blocks = np.ascontiguousarray(np.stack(blocks), np.uint32)
        counts = np.zeros(2, np.uint32)
        dec = np.zeros(len(blocks) * C, np.uint8)
        lib.emul_key_share_adopt(ptr(blocks), len(blocks), self_part, n_slots, ptr(tab_addr), ptr(tab_ref), ptr(tab_n), stride,
                                 ptr(self.state), ptr(self.xy), ptr(self.addr), ptr(self.shared), ptr(counts), ptr(dec))
        # the big-integer model
        want_dec, adopted, refused = np.full(len(blocks) * C, 0xFF, np.uint8), 0, 0
        for p, blk in enumerate(blocks):
            if p == self_part:
                continue
            if blk[0] > C:
                refused += 1
                continue
            for i in range(blk[0]):
                rec = blk[1 + REC * i: 1 + REC * (i + 1)]
                a = rec[:5].tobytes()
                r = next((t[a] for t in self.tables if a in t), None)
                x = sum(int(w) << (32 * k) for k, w in enumerate(rec[5:13]))
                y = sum(int(w) << (32 * k) for k, w in enumerate(rec[13:21]))
                if r is None:
                    d = DROP
                elif not oracle_accepts(x, y, self.addr[r].tobytes()):
                    d = REFUSE
                    refused += 1
                elif model_state[r] != UNKNOWN:
                    d = KNOWN
                else:
                    d = ADOPT
                    adopted += 1
                    model_state[r], model_shared[r] = LEARNED, 1
                    model_xy[r] = rec[5:]
                want_dec[p * C + i] = d
        assert np.array_equal(dec, want_dec)
        assert counts.tolist() == [adopted, refused]
        assert np.array_equal(self.state, model_state) and np.array_equal(self.shared, model_shared)
        assert np.array_equal(self.xy, model_xy)
        return dec.reshape(len(blocks), C), counts.tolist()


def fake_addr(r):
    return bytes([0xEE]) + r.to_bytes(19, "big")


def test_export_order_cap_and_carry_over(lib):
    """2,500 entries in every state: three exports take the exportable ones in ascending entry order, 1,024 at most each; the
    fourth finds nothing.  Entries learned between exports go at the next one, behind the carried-over ones."""
    rng = np.random.default_rng(7)
    n = 2500
    R = Registry(n)
    for r in range(n):
        st = int(rng.choice([UNKNOWN, LEARNED, READY, BUILDING, EVICTED], p=[0.1, 0.4, 0.3, 0.05, 0.15]))
        R.put(r, fake_addr(r), (int.from_bytes(rng.bytes(32), "big") % P, int.from_bytes(rng.bytes(32), "big") % P), st)
        R.state[r] = st
    exportable = [r for r in range(n) if R.state[r] in (LEARNED, READY, EVICTED)]
    assert len(exportable) > 2 * C
    _, first = R.export(lib)
    assert first == exportable[:C]
    late = [r for r in range(first[-1]) if R.state[r] == UNKNOWN][:5]   # learned below the first export's last entry
    for r in late:
        R.state[r] = LEARNED
    _, second = R.export(lib)
    assert second == sorted(late + exportable[C:])[:C] and late[0] in second
    _, third = R.export(lib)
    assert sorted(first + second + third) == sorted(exportable + late)
    assert R.export(lib)[1] == []


def test_no_echo_of_adopted_keys(lib, keys):
    """Rank A learned keys 0-9, rank B keys 5-14 (entries numbered differently).  B adopts A's 0-4, finds 5-9 known; its next
    export holds only the keys it learned itself, and A adopts exactly 10-14 from it."""
    A, B = Registry(N_KEYS), Registry(N_KEYS)
    for i, (a, Q) in enumerate(keys):
        A.put(i, a, Q if i < 10 else None)
        B.put(N_KEYS - 1 - i, a, Q if 5 <= i < 15 else None)
    A.tables = [{a: i for i, (a, _) in enumerate(keys)}]
    B.tables = [{a: N_KEYS - 1 - i for i, (a, _) in enumerate(keys)}]
    blk_a, _ = A.export(lib)
    blk_b, _ = B.export(lib)
    dec, counts = B.adopt(lib, [blk_a, blk_b], 1)
    assert counts == [5, 0] and dec[0][:10].tolist() == [ADOPT] * 5 + [KNOWN] * 5
    blk_b2, sent = B.export(lib)
    assert sent == []                                             # B exported 5-14 already, and adopted 0-4
    dec, counts = A.adopt(lib, [blk_a, blk_b], 0)
    assert counts == [5, 0]
    assert sorted(A.state.nonzero()[0].tolist()) == list(range(15))
    assert A.export(lib)[1] == []                                 # nothing goes back to B


def test_readdressed_entry(lib, keys):
    """An exported entry that ibft_set_validators gives to another address (k_key_share_forget, then k_adopt_entries): it is
    not exported while its new key is unknown, and then exported with the new address and key, never the old key."""
    (a0, Q0), (a1, Q1) = keys[0], keys[1]
    R = Registry(4)
    R.put(2, a0, Q0)
    assert R.export(lib)[1] == [2]
    R.shared[2], R.state[2] = 0, UNKNOWN                           # forget + reset on re-addressing
    R.addr[2] = np.frombuffer(a1, np.uint8)
    assert R.export(lib)[1] == []
    R.put(2, a1, Q1)                                                # learned by recovery
    blk, sent = R.export(lib)
    assert sent == [2]
    assert blk[1:6].tobytes() == a1 and np.array_equal(blk[6:22], np.array(words_of(Q1[0]) + words_of(Q1[1]), np.uint32))


def test_slots_and_unlisted_addresses(lib, keys):
    """A record whose address only the second resident table lists is adopted into that table's entry; one no table lists is
    dropped (neither adopted nor refused)."""
    src = Registry(N_KEYS)
    for i, (a, Q) in enumerate(keys):
        src.put(i, a, Q)
    blk, _ = src.export(lib)
    R = Registry(N_KEYS)
    for i, (a, _) in enumerate(keys):
        R.put(i, a)
    R.tables = [{keys[i][0]: i for i in range(0, 8)}, {keys[i][0]: i for i in range(4, 16)}]   # 16-23 unlisted
    dec, counts = R.adopt(lib, [np.zeros(WORDS, np.uint32), blk], 0)
    assert counts == [16, 0]
    assert dec[1][:N_KEYS].tolist() == [ADOPT] * 16 + [DROP] * 8
    assert R.state[:16].tolist() == [LEARNED] * 16 and not R.state[16:].any()


def forged_block(recs):
    blk = np.zeros(WORDS, np.uint32)
    blk[0] = len(recs)
    for i, (a, x, y) in enumerate(recs):
        blk[1 + REC * i: 6 + REC * i] = np.frombuffer(a, np.uint32)
        blk[6 + REC * i: 1 + REC * (i + 1)] = words_of(x) + words_of(y)
    return blk


def test_refusals(lib, keys):
    """x >= p, y >= p, a point off the curve, another validator's key, and a block whose count word exceeds the cap: every one
    refused, the entries stay unknown.  A known entry refuses a forged key as well."""
    edge = [(ec.pubkey_to_address(Q), Q) for Q in A.known_points()]      # keys at the coordinate edges: x or y < 2^256 - p
    keys = keys + [next(k for k in edge if k[1][0] + P < 1 << 256), next(k for k in edge if k[1][1] + P < 1 << 256)]
    small_x, small_y = len(keys) - 2, len(keys) - 1
    R = Registry(len(keys))
    for i, (a, _) in enumerate(keys):
        R.put(i, a)
    R.put(7, keys[7][0], keys[7][1])
    R.tables = [{a: i for i, (a, _) in enumerate(keys)}]
    recs = [
        (keys[small_x][0], keys[small_x][1][0] + P, keys[small_x][1][1]),   # x >= p
        (keys[small_y][0], keys[small_y][1][0], keys[small_y][1][1] + P),   # y >= p
        (keys[2][0], keys[2][1][0], (keys[2][1][1] + 1) % P),                # off the curve
        (keys[3][0], *keys[4][1]),                                           # validator 4's key under validator 3's address
        (keys[7][0], *keys[8][1]),                                           # a forged key for a known entry
    ]
    over = forged_block([(keys[5][0], *keys[5][1])])
    over[0] = C + 1
    dec, counts = R.adopt(lib, [forged_block(recs), over], 2)
    assert counts == [0, len(recs) + 1]
    assert dec[0][: len(recs)].tolist() == [REFUSE] * len(recs)
    assert R.state.tolist() == [LEARNED if i == 7 else UNKNOWN for i in range(len(keys))]
    assert R.export(lib)[1] == [7]
