"""The bounded key registry's table policy (go-ibft_b200/csrc/key_budget.hpp, ibft_set_key_table_budget) against a Python model of
its ranking, over seeded random sequences of listed sets, used flags, keys learned between reclaim points and budget changes.

At a reclaim point the entries with a known key that a resident table lists are ranked by the reclaim point at which they were
last used (newest first), then those holding a table before those that do not, then by address; the first max_tables keep or
get a table.  Between reclaim points, keys learned since take free slots in ascending address order."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

NO = 0xFFFFFFFF
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def kb(tmp_path_factory):
    cxx = shutil.which(os.environ.get("CXX", "g++"))
    if cxx is None:
        pytest.fail("no C++ compiler to build the policy driver")
    so = str(tmp_path_factory.mktemp("key_budget") / "libkb.so")
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-Wall", "-Wextra", "-fPIC", "-shared", "-o", so,
                           os.path.join(HERE, "emul", "key_budget_driver.cpp")])
    lib = ctypes.CDLL(so)
    lib.kb_new.restype = ctypes.c_void_p
    lib.kb_free.argtypes = [ctypes.c_void_p]
    P = ctypes.c_void_p
    U32P = ctypes.POINTER(ctypes.c_uint32)
    lib.kb_reclaim.restype = ctypes.c_uint32
    lib.kb_reclaim.argtypes = [P, ctypes.c_uint32, P, P, P, P, ctypes.c_uint32, P, U32P, U32P, U32P]
    lib.kb_take_free.restype = ctypes.c_uint32
    lib.kb_take_free.argtypes = [P, ctypes.c_uint32, ctypes.c_uint32]
    lib.kb_live.restype = ctypes.c_uint32
    lib.kb_live.argtypes = [P]
    return lib


def ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


class Model:
    """the ranking, restated"""

    def __init__(self):
        self.clock = 0
        self.stamp = {}
        self.holds = set()
        self.max = 0

    def reclaim(self, listed, known, used, addr, new_max):
        self.clock += 1
        for r in np.flatnonzero(used):
            self.stamp[int(r)] = self.clock
        for r in np.flatnonzero(~listed):
            self.stamp.pop(int(r), None)
            self.holds.discard(int(r))
        cand = [int(r) for r in np.flatnonzero(listed & known)]
        cand.sort(key=lambda r: (-self.stamp.get(r, 0), r not in self.holds, bytes(addr[r]), r))
        before = set(self.holds)
        self.holds = set(cand[:new_max])
        self.max = new_max
        return before

    def learn(self, fresh, addr):
        """keys learned between reclaim points take the free slots, lowest address first"""
        free = self.max - len(self.holds)
        got = sorted(fresh, key=lambda r: bytes(addr[r]))[:max(free, 0)]
        self.holds |= set(got)
        return got


@pytest.mark.parametrize("seed", range(12))
def test_policy_matches_the_model(kb, seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(20, 400))
    addr = rng.integers(0, 256, size=(n, 20), dtype=np.uint8)
    if seed % 3 == 0:
        addr[:, :18] = 0                             # near-equal addresses: the order comes from the last bytes
    h = kb.kb_new()
    model = Model()
    listed = np.zeros(n, bool)
    known = np.zeros(n, bool)
    table = np.full(n, NO, np.uint32)
    ev, ad, rt = ctypes.c_uint32(), ctypes.c_uint32(), ctypes.c_uint32()
    try:
        for step in range(60):
            # a new validator set: some entries leave every table (their keys are forgotten), some arrive
            flip = rng.random(n) < rng.choice([0.0, 0.05, 0.3])
            leaving = flip & listed
            listed ^= flip
            known[leaving] = False
            known |= listed & (rng.random(n) < 0.3)
            used = (listed & (rng.random(n) < rng.choice([0.0, 0.1, 0.5, 1.0]))).astype(np.uint8)
            if step % 7 == 3:
                used[:] = used.any()  # everybody equally hot (or cold)
                used &= listed
            new_max = int(rng.choice([0, 1, 8, n // 4, n // 2, n, n + 30])) if step % 4 == 0 else model.max
            was = table.copy()
            before = model.reclaim(listed, known, used.astype(bool), addr, new_max)
            moves = kb.kb_reclaim(h, n, ptr(listed.astype(np.uint8)), ptr(known.astype(np.uint8)), ptr(used), ptr(addr), new_max,
                                  ptr(table), ctypes.byref(ev), ctypes.byref(ad), ctypes.byref(rt))
            assert moves != NO, "a move left a table above the budget or at the wrong slot"
            holds = set(np.flatnonzero(table != NO).tolist())
            assert holds == model.holds, f"step {step}: selection differs"
            assert len(holds) <= new_max and kb.kb_live(h) == len(holds)
            slots = table[table != NO]
            assert len(set(slots.tolist())) == len(slots) and (slots < max(new_max, 1)).all()
            # a retired entry's slot is freed
            assert (table[~listed] == NO).all()
            assert rt.value == int(((was != NO) & ~listed).sum())
            # with equal stamps no incumbent is displaced: everything admitted was used more recently than everything evicted
            evicted = (before - holds) & set(np.flatnonzero(listed & known).tolist())
            admitted = holds - before
            if evicted and admitted:
                assert min(model.stamp.get(a, 0) for a in admitted) > max(model.stamp.get(e, 0) for e in evicted)
            # keys learned before the next reclaim point take free slots in ascending address order
            fresh = [int(r) for r in np.flatnonzero(listed & ~known & (rng.random(n) < 0.4))]
            known[fresh] = True
            want = model.learn(fresh, addr)
            got = []
            for r in sorted(fresh, key=lambda r: bytes(addr[r])):
                t = kb.kb_take_free(h, n, r)
                if t == NO:
                    break
                assert t < new_max and t not in set(table[table != NO].tolist())
                table[r] = t
                got.append(r)
            assert got == want
            assert kb.kb_live(h) <= new_max
    finally:
        kb.kb_free(h)


def test_lowering_moves_tables_below_the_budget(kb):
    """32 keys in 32 slots, budget lowered to 8: the 8 most recently used keep a table, every kept table sits below 8"""
    n = 32
    addr = np.arange(n, dtype=np.uint8)[:, None].repeat(20, 1)
    h = kb.kb_new()
    try:
        ones = np.ones(n, np.uint8)
        table = np.full(n, NO, np.uint32)
        ev, ad, rt = ctypes.c_uint32(), ctypes.c_uint32(), ctypes.c_uint32()
        kb.kb_reclaim(h, n, ptr(ones), ptr(ones), ptr(np.zeros(n, np.uint8)), ptr(addr), n, ptr(table), ctypes.byref(ev),
                      ctypes.byref(ad), ctypes.byref(rt))
        assert sorted(table.tolist()) == list(range(n))
        used = np.zeros(n, np.uint8)
        hot = [3, 9, 12, 17, 22, 27, 30, 31]
        used[hot] = 1
        moves = kb.kb_reclaim(h, n, ptr(ones), ptr(ones), ptr(used), ptr(addr), 8, ptr(table), ctypes.byref(ev),
                              ctypes.byref(ad), ctypes.byref(rt))
        assert sorted(np.flatnonzero(table != NO).tolist()) == hot
        assert (table[hot] < 8).all() and moves == sum(1 for r in hot if r >= 8)
        assert ev.value == n - 8 and ad.value == 0
    finally:
        kb.kb_free(h)
