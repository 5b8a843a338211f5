"""The multi-device engine's shard planner (go-ibft_b200/csrc/shard_plan.hpp) on random and hand-made item sets: every item's
shard-local bytes equal its bytes in the call's arena (both spans of IBFT_KIND_PAYLOAD2), a shard's arena is never longer than
the call's, spans outside the call's arena stay outside the shard's, the shard bounds are sharding.shard_bounds', and empty
shards plan to nothing."""
import ctypes
import importlib
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
eng = importlib.import_module("go-ibft_b200.engine")
sharding = importlib.import_module("go-ibft_b200.sharding")
ITEM = eng.ITEM_DTYPE
PAYLOAD_KINDS = (eng.KIND_PAYLOAD, eng.KIND_WIRE, eng.KIND_WIRE_SEAL, eng.KIND_PAYLOAD2)


@pytest.fixture(scope="module")
def sp(tmp_path_factory):
    cxx = shutil.which(os.environ.get("CXX", "g++"))
    if cxx is None:
        pytest.fail("no C++ compiler to build the planner driver")
    so = str(tmp_path_factory.mktemp("shard_plan") / "libsp.so")
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-Wall", "-Wextra", "-fPIC", "-shared", "-o", so,
                           os.path.join(HERE, "emul", "shard_plan_driver.cpp")])
    lib = ctypes.CDLL(so)
    P, U32 = ctypes.c_void_p, ctypes.c_uint32
    lib.sp_devices.restype = U32
    lib.sp_devices.argtypes = [U32, U32]
    lib.sp_bounds.argtypes = [U32, U32, U32, ctypes.POINTER(U32), ctypes.POINTER(U32)]
    lib.sp_plan.restype = ctypes.c_size_t
    lib.sp_plan.argtypes = [P, U32, U32, P, ctypes.c_size_t, P, P]
    return lib


def off2(it):
    return int.from_bytes(bytes(it["digest"][:8]), "little"), int.from_bytes(bytes(it["digest"][8:12]), "little")


def set_off2(it, off, ln):
    it["digest"][:8] = np.frombuffer(int(off).to_bytes(8, "little"), np.uint8)
    it["digest"][8:12] = np.frombuffer(int(ln).to_bytes(4, "little"), np.uint8)


def plan(sp, items, lo, hi, arena):
    local = np.zeros(max(1, hi - lo), dtype=ITEM)
    out = np.full(max(16, len(arena)), 0xEE, dtype=np.uint8)
    ln = sp.sp_plan(items.ctypes.data, lo, hi, arena.ctypes.data if len(arena) else None, len(arena), local.ctypes.data, out.ctypes.data)
    return local[: hi - lo], out[:ln], ln


def spans(it, arena_len):
    """(global span, in range) pairs the kernels read for one tuple"""
    k = int(it["kind"])
    if k not in PAYLOAD_KINDS:
        return []
    off, ln = int(it["payload_off"]), int(it["payload_len"])
    out = [((off, ln), off + ln <= arena_len)]
    if k == eng.KIND_PAYLOAD2:
        o2, l2 = off2(it)
        out.append(((o2, l2), o2 <= arena_len and l2 <= arena_len - o2))
    return out


def check_shard(items, arena, lo, hi, local, shard_arena):
    assert len(shard_arena) <= len(arena)
    for i in range(hi - lo):
        g, l = items[lo + i], local[i]
        # everything but the offsets is the caller's tuple
        for f in ("r", "s", "signer", "v", "kind", "group", "payload_len"):
            assert np.array_equal(g[f], l[f]), f
        if int(g["kind"]) != eng.KIND_PAYLOAD2:
            assert np.array_equal(g["digest"], l["digest"])
        else:
            assert np.array_equal(g["digest"][8:], l["digest"][8:])
        if int(g["kind"]) not in PAYLOAD_KINDS:
            assert g["payload_off"] == l["payload_off"]
            continue
        for ((go, gl), inr), ((lo_, ll), local_inr) in zip(spans(g, len(arena)), spans(l, len(shard_arena))):
            assert gl == ll and local_inr == inr   # out-of-range spans stay out of range
            if inr:
                assert bytes(shard_arena[lo_:lo_ + ll]) == bytes(arena[go:go + gl])
                if gl:
                    assert lo_ % 16 == go % 16   # the sponge sees the same alignment


def random_call(rng, n, arena_len):
    arena = rng.integers(0, 256, arena_len, dtype=np.uint8)
    items = np.zeros(n, dtype=ITEM)
    items["r"] = rng.integers(0, 256, (n, 32))
    items["digest"] = rng.integers(0, 256, (n, 32))
    kinds = np.array([0, 1, 2, 3, 4, 5, 255, 7])
    items["kind"] = rng.choice(kinds, n, p=[.1, .25, .1, .15, .1, .2, .05, .05])
    tails = [(int(o), int(rng.integers(0, 300))) for o in rng.integers(0, arena_len, 4)]
    for i in range(n):
        r = rng.random()
        if r < 0.05:
            off, ln = int(rng.integers(arena_len - 5, arena_len + 50)), int(rng.integers(1, 60))   # past the end
        elif r < 0.1:
            off, ln = int(rng.integers(0, arena_len + 1)), 0
        else:
            off = int(rng.integers(0, arena_len))
            ln = int(rng.integers(0, min(400, arena_len - off) + 1))
        items[i]["payload_off"], items[i]["payload_len"] = off, ln
        if items[i]["kind"] == eng.KIND_PAYLOAD2:
            o2, l2 = tails[int(rng.integers(0, len(tails)))]
            if rng.random() < 0.1:
                o2 = arena_len + int(rng.integers(0, 3))
            set_off2(items[i], o2, l2)
    return items, arena


@pytest.mark.parametrize("seed", range(12))
def test_random_calls(sp, seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(0, 5000))
    items, arena = random_call(rng, n, int(rng.integers(1, 20000)))
    for world in (1, 2, 3, 8):
        for rank in range(world):
            lo, hi = sharding.shard_bounds(n, world, rank)
            local, shard_arena, _ = plan(sp, items, lo, hi, arena)
            check_shard(items, arena, lo, hi, local, shard_arena)


def test_bounds_match_sharding(sp):
    lo, hi = ctypes.c_uint32(), ctypes.c_uint32()
    for n in list(range(0, 200)) + [1023, 1024, 1025, 2047, 2049, 10000, 144953, (1 << 17) + 1, 1 << 20]:
        for world in range(1, 9):
            for rank in range(world):
                sp.sp_bounds(n, world, rank, ctypes.byref(lo), ctypes.byref(hi))
                assert (lo.value, hi.value) == sharding.shard_bounds(n, world, rank)
        for devices in range(1, 9):
            assert sp.sp_devices(n, devices) == max(1, min(devices, -(-n // 1024)))


def test_empty_shards(sp):
    items, arena = random_call(np.random.default_rng(5), 40, 1000)
    # 40 items over 8 shards: two words, so shards 2..7 are empty
    for rank in range(8):
        lo, hi = sharding.shard_bounds(40, 8, rank)
        local, shard_arena, ln = plan(sp, items, lo, hi, arena)
        if rank >= 2:
            assert lo == hi == 40 and ln == 0 and len(local) == 0
        else:
            check_shard(items, arena, lo, hi, local, shard_arena)
    local, shard_arena, ln = plan(sp, np.zeros(1, dtype=ITEM), 0, 0, np.zeros(0, np.uint8))
    assert ln == 0


def test_nested_frames_and_shared_tails_fit(sp):
    """Certificates: an outer frame and the PREPARE frames nested inside it, and ROUND_CHANGE heads sharing one tail.  The union
    never exceeds the call's arena, where per-item copies (sharding.rebase_shard) would hold the nested bytes twice."""
    rng = np.random.default_rng(7)
    outer = 4000
    arena = rng.integers(0, 256, outer + 64 * 100, dtype=np.uint8)
    items = np.zeros(1 + 40 + 100, dtype=ITEM)
    items[0]["kind"], items[0]["payload_off"], items[0]["payload_len"] = eng.KIND_WIRE, 0, outer
    for j in range(40):  # nested frames inside the outer one
        it = items[1 + j]
        it["kind"], it["payload_off"], it["payload_len"] = eng.KIND_WIRE, 100 * j + 3, 97
    for j in range(100):  # heads after the certificate, each with the certificate as its tail
        it = items[41 + j]
        it["kind"], it["payload_off"], it["payload_len"] = eng.KIND_PAYLOAD2, outer + 64 * j, 64
        set_off2(it, 0, outer)
    n = len(items)
    local, shard_arena, ln = plan(sp, items, 0, n, arena)
    assert ln == len(arena)
    check_shard(items, arena, 0, n, local, shard_arena)
    _, per_item = sharding.rebase_shard(items, arena, 0, n)
    assert len(per_item) > len(arena)
    for world in (2, 3):
        for rank in range(world):
            lo, hi = sharding.shard_bounds(n, world, rank)
            local, shard_arena, ln = plan(sp, items, lo, hi, arena)
            assert ln <= len(arena)
            check_shard(items, arena, lo, hi, local, shard_arena)


def test_hand_made_edges(sp):
    arena = np.arange(256, dtype=np.uint8)
    rows = [  # (kind, off, len, off2, len2)
        (eng.KIND_PAYLOAD, 250, 6, 0, 0),      # ends exactly at the arena's end
        (eng.KIND_PAYLOAD, 250, 7, 0, 0),      # one byte past it
        (eng.KIND_PAYLOAD, 256, 0, 0, 0),      # empty, at the end
        (eng.KIND_PAYLOAD, 0xFFFFFFFF, 1, 0, 0),
        (eng.KIND_PAYLOAD2, 10, 5, 256, 0),    # empty tail at the end
        (eng.KIND_PAYLOAD2, 10, 5, 257, 0),    # tail past the end
        (eng.KIND_PAYLOAD2, 10, 5, 1 << 63, 2),
        (eng.KIND_PAYLOAD2, 300, 5, 12, 20),   # head past the end, tail inside
        (eng.KIND_WIRE_SEAL, 17, 33, 0, 0),
        (eng.KIND_DIGEST, 9999, 9999, 0, 0),   # kinds without a payload keep their fields
        (eng.KIND_SEAL, 5, 5, 0, 0),
        (eng.KIND_INVALID, 5, 5, 0, 0),
    ]
    items = np.zeros(len(rows), dtype=ITEM)
    for it, (k, o, ln, o2, l2) in zip(items, rows):
        it["kind"], it["payload_off"], it["payload_len"] = k, o, ln
        if k == eng.KIND_PAYLOAD2:
            set_off2(it, o2, l2)
    for lo in range(len(rows)):
        for hi in range(lo, len(rows) + 1):
            local, shard_arena, _ = plan(sp, items, lo, hi, arena)
            check_shard(items, arena, lo, hi, local, shard_arena)
