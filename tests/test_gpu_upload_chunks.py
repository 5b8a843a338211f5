"""Host-buffer calls across upload chunks (tests/upload_shapes.py): one to five chunks, last chunks staged in one to four parts,
synchronous and submit / wait, from pageable and from page-locked memory, on every recover kernel, with the key registry and with
hash-bound groups, while another call is pending, and over two devices -- every output against the oracle's expectations.  An
asynchronous call's tuples are overwritten as soon as it returns: its outputs must be those of the batch as submitted."""
import itertools

import numpy as np
import pytest

import ibft_b200 as ib
import upload_shapes as U
from test_gpu_adversarial import expected_handed_back

pytestmark = pytest.mark.gpu
E = ib.Engine
EM = ib.engine                 # the ctypes binding: raw ABI calls whose outputs are checked untouched
C = U.C
ARENA_CAP = 32 << 20
CAP = dict(device=0, max_items=5 * C, max_payload_bytes=ARENA_CAP, max_groups=4, max_table_slots=1, max_validators=16384)
calls = itertools.count()      # every call uploads a rotation of its own: no two consecutive calls send the same bytes


@pytest.fixture(scope="module")
def up():
    return U.uploads()


def make_engine(up, **kw):
    e = E(**{**CAP, **kw})
    e.set_validators(0, up.height, up.addrs, up.powers)
    return e


@pytest.fixture(scope="module")
def eng(up):
    e = make_engine(up)
    yield e
    e.close()


def groups_of(eng):
    return eng.groups(len(U.SLOTS), slot=U.SLOTS)


def bits(bm, n):
    return np.unpackbits(np.ascontiguousarray(bm, dtype=np.uint32).view(np.uint8), bitorder="little")[:n].astype(bool)


def pinned(items, offset=0):
    """(tensor, view): a copy of items in page-locked memory, starting `offset` bytes into the allocation"""
    import torch
    t = torch.empty(offset + items.nbytes, dtype=torch.uint8, pin_memory=True)
    a = t.numpy()[offset:offset + items.nbytes].view(ib.ITEM_DTYPE)
    a[:] = items
    return t, a


def where(i, n):
    c = i // C
    return f"item {i} (chunk {c}, +{i - c * C})"


def check(eng, up, e, label, bm, res, st, rec=None, voted=None, counted=None, flags=None):
    """bitmap, status, recovered addresses, every group's result (all five power limbs) and voted set against the expectations"""
    n = len(e["bit"])
    got = bits(bm, n)
    bad = np.nonzero(got != e["bit"])[0]
    assert len(bad) == 0, (label, len(bad), [(where(int(i), n), bool(got[i])) for i in bad[:6]])
    bad = np.nonzero(st != e["status"])[0]
    assert len(bad) == 0, (label, "status", [where(int(i), n) for i in bad[:6]])
    if rec is not None:
        bad = np.nonzero((rec != e["rec"]).any(axis=1))[0]
        assert len(bad) == 0, (label, "recovered", [where(int(i), n) for i in bad[:6]])
    if counted is not None:
        got = bits(counted, n)
        bad = np.nonzero(got != flags)[0]
        assert len(bad) == 0, (label, "counted", [where(int(i), n) for i in bad[:6]])
    n_val = len(up.members)
    for g, (nv, vs, power, hq) in enumerate(e["groups"]):
        r = res[g]
        have = (int(r["n_valid"]), int(r["n_distinct"]), sum(int(r["power"][k]) << (64 * k) for k in range(5)), bool(r["has_quorum"]))
        assert have == (nv, len(vs), power, hq), (label, g, have, (nv, len(vs), power, hq))
        if vs:
            words = voted[g] if voted is not None else eng.voted_bitmap(g, n_val)
            assert set(np.nonzero(bits(words, n_val))[0].tolist()) == vs, (label, g)


def run(eng, up, n, sync, memory, label, arena=None):
    """one call of n tuples: synchronous (verify_batch) or verify_submit + wait, from pageable numpy memory, a pinned tensor or a
    view that starts 448 bytes into a pinned allocation; every output checked"""
    items, src, grp = up.batch(n, next(calls))
    e = up.expect(src, grp)
    keep = None
    if memory == "pinned":
        keep, items = pinned(items)
    elif memory == "pinned_view":
        keep, items = pinned(items, offset=448)
    arena = up.arena if arena is None else arena
    groups = groups_of(eng)
    if sync:
        bm, res, rec = eng.verify_batch(items, arena, groups, want_recovered=True)
    else:
        bm = np.zeros((n + 31) // 32, np.uint32)
        res = np.zeros(len(groups), ib.RESULT_DTYPE)
        rec = np.zeros((n, 20), np.uint8)
        eng.verify_submit(items, np.frombuffer(arena, np.uint8), groups, bm, res, rec)
        eng.wait()
    st = eng.last_item_status(n)
    check(eng, up, e, label, bm, res, st, rec)
    del keep


WAYS = [(True, "pageable"), (False, "pageable"), (True, "pinned"), (False, "pinned_view")]


@pytest.mark.parametrize("shape", list(U.SHAPES))
def test_auto_every_shape_four_ways(eng, up, shape):
    """AUTO at every shape: synchronous and submit / wait, from pageable and from page-locked memory"""
    eng.set_recover_path(E.PATH_AUTO)
    for sync, memory in WAYS:
        run(eng, up, U.SHAPES[shape], sync, memory, (shape, "sync" if sync else "async", memory))


def test_forced_paths_past_one_chunk(eng, up):
    """each recover kernel at C + 1: chunk 1 starts at lo = 2^17, which is 8 mod 24 and 32 mod 96 -- off the qsplit and split
    CTA grids"""
    assert C % 24 == 8 and C % 96 == 32
    try:
        for path in (E.PATH_THREAD, E.PATH_QUAD, E.PATH_SPLIT, E.PATH_QSPLIT):
            eng.set_recover_path(path)
            run(eng, up, C + 1, True, "pageable", ("path", path))
    finally:
        eng.set_recover_path(E.PATH_AUTO)


# ------------------------------------------------------------------------------------------------------------ key registry
@pytest.fixture(scope="module")
def known(up):
    """a key-registry engine that has learned the keys of config 3's valid signers and of the sweep's known classes (by a call that
    asks for recovered addresses: the plain recover kernels)"""
    S = up.S
    eng = make_engine(up, key_cache=True)
    learn2 = U.PS.wl.make_item(U.PS.wl.sign(S.reason_vs.keys[2], b"\x01" * 32), S.reason_vs.addrs[2], 0, b"\x01" * 32)
    warm = np.concatenate([up.fillers, S.classes["valid_low_s"], S.known_warm[0], S.known_warm[1], learn2])
    warm["group"][up.F:] = 0
    bm, _, _ = eng.verify_batch(warm, up.arena, groups_of(eng), want_recovered=True)
    ok = bits(bm, len(warm))
    assert ok[up.F:].all() and np.array_equal(ok[:up.F], up.filler_gold)
    eng.refresh_key_tables()
    yield eng, {bytes(warm[i]["signer"]) for i in np.nonzero(ok)[0]}
    eng.close()


def test_key_registry_across_chunks(known, up):
    """known, misattributed, unknown-signer, x = r + n, cancelling and flipped items at the odd slots.  C + 1 (worklists 0 and 1):
    the count handed to the recover pass is the expected one.  3C + 49,153 (worklist 0 filled by chunks 0 and 2): the count is
    refused, and the outputs still equal the oracle's."""
    eng, known_signers = known
    members = set(up.members)
    for shape in ("C+1", "4chunks"):
        n = U.SHAPES[shape]
        items, src, grp = up.batch(n, next(calls), known=True)
        e = up.expect(src, grp)
        bm, res, _ = eng.verify_batch(items, up.arena, groups_of(eng))
        st = eng.last_item_status(n)
        if shape == "C+1":
            handed = eng.known_handed_back()
            assert handed == expected_handed_back(items, len(up.arena), members, e["bit"], known_signers) > 0
        else:
            with pytest.raises(ib.EngineError):
                eng.known_handed_back()
        check(eng, up, e, ("known", shape), bm, res, st)
        known_signers |= {bytes(items[i]["signer"]) for i in np.nonzero(e["bit"])[0]}   # recovered, hence learned


# ------------------------------------------------------------------------------------------------------------ hashed groups
@pytest.mark.parametrize("shape", ["C+1", "5chunks"])
def test_hashed_groups_across_chunks(eng, up, shape):
    """verify_batch_ex with group 0 bound to config 3's proposal and group 1 to another hash: the counted bits against
    tests/group_hash_model.py, and the results and voted sets over the counted items"""
    n = U.SHAPES[shape]
    items, src, grp = up.batch(n, next(calls))
    h = up.hashes()
    flags = up.counted(src, grp, h)
    e = up.expect(src, grp, flags=flags)
    stride = (len(up.members) + 31) // 32
    bm, res, st, voted, counted = eng.verify_batch_ex(items, up.arena, groups_of(eng), voted_stride_words=stride, group_hashes=h)
    check(eng, up, e, ("hashed", shape), bm, res, st, voted=voted, counted=counted, flags=flags)


# ------------------------------------------------------------------------------------------------------------ async inputs
@pytest.mark.parametrize("memory", ["pageable", "pinned"])
def test_submitted_inputs_overwritten_at_once(eng, up, memory):
    """A four-chunk call behind a 32 MiB arena: as soon as verify_submit returns, the first and last 1,024 tuples of every chunk
    are overwritten with rejected items and the arena's first 64 KiB with 0xFF.  Every one of those tuples goes up only after the
    arena, so a call that still read the caller's memory would verify the new bytes.  The outputs must be those of the batch as
    submitted."""
    n = U.SHAPES["4chunks"]
    items, src, grp = up.batch(n, next(calls))
    e = up.expect(src, grp)
    arena = np.zeros(ARENA_CAP, np.uint8)
    arena[:len(up.arena)] = np.frombuffer(up.arena, np.uint8)
    keep = None
    if memory == "pinned":
        keep, items = pinned(items)
    junk = np.tile(up.S.invalid, 1024)
    junk["group"] = 0
    groups = groups_of(eng)
    bm = np.zeros((n + 31) // 32, np.uint32)
    res = np.zeros(len(groups), ib.RESULT_DTYPE)
    rec = np.zeros((n, 20), np.uint8)
    eng.verify_submit(items, arena, groups, bm, res, rec)
    for lo, hi in U.chunks(n):
        items[lo:lo + 1024] = junk
        items[hi - 1024:hi] = junk
    arena[:1 << 16] = 0xFF
    eng.wait()
    check(eng, up, e, ("overwritten", memory), bm, res, eng.last_item_status(n), rec)
    del keep


# ------------------------------------------------------------------------------------------------------------ lanes
def test_small_lane_beside_a_pending_call(eng, up):
    """With a five-chunk call pending on lane 0: 16,384 tuples with a 4 MiB arena run on the small lane and are exact; 16,385
    tuples, or a 4 MiB + 1 arena, need lane 0 and are refused with IBFT_ERR_INVALID_ARG, their outputs untouched; then the pending
    call's outputs are exact."""
    lib = eng.lib
    n = U.SHAPES["5chunks"]
    items, src, grp = up.batch(n, next(calls))
    e = up.expect(src, grp)
    groups = groups_of(eng)
    big_arena = np.zeros(ARENA_CAP, np.uint8)
    big_arena[:len(up.arena)] = np.frombuffer(up.arena, np.uint8)
    bm = np.zeros((n + 31) // 32, np.uint32)
    res = np.zeros(len(groups), ib.RESULT_DTYPE)
    rec = np.zeros((n, 20), np.uint8)
    eng.verify_submit(items, big_arena, groups, bm, res, rec)
    small, ssrc, sgrp = up.batch(16385, next(calls))
    small_arena = np.zeros(4 << 20, np.uint8)
    small_arena[:len(up.arena)] = np.frombuffer(up.arena, np.uint8)
    stride = (len(up.members) + 31) // 32
    try:
        sbm, sres, sst, svoted = eng.verify_batch_ex(small[:16384], small_arena, groups, voted_stride_words=stride)
        check(eng, up, up.expect(ssrc[:16384], sgrp[:16384]), ("small lane", 16384), sbm, sres, sst, voted=svoted)
        for m, ar in ((16385, small_arena), (16, np.concatenate([small_arena, np.zeros(1, np.uint8)]))):
            it = np.ascontiguousarray(small[:m])
            obm = np.full((m + 31) // 32, 0xA5A5A5A5, np.uint32)
            ores = np.frombuffer(b"\xa5" * (len(groups) * ib.RESULT_DTYPE.itemsize), ib.RESULT_DTYPE).copy()
            ost = np.full(m, 0xA5, np.uint8)
            ovoted = np.full((len(groups), stride), 0xA5A5A5A5, np.uint32)
            rc = lib.ibft_verify_batch_ex(eng.handle, EM._ptr(it), m, EM._ptr(ar), len(ar), EM._ptr(groups),
                                          len(groups), EM._ptr(obm), EM._ptr(ores), None, EM._ptr(ost),
                                          EM._ptr(ovoted), stride)
            assert rc == EM.ERR_INVALID_ARG, (m, len(ar), rc)
            assert (obm == 0xA5A5A5A5).all() and ores.tobytes() == b"\xa5" * ores.nbytes and (ost == 0xA5).all()
            assert (ovoted == 0xA5A5A5A5).all()
    finally:
        eng.wait()
    check(eng, up, e, ("pending lane 0", n), bm, res, eng.last_item_status(n), rec)


# ------------------------------------------------------------------------------------------------------------ two devices
def test_two_devices_chunked_shards(up):
    """An engine over devices [0, 0] with 2C + 2 tuples: each device's shard of C + 1 is chunked.  Synchronous and submit / wait,
    pageable and page-locked, against the oracle's expectations."""
    eng = make_engine(up, devices=[0, 0])
    try:
        for sync, memory in WAYS:
            run(eng, up, 2 * C + 2, sync, memory, ("two devices", "sync" if sync else "async", memory))
    finally:
        eng.close()
