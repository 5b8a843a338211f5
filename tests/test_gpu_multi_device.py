"""One engine over several devices (ibft_engine_create_multi) against a single-device engine and the golden / oracle answers.

On one GPU the sub-engines repeat ordinal 0 ([0, 0], [0, 0, 0], [0] * 8): every shard, arena plan, peer copy and merge runs as
on distinct devices.  Every comparison is byte for byte: verdict bitmap, group results (the five power limbs, counts,
has_quorum), voted sets, item statuses and recovered addresses."""
import threading

import numpy as np
import pytest

import ibft_b200 as ib
import workloads as wl
from oracle import coracle as co

pytestmark = pytest.mark.gpu

CAP = dict(max_items=(1 << 17) + 64, max_payload_bytes=1 << 24, max_groups=16, max_table_slots=4, max_validators=10_000)


def _copy(x):
    return None if x is None else np.array(x, copy=True)


@pytest.fixture(scope="module")
def fixtures():
    return {"config2": wl.config2(), "config3": wl.config3()}


@pytest.fixture(scope="module")
def engines():
    single = ib.Engine(device=0, **CAP)
    multi = {k: ib.Engine(devices=[0] * k, **CAP) for k in (2, 3)}
    yield single, multi
    single.close()
    for e in multi.values():
        e.close()


def setup_round(e, w, slot=0):
    e.set_validators(slot, w["height"], w["addrs"], w["powers"])
    return e.groups(len(w["groups"]), slot=slot)


def run_ex(e, items, arena, groups, stride=None):
    stride = stride if stride is not None else (CAP["max_validators"] + 31) // 32
    bm, res, st, voted = e.verify_batch_ex(items, arena, groups, voted_stride_words=stride)
    _, _, rec = e.verify_batch(items, arena, groups, want_recovered=True)
    return [_copy(bm), _copy(res), _copy(st), _copy(voted), _copy(rec)]


def assert_same(a, b):
    for x, y, what in zip(a, b, ("bitmap", "results", "status", "voted", "recovered")):
        if x is None or y is None:
            assert x is None and y is None, what
        else:
            assert x.tobytes() == y.tobytes(), what


def sample(w, n, seed=0):
    items, arena = w["items"], w["arena"]
    if n <= len(items):
        idx = np.sort(np.random.default_rng(seed).choice(len(items), n, replace=False)) if n < len(items) else np.arange(n)
    else:
        idx = np.arange(n) % len(items)
    return np.ascontiguousarray(items[idx]), arena


SIZES = [0, 1, 31, 32, 33, 1023, 1024, 1025, 2049, 3000]


@pytest.mark.parametrize("name", ["config2", "config3"])
def test_fixtures_match_single_engine(engines, fixtures, name):
    single, multi = engines
    w = fixtures[name]
    rng = np.random.default_rng(11)
    sizes = SIZES + [int(x) for x in rng.integers(0, 1001, 6)] + ([len(w["items"])] if name == "config3" else [])
    for e in [single] + list(multi.values()):
        groups = setup_round(e, w)
    for n in sizes:
        items, arena = sample(w, n, seed=n)
        want = run_ex(single, items, arena, groups)
        if n and n == len(w["items"]):
            assert np.array_equal(want[0], wl.oracle_bitmap(w))
        for k, e in multi.items():
            assert_same(run_ex(e, items, arena, groups), want)
            assert np.array_equal(e.last_item_status(n), want[2])


def test_chunked_path_on_every_sub_engine(engines, fixtures):
    """2^17 + 1 tuples: every shard of [0, 0] is a chunked call of its own sub-engine; [0] * 8 with small capacities splits
    the same batch eight ways (the last device's shard is ragged)."""
    single, multi = engines
    w = fixtures["config3"]
    items, arena = sample(w, (1 << 17) + 1)
    groups = setup_round(single, w)
    want = run_ex(single, items, arena, groups)
    e = multi[2]
    assert_same(run_ex(e, items, arena, setup_round(e, w)), want)
    e8 = ib.Engine(devices=[0] * 8, max_items=(1 << 17) + 64, max_payload_bytes=len(arena), max_groups=4, max_table_slots=1,
                   max_validators=10_000)
    try:
        assert e8.device_count() == 8
        assert_same(run_ex(e8, items, arena, setup_round(e8, w)), want)
        # fewer items than devices x 1,024: the trailing devices get nothing
        small, _ = sample(w, 2500)
        assert_same(run_ex(e8, small, arena, groups), run_ex(single, small, arena, groups))
    finally:
        e8.close()


def test_config5_pin_on_two_and_three_devices():
    w, pin = wl.load_full("config5")
    for k in (2, 3):
        e = ib.Engine(devices=[0] * k, max_items=1 << 18, max_payload_bytes=1 << 25, max_groups=128, max_table_slots=16,
                      max_validators=10_000)
        try:
            for s in range(16):
                e.set_validators(s, w["heights"][s], w["tables"][s], w["powers"])
            groups = e.groups(w["n_groups"], slot=w["group_table"])
            bitmap, results, _ = e.verify_batch(w["items"], w["arena"], groups)
            assert np.array_equal(bitmap, pin["bitmap"])
            for g in range(len(pin["results"])):
                r = results[g]
                assert (int(r["n_valid"]), int(r["n_distinct"]), int(r["has_quorum"])) == tuple(int(x) for x in pin["results"][g, :3])
                assert [int(x) for x in r["power"]] == [int(x) for x in pin["results"][g, 4:9]]
        finally:
            e.close()


def certificate_batch(w, n_certs=3):
    """Raw PREPARE frames nested inside certificate blobs, an IBFT_KIND_WIRE item per nested frame (its span inside the blob),
    an outer item per blob, and ROUND_CHANGE-like heads whose tail is a shared blob (IBFT_KIND_PAYLOAD2, signed over
    head || blob)."""
    frames = w["wire"][: w["n"]]             # the PREPARE frames of config 2
    arena, items, blobs = bytearray(), [], []
    per = len(frames) // n_certs
    for c in range(n_certs):
        start = len(arena)
        for j, f in enumerate(frames[c * per:(c + 1) * per]):
            arena.extend(f)
            it = np.zeros(1, dtype=ib.ITEM_DTYPE)
            it["kind"], it["group"], it["payload_off"], it["payload_len"] = ib.KIND_WIRE, 0, len(arena) - len(f), len(f)
            items.append(it)
        blobs.append((start, len(arena) - start))
        it = np.zeros(1, dtype=ib.ITEM_DTYPE)      # the outer frame: not a canonical PREPARE/COMMIT, so it is handed back
        it["kind"], it["group"], it["payload_off"], it["payload_len"] = ib.KIND_WIRE, 1, start, len(arena) - start
        items.append(it)
    keys = [wl.privkey(1, i) for i in range(w["n"])]
    for i in range(0, w["n"], 7):
        off2, len2 = blobs[i % n_certs]
        head = b"round-change head %d" % i
        sig = wl.sign(keys[i], co.keccak256(head + bytes(arena[off2:off2 + len2])))
        it = wl.make_item(sig, bytes(w["addrs"][i]), ib.KIND_PAYLOAD2, b"", 1, len(arena), len(head))
        it["digest"][0][:8] = np.frombuffer(off2.to_bytes(8, "little"), np.uint8)
        it["digest"][0][8:12] = np.frombuffer(len2.to_bytes(4, "little"), np.uint8)
        arena.extend(head)
        items.append(it)
    return np.concatenate(items).view(ib.ITEM_DTYPE), bytes(arena)


def test_raw_frames_and_shared_tails_fit_the_arena_exactly(engines, fixtures):
    single, _ = engines
    w = fixtures["config2"]
    items, arena = certificate_batch(w)
    groups = setup_round(single, w)[:2]
    want = run_ex(single, items, arena, groups)
    assert int(np.unpackbits(want[0].view(np.uint8)).sum()) > 900
    for k in (2, 3):
        e = ib.Engine(devices=[0] * k, max_items=4096, max_payload_bytes=len(arena), max_groups=4, max_table_slots=1,
                      max_validators=1024)
        try:
            got = run_ex(e, items, arena, setup_round(e, w)[:2], stride=32)
            assert_same(got, run_ex(single, items, arena, groups, stride=32))
        finally:
            e.close()


def test_groups_across_shards(engines, fixtures):
    """Groups re-assigned over config 2's 3,000 tuples so that their valid items sit on one device or straddle devices: every
    quorum rule, a PREPARE proposer whose own PREPARE lands on another device, PROPOSER_NONE / _UNSET, IBFT_NO_TABLE groups."""
    single, multi = engines
    w = fixtures["config2"]
    items = w["items"].copy()
    n = len(items)
    g = np.zeros(n, dtype=np.uint16)
    g[: n // 2] = 0                   # first half
    g[n // 2:] = 1                    # second half: on the last device of [0, 0, 0]
    g[2500:] = 2                      # all on the last device
    g[::97] = 3                       # spread over every device
    g[5] = 4                          # the proposer's PREPARE (validator 5) alone on device 0
    g[1200:1400] = 4                  # the other PREPAREs of that group on device 1
    g[2000:2050] = 5
    items["group"] = g
    arena = w["arena"]
    for e in [single] + list(multi.values()):
        setup_round(e, w)
    rules = [(ib.QUORUM_DEFAULT, 0), (ib.QUORUM_PREPARE, 5), (ib.QUORUM_PREPARE, ib.PROPOSER_NONE),
             (ib.QUORUM_PREPARE, ib.PROPOSER_UNSET), (ib.QUORUM_PREPREPARE, 0)]
    for shift in range(len(rules)):
        rs = [rules[(i + shift) % len(rules)] for i in range(6)]
        slots = [0] * 6
        if shift == 0:
            slots[5], rs[5] = ib.NO_TABLE, (ib.QUORUM_DEFAULT, 0)
        groups = single.groups(6, slot=slots, rule=[r for r, _ in rs], proposer=[p for _, p in rs])
        want = run_ex(single, items, arena, groups)
        for e in multi.values():
            assert_same(run_ex(e, items, arena, groups), want)


def test_errors_leave_outputs_untouched(engines, fixtures):
    single, multi = engines
    w = fixtures["config2"]
    items, arena = w["items"], w["arena"]
    good = setup_round(single, w)
    for e in multi.values():
        setup_round(e, w)
    bad_height = good.copy()
    bad_height[1]["height"] += 1
    rule3 = good.copy()
    rule3[0]["flags"] = 3
    proposer = single.groups(len(good), rule=ib.QUORUM_PREPARE, proposer=len(w["addrs"]))
    big = np.concatenate([items] * 44)     # > max_items
    cases = [(items, bad_height), (items, rule3), (items, proposer), (big, good)]
    for it, groups in cases:
        codes = []
        for e in [single] + list(multi.values()):
            n, ng = len(it), len(groups)
            bm = np.full((n + 31) // 32, 0xA5A5A5A5, dtype=np.uint32)
            res = np.zeros(ng, dtype=ib.RESULT_DTYPE)
            res.view(np.uint8)[:] = 0x5A
            rec = np.full((n, 20), 0x3C, dtype=np.uint8)
            st = np.full(n, 0x77, dtype=np.uint8)
            voted = np.full((ng, 40), 0x11, dtype=np.uint32)
            rc = e.lib.ibft_verify_batch_ex(e.handle, ib.engine._ptr(it), n, ib.engine._ptr(np.frombuffer(arena, np.uint8)), len(arena),
                                            ib.engine._ptr(groups), ng, ib.engine._ptr(bm), ib.engine._ptr(res), ib.engine._ptr(rec),
                                            ib.engine._ptr(st), ib.engine._ptr(voted), 40)
            codes.append(rc)
            assert (bm == 0xA5A5A5A5).all() and (res.view(np.uint8) == 0x5A).all() and (rec == 0x3C).all()
            assert (st == 0x77).all() and (voted == 0x11).all()
        assert codes[0] != ib.engine.IBFT_OK and len(set(codes)) == 1, codes


def test_async_and_concurrent_callers(engines, fixtures):
    single, multi = engines
    w2, w3 = fixtures["config2"], fixtures["config3"]
    e = multi[3]
    g2 = setup_round(single, w2, slot=0)
    g3 = setup_round(single, w3, slot=1)
    setup_round(e, w2, slot=0)
    setup_round(e, w3, slot=1)
    big, _ = sample(w3, 20_000)              # bulk lane (more than the small lane's 16,384)
    small = w2["items"]
    want_big = single.verify_batch(big, w3["arena"], g3)[:2]
    want_small = single.verify_batch(small, w2["arena"], g2)[:2]
    # submit / poll / wait
    bm = np.zeros((len(big) + 31) // 32, dtype=np.uint32)
    res = np.zeros(len(g3), dtype=ib.RESULT_DTYPE)
    arena3 = np.frombuffer(w3["arena"], np.uint8)
    e.verify_submit(big, arena3, g3, bm, res)
    while not e.poll():
        pass
    e.wait()
    assert bm.tobytes() == want_big[0].tobytes() and res.tobytes() == want_big[1].tobytes()
    # two threads at once, on the bulk and the small lane
    out, errs = {}, []

    def call(key, items, arena, groups):
        try:
            for r in range(3):
                out[(key, r)] = e.verify_batch(items, arena, groups)[:2]
        except Exception as ex:  # noqa: BLE001
            errs.append(ex)
    th = [threading.Thread(target=call, args=("big", big, w3["arena"], g3)),
          threading.Thread(target=call, args=("small", small, w2["arena"], g2))]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs
    for r in range(3):
        for key, want in (("big", want_big), ("small", want_small)):
            got = out[(key, r)]
            assert got[0].tobytes() == want[0].tobytes() and got[1].tobytes() == want[1].tobytes()


def test_key_registry_per_device(fixtures):
    w = fixtures["config3"]
    kw = dict(max_items=1 << 15, max_payload_bytes=1 << 23, max_groups=4, max_table_slots=2, max_validators=10_000, key_cache=True)
    single = ib.Engine(device=0, **kw)
    multi = ib.Engine(devices=[0, 0], **kw)
    try:
        groups = setup_round(single, w)
        setup_round(multi, w)
        commit = w["items"]
        for r in range(3):
            a = single.verify_batch_ex(commit, w["arena"], groups, voted_stride_words=313)
            b = multi.verify_batch_ex(commit, w["arena"], groups, voted_stride_words=313)
            for x, y in zip(a, b):
                assert x.tobytes() == y.tobytes()
            subs = [multi.sub(k) for k in range(2)]
            assert multi.known_handed_back() == sum(s.known_handed_back() for s in subs)
        known = multi.refresh_key_tables()
        assert known == single.refresh_key_tables()
        for s in subs:
            used, ready, _ = s.key_registry()
            assert used == 10_000 and 0 < ready <= 10_000
        # a budget bounds every device's pool
        multi.set_key_table_budget(300)
        multi.verify_batch(commit, w["arena"], groups)
        multi.refresh_key_tables()
        for s in subs:
            assert s.key_registry()[2] <= 300 * 136 * 1024
        assert multi.verify_batch(commit, w["arena"], groups)[0].tobytes() == single.verify_batch(commit, w["arena"], groups)[0].tobytes()
    finally:
        single.close()
        multi.close()


def test_validator_tables_are_replicated(engines, fixtures):
    _, multi = engines
    w = fixtures["config2"]
    e = multi[3]
    setup_round(e, w, slot=2)
    want = e.get_quorum(2)
    assert [e.sub(k).get_quorum(2) for k in range(3)] == [want] * 3
    with pytest.raises(ib.EngineError) as ex:
        e.set_validators(2, 7, w["addrs"], np.zeros((len(w["addrs"]), 32), np.uint8))
    assert ex.value.code == ib.engine.ERR_VOTING_POWER
    assert [e.sub(k).get_quorum(2) for k in range(3)] == [want] * 3


def test_hashing_and_signing_match_single_engine(engines):
    single, multi = engines
    rng = np.random.default_rng(3)
    for n in (1, 33, 10_000):
        msgs = [rng.integers(0, 256, int(rng.integers(0, 300)), dtype=np.uint8).tobytes() for _ in range(n)]
        rounds = [int(x) for x in rng.integers(0, 1 << 40, n)]
        keys = [int.from_bytes(rng.bytes(32), "big") for _ in range(n)]
        digests = [rng.bytes(32) for _ in range(n)]
        nonces = [int.from_bytes(rng.bytes(32), "big") for _ in range(n)]
        want = (single.keccak256_batch(msgs), single.proposal_hash_batch(msgs, rounds), single.sign_batch(keys, digests),
                single.sign_batch(keys, digests, nonces), single.sign_batch_rfc6979(keys, digests))
        for e in multi.values():
            got = (e.keccak256_batch(msgs), e.proposal_hash_batch(msgs, rounds), e.sign_batch(keys, digests),
                   e.sign_batch(keys, digests, nonces), e.sign_batch_rfc6979(keys, digests))
            assert got == want


def test_refusals(engines):
    _, multi = engines
    e = multi[2]
    lib, h = e.lib, e.handle
    assert lib.ibft_bind_groups(h, None, 0) == ib.engine.ERR_INVALID_ARG
    assert lib.ibft_verify_batch_device(h, None, 0, None, 0, 0, 0, None, None, None) == ib.engine.ERR_INVALID_ARG
    assert lib.ibft_quorum_reduce_device(h, None, 0, None, None, 0, None, None) == ib.engine.ERR_INVALID_ARG
    w = ib.engine.c_uint32()
    assert lib.ibft_quorum_partial_words(h, ib.engine.ctypes.byref(w)) == ib.engine.ERR_INVALID_ARG
    assert lib.ibft_quorum_mark_device(h, None, 0, 0, 0, None, None, None) == ib.engine.ERR_INVALID_ARG
    assert lib.ibft_quorum_merge_device(h, None, 1, 0, None, None) == ib.engine.ERR_INVALID_ARG
    with pytest.raises(ib.EngineError, match="one engine per device"):
        e.exchange_alloc(64)
    for f in (lambda: e.exchange_open(bytes(64)), lambda: e.exchange_close(1), lambda: e.exchange_free(1),
              lambda: e.exchange_clear(1, 0, 1), lambda: e.quorum_exchange_device([1, 2], 0, 8, 1, 1, 1, 1, 1)):
        with pytest.raises(ib.EngineError) as ex:
            f()
        assert ex.value.code == ib.engine.ERR_INVALID_ARG
    s = e.sub(1)
    assert s.device_info()["name"] and s.device_count() == 1
    items = np.zeros(1, dtype=ib.ITEM_DTYPE)
    refused = [lambda: s.set_validators(0, 1, np.zeros((1, 20), np.uint8)), lambda: s.verify_batch(items),
               lambda: s.verify_batch_ex(items), lambda: s.verify_submit(items, b"", None, np.zeros(1, np.uint32), None),
               lambda: s.poll(), lambda: s.wait(), lambda: s.keccak256_batch([b"x"]), lambda: s.proposal_hash_batch([b"x"], [0]),
               lambda: s.sign_batch([1], [bytes(32)]), lambda: s.sign_batch_rfc6979([1], [bytes(32)]), lambda: s.refresh_key_tables(),
               lambda: s.set_key_table_budget(1), lambda: s.set_recover_path(0), lambda: s.bind_groups(None),
               lambda: s.exchange_alloc(64)]
    for f in refused:
        with pytest.raises(ib.EngineError) as ex:
            f()
        assert ex.value.code == ib.engine.ERR_INVALID_ARG
    s.close()                                   # a borrowed handle: closing it leaves the engine alone
    assert e.sub(1).device_info()["name"]


def test_create_arguments_and_launch_count(engines):
    _, multi = engines
    lib = ib.engine.load_library()
    p = ib.engine.EngineParams(0, 1024, 1 << 16, 4, 1, 64, 0)
    h = ib.engine.c_void_p()
    for devs, code in (([], ib.engine.ERR_INVALID_ARG), ([0] * 9, ib.engine.ERR_INVALID_ARG), ([0, 999], ib.engine.ERR_INVALID_ARG), ([0, -1], ib.engine.ERR_INVALID_ARG)):
        arr = (ib.engine.c_int32 * max(1, len(devs)))(*devs)
        assert lib.ibft_engine_create_multi(ib.engine.ctypes.byref(p), arr, len(devs), ib.engine.ctypes.byref(h)) == code
        assert not h.value
    one = ib.Engine(devices=[0], max_items=1024, max_payload_bytes=1 << 16, max_groups=4, max_table_slots=1, max_validators=64)
    try:
        assert one.device_count() == 1 and one.sub(0).handle.value == one.handle.value
    finally:
        one.close()
    for e in multi.values():
        assert e.launch_count() == sum(e.sub(k).launch_count() for k in range(e.device_count())) > 0
