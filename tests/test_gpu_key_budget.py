"""A bounded key registry (ibft_set_key_table_budget): at most max_tables comb tables, for the keys used most recently.  Every
bitmap, quorum result and voted set must equal a plain engine's and the oracle's; known_handed_back() must be what the tables
predict (members whose key has no table, plus rejected signatures); ibft_set_validators never fails for table memory."""
import threading

import numpy as np
import pytest
import torch

import adversarial as A
import ibft_b200 as ib
from oracle import coracle as co
from test_gpu_adversarial import bits, check_whole_key_table, expected_handed_back, known_addrs, known_batch, valid_known_items
from test_gpu_key_registry import make_engine, round_items, same_as_plain

pytestmark = pytest.mark.gpu
TAB = 17 * 128 * 64           # one comb table: 136 KiB
CHUNK = 256 * TAB


def ready_set(eng, slot, addrs):
    """addresses of `slot` whose comb table is built (ibft_debug_keytab state 2)"""
    return {bytes(addrs[v]) for v in range(len(addrs)) if eng.key_table(slot, v)[0] == 2}


def check_round(eng, plain, items, addrs, slot, with_table, rule=ib.QUORUM_DEFAULT):
    """verify on both engines and against the oracle; the known-key pass hands back every member without a table"""
    groups = eng.groups(1, slot, rule)
    a, ra, _ = eng.verify_batch(items, b"", groups)
    handed = eng.known_handed_back()
    b, rb, _ = plain.verify_batch(items, b"", plain.groups(1, slot, rule))
    assert np.array_equal(a, b) and ra.tobytes() == rb.tobytes()
    assert np.array_equal(eng.voted_bitmap(0, len(addrs)), plain.voted_bitmap(0, len(addrs)))
    want = co.verify_batch(items, b"", tables=[addrs], group_table=[0], n_threads=8)
    assert np.array_equal(a, want)
    valid = bits(want, len(items))
    assert handed == expected_handed_back(items, 0, {bytes(x) for x in addrs}, valid, with_table)
    return valid


def keys(seed, n):
    privs = co.privkeys(seed, n)
    return privs, co.addresses(privs)


def test_budget_below_the_set():
    """Config-2 size (1,000 validators) at budget 256: after the first call exactly 256 tables exist (the lowest addresses), the
    pool is exactly 256 tables, every valid signer's key is known, and the next height verifies exactly."""
    privs, addrs = keys(801, 1000)
    eng, plain = make_engine(slots=2, max_validators=1024, key_cache=True, key_table_budget=256), make_engine(slots=2, max_validators=1024)
    try:
        for e in (eng, plain):
            e.set_validators(0, 1, addrs)
            e.set_validators(1, 2, addrs)
        items = round_items(privs, addrs, co.keccak256(b"budget-1"))
        assert check_round(eng, plain, items, addrs, 0, set()).all()
        assert eng.key_registry() == (1000, 256, 256 * TAB)
        assert ready_set(eng, 0, addrs) == set(sorted(bytes(a) for a in addrs)[:256])
        assert all(eng.key_table(0, v)[0] in (1, 2) for v in range(1000))
        tables = ready_set(eng, 1, addrs)
        assert check_round(eng, plain, round_items(privs, addrs, co.keccak256(b"budget-2")), addrs, 1, tables).all()
        assert eng.key_registry() == (1000, 256, 256 * TAB)
    finally:
        eng.close()
        plain.close()


def test_hot_set_wins():
    """200 validators sign every round, the other 800 rotate 50 at a time.  After the reclaim points, all 200 hold a table and a
    round of theirs hands back nothing."""
    privs, addrs = keys(802, 1000)
    hot = np.arange(0, 1000, 5)
    cold = np.setdiff1d(np.arange(1000), hot)
    eng, plain = make_engine(slots=2, max_validators=1024, key_cache=True, key_table_budget=256), make_engine(slots=2, max_validators=1024)
    try:
        for e in (eng, plain):
            e.set_validators(0, 1, addrs)
        for k in range(4):
            sel = np.concatenate([hot, cold[50 * k:50 * (k + 1)]])
            items = round_items([privs[i] for i in sel], addrs[sel], co.keccak256(b"hot-%d" % k))
            check_round(eng, plain, items, addrs, 0, ready_set(eng, 0, addrs))
            eng.refresh_key_tables()                              # reclaim point
        assert {bytes(addrs[i]) for i in hot} <= ready_set(eng, 0, addrs)
        items = round_items([privs[i] for i in hot], addrs[hot], co.keccak256(b"hot-only"))
        launches = eng.launch_count()
        assert check_round(eng, plain, items, addrs, 0, ready_set(eng, 0, addrs)).all()
        assert eng.known_handed_back() == 0 and eng.launch_count() - launches == 3
    finally:
        eng.close()
        plain.close()


def test_no_thrash_when_everybody_is_equally_hot():
    """All 1,000 sign every round at budget 256 over 5 heights: after the first refresh no table is ever built again (3 launches
    per call) and the same 256 validators keep their tables."""
    privs, addrs = keys(803, 1000)
    eng, plain = make_engine(slots=2, max_validators=1024, key_cache=True, key_table_budget=256), make_engine(slots=2, max_validators=1024)
    try:
        for e in (eng, plain):
            e.set_validators(0, 1, addrs)
        check_round(eng, plain, round_items(privs, addrs, co.keccak256(b"warm")), addrs, 0, set())
        first = ready_set(eng, 0, addrs)
        assert len(first) == 256
        for h in range(2, 7):
            for e in (eng, plain):
                e.set_validators(h % 2, h, addrs)
            launches = eng.launch_count()
            check_round(eng, plain, round_items(privs, addrs, co.keccak256(b"h%d" % h)), addrs, h % 2, first)
            assert eng.launch_count() - launches == 3
            assert ready_set(eng, h % 2, addrs) == first
    finally:
        eng.close()
        plain.close()


def test_set_validators_is_never_refused():
    """Budget 256, 16 slots of 1,000 distinct new addresses each: every set_validators succeeds, 16,000 entries are in use, the
    pool stays within 256 tables and every slot's batch is exact."""
    eng = make_engine(slots=16, max_validators=1000, key_cache=True, key_table_budget=256)
    plain = make_engine(slots=16, max_validators=1000)
    try:
        sets = [keys(900 + k, 1000) for k in range(16)]
        for k, (_, addrs) in enumerate(sets):
            for e in (eng, plain):
                e.set_validators(k, 10 + k, addrs)
        assert eng.key_registry()[0] == 16000 and eng.key_registry()[2] <= 256 * TAB
        for k, (privs, addrs) in enumerate(sets):
            items = round_items(privs, addrs, co.keccak256(b"never-%d" % k))
            check_round(eng, plain, items, addrs, k, ready_set(eng, k, addrs) if k else set())
            used, ready, nbytes = eng.key_registry()
            assert used == 16000 and ready <= 256 and nbytes <= 256 * TAB
    finally:
        eng.close()
        plain.close()


def test_reassigned_slot_never_verifies_against_its_old_key():
    """Budget 16: A (16 validators) is learned and built, leaves, and B takes its table slots.  Every A key's signature attributed
    to every B validator is rejected, before and after B is built.  A rejoins and is accepted again once relearned."""
    pa, A = keys(811, 16)
    pb, B = keys(812, 16)
    eng, plain = make_engine(slots=2, max_validators=64, key_cache=True, key_table_budget=16), make_engine(slots=2, max_validators=64)
    d = co.keccak256(b"reassign")
    cross = np.concatenate([round_items(pa, np.repeat(B[j:j + 1], 16, 0), d) for j in range(16)])
    try:
        for e in (eng, plain):
            e.set_validators(0, 1, A)
        assert check_round(eng, plain, round_items(pa, A, d), A, 0, set()).all()
        assert eng.key_registry() == (16, 16, 16 * TAB)
        for e in (eng, plain):
            e.set_validators(0, 2, B)
        assert not check_round(eng, plain, cross, B, 0, set()).any()
        assert check_round(eng, plain, round_items(pb, B, d), B, 0, set()).all()
        assert eng.key_registry() == (16, 16, 16 * TAB)
        assert not check_round(eng, plain, cross, B, 0, {bytes(b) for b in B}).any()
        for e in (eng, plain):
            e.set_validators(0, 3, A)
        assert check_round(eng, plain, round_items(pa, A, d), A, 0, set()).all()
        assert check_round(eng, plain, round_items(pa, A, d), A, 0, {bytes(a) for a in A}).all()
    finally:
        eng.close()
        plain.close()


def test_budget_changes_at_run_time():
    """All 1,000 hold tables at budget 1,024; lowered to 256 the pool shrinks (and the device gets the memory back) and the 256
    used last keep theirs; raised again the tables are rebuilt after use; at budget 0 every member is handed back."""
    privs, addrs = keys(804, 1000)
    eng, plain = make_engine(slots=2, max_validators=1024, key_cache=True, key_table_budget=1024), make_engine(slots=2, max_validators=1024)
    try:
        for e in (eng, plain):
            e.set_validators(0, 1, addrs)
        check_round(eng, plain, round_items(privs, addrs, co.keccak256(b"rt-0")), addrs, 0, set())
        assert eng.key_registry() == (1000, 1000, 1024 * TAB)
        eng.refresh_key_tables()                                  # clears the used flags
        last = np.random.default_rng(1).choice(1000, 256, replace=False)
        check_round(eng, plain, round_items([privs[i] for i in last], addrs[last], co.keccak256(b"rt-1")), addrs, 0,
                    {bytes(a) for a in addrs})
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        eng.set_key_table_budget(256)
        free1 = torch.cuda.mem_get_info()[0]
        assert eng.key_registry() == (1000, 256, 256 * TAB)
        assert free1 - free0 >= 3 * CHUNK - (64 << 20)
        assert ready_set(eng, 0, addrs) == {bytes(addrs[i]) for i in last}
        check_round(eng, plain, round_items(privs, addrs, co.keccak256(b"rt-2")), addrs, 0, {bytes(addrs[i]) for i in last})
        eng.set_key_table_budget(1024)
        assert eng.refresh_key_tables() == 1000                   # reclaim point: all 1,000 used, admitted and built
        assert eng.key_registry() == (1000, 1000, 1024 * TAB)
        check_round(eng, plain, round_items(privs, addrs, co.keccak256(b"rt-3")), addrs, 0, {bytes(a) for a in addrs})
        eng.set_key_table_budget(0)
        assert eng.key_registry() == (1000, 0, 0)
        assert check_round(eng, plain, round_items(privs, addrs, co.keccak256(b"rt-4")), addrs, 0, set()).all()
        assert eng.known_handed_back() == 1000
    finally:
        eng.close()
        plain.close()


def test_edge_keys_evicted_readmitted_and_moved_down():
    """The crafted known-key set of tests/adversarial.py (its coordinate-edge keys: coordinates below 2^256 - p or near p; and the
    keys of the x = r + n forgeries) at a budget 16 below its size.  The keys without a table sign and take tables from 16 others at
    the reclaim point (EVICTED: state 1); those sign and are readmitted; then the budget is lowered, so that kept tables above it
    move down.  After each step every verdict equals a plain engine's and the oracle's, the known-key pass hands back what the
    tables predict -- every forgery among them -- and every edge key holding a table holds the big-int oracle's whole table."""
    pts = A.known_points()
    addrs = known_addrs()
    edge = {bytes(A.known_addr(i)): Q for i, Q in enumerate(pts) if i >= len(A.KNOWN_KEYS)}
    by_key: dict[int, list] = {}
    for v in A.known_vectors():
        by_key.setdefault(v.key_index, []).append(v)
    mixed, _ = known_batch()

    def signing(keys):
        return valid_known_items([v for i in sorted(keys) for v in by_key[i]])

    def check_tables(ready):
        assert ready & set(edge)
        for v in range(len(addrs)):
            a = bytes(addrs[v])
            if a in edge and a in ready:
                check_whole_key_table(eng.key_table(0, v, 0, 17 * 128)[2], edge[a])

    budget = len(pts) - 16
    eng = make_engine(slots=2, max_validators=1024, key_cache=True, key_table_budget=budget)
    plain = make_engine(slots=2, max_validators=1024)
    try:
        for e in (eng, plain):
            e.set_validators(0, 1, addrs)
        assert check_round(eng, plain, signing(range(len(pts))), addrs, 0, set()).all()  # every key learned
        eng.refresh_key_tables()                                  # reclaim point: clears the used flags
        first = ready_set(eng, 0, addrs)
        assert len(first) == budget
        check_tables(first)
        cold = [i for i in range(len(pts)) if bytes(addrs[i]) not in first]
        assert check_round(eng, plain, signing(cold), addrs, 0, first).all()
        eng.refresh_key_tables()                                  # reclaim point: the cold keys take 16 tables
        second = ready_set(eng, 0, addrs)
        evicted = first - second
        assert len(second) == budget and {bytes(addrs[i]) for i in cold} <= second and len(evicted) == 16
        assert evicted & set(edge)
        assert all(eng.key_table(0, v)[0] == 1 for v in range(len(addrs)) if bytes(addrs[v]) in evicted)
        check_tables(second)
        check_round(eng, plain, mixed, addrs, 0, second)
        eng.refresh_key_tables()                                  # every key used alike: nothing moves
        assert ready_set(eng, 0, addrs) == second
        back = [i for i in range(len(pts)) if bytes(addrs[i]) in evicted]
        assert check_round(eng, plain, signing(back), addrs, 0, second).all()
        eng.refresh_key_tables()                                  # reclaim point: the evicted keys are readmitted
        third = ready_set(eng, 0, addrs)
        assert len(third) == budget and evicted <= third
        check_tables(third)
        check_round(eng, plain, mixed, addrs, 0, third)
        eng.set_key_table_budget(budget - 16)                     # kept tables in the top 16 slots move down
        fourth = ready_set(eng, 0, addrs)
        assert len(fourth) == budget - 16 and fourth <= third and eng.key_registry()[1] == budget - 16
        check_tables(fourth)
        check_round(eng, plain, mixed, addrs, 0, fourth)
        assert check_round(eng, plain, signing(range(len(pts))), addrs, 0, fourth).all()
    finally:
        eng.close()
        plain.close()


@pytest.mark.parametrize("rule", [ib.QUORUM_DEFAULT, ib.QUORUM_PREPREPARE, ib.QUORUM_PREPARE])
def test_every_path(rule):
    """Small AUTO batches, large AUTO batches, forced SPLIT and the device-resident entry point (ibft_refresh_key_tables as the
    reclaim point) on a budget below the set, under each quorum rule."""
    privs, addrs = keys(805, 1000)
    eng, plain = make_engine(slots=2, max_validators=1024, key_cache=True, key_table_budget=300), make_engine(slots=2, max_validators=1024)
    try:
        for e in (eng, plain):
            e.set_validators(0, 1, addrs)
        small = round_items(privs[:200], addrs[:200], co.keccak256(b"small"))
        full = round_items(privs, addrs, co.keccak256(b"full"))
        big = np.concatenate([full] * 24)
        check_round(eng, plain, small, addrs, 0, set(), rule)
        eng.refresh_key_tables()
        for items in (small, big, full):
            check_round(eng, plain, items, addrs, 0, ready_set(eng, 0, addrs), rule)
        eng.set_recover_path(ib.Engine.PATH_SPLIT)
        check_round(eng, plain, full, addrs, 0, ready_set(eng, 0, addrs), rule)
        eng.set_recover_path(ib.Engine.PATH_AUTO)
        want = co.verify_batch(big, b"", tables=[addrs], group_table=[0], n_threads=8)
        eng.bind_groups(eng.groups(1, 0, rule))
        t_items = torch.from_numpy(big.view(np.uint8).reshape(-1, 128).copy()).cuda()
        t_arena = torch.zeros(16, dtype=torch.uint8, device="cuda")
        for k in range(3):
            t_bm = torch.zeros((len(big) + 31) // 32, dtype=torch.int32, device="cuda")
            st = torch.cuda.current_stream().cuda_stream
            eng.verify_device(t_items.data_ptr(), len(big), t_arena.data_ptr(), 0, 0, len(big), t_bm.data_ptr(), 0, st)
            torch.cuda.synchronize()
            assert np.array_equal(t_bm.cpu().numpy().view(np.uint32), want), k
            eng.refresh_key_tables()
        eng.bind_groups(None)
        assert eng.key_registry()[1] == 300
    finally:
        eng.close()
        plain.close()


def test_two_lanes():
    """One thread verifies small batches (lane 1) while another replaces tables, refreshes and changes the budget."""
    privs, addrs = keys(806, 512)
    eng = make_engine(slots=4, max_validators=512, key_cache=True, key_table_budget=128)
    try:
        for s in range(4):
            eng.set_validators(s, 1 + s, addrs)
        items = round_items(privs[:96], addrs[:96], co.keccak256(b"lanes"))
        items[5]["s"][31] ^= 1                                    # one rejected signature
        want = co.verify_batch(items, b"", tables=[addrs], group_table=[0], n_threads=8)
        stop, errors = threading.Event(), []

        def verifier():
            try:
                while not stop.is_set():
                    bm, _, _ = eng.verify_batch(items, b"", eng.groups(1, 0))
                    if not np.array_equal(bm, want):
                        errors.append("bitmap")
            except Exception as ex:  # noqa: BLE001 -- reported below
                errors.append(repr(ex))

        t = threading.Thread(target=verifier)
        t.start()
        try:
            for k in range(12):
                eng.set_validators(1 + k % 3, 10 + k, addrs[::-1] if k % 2 else addrs)
                eng.refresh_key_tables()
                eng.set_key_table_budget([128, 16, 0, 512][k % 4])
        finally:
            stop.set()
            t.join()
        assert not errors, errors[:3]
    finally:
        eng.close()
