"""One key registry across the devices of a multi-device engine (ibft_engine_create_multi with IBFT_FLAG_KEY_CACHE).

After every host-buffer call the devices adopt the keys any device learned (k_adopt_peer_keys, each key checked against the
entry's address on the device), then build their tables.  Every sub-engine must therefore hold what a single-device engine
fed the same calls holds: the same keys and states, the same comb tables, the same tables under a budget, and the same
handed-back count from the second round on.  On one GPU the sub-engines repeat ordinal 0."""
import importlib
import os
import threading

import numpy as np
import pytest

import adversarial as A
import ibft_b200 as ib
from oracle import coracle as co
from test_emul_key_share import key_check_cases, oracle_accepts
from test_gpu_adversarial import ENTRIES, POSITIONS, bits, known_addrs, known_batch

pytestmark = pytest.mark.gpu
sharding = importlib.import_module("go-ibft_b200.sharding")

KW = dict(max_items=1 << 15, max_payload_bytes=1 << 23, max_groups=4, max_table_slots=2, max_validators=10_000, key_cache=True)
ROUNDS = 5


@pytest.fixture(scope="module")
def rnd():
    """config 3's COMMIT round (10,000 validators, slot 0) plus the crafted known-key batch (the coordinate-edge and x = r + n
    forgery keys with their rejected variants, slot 1, the last group), its oracle bitmap and the members of each slot"""
    d = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "config3.npz"))
    c3 = np.ascontiguousarray(d["items"]).view(ib.ITEM_DTYPE).reshape(-1)
    kitems, _ = known_batch()
    kaddrs = known_addrs()
    kwant = bits(co.verify_batch(kitems, b"", tables=[kaddrs], group_table=[0], n_threads=8), len(kitems))
    n_g = len(d["groups"])
    kitems = kitems.copy()
    kitems["group"] = n_g
    items = np.concatenate([c3, kitems]).view(ib.ITEM_DTYPE)
    want = np.concatenate([bits(d["bitmap"], len(c3)), kwant])
    return dict(items=items, arena=d["arena"].tobytes(), want=want, addrs=d["addrs"], powers=d["powers"], height=int(d["meta"][2]),
                kaddrs=kaddrs, n_groups=n_g + 1, n_c3=len(c3))


def setup(e, r):
    e.set_validators(0, r["height"], r["addrs"], r["powers"])
    e.set_validators(1, 3, r["kaddrs"], None)
    return e.groups(r["n_groups"], slot=[0] * (r["n_groups"] - 1) + [1])


def subs(e):
    return [e.sub(k) for k in range(e.device_count())]


def sample_members(r):
    """(slot, validator) pairs whose whole comb table is compared: a spread of config 3 and every coordinate-edge key"""
    return [(0, int(v)) for v in np.linspace(0, len(r["addrs"]) - 1, 12).astype(int)] + \
           [(1, v) for v in range(len(A.KNOWN_KEYS), len(r["kaddrs"]))]


def snapshot(e, r, tables=True):
    """(registry summary, state and key of every member of both slots, whole comb tables of the sample)"""
    reg = e.key_registry()
    rows = []
    for slot, n in ((0, len(r["addrs"])), (1, len(r["kaddrs"]))):
        for v in range(n):
            st, key, _ = e.key_table(slot, v)
            rows.append((st, key.tobytes() if st else b""))
    tabs = []
    if tables:
        for slot, v in sample_members(r):
            st, _, _ = e.key_table(slot, v)
            tabs.append(e.key_table(slot, v, 0, POSITIONS * ENTRIES)[2].tobytes() if st == 2 else None)
    return reg, rows, tabs


def perms(n, rounds, seed=7):
    rng = np.random.default_rng(seed)
    return [rng.permutation(n) for _ in range(rounds)]


def run(e, r, groups, idx):
    bm, res, _ = e.verify_batch(r["items"][idx], r["arena"], groups)
    return bm.tobytes(), res.tobytes()


def test_registries_match_a_single_engine_round_after_round(rnd):
    """Five permuted rounds on [0, 0] and [0] * 4: after every call every sub-engine holds the single engine's registry, keys,
    states and sampled comb tables; from round 2 on the known-key pass hands back only the rejects, as on the single engine."""
    r = rnd
    order = perms(len(r["items"]), ROUNDS)
    single = ib.Engine(device=0, **KW)
    want = []
    try:
        g = setup(single, r)
        for idx in order:
            out = run(single, r, g, idx)
            assert np.array_equal(bits(np.frombuffer(out[0], np.uint32), len(idx)), r["want"][idx])
            want.append((out, single.known_handed_back(), snapshot(single, r)))
    finally:
        single.close()
    rejects = int((~r["want"]).sum())
    assert want[-1][1] <= rejects
    for devs in ([0, 0], [0] * 4):
        e = ib.Engine(devices=devs, **KW)
        try:
            g = setup(e, r)
            for k, idx in enumerate(order):
                out = run(e, r, g, idx)
                w_out, w_handed, w_snap = want[k]
                assert out == w_out, (devs, k)
                assert e.known_handed_back() == w_handed, (devs, k)
                for j, s in enumerate(subs(e)):
                    got = snapshot(s, r)
                    assert got[0] == w_snap[0], (devs, k, j)
                    assert got[1] == w_snap[1], (devs, k, j)
                    assert got[2] == w_snap[2], (devs, k, j)
        finally:
            e.close()


def _validator_of(r):
    where = {bytes(a): i for i, a in enumerate(r["addrs"])}
    return np.array([where.get(bytes(it["signer"]), len(r["addrs"])) for it in r["items"][: r["n_c3"]]])


def test_disjoint_shards_teach_every_device(rnd):
    """Config 3's items sorted by validator: device k of [0] * 4 verifies (nearly) only its own quarter of the validators, and
    after the one call every device knows every key the single engine knows."""
    r = rnd
    v_of = _validator_of(r)
    idx = np.argsort(v_of, kind="stable")
    single = ib.Engine(device=0, **KW)
    e = ib.Engine(devices=[0] * 4, **KW)
    try:
        gs, ge = setup(single, r), setup(e, r)
        seen = [set(v_of[idx[slice(*sharding.shard_bounds(r["n_c3"], 4, k))]].tolist()) for k in range(4)]
        assert all(len(s) < 0.3 * len(r["addrs"]) for s in seen)
        items = r["items"][idx]
        assert single.verify_batch(items, r["arena"], gs)[0].tobytes() == e.verify_batch(items, r["arena"], ge)[0].tobytes()
        want = snapshot(single, r, tables=False)
        assert sum(st != 0 for st, _ in want[1]) > 9000
        for s in subs(e):
            assert snapshot(s, r, tables=False) == want
    finally:
        single.close()
        e.close()


def test_lead_only_calls_teach_every_device(rnd):
    """Calls of fewer than 1,024 items run on the lead alone; their keys reach the other devices before the call returns, so
    the next large call hands back only what the single engine hands back."""
    r = rnd
    single = ib.Engine(device=0, **KW)
    e = ib.Engine(devices=[0, 0, 0], **KW)
    try:
        gs, ge = setup(single, r), setup(e, r)
        order = perms(len(r["items"]), 1, seed=3)[0]
        first = True
        for lo in range(0, len(order), 1000):
            idx = order[lo:lo + 1000]
            assert run(single, r, gs, idx) == run(e, r, ge, idx)
            if first:
                want = snapshot(single, r, tables=False)
                assert sum(st != 0 for st, _ in want[1]) > 300
                for s in subs(e):
                    assert snapshot(s, r, tables=False) == want
                first = False
        idx = perms(len(r["items"]), 1, seed=4)[0]
        assert run(single, r, gs, idx) == run(e, r, ge, idx)
        assert e.known_handed_back() == single.known_handed_back() <= int((~r["want"]).sum())
        want = snapshot(single, r)
        for s in subs(e):
            assert snapshot(s, r) == want
    finally:
        single.close()
        e.close()


def test_bounded_registry_keeps_the_same_tables(rnd):
    """A 300-table budget: permuted calls alternate with set_validators reclaim points.  The validators holding a table are the
    same on every sub-engine and the single engine's, and the pool stays within the budget."""
    r = rnd
    single = ib.Engine(device=0, **KW)
    e = ib.Engine(devices=[0, 0], **KW)
    budget = 300
    try:
        gs, ge = setup(single, r), setup(e, r)
        single.set_key_table_budget(budget)
        e.set_key_table_budget(budget)
        order = perms(len(r["items"]), 4, seed=11)
        for k, idx in enumerate(order):
            # each round sees a different part of the validators, so the ranking by use moves
            part = idx[: len(idx) * (k + 2) // 6]
            assert run(single, r, gs, part) == run(e, r, ge, part), k
            want = snapshot(single, r, tables=False)
            ready = [i for i, (st, _) in enumerate(want[1]) if st == 2]
            assert 0 < len(ready) <= budget
            for s in subs(e):
                got = snapshot(s, r, tables=False)
                assert [i for i, (st, _) in enumerate(got[1]) if st == 2] == ready, k
                assert got == want, k
                assert got[0][2] <= budget * 136 * 1024
            for eng in (single, e):
                setup(eng, r)                       # a reclaim point
        assert single.refresh_key_tables() == e.refresh_key_tables()
        want = snapshot(single, r, tables=False)
        for s in subs(e):
            assert snapshot(s, r, tables=False) == want
    finally:
        single.close()
        e.close()


def test_small_and_bulk_lane_calls_at_once(rnd):
    """Two threads on [0, 0] while keys are being learned: one makes lead-only small-lane calls, the other bulk-lane calls of
    every item.  No deadlock, every output the single engine's, and after refresh_key_tables() the registries agree."""
    r = rnd
    single = ib.Engine(device=0, **KW)
    e = ib.Engine(devices=[0, 0], **KW)
    try:
        gs, ge = setup(single, r), setup(e, r)
        n = len(r["items"])
        small = [np.arange(lo, min(n, lo + 700)) for lo in range(0, n, 700)]
        bulk = perms(n, 3, seed=5)
        assert len(bulk[0]) > 16384                   # more than the small lane holds
        want = {("s", k): run(single, r, gs, idx) for k, idx in enumerate(small)}
        want.update({("b", k): run(single, r, gs, idx) for k, idx in enumerate(bulk)})
        got, errs = {}, []

        def call(tag, batches):
            try:
                for k, idx in enumerate(batches):
                    got[(tag, k)] = run(e, r, ge, idx)
            except Exception as ex:  # noqa: BLE001
                errs.append(ex)
        th = [threading.Thread(target=call, args=("s", small), daemon=True),
              threading.Thread(target=call, args=("b", bulk), daemon=True)]
        for t in th:
            t.start()
        for t in th:
            t.join(timeout=600)
        assert not any(t.is_alive() for t in th), "deadlock"
        assert not errs, errs
        assert got == want
        assert e.refresh_key_tables() == single.refresh_key_tables()
        want = snapshot(single, r)
        for s in subs(e):
            assert snapshot(s, r) == want
    finally:
        single.close()
        e.close()


def test_device_key_check_matches_the_emulation():
    """IBFT_DBG_KEY_ADDRESS runs key_matches_address on the device: the answers of tests/test_emul_key_share.py's set, which the
    host emulation gives too."""
    cases = key_check_cases()
    e = ib.Engine(device=0, max_items=64, max_payload_bytes=1 << 10, max_groups=1, max_table_slots=1, max_validators=16)
    try:
        out = e.debug_op("KEY_ADDRESS", [x for _, x, _, _ in cases], [y for _, _, y, _ in cases], [a + bytes(44) for *_, a in cases])
        for (tag, x, y, a), o in zip(cases, out):
            assert o[0] == int(oracle_accepts(x, y, a)), tag
        assert sum(o[0] for o in out) == sum(oracle_accepts(x, y, a) for _, x, y, a in cases) > 0
    finally:
        e.close()
