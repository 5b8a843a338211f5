"""Every verify kernel with each rejection class, each crafted valid item and a valid item of each kind at every signature slot of
its CTA (tests/position_sweep.py), against the oracle's expectations: verdict bits, item status, recovered addresses, the quorum
results and voted sets of every group; the known-key kernels with known, misattributed, flipped, unknown, cancelling and x = r + n
items at every slot and worklists whose length crosses the consumers' CTAs; device-resident shards that start off the CTA grid;
the explain pass over compacted rejections; and a two-device engine."""
import numpy as np
import pytest

import ibft_b200 as ib
import position_sweep as PS
from test_gpu_adversarial import expected_handed_back, sm_count

pytestmark = pytest.mark.gpu
E = ib.Engine
CAP = dict(device=0, max_items=1 << 16, max_payload_bytes=1 << 22, max_groups=512, max_table_slots=2, max_validators=4096)


@pytest.fixture(scope="module")
def S():
    return PS.sweep()


@pytest.fixture(scope="module")
def sms():
    return sm_count()


def set_tables(eng, S, W):
    (a0, p0), (a1, p1) = S.tables(W)
    eng.set_validators(0, 1, a0, p0)
    eng.set_validators(1, 2, a1, p1)


def where(i, W):
    return f"item {i} (block {i // W}, position {i % W})"


def check_groups(eng, res, e, label, voted_sets=True):
    n_val = len(PS.sweep().members)
    for g, (nv, voted, power, hq) in enumerate(e["groups"]):
        r = res[g]
        got = (int(r["n_valid"]), int(r["n_distinct"]), sum(int(r["power"][k]) << (64 * k) for k in range(5)), bool(r["has_quorum"]))
        assert got == (nv, len(voted), power, hq), (label, g, got, (nv, len(voted), power, hq))
        if voted_sets and voted:
            words = eng.voted_bitmap(g, n_val)
            assert set(np.nonzero(PS.bits(words, n_val))[0].tolist()) == voted, (label, g)


def run_and_check(eng, S, items, n_blocks, W, label, arena=None):
    """one host-buffer call with recovered addresses, every output against the expectations"""
    n = len(items)
    groups = eng.groups(S.n_groups(n_blocks), slot=S.group_slots(n_blocks))
    bm, res, rec = eng.verify_batch(items, S.arena if arena is None else arena, groups, want_recovered=True)
    st = eng.last_item_status(n)
    e = S.expect(items, n_blocks, W)
    got = PS.bits(bm, n)
    bad = np.nonzero(got != e["bit"])[0]
    assert len(bad) == 0, (label, [(where(int(i), W), bool(got[i])) for i in bad[:6]])
    bad = np.nonzero(st != e["status"])[0]
    assert len(bad) == 0, (label, "status", [where(int(i), W) for i in bad[:6]])
    bad = np.nonzero((rec != e["rec"]).any(axis=1))[0]
    assert len(bad) == 0, (label, "recovered", [where(int(i), W) for i in bad[:6]])
    check_groups(eng, res, e, label)
    return bm, res, rec


@pytest.fixture(scope="module")
def eng(S):
    e = E(**CAP)
    yield e
    e.close()


# (geometry, path, window)
RECOVER = [("thread32", E.PATH_THREAD, 32), ("thread128", E.PATH_THREAD, 128), ("quad", E.PATH_QUAD, 32), ("split", E.PATH_SPLIT, 96),
           ("qsplit", E.PATH_QSPLIT, 96)]


@pytest.mark.parametrize("geom,path,W", RECOVER, ids=[r[0] for r in RECOVER])
def test_every_class_at_every_slot(eng, S, sms, geom, path, W):
    """patterns (a), (b) and (c) on one forced recover kernel.  k_recover<128> needs more than SMs x 256 items: its calls are
    padded with fillers after the blocks, and its tails are preceded by a CTA-aligned run of fillers."""
    eng.set_recover_path(path)
    set_tables(eng, S, W)
    big = sms * 256 + 1
    fit = (lambda it, nb: S.pad(it, nb, big)) if geom == "thread128" else (lambda it, nb: it)
    if geom == "thread32":
        assert W * W <= sms * 256
    for name in S.names:
        run_and_check(eng, S, fit(S.pattern_a(W, name), W), W, W, (geom, "a", name))
    run_and_check(eng, S, fit(S.pattern_b(W), W), W, W, (geom, "b"))
    if geom == "thread128":
        k = -(-big // 128) * 128
        for p in range(W):
            name = S.names[p % len(S.names)]
            it = S.prefix(S.pattern_c(W, name, p), 1, k)
            run_and_check(eng, S, it, 1, W, (geom, "c", name, p))
    else:
        for name in S.names:
            for p in range(W):
                run_and_check(eng, S, S.pattern_c(W, name, p), 1, W, (geom, "c", name, p))
    eng.set_recover_path(E.PATH_AUTO)


def test_auto_in_each_range(eng, S, sms):
    """AUTO at one size in each of its ranges: four-lane chain + helper (<= SMs x 48), the four-piece upload on chain + helper warps
    (<= SMs x 96), chain + helper warps (<= SMs x 192), one thread per signature (beyond)"""
    W = 96
    eng.set_recover_path(E.PATH_AUTO)
    set_tables(eng, S, W)
    cat = np.concatenate([S.pattern_a(W, name) for name in S.names[:4]])
    for n in (sms * 48 - 7, sms * 72 + 5, sms * 150 + 3, sms * 192 + 77):
        it = cat[:n] if n <= len(cat) else S.pad(cat, W, n)
        run_and_check(eng, S, it, W, W, ("auto", n))


# ------------------------------------------------------------------------------------------------------------ key registry
@pytest.fixture(scope="module")
def known(S):
    """a key-registry engine and a plain one over the same tables; the registry has learned the fillers', the signers of the
    known classes' and the two crafted keys' keys (every validator but the unknown signer and the fresh ones).  The keys are
    learned by a call that asks for the recovered addresses, which takes the plain recover kernels: no worklist is involved before
    the tests that sweep them."""
    eng, plain = E(**CAP, key_cache=True), E(**CAP)
    for e in (eng, plain):
        set_tables(e, S, 96)
    warm = np.concatenate([S.fillers, S.classes["valid_low_s"], S.known_warm[0], S.known_warm[1],
                           PS.wl.make_item(PS.wl.sign(S.reason_vs.keys[2], b"\x01" * 32), S.reason_vs.addrs[2], 0, b"\x01" * 32)])
    groups = eng.groups(1, slot=0)
    bm, _, _ = eng.verify_batch(warm, b"", groups, want_recovered=True)
    assert PS.bits(bm, len(warm)).all()
    eng.refresh_key_tables()
    known_signers = {bytes(a) for a in warm["signer"]}
    yield eng, plain, known_signers
    eng.close()
    plain.close()


KNOWN = [("verify_known32", E.PATH_THREAD, 32), ("verify_known128", E.PATH_THREAD, 128), ("verify_split", E.PATH_SPLIT, 96)]


@pytest.mark.parametrize("geom,path,W", KNOWN, ids=[k[0] for k in KNOWN])
def test_known_key_classes_at_every_slot(known, S, sms, geom, path, W):
    """k_verify_known<32>, k_verify_known<128> (padded past SMs x 256) and k_verify_split with each known-key class at every slot:
    the bitmap against the oracle, the quorum results byte for byte against a plain engine and against the expectations, and the
    number of items handed to the recover pass exactly the expected one"""
    eng, plain, known_signers = known
    for e in (eng, plain):
        e.set_recover_path(path)
        set_tables(e, S, W)
    members = set(S.members)
    for name, odd in S.known_classes.items():
        if name == "known_no_table":              # test_known_key_without_table_at_every_slot
            continue
        items = np.concatenate([S.block(W, p, W, odd, p, "a") for p in range(W)])
        if geom == "verify_known128":
            items = S.pad(items, W, sms * 256 + 1)
        groups = eng.groups(S.n_groups(W), slot=S.group_slots(W))
        bm, res, _ = eng.verify_batch(items, b"", groups)
        handed = eng.known_handed_back()
        e = S.expect(items, W, W)
        got = PS.bits(bm, len(items))
        bad = np.nonzero(got != e["bit"])[0]
        assert len(bad) == 0, (geom, name, [(where(int(i), W), bool(got[i])) for i in bad[:6]])
        check_groups(eng, res, e, (geom, name))
        bp, rp, _ = plain.verify_batch(items, b"", groups)
        assert np.array_equal(bm, bp) and res.tobytes() == rp.tobytes(), (geom, name)
        assert handed == expected_handed_back(items, 0, members, e["bit"], known_signers, split=path == E.PATH_SPLIT), (geom, name)
        if name != "known_valid" and name != "unknown_signer":
            assert handed == W, (geom, name)
        if name == "unknown_signer":              # recovered, hence learned: known from the next geometry on
            known_signers.add(bytes(odd["signer"][0]))
            eng.refresh_key_tables()
    for e in (eng, plain):
        e.set_recover_path(E.PATH_AUTO)


def test_known_key_without_table_at_every_slot(S, sms):
    """A member whose key is known but whose comb table a small key-table budget evicted, at every slot of k_verify_known<32>,
    <128> and k_verify_split among fillers whose tables are kept: the known-key pass must hand exactly that member's items back
    (expected_handed_back with the member counted as not known), and the recover pass must accept them -- bitmap against the
    oracle's expectations and a plain engine, quorum results byte for byte."""
    vs = S.reason_vs
    victim = bytes(S.known_classes["known_no_table"]["signer"][0])
    dig = b"\x02" * 32
    others = np.concatenate([S.fillers] + [PS.wl.make_item(PS.wl.sign(vs.keys[i], dig), vs.addrs[i], 0, dig) for i in (2, 3)])
    learn_victim = PS.wl.make_item(PS.wl.sign(vs.keys[1], dig), vs.addrs[1], 0, dig)
    want_tabled = {bytes(a) for a in others["signer"]}
    eng, plain = E(**CAP, key_cache=True, key_table_budget=4 * len(others)), E(**CAP)
    members = set(S.members)
    try:
        for e in (eng, plain):
            set_tables(e, S, 128)
        bm, _, _ = eng.verify_batch(np.concatenate([others, learn_victim]), b"", eng.groups(1, slot=0), want_recovered=True)
        assert PS.bits(bm, len(others) + 1).all()
        for geom, path, W in KNOWN:
            for e in (eng, plain):
                e.set_recover_path(E.PATH_AUTO)
                set_tables(e, S, W)
            eng.set_key_table_budget(4 * len(others))
            eng.refresh_key_tables()                          # every learned key tabled; the used flags cleared
            bm, _, _ = eng.verify_batch(others, b"", eng.groups(1, slot=0))   # every key but the victim's used since
            assert PS.bits(bm, len(others)).all() and eng.known_handed_back() == 0, geom
            eng.set_key_table_budget(len(others))             # room for the used ones only: the victim's table goes
            tabled = {bytes(S.members[v]) for v in range(len(S.members)) if eng.key_table(0, v)[0] == 2}
            assert tabled == want_tabled, geom
            for e in (eng, plain):
                e.set_recover_path(path)
            items = np.concatenate([S.block(W, p, W, S.known_classes["known_no_table"], p, "a") for p in range(W)])
            if geom == "verify_known128":
                items = S.pad(items, W, sms * 256 + 1)
            groups = eng.groups(S.n_groups(W), slot=S.group_slots(W))
            bm, res, _ = eng.verify_batch(items, b"", groups)
            handed = eng.known_handed_back()
            e = S.expect(items, W, W)
            got = PS.bits(bm, len(items))
            bad = np.nonzero(got != e["bit"])[0]
            assert len(bad) == 0, (geom, [(where(int(i), W), bool(got[i])) for i in bad[:6]])
            check_groups(eng, res, e, (geom, "known_no_table"))
            bp, rp, _ = plain.verify_batch(items, b"", groups)
            assert np.array_equal(bm, bp) and res.tobytes() == rp.tobytes(), geom
            assert handed == expected_handed_back(items, 0, members, e["bit"], want_tabled, split=path == E.PATH_SPLIT) == W, geom
    finally:
        eng.close()
        plain.close()


WORKLIST_COUNTS = [1, 23, 24, 25, 47, 48, 49, 95, 96, 97, 127, 128, 129]


@pytest.mark.parametrize("consumer", ["qsplit", "recover128_long_payloads", "recover128_large"])
def test_worklist_counts_across_consumer_ctas(known, S, sms, consumer):
    """k items handed back per call, k crossing k_recover_qsplit's 24-signature CTA and recover_kernel<128>'s CTA: valid signatures
    of validators whose keys are not known yet, spread over a batch of known fillers.  Every one must be recovered (bit 1) and the
    count handed back must be k.  qsplit: a small batch of short items; recover_kernel<128>: a small batch of long PAYLOAD items
    (more than 256 arena bytes per item), and a batch beyond SMs x 256."""
    eng, plain, known_signers = known
    eng.set_recover_path(E.PATH_THREAD)
    offset = {"qsplit": 0, "recover128_long_payloads": 900, "recover128_large": 1800}[consumer]
    n = 300 if consumer != "recover128_large" else sms * 256 + 300
    long_payloads = consumer == "recover128_long_payloads"
    fresh = S.fresh
    used = 0
    for k in WORKLIST_COUNTS:
        items = np.tile(S.fillers, -(-n // len(S.fillers)))[:n].copy()
        items["group"] = 0
        pos = np.linspace(0, n - 1, k).astype(int) if k > 1 else np.array([n // 2])
        assert len(set(pos.tolist())) == k
        dig = bytes([k]) * 32
        arena = bytearray()
        for t, i in enumerate(pos):
            v = offset + used + t
            if long_payloads:                     # PAYLOAD items of 600 to 1,200 bytes: the consumer hashes them
                msg = bytes([k, t & 0xFF]) * (300 + (t * 37) % 300)
                items[i] = PS.wl.make_item(PS.wl.sign(fresh.keys[v], PS.co.keccak256(msg)), fresh.addrs[v], PS.wl.KIND_PAYLOAD, b"", 0,
                                           len(arena), len(msg))[0]
                arena.extend(msg)
            else:
                items[i] = PS.wl.make_item(PS.wl.sign(fresh.keys[v], dig), fresh.addrs[v], 0, dig)[0]
        if long_payloads:
            arena.extend(bytes(max(0, 257 * n - len(arena))))   # more than 256 arena bytes per item: recover_kernel<128>
        used += k
        groups = eng.groups(1, slot=0)
        bm, res, _ = eng.verify_batch(items, bytes(arena), groups)
        assert PS.bits(bm, n).all(), (consumer, k, np.nonzero(~PS.bits(bm, n))[0][:6])
        assert eng.known_handed_back() == k, (consumer, k)
        assert int(res[0]["n_valid"]) == n, (consumer, k)
    assert used <= 900
    eng.set_recover_path(E.PATH_AUTO)


# ------------------------------------------------------------------------------------------------------------ device shards
@pytest.mark.parametrize("path", [E.PATH_QSPLIT, E.PATH_SPLIT, E.PATH_THREAD], ids=["qsplit", "split", "thread"])
def test_device_shards_off_the_cta_grid(eng, S, path):
    """n = 32 + 96 k + 17 items through verify_device as the shard [32, n) and as the shards [0, 64) + [64, n): the CTA grids
    start off the 96- and 24-signature grids and hi = n is ragged; then quorum_mark_device per shard + quorum_merge_device"""
    import torch
    W = 96
    eng.set_recover_path(path)
    set_tables(eng, S, W)
    cat = np.concatenate([S.pattern_b(W)[:W * 2], S.pattern_a(W, "u1_zero_z0")[:W * 2]])
    n = 32 + 96 * 3 + 17
    items = cat[:n].copy()
    ng = S.n_groups(W)
    groups = eng.groups(ng, slot=S.group_slots(W))
    eng.bind_groups(groups)
    t_items = torch.from_numpy(items.view(np.uint8).reshape(-1, 128).copy()).cuda()
    t_arena = torch.from_numpy(np.frombuffer(S.arena, np.uint8).copy()).cuda()
    st = torch.cuda.current_stream().cuda_stream
    Wp = eng.quorum_partial_words()
    for shards in ([(32, n)], [(0, 64), (64, n)]):
        t_bm = torch.zeros((n + 31) // 32, dtype=torch.int32, device="cuda")
        parts = torch.full((len(shards), Wp), -1, dtype=torch.int32, device="cuda")
        for lo, hi in shards:
            eng.verify_device(t_items.data_ptr(), n, t_arena.data_ptr(), t_arena.numel(), lo, hi, t_bm.data_ptr(), 0, st)
        for r, (lo, hi) in enumerate(shards):
            eng.quorum_mark_device(t_items.data_ptr(), n, lo, hi, t_bm.data_ptr(), parts[r].data_ptr(), st)
        t_res = torch.zeros(ng * ib.RESULT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
        eng.quorum_merge_device(parts.data_ptr(), len(shards), Wp, t_res.data_ptr(), st)
        torch.cuda.synchronize()
        lo0 = shards[0][0]
        got = PS.bits(t_bm.cpu().numpy().view(np.uint32), n)
        sub = items[lo0:]
        e = S.expect(sub, W, W)
        want = np.concatenate([np.zeros(lo0, bool), e["bit"]])
        bad = np.nonzero(got != want)[0]
        assert len(bad) == 0, (path, shards, bad[:8])
        res = t_res.cpu().numpy().view(ib.RESULT_DTYPE)
        check_groups(eng, res, e, (path, shards), voted_sets=False)
    eng.bind_groups(None)
    eng.set_recover_path(E.PATH_AUTO)


# ------------------------------------------------------------------------------------------------------------ explain
@pytest.mark.parametrize("W", [32, 96])
def test_explain_compacted_rejections(eng, S, W):
    """explain_batch behind a verify call: pattern (b) compacts to whole one-warp CTAs of rejected items with one accepted item
    missing at every slot; pattern (a) of each class to one item per block.  Reasons = the reference; recovered addresses = the
    reference's for the rejected items (the accepted ones are not explained: zero)."""
    set_tables(eng, S, W)
    batches = [S.pattern_b(W)] + [S.pattern_a(W, name) for name in S.names]
    for items in batches:
        groups = eng.groups(S.n_groups(W), slot=S.group_slots(W))
        bm, _, _ = eng.verify_batch(items, S.arena, groups)
        reasons, rec = eng.explain_batch(items, S.arena, groups, bitmap=bm)
        e = S.expect(items, W, W)
        bad = np.nonzero(reasons != e["reason"])[0]
        assert len(bad) == 0, [(where(int(i), W), int(reasons[i]), int(e["reason"][i])) for i in bad[:6]]
        assert np.array_equal(rec, np.where(e["bit"][:, None], 0, e["xrec"]))   # accepted items: REASON_OK without device work


# ------------------------------------------------------------------------------------------------------------ two devices
def test_two_device_engine_matches(S):
    """an engine over devices [0, 0] on pattern (a), qsplit and one thread per signature: byte for byte the one-device results"""
    W = 96
    multi, single = E(devices=[0, 0], **CAP), E(**CAP)
    try:
        for e in (multi, single):
            set_tables(e, S, W)
        for path in (E.PATH_QSPLIT, E.PATH_THREAD):
            for e in (multi, single):
                e.set_recover_path(path)
            for name in S.names:
                items = S.pattern_a(W, name)
                got = run_and_check(multi, S, items, W, W, ("multi", path, name))
                groups = single.groups(S.n_groups(W), slot=S.group_slots(W))
                want = single.verify_batch(items, S.arena, groups, want_recovered=True)
                assert all(a.tobytes() == b.tobytes() for a, b in zip(got, want)), (path, name)
    finally:
        multi.close()
        single.close()
