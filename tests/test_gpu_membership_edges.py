"""The signer lookup at table-size and address-order edges (tests/membership_edges.py) on every path that looks a signer up,
against a dict from address to index (go-ibft's map): bitmaps, recovered addresses, per-group results and voted sets on the four
recover kernels and AUTO, the known-key kernels and the key registry entry by entry, k_quorum_mark's own lookup of raw frames,
the reject reasons, a multi-device engine, max_groups groups packed back to back, and the C++ host mirror.  Also: a table that
lists an address twice is refused, and nothing changes."""
import functools
import importlib

import numpy as np
import pytest
import torch

import explain_oracle as eo
import ibft_b200 as ib
import membership_edges as me
import workloads as wl
from oracle import coracle as co
from oracle import ibft_logic as L
from oracle import ibft_proto as ip
from oracle import secp256k1 as ec
from test_gpu_adversarial import sm_count
from test_gpu_exchange_ranks import DeviceBatch, assert_results
from test_gpu_host import oracle_backend

pytestmark = pytest.mark.gpu
host = importlib.import_module("go-ibft_b200.host")
PATHS = {"thread": ib.Engine.PATH_THREAD, "quad": ib.Engine.PATH_QUAD, "split": ib.Engine.PATH_SPLIT, "qsplit": ib.Engine.PATH_QSPLIT}
STRIDE = me.MAX_VALIDATORS // 32
ERR_INVALID_ARG = 1  # IBFT_ERR_INVALID_ARG


def params(**kw):
    T = me.tables()
    return dict(dict(device=0, max_items=1 << 16, max_payload_bytes=1 << 20, max_groups=len(T), max_table_slots=len(T),
                     max_validators=me.MAX_VALIDATORS), **kw)


def load(e):
    for slot, t in enumerate(me.tables()):
        e.set_validators(slot, me.HEIGHT, t.addr_array(), t.power_array())
    return e


def groups_of(e, rule=me.DEFAULT):
    T = me.tables()
    return e.groups(len(T), list(range(len(T))), rule=rule, proposer=[t.proposer for t in T])


def bits(bm, n):
    return np.unpackbits(np.ascontiguousarray(bm).view(np.uint8), bitorder="little")[:n].astype(bool)


def tile(b: me.Batch, n: int) -> me.Batch:
    reps = -(-n // len(b.items))
    return me.Batch(np.tile(b.items, reps)[:n], (b.tags * reps)[:n], (b.recovered * reps)[:n])


def recovered_of(b: me.Batch) -> np.ndarray:
    return np.frombuffer(b"".join(r or bytes(20) for r in b.recovered), np.uint8).reshape(-1, 20)


@functools.lru_cache(maxsize=None)
def base():
    return me.digest_batch()


def check_call(e, b: me.Batch, rule=me.DEFAULT, what=""):
    """one host-buffer call against the dict reference: bitmap, per-group results and voted sets"""
    want_bits, want_res, want_voted = me.reference(b, rule=rule)
    bm, res, _, voted = e.verify_batch_ex(b.items, b"", groups_of(e, rule), voted_stride_words=STRIDE)
    assert np.array_equal(bits(bm, len(b.items)), want_bits), what
    assert_results(res, want_res, what)
    assert np.array_equal(voted, me.voted_words(want_voted)), what
    return bm


# ------------------------------------------------------------------------------------------- recover paths and AUTO
@pytest.mark.parametrize("path", list(PATHS))
def test_lookup_edges_on_every_recover_kernel(path):
    e = load(ib.Engine(**params()))
    try:
        e.set_recover_path(PATHS[path])
        b = base()
        for rule in (me.DEFAULT, me.PREPREPARE, me.PREPARE):
            check_call(e, b, rule, (path, rule))
        bm, _, rec = e.verify_batch(b.items, b"", groups_of(e), want_results=False, want_recovered=True)
        assert np.array_equal(rec, recovered_of(b)), path
    finally:
        e.close()


def test_lookup_edges_through_auto():
    """<= SMs x 48 (four-lane chain + helper), the four-piece range (SMs x 48, SMs x 96], the chain + helper range (SMs x 96,
    SMs x 192], > SMs x 192 (one thread per signature): the batch replicated to one size in each"""
    sms = sm_count()
    e = load(ib.Engine(**params()))
    try:
        for n in (sms * 24 - 5, sms * 72 + 3, sms * 144 + 7, sms * 192 + 40):
            b = tile(base(), n)
            check_call(e, b, me.PREPARE, n)
            bm, _, rec = e.verify_batch(b.items, b"", groups_of(e), want_results=False, want_recovered=True)
            assert np.array_equal(bits(bm, n), me.reference(b)[0]) and np.array_equal(rec, recovered_of(b)), n
    finally:
        e.close()


def test_packed_groups_keep_their_votes():
    """max_groups groups in one call, on tables of n = 0, 1 and 31 (mod 32) whose signer is validator n - 1: the voted sets lie
    back to back, and the vote for validator n - 1 of group g must not reach group g + 1"""
    T = me.tables()
    edge = [g for g, t in enumerate(T) if t.n % 32 in (0, 1, 31) and t.index[t.signer_addr] == t.n - 1]
    assert {T[g].n % 32 for g in edge} == {0, 1, 31}
    e = load(ib.Engine(**params()))
    try:
        assert len(groups_of(e)) == e.params.max_groups
        check_call(e, base())
        _, _, voted = me.reference(base())
        for g, t in enumerate(T):
            assert np.array_equal(e.voted_bitmap(g, t.n), me.voted_words(voted)[g, : (t.n + 31) // 32]), g
    finally:
        e.close()


# ------------------------------------------------------------------------------------------------------ key registry
def check_registry(e):
    """every signer's entry holds exactly its key; every other member's entry (decoys, the absent signers' neighbours, filler,
    the zero address) is still unknown"""
    for slot, t in enumerate(me.tables()):
        for v, a in enumerate(t.addrs):
            st, key, _ = e.key_table(slot, v)
            if a == t.signer_addr:
                x = sum(int(key[i]) << (32 * i) for i in range(8))
                y = sum(int(key[8 + i]) << (32 * i) for i in range(8))
                assert st in (1, 2) and ec.pubkey_to_address((x, y)) == a, (slot, v)
            else:
                assert st == 0, (slot, v, a.hex())


@pytest.mark.parametrize("budget", [None, 4], ids=["unbounded", "budget4"])
def test_key_registry_learns_only_the_signers(budget):
    sms = sm_count()
    e = load(ib.Engine(**params(key_cache=True, key_table_budget=budget)))
    try:
        b = base()
        check_call(e, b, me.DEFAULT, "learn")
        e.refresh_key_tables()
        check_call(e, b, me.PREPARE, "refresh")
        # k_verify_known<32> (AUTO, one-warp CTAs), k_verify_known<128> (AUTO above SMs x 256), forced SPLIT (k_verify_split),
        # and the four-piece AUTO range
        for path, n in ((ib.Engine.PATH_AUTO, sms * 24 - 5), (ib.Engine.PATH_AUTO, sms * 256 + 100),
                        (ib.Engine.PATH_SPLIT, len(b.items)), (ib.Engine.PATH_AUTO, sms * 72 + 3)):
            e.set_recover_path(path)
            check_call(e, tile(b, n), me.DEFAULT, (path, n))
        e.set_recover_path(ib.Engine.PATH_AUTO)
        check_registry(e)
    finally:
        e.close()


# -------------------------------------------------------------------------------------------- device-resident quorum
def test_quorum_mark_looks_up_frame_signers():
    """verify_device + quorum_mark_device on IBFT_KIND_WIRE frames (k_quorum_mark resolves the signer from the frame), then
    quorum_merge_device over two 32-aligned shards that split one group"""
    wb, arena = me.wire_batch()
    n = len(wb.items)
    want_bits, want_res, want_voted = me.reference(wb)
    grp = wb.items["group"]
    mid = next(m for m in range(32 * (n // 64), n, 32) if grp[m - 1] == grp[m])
    e = load(ib.Engine(**params()))
    try:
        groups = groups_of(e)
        bm, res, _, voted = e.verify_batch_ex(wb.items, arena, groups, voted_stride_words=STRIDE)
        assert np.array_equal(bits(bm, n), want_bits)
        assert_results(res, want_res, "host-buffer")
        assert np.array_equal(voted, me.voted_words(want_voted))
        db = DeviceBatch(wb.items, arena)
        t_bm = torch.zeros((n + 31) // 32, dtype=torch.int32, device="cuda")
        t_res = torch.zeros(len(groups) * ib.RESULT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
        e.bind_groups(groups)
        W = e.quorum_partial_words()    # of the bound groups
        t_parts = torch.zeros((2, W), dtype=torch.int32, device="cuda")
        e.verify_device(db.items.data_ptr(), n, db.arena.data_ptr(), db.arena_len, 0, n, t_bm.data_ptr())
        for r, (lo, hi) in enumerate(((0, mid), (mid, n))):
            e.quorum_mark_device(db.items.data_ptr(), n, lo, hi, t_bm.data_ptr(), t_parts[r].data_ptr())
        e.quorum_merge_device(t_parts.data_ptr(), 2, W, t_res.data_ptr())
        torch.cuda.synchronize()
        assert np.array_equal(bits(t_bm.cpu().numpy().view(np.uint32), n), want_bits)
        assert_results(t_res.cpu().numpy().view(ib.RESULT_DTYPE), want_res, "marks + merge")
        # each shard's partial: the groups' voted sets back to back ((n + 31) // 32 words each), then the valid counts; together
        # the two shards hold exactly the reference's voted sets
        packed = np.concatenate([me.voted_words(want_voted)[g, : (t.n + 31) // 32] for g, t in enumerate(me.tables())])
        parts = t_parts.cpu().numpy().view(np.uint32)
        assert np.array_equal(parts[0, : len(packed)] | parts[1, : len(packed)], packed)
        counts = parts[0, len(packed): len(packed) + len(groups)] + parts[1, len(packed): len(packed) + len(groups)]
        assert counts.tolist() == [r[0] for r in want_res]
        e.bind_groups(None)
    finally:
        e.close()


# ------------------------------------------------------------------------------------------------------------ explain
def test_explain_reasons_at_the_lookup_edges():
    b = base()
    e = load(ib.Engine(**params()))
    try:
        groups = groups_of(e)
        bm, _, _ = e.verify_batch(b.items, b"", groups)
        reasons, rec = e.explain_batch(b.items, b"", groups, bm)
        want_r, want_rec = eo.explain_batch(b.items, b"", [t.addr_array() for t in me.tables()], list(range(len(me.tables()))))
        assert np.array_equal(reasons, want_r)
        # accepted items get OK without device work, so only the rejected ones carry a recovered address
        rejected = ~bits(bm, len(b.items))
        assert np.array_equal(rec[rejected], want_rec[rejected])
        assert not rec[~rejected].any()
        by_case = {}
        for i, (case, _) in enumerate(b.tags):
            by_case.setdefault(case, set()).add(int(reasons[i]))
        assert by_case["a"] == {eo.OK} and by_case["b"] == {eo.SIGNER_MISMATCH}
        assert by_case["c"] == {eo.NOT_VALIDATOR, eo.SIGNER_MISMATCH}
        assert by_case["d"] == {eo.R_RANGE, eo.R_NOT_X, eo.NO_KEY}
    finally:
        e.close()


# ------------------------------------------------------------------------------------------------------- multi-device
def test_multi_device_engine_gives_the_single_engines_bytes():
    b = tile(base(), 2 * len(base().items))
    single, multi = load(ib.Engine(**params())), load(ib.Engine(**params(devices=[0, 0])))
    try:
        for rule in (me.DEFAULT, me.PREPARE):
            one = single.verify_batch_ex(b.items, b"", groups_of(single, rule), voted_stride_words=STRIDE)
            two = multi.verify_batch_ex(b.items, b"", groups_of(multi, rule), voted_stride_words=STRIDE)
            for x, y in zip(one, two):
                assert np.array_equal(x, y), rule
        check_call(multi, b, me.PREPARE, "multi")
    finally:
        single.close()
        multi.close()


# --------------------------------------------------------------------------------------------------------- host mirror
def test_host_mirror_commit_round_on_a_decoy_dense_table():
    """33 validators: the 12 signers, the +-1 neighbours of most of them and of one absent key; COMMITs from every signer, seals
    claiming a neighbour, and the absent key's valid COMMIT -- the decisions equal oracle/ibft_logic.py's"""
    S = me.signers()
    height = me.HEIGHT
    absent_key = wl.privkey(me.SEED, me.SCAN + 1)
    absent = wl.address_of(absent_key)
    addrs = [a for _, _, a in S] + [me.i2a(me.a2i(absent) - 1), me.i2a(me.a2i(absent) + 1)]
    for _, _, a in S:
        for y in (me.a2i(a) - 1, me.a2i(a) + 1):
            if len(addrs) < 33:
                addrs.append(me.i2a(y))
    assert len(set(addrs)) == 33 and absent not in addrs
    powers = [10**6 + i if i < len(S) else 1000 + i for i in range(33)]   # the signers alone reach quorum
    raw = b"membership" * 20
    ph = wl.proposal_hash(raw, 0)
    view = ip.View(height, 0)
    keys = {a: d for _, d, a in S}
    keys[absent] = absent_key

    def signed(m, d):
        m.signature = wl.sign(d, co.keccak256(m.payload_no_sig()))
        return m
    pp = signed(ip.IbftMessage(view, S[0][2], b"", ip.PREPREPARE, ip.PrePrepareMessage(ip.Proposal(raw, 0), ph, None)), S[0][1])
    commits = [signed(ip.IbftMessage(view, a, b"", ip.COMMIT, ip.CommitMessage(ph, wl.sign(keys[a], wl.seal_digest(ph)))), keys[a])
               for a in [a for _, _, a in S] + [absent]]
    # a signer's COMMIT claiming its +1 neighbour (frame and seal signed by the signer)
    for _, d, a in S[:4]:
        nb = me.i2a(me.a2i(a) + 1)
        commits.append(signed(ip.IbftMessage(view, nb, b"", ip.COMMIT, ip.CommitMessage(ph, wl.sign(d, wl.seal_digest(ph)))), d))
    proposer_of = lambda a, h, r: a == S[0][2]  # noqa: E731
    o = L.IBFT(oracle_backend({height: set(addrs)}, height, proposer_of), L.ValidatorManager(lambda h: dict(zip(addrs, powers))))
    o.vm.init(height)
    c = host.HostContext("gpu", {"is_proposer": proposer_of}, b"", host.EngineParams(0, 1 << 14, 1 << 24, 32, 8, 4096, 0))
    try:
        assert c.set_validators(height, addrs, powers) == 0
        o.state.view, o.state.name, o.state.proposal_message = view, L.COMMIT_STATE, pp
        c.set_state(height, 0, L.COMMIT_STATE, enc(pp))
        for m in commits:
            o.messages.add_message(m)
            c.store_add(enc(m))
        assert o.handle_commit(view) == c.handle_commit(height, 0)
        assert c.store_senders(height, 0, ip.COMMIT) == sorted(m.from_ for m in o.messages.maps[ip.COMMIT][height][0].values())
        assert c.seal_count() == len(o.state.seals) == len(S)
    finally:
        c.close()


enc = ip.encode_ibft_message


# ------------------------------------------------------------------------------------------- duplicate addresses refused
def dup_table(n, where):
    t = me.tables()[-1] if n == me.MAX_VALIDATORS else None
    addrs = [bytes(a) for a in (t.addr_array() if t else me.tables()[1].addr_array())][:n]
    j = 1 if where == "adjacent" else n - 1
    # "adjacent": the duplicate sits at the next validator index and, once sorted, next to its twin; "far": index n - 1
    addrs[j] = addrs[0]
    return np.frombuffer(b"".join(addrs), np.uint8).reshape(n, 20).copy(), j


@pytest.mark.parametrize("devices", [None, [0, 0]], ids=["single", "multi"])
def test_a_table_that_lists_an_address_twice_is_refused(devices):
    e = load(ib.Engine(**params(key_cache=True, devices=devices)))
    try:
        b = base()
        bm0 = check_call(e, b, me.DEFAULT, "before")
        e.refresh_key_tables()
        reg = e.key_registry()
        quorums = [e.get_quorum(s) for s in range(len(me.tables()))]
        for slot, n in ((1, 2), (len(me.tables()) - 1, me.MAX_VALIDATORS)):
            for where in ("adjacent", "far"):
                addrs, j = dup_table(n, where)
                for powers in (None, me.tables()[slot].power_array()[:n] if n == me.tables()[slot].n else None):
                    with pytest.raises(ib.EngineError) as ex:
                        e.set_validators(slot, me.HEIGHT + 1, addrs, powers)
                    assert ex.value.code == ERR_INVALID_ARG and f"validators 0 and {j}" in str(ex.value), str(ex.value)
                    assert e.key_registry() == reg
                    assert [e.get_quorum(s) for s in range(len(me.tables()))] == quorums
        assert np.array_equal(check_call(e, b, me.DEFAULT, "after"), bm0)
    finally:
        e.close()


@pytest.mark.parametrize("devices", [None, [0, 0]], ids=["single", "multi"])
def test_host_gpu_context_refuses_a_duplicate(devices):
    """GpuVerifier::SetValidators returns false when the engine refuses the table; the context keeps answering for the height it
    had -- IsValidValidator through the device and the quorum through the ValidatorManager"""
    T = me.tables()[30]
    S = me.signers()
    addrs, powers = list(T.addrs), list(T.powers)
    c = host.HostContext("gpu", {}, b"", host.EngineParams(0, 1 << 12, 1 << 20, 8, 4, 4096, 0), devices=devices)
    try:
        assert c.set_validators(1, addrs, powers) == 0
        m = ip.IbftMessage(ip.View(1, 0), T.signer_addr, b"", ip.PREPARE, ip.PrepareMessage(me.DIGEST))
        m.signature = wl.sign(S[T.signer][1], co.keccak256(m.payload_no_sig()))
        frame = ip.encode_ibft_message(m)
        assert powers[T.index[T.signer_addr]] >= 1 << 255      # the signer alone holds a quorum of this table
        assert c.is_valid_validator(frame) and c.has_quorum_senders([T.signer_addr])
        quorum_before = c.has_quorum_senders(addrs[: 2 * T.n // 3 + 1])
        for h in (1, 5):      # the same height, and one whose slot (5 mod 4) is the same
            dup = addrs[:-1] + [addrs[0]]
            assert c.set_validators(h, dup, powers) == ERR_INVALID_ARG
            assert c.set_validators(h, dup, None) == ERR_INVALID_ARG
            assert c.is_valid_validator(frame), h
            assert c.has_quorum_senders(addrs[: 2 * T.n // 3 + 1]) == quorum_before
            assert c.has_quorum_senders([T.signer_addr])
    finally:
        c.close()
