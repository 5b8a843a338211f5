"""Groups bound to the accepted proposal's hash (ibft_group_hash): only the PREPAREs and COMMITs that name it count, as in go-ibft's
handlePrepare / handleCommit.  Every case checks the counted bits, the voted sets and every ibft_group_result against the model of
tests/group_hash_model.py (itself checked against oracle.ibft_logic by tests/test_emul_group_hash.py), and that the verdict bitmap
and item statuses are byte-identical to the same call without hashes, on every kernel path, with and without the key registry, on
a multi-device engine, through the device-resident reduce, the shard marks + merge, the peer-memory exchange and ShardedVerifier."""
import functools
import importlib

import numpy as np
import pytest
import torch

import group_hash_model as M
import ibft_b200 as ib
from oracle import coracle as co
from oracle import ibft_proto as ip

pytestmark = pytest.mark.gpu
sharding = importlib.import_module("go-ibft_b200.sharding")

HEIGHT, ROUND = 4_200_000, 2
SLOT = 3


def seal_digest(h: bytes) -> bytes:
    return co.keccak256(h + b"\x02")


class Keys:
    def __init__(self, seed, n, weighted):
        self.privs = co.privkeys(seed, n)
        self.addrs = co.addresses(self.privs)
        self.powers = [1 + (i % 7) if weighted else 1 for i in range(n)]
        self.powers_be = np.frombuffer(b"".join(p.to_bytes(32, "big") for p in self.powers), np.uint8).reshape(n, 32).copy()
        self.n = n
        self.table = M.Table(self.addrs, self.powers)

    def addr(self, i):
        return bytes(self.addrs[i])

    def take(self, target, exclude=()):
        """validators outside `exclude` whose powers sum to exactly `target`"""
        out, acc = [], 0
        for i in sorted(range(self.n), key=lambda i: (-self.powers[i], i)):
            if i in exclude or acc + self.powers[i] > target:
                continue
            out.append(i)
            acc += self.powers[i]
            if acc == target:
                return out
        raise AssertionError("no validator set of that power")


@functools.lru_cache(maxsize=None)
def keys(name):
    return {"c2": lambda: Keys(1, 1000, False), "c3": lambda: Keys(2, 10_000, False), "c3w": lambda: Keys(2, 10_000, True)}[name]()


ACCEPTED = co.keccak256(b"accepted proposal")
COMPETING = co.keccak256(b"competing proposal")
STALE = co.keccak256(b"proposal of round 1")


class Batch:
    """items + arena built from entries (validator, kind, msg_type, hash, group, valid); signatures by the C oracle's signer"""

    def __init__(self, K):
        self.K, self.entries = K, []

    def add(self, validators, kind, msg_type, h, group, valid=True, noncanonical=False):
        for v in validators:
            self.entries.append((v, kind, msg_type, h, group, valid, noncanonical))
        return self

    def build(self):
        K, E = self.K, self.entries
        view = ip.View(HEIGHT, ROUND)
        # pass 1: committed seals over Keccak(hash || 0x02)
        seal_d = np.frombuffer(b"".join(seal_digest(e[3]) for e in E), np.uint8).reshape(-1, 32)
        seals = co.sign_derived_batch(K.privs[[e[0] for e in E]], seal_d) if E else np.zeros((0, 65), np.uint8)
        # pass 2: the signed bytes of every item that signs a message
        spans, digests = [], []
        for k, (v, kind, mt, h, g, valid, nc) in enumerate(E):
            payload = ip.PrepareMessage(h) if mt == M.HASH_PREPARE else ip.CommitMessage(h, bytes(seals[k]))
            m = ip.IbftMessage(view, K.addr(v), b"", ip.PREPARE if mt == M.HASH_PREPARE else ip.COMMIT, payload)
            body = ip.encode_ibft_message(m, with_signature=False)
            if nc:  # PayloadNoSig a Go node re-marshalled from a non-canonical frame: unknown field and a second, merged member
                member = 6 if mt == M.HASH_PREPARE else 7
                body += ip._f_bytes(13, b"unknown") + ip._f_msg(member, b"")
            spans.append(body)
            digests.append(co.keccak256(body) if kind != M.KIND_SEAL else seal_digest(h))
        sigs = co.sign_derived_batch(K.privs[[e[0] for e in E]], np.frombuffer(b"".join(digests), np.uint8).reshape(-1, 32)) \
            if E else np.zeros((0, 65), np.uint8)
        items, arena, expect = np.zeros(len(E), dtype=ib.ITEM_DTYPE), bytearray(), []
        for k, (v, kind, mt, h, g, valid, nc) in enumerate(E):
            it = items[k]
            sig = bytes(seals[k]) if kind in (M.KIND_SEAL, M.KIND_WIRE_SEAL) else bytes(sigs[k])  # the signature the item checks
            if not valid:
                sig = sig[:5] + bytes([sig[5] ^ 1]) + sig[6:]
            it["group"], it["kind"] = g, kind
            it["signer"] = np.frombuffer(K.addr(v), np.uint8)
            it["r"], it["s"], it["v"] = np.frombuffer(sig[:32], np.uint8), np.frombuffer(sig[32:64], np.uint8), sig[64]
            if kind == M.KIND_SEAL:
                it["digest"] = np.frombuffer(h, np.uint8)
            elif kind in (M.KIND_WIRE, M.KIND_WIRE_SEAL):
                payload = ip.PrepareMessage(h) if mt == M.HASH_PREPARE else ip.CommitMessage(h, sig if kind == M.KIND_WIRE_SEAL else bytes(seals[k]))
                m = ip.IbftMessage(view, K.addr(v), sig if kind == M.KIND_WIRE else bytes(sigs[k]),
                                   ip.PREPARE if mt == M.HASH_PREPARE else ip.COMMIT, payload)
                frame = ip.encode_ibft_message(m)
                it["payload_off"], it["payload_len"] = len(arena), len(frame)
                arena += frame
            elif kind == 0:  # DIGEST: z given
                it["digest"] = np.frombuffer(digests[k], np.uint8)
            elif kind == 5:  # PAYLOAD2: PayloadNoSig in two spans
                half = len(spans[k]) // 2
                it["payload_off"], it["payload_len"] = len(arena), half
                off2 = len(arena) + half
                it["digest"][:8] = np.frombuffer(off2.to_bytes(8, "little"), np.uint8)
                it["digest"][8:12] = np.frombuffer((len(spans[k]) - half).to_bytes(4, "little"), np.uint8)
                arena += spans[k]
            else:  # PAYLOAD
                it["payload_off"], it["payload_len"] = len(arena), len(spans[k])
                arena += spans[k]
            expect.append(valid)
        return items, bytes(arena), M.pack_bits(np.array(expect, dtype=bool))


def hashes_for(n_groups, bound):
    return ib.group_hashes(n_groups, bound)


def new_engine(K, max_items=1 << 16, key_cache=False, devices=None, max_groups=8):
    e = ib.Engine(max_items=max_items, max_payload_bytes=1 << 24, max_groups=max_groups, max_table_slots=4,
                  max_validators=max(1024, K.n), key_cache=key_cache, devices=devices)
    e.set_validators(SLOT, HEIGHT, K.addrs, K.powers_be)
    return e


def check_call(e, K, items, arena, groups, hashes, want_bitmap=None):
    """the hashed call against the unbound one and the model; returns (results, counted flags)"""
    stride = (K.n + 31) // 32
    b0, r0, s0, v0 = e.verify_batch_ex(items, arena, groups, stride)
    b1, r1, s1, v1, c1 = e.verify_batch_ex(items, arena, groups, stride, group_hashes=hashes)
    assert np.array_equal(b1, b0) and np.array_equal(s1, s0)
    if want_bitmap is not None:
        assert np.array_equal(b1, want_bitmap)
    flags = M.counted(items, arena, b1, len(groups), hashes)
    assert np.array_equal(c1, M.pack_bits(flags))
    check_results(r1, v1, M.group_results(items, arena, flags, groups, {SLOT: K.table}))
    check_results(r0, v0, M.group_results(items, arena, M.counted(items, arena, b0, len(groups), None), groups, {SLOT: K.table}))
    for g in range(len(groups)):
        if int(hashes[g]["msg_type"]) == M.HASH_UNBOUND:
            assert r1[g].tobytes() == r0[g].tobytes() and np.array_equal(v1[g], v0[g]), g
    return r1, flags


def check_results(res, voted, model):
    mres, mvoted = model
    for g, m in enumerate(mres):
        got = dict(power=M.power_of(res[g]), n_valid=int(res[g]["n_valid"]), n_distinct=int(res[g]["n_distinct"]),
                   has_quorum=int(res[g]["has_quorum"]))
        assert got == m, (g, got, m)
        if voted is not None:
            assert M.voted_set(voted[g]) == mvoted[g], g


def commit_round(K, matching_power, pad_with_mismatch=True):
    """A COMMIT round bound to ACCEPTED in group 0: seals over ACCEPTED worth `matching_power`; equivocators among them also seal
    COMPETING; further validators seal only a stale round's hash or the competing proposal, enough to push the unfiltered sum
    over the quorum; a few invalid seals.  Group 1 repeats the matching seals unbound."""
    match = K.take(matching_power)
    rest = [i for i in range(K.n) if i not in set(match)]
    b = Batch(K).add(match, M.KIND_SEAL, M.HASH_COMMIT, ACCEPTED, 0)
    b.add(match[::9], M.KIND_SEAL, M.HASH_COMMIT, COMPETING, 0)                # equivocators: two COMMITs
    if pad_with_mismatch:
        b.add(rest[0::2][:40], M.KIND_SEAL, M.HASH_COMMIT, STALE, 0)            # a stale round
        b.add(rest[1::2][:40], M.KIND_SEAL, M.HASH_COMMIT, COMPETING, 0)        # a competing proposal
    b.add(rest[100:104], M.KIND_SEAL, M.HASH_COMMIT, ACCEPTED, 0, valid=False)
    b.add(match[:50], M.KIND_SEAL, M.HASH_COMMIT, STALE, 1)
    return b.build(), 2


@pytest.mark.parametrize("name", ["c2", "c3", "c3w"])
def test_commit_boundary(name):
    K = keys(name)
    e = new_engine(K)
    groups = e.groups(2, slot=SLOT)
    hashes = hashes_for(2, {0: (ib.HASH_COMMIT, ACCEPTED)})
    for power, bound_q, unbound_q in ((K.table.quorum - 1, 0, 1), (K.table.quorum, 1, 1)):
        (items, arena, want), _ = commit_round(K, power)
        r1, flags = check_call(e, K, items, arena, groups, hashes, want)
        assert int(r1[0]["has_quorum"]) == bound_q and M.power_of(r1[0]) == power
        _, r0, _, _ = e.verify_batch_ex(items, arena, groups)
        assert int(r0[0]["has_quorum"]) == unbound_q
    e.close()


def mixed_batch(K, proposer_in):
    """every item kind in bound and unbound groups of one call.  Groups: 0 COMMIT bound (rule 0), 1 PREPARE bound (rule 2,
    proposer p), 2 PREPARE bound (rule 0), 3 unbound COMMIT, 4 unbound PREPARE rule 2"""
    n = min(K.n, 1000)
    p = 5
    q = K.table.quorum
    prep_match = K.take(q - K.powers[p] - 3, exclude={p}) if K.n <= 1000 else list(range(6, 600))
    b = Batch(K)
    third = n // 3
    for kind in (M.KIND_SEAL, M.KIND_WIRE_SEAL, M.KIND_WIRE, M.KIND_PAYLOAD):
        b.add(range(kind, third, 4), kind, M.HASH_COMMIT, ACCEPTED, 0)
        b.add(range(third + kind, third + 60, 4), kind, M.HASH_COMMIT, COMPETING, 0)
        b.add(range(kind, 80, 4), kind, M.HASH_COMMIT, ACCEPTED, 3)
    b.add(range(2 * third, 2 * third + 40), M.KIND_PAYLOAD, M.HASH_COMMIT, ACCEPTED, 0, noncanonical=True)
    b.add(range(2 * third + 40, 2 * third + 60), M.KIND_PAYLOAD, M.HASH_COMMIT, COMPETING, 0, noncanonical=True)
    b.add(range(2 * third + 60, 2 * third + 80), 0, M.HASH_COMMIT, ACCEPTED, 0)        # DIGEST: never counts when bound
    b.add(range(2 * third + 80, 2 * third + 100), 5, M.HASH_COMMIT, ACCEPTED, 0)      # PAYLOAD2: never counts when bound
    b.add(range(2 * third + 60, 2 * third + 70), 0, M.HASH_COMMIT, ACCEPTED, 3)
    for half, kind in enumerate((M.KIND_WIRE, M.KIND_PAYLOAD)):
        for g in (1, 2, 4):
            b.add(prep_match[half::2], kind, M.HASH_PREPARE, ACCEPTED, g)
    b.add([x for x in range(n) if x not in set(prep_match) and x != p][:30], M.KIND_WIRE, M.HASH_PREPARE, STALE, 1)
    b.add(prep_match[:5], M.KIND_SEAL, M.HASH_COMMIT, ACCEPTED, 1)                    # a seal never counts in a PREPARE group
    b.add([p], M.KIND_WIRE, M.HASH_PREPARE, ACCEPTED if proposer_in else COMPETING, 1)  # the proposer's own PREPARE
    b.add([p], M.KIND_WIRE, M.HASH_PREPARE, COMPETING, 4)
    return b.build()


@pytest.mark.parametrize("name", ["c2", "c3w"])
@pytest.mark.parametrize("proposer_in", [False, True])
def test_every_kind_mixed_groups_and_prepare_rule(name, proposer_in):
    K = keys(name)
    e = new_engine(K)
    groups = e.groups(5, slot=SLOT, rule=[0, ib.QUORUM_PREPARE, 0, 0, ib.QUORUM_PREPARE], proposer=[0, 5, 0, 0, 5])
    hashes = hashes_for(5, {0: (ib.HASH_COMMIT, ACCEPTED), 1: (ib.HASH_PREPARE, ACCEPTED), 2: (ib.HASH_PREPARE, ACCEPTED)})
    items, arena, want = mixed_batch(K, proposer_in)
    r1, flags = check_call(e, K, items, arena, groups, hashes, want)
    kinds = items["kind"]
    assert not flags[(kinds == 0) | (kinds == 5)][items["group"][(kinds == 0) | (kinds == 5)] == 0].any()
    assert flags[(kinds == M.KIND_WIRE_SEAL) & (items["group"] == 0)].any()
    assert int(r1[1]["has_quorum"]) == (0 if proposer_in else int(M.power_of(r1[1]) >= K.table.quorum))
    e.close()


def forced_paths():
    return [ib.Engine.PATH_THREAD, ib.Engine.PATH_QUAD, ib.Engine.PATH_SPLIT, ib.Engine.PATH_QSPLIT]


@pytest.mark.parametrize("key_cache", [False, True])
def test_every_path_and_the_key_registry(key_cache):
    """AUTO at qsplit (config-2 round), split (10k round) and thread (> SMs x 192 items) sizes, then each forced path; with the
    key registry every call runs twice, keys unknown and then known"""
    K = keys("c3w")
    e = new_engine(K, key_cache=key_cache)
    groups = e.groups(3, slot=SLOT)
    hashes = hashes_for(3, {0: (ib.HASH_COMMIT, ACCEPTED), 1: (ib.HASH_COMMIT, COMPETING)})
    sm = e.device_info()["sm_count"]
    small = Batch(K).add(range(0, 3000, 2), M.KIND_SEAL, M.HASH_COMMIT, ACCEPTED, 0).add(range(1, 1500, 2), M.KIND_SEAL, M.HASH_COMMIT,
                                                                                           COMPETING, 0).build()
    mid = Batch(K).add(range(K.n), M.KIND_SEAL, M.HASH_COMMIT, ACCEPTED, 0).add(range(0, K.n, 20), M.KIND_SEAL, M.HASH_COMMIT,
                                                                                 COMPETING, 0).add(range(1, K.n, 20), M.KIND_SEAL,
                                                                                                   M.HASH_COMMIT, STALE, 2).build()
    big = Batch(K).add(range(K.n), M.KIND_SEAL, M.HASH_COMMIT, ACCEPTED, 0).add(range(K.n), M.KIND_SEAL, M.HASH_COMMIT, COMPETING, 1)
    big = big.add(range(K.n), M.KIND_SEAL, M.HASH_COMMIT, STALE, 0).add(range(0, K.n, 2), M.KIND_SEAL, M.HASH_COMMIT, ACCEPTED, 2).build()
    assert len(small[0]) <= sm * 48 < len(mid[0]) <= sm * 192 < len(big[0])
    for items, arena, want in (small, mid, big):
        for _ in range(2 if key_cache else 1):
            check_call(e, K, items, arena, groups, hashes, want)
    for path in forced_paths():
        e.set_recover_path(path)
        check_call(e, K, *mid[:2], groups, hashes, mid[2])
    e.close()


def test_multi_device_engine():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two devices")
    K = keys("c3w")
    e = new_engine(K, devices=[0, 1])
    groups = e.groups(2, slot=SLOT)
    hashes = hashes_for(2, {0: (ib.HASH_COMMIT, ACCEPTED)})
    (items, arena, want), _ = commit_round(K, K.table.quorum - 1)
    r1, _ = check_call(e, K, items, arena, groups, hashes, want)
    assert int(r1[0]["has_quorum"]) == 0
    e.close()


def test_multi_device_engine_repeated_ordinal():
    """the multi-device code path on one device: shards apply the filter and the lead merges their counted votes"""
    K = keys("c3w")
    e = new_engine(K, devices=[0, 0])
    groups = e.groups(5, slot=SLOT, rule=[0, ib.QUORUM_PREPARE, 0, 0, ib.QUORUM_PREPARE], proposer=[0, 5, 0, 0, 5])
    hashes = hashes_for(5, {0: (ib.HASH_COMMIT, ACCEPTED), 1: (ib.HASH_PREPARE, ACCEPTED), 2: (ib.HASH_PREPARE, ACCEPTED)})
    items, arena, want = mixed_batch(K, False)
    big = np.concatenate([items] * 2)  # more than 1,024 items per device: two shards
    check_call(e, K, big, arena, groups, hashes, np.concatenate([want, want]) if len(items) % 32 == 0 else None)
    e.close()


def device_round(K):
    (items, arena, want), ng = commit_round(K, K.table.quorum - 1)
    return items, arena, want, ng


def test_device_resident_reduce_and_shard_marks():
    K = keys("c3w")
    e = new_engine(K)
    items, arena, want, ng = device_round(K)
    n = len(items)
    groups = e.groups(ng, slot=SLOT)
    hashes = hashes_for(ng, {0: (ib.HASH_COMMIT, ACCEPTED)})
    dev = torch.device("cuda", 0)
    d_items = torch.from_numpy(items.view(np.uint8).reshape(-1).copy()).to(dev)
    d_arena = torch.from_numpy(np.frombuffer(arena, np.uint8).copy()).to(dev)
    d_bitmap = torch.zeros((n + 31) // 32, dtype=torch.int32, device=dev)
    d_results = torch.zeros(ng * ib.RESULT_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    d_counted = torch.full(((n + 31) // 32,), -1, dtype=torch.int32, device=dev)
    e.bind_groups(groups)
    e.bind_group_hashes(hashes)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        e.verify_device(d_items.data_ptr(), n, d_arena.data_ptr(), len(arena), 0, n, d_bitmap.data_ptr(), 0, st.cuda_stream)
        e.quorum_reduce_device(d_items.data_ptr(), n, d_bitmap.data_ptr(), ng, d_results.data_ptr(), st.cuda_stream, d_counted.data_ptr())
    st.synchronize()
    bitmap = d_bitmap.cpu().numpy().view(np.uint32)
    assert np.array_equal(bitmap, want)
    flags = M.counted(items, arena, bitmap, ng, hashes)
    counted = d_counted.cpu().numpy().view(np.uint32).copy()
    if n % 32:
        counted[-1] &= (1 << (n % 32)) - 1
    assert np.array_equal(counted, M.pack_bits(flags))
    model = M.group_results(items, arena, flags, groups, {SLOT: K.table})
    check_results(d_results.cpu().numpy().view(ib.RESULT_DTYPE), None, model)
    assert int(model[0][0]["has_quorum"]) == 0
    # the same through three shard marks and the merge
    W = e.quorum_partial_words()
    parts = torch.zeros(3 * W, dtype=torch.int32, device=dev)
    d_counted.fill_(-1)
    bounds = [0, n // 3 + 5, 2 * n // 3 + 1, n]  # any bounds: counted bits are set one by one
    with torch.cuda.stream(st):
        for k in range(3):
            e.quorum_mark_device(d_items.data_ptr(), n, bounds[k], bounds[k + 1], d_bitmap.data_ptr(), parts.data_ptr() + 4 * k * W,
                                 st.cuda_stream, d_counted.data_ptr())
        e.quorum_merge_device(parts.data_ptr(), 3, W, d_results.data_ptr(), st.cuda_stream)
    st.synchronize()
    counted = d_counted.cpu().numpy().view(np.uint32).copy()
    if n % 32:
        counted[-1] &= (1 << (n % 32)) - 1
    assert np.array_equal(counted, M.pack_bits(flags))
    check_results(d_results.cpu().numpy().view(ib.RESULT_DTYPE), None, model)
    # unbinding restores the unfiltered decision; ibft_bind_groups drops the hashes too
    e.bind_group_hashes(None)
    with torch.cuda.stream(st):
        e.quorum_reduce_device(d_items.data_ptr(), n, d_bitmap.data_ptr(), ng, d_results.data_ptr(), st.cuda_stream)
    st.synchronize()
    assert int(d_results.cpu().numpy().view(ib.RESULT_DTYPE)[0]["has_quorum"]) == 1
    e.close()


@pytest.mark.parametrize("world,exchange", [(1, "nccl"), (2, "nccl"), (2, "p2p")])
def test_sharded_verifier(monkeypatch, world, exchange):
    """ShardedVerifier with bound hashes: ranks as threads of this process on one device, as test_gpu_exchange_ranks.py runs them"""
    from test_gpu_exchange_ranks import ThreadDist, run_ranks, share_exchange_buffers
    K = keys("c3w")
    items, arena, want, ng = device_round(K)
    n = len(items)
    hashes = hashes_for(ng, {0: (ib.HASH_COMMIT, ACCEPTED)})
    fake = ThreadDist(world)
    monkeypatch.setattr(sharding, "dist", fake)
    registry, out = {}, [None] * world

    def rank_main(r):
        fake.local.rank = r
        torch.cuda.set_device(0)
        e = new_engine(K)
        if exchange == "p2p":
            share_exchange_buffers(e, registry)
        lo, hi = sharding.shard_bounds(n, world, r)
        li, la = sharding.rebase_shard(items, np.frombuffer(arena, np.uint8), lo, hi)
        sv = sharding.ShardedVerifier(e, n, e.groups(ng, slot=SLOT), world, r, li, la, torch.cuda.Stream(), exchange=exchange,
                                      group_hashes=hashes)
        try:
            res, bm = sv.run()
            out[r] = (res, bm, sv.counted, lo, hi)
        finally:
            sv.close()
            e.close()
    run_ranks(world, rank_main)
    groups = ib.group_descs(ng, SLOT, slot_height={SLOT: HEIGHT})
    flags = M.counted(items, arena, want, ng, hashes)
    model = M.group_results(items, arena, flags, groups, {SLOT: K.table})
    assert int(model[0][0]["has_quorum"]) == 0
    for res, bm, counted, lo, hi in out:
        assert np.array_equal(bm, want)
        assert np.array_equal(counted, M.pack_bits(flags[lo:hi]))
        check_results(res, None, model)


def test_peer_memory_exchange_world_two_one_device():
    """both ranks' shard marks + the exchange kernel, ranks driven from one process on one device (as test_gpu_exchange_ranks)"""
    K = keys("c3w")
    items, arena, want, ng = device_round(K)
    n = len(items)
    hashes = hashes_for(ng, {0: (ib.HASH_COMMIT, ACCEPTED)})
    dev = torch.device("cuda", 0)
    world = 2
    engines = [new_engine(K) for _ in range(world)]
    groups = engines[0].groups(ng, slot=SLOT)
    per = sharding.shard_words(n, world)
    W = None
    bufs, ptrs = [], []
    for e in engines:
        e.bind_groups(groups)
        e.bind_group_hashes(hashes)
        W = e.quorum_partial_words()
    wpr = (per + W + 63) // 64 * 64
    for e in engines:
        p, _ = e.exchange_alloc(2 * wpr + 64)
        ptrs.append(p)
    d_items = torch.from_numpy(items.view(np.uint8).reshape(-1).copy()).to(dev)
    d_arena = torch.from_numpy(np.frombuffer(arena, np.uint8).copy()).to(dev)
    d_counted = torch.zeros((n + 31) // 32, dtype=torch.int32, device=dev)
    fulls = [torch.zeros(world * per, dtype=torch.int32, device=dev) for _ in range(world)]
    results = [torch.zeros(ng * ib.RESULT_DTYPE.itemsize, dtype=torch.uint8, device=dev) for _ in range(world)]
    tflags = [torch.zeros(1, dtype=torch.int32, device=dev) for _ in range(world)]
    streams = [torch.cuda.Stream() for _ in range(world)]
    epoch, par = 1, 1
    for r, e in enumerate(engines):
        lo, hi = sharding.shard_bounds(n, world, r)
        base = ptrs[r] + par * wpr * 4
        st = streams[r].cuda_stream
        e.exchange_clear(ptrs[r], par * wpr, wpr, st)
        e.verify_device(d_items.data_ptr(), n, d_arena.data_ptr(), len(arena), lo, hi, base - (lo // 32) * 4, 0, st)
        e.quorum_mark_device(d_items.data_ptr(), n, lo, hi, base - (lo // 32) * 4, base + per * 4, st, d_counted.data_ptr())
    for r, e in enumerate(engines):  # both exchange kernels run concurrently on their own streams
        e.quorum_exchange_device(ptrs, r, wpr, per, epoch, fulls[r].data_ptr(), results[r].data_ptr(), tflags[r].data_ptr(),
                                 streams[r].cuda_stream)
    for s in streams:
        s.synchronize()
    bitmap = fulls[0].cpu().numpy().view(np.uint32)[: (n + 31) // 32]
    assert np.array_equal(bitmap, want)
    flags = M.counted(items, arena, bitmap, ng, hashes)
    counted = d_counted.cpu().numpy().view(np.uint32).copy()
    assert np.array_equal(counted, M.pack_bits(flags))
    model = M.group_results(items, arena, flags, groups, {SLOT: K.table})
    for r in range(world):
        assert int(tflags[r].item()) == 0
        check_results(results[r].cpu().numpy().view(ib.RESULT_DTYPE), None, model)
    for r, e in enumerate(engines):
        e.exchange_free(ptrs[r])
        e.close()


def test_refused_bindings_launch_nothing():
    K = keys("c2")
    e = new_engine(K)
    groups = e.groups(3, slot=SLOT, rule=[0, ib.QUORUM_PREPARE, ib.QUORUM_PREPREPARE], proposer=[0, 5, 0])
    (items, arena, _), _ = commit_round(K, 10, pad_with_mismatch=False)
    items["group"] = 0
    bad = []
    h = hashes_for(3, {0: (ib.HASH_COMMIT, ACCEPTED)})
    h[0]["msg_type"] = 3
    bad.append(h)                                              # unknown msg_type
    bad.append(hashes_for(3, {2: (ib.HASH_PREPARE, ACCEPTED)}))  # PREPREPARE rule
    bad.append(hashes_for(3, {2: (ib.HASH_COMMIT, ACCEPTED)}))
    bad.append(hashes_for(3, {1: (ib.HASH_COMMIT, ACCEPTED)}))   # PREPARE rule with COMMIT hashes
    h = hashes_for(3, {0: (ib.HASH_COMMIT, ACCEPTED)})
    h[1]["reserved"][2] = 1
    bad.append(h)                                              # reserved words, in an unbound entry too
    e.bind_groups(groups)
    lib = e.lib
    n, ng = len(items), len(groups)
    a = np.frombuffer(arena, np.uint8)
    for h in bad:
        before = e.launch_count()
        bitmap = np.full((n + 31) // 32, 0xDEADBEEF, np.uint32)
        counted = bitmap.copy()
        results = np.full(ng, 0xAB, np.uint8).repeat(ib.RESULT_DTYPE.itemsize)
        rc = lib.ibft_verify_batch_hashed(e.handle, items.ctypes.data, n, a.ctypes.data, len(a), groups.ctypes.data, ng,
                                          bitmap.ctypes.data, results.ctypes.data, None, None, None, 0, h.ctypes.data, counted.ctypes.data)
        assert rc == ib.engine.ERR_INVALID_ARG
        assert (bitmap == 0xDEADBEEF).all() and (counted == 0xDEADBEEF).all() and (results == 0xAB).all()
        with pytest.raises(ib.EngineError) as ei:
            e.bind_group_hashes(h)
        assert ei.value.code == ib.engine.ERR_INVALID_ARG
        assert e.launch_count() == before
    with pytest.raises(ib.EngineError):
        e.bind_group_hashes(hashes_for(2, {0: (ib.HASH_COMMIT, ACCEPTED)}))  # not the bound groups' count
    # the accepted forms: COMMIT on rule 0, PREPARE on rules 0 and 2
    ok = hashes_for(3, {0: (ib.HASH_COMMIT, ACCEPTED), 1: (ib.HASH_PREPARE, ACCEPTED)})
    e.bind_group_hashes(ok)
    e.verify_batch_ex(items, arena, groups, 0, group_hashes=ok)
    e.close()
