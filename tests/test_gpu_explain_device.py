"""ibft_explain_batch_device on the H100: the reasons and recovered addresses of device-resident items, after
ibft_verify_batch_device, byte for byte what ibft_explain_batch and the reference of tests/explain_oracle.py give -- over whole
batches and 32-aligned sub-shards, with and without bound groups, on key-registry engines, in chunks larger than the engine's
max_items -- plus the shard-only writes, NEEDS_HOST on raw frames, the errors, and ShardedVerifier.explain with ranks as threads."""
import importlib

import numpy as np
import pytest
import torch

import explain_oracle as X
import ibft_b200 as ib
from test_explain_oracle import edge_frame_batch
from test_gpu_exchange_ranks import ThreadDist, case, run_ranks, share_exchange_buffers
from test_gpu_explain import crafted_cases, fixture_case, groups_for, new_engine, set_fixture

pytestmark = pytest.mark.gpu
sharding = importlib.import_module("go-ibft_b200.sharding")
REASON_SENTINEL, REC_SENTINEL, COUNT_SENTINEL = 0xAB, 0xCD, 0x5A5A5A5A


def to_dev(a) -> torch.Tensor:
    b = np.frombuffer(a, np.uint8) if isinstance(a, (bytes, bytearray)) else np.ascontiguousarray(a).view(np.uint8).reshape(-1)
    return torch.from_numpy(b.copy() if b.size else np.zeros(16, np.uint8)).cuda()


class DeviceCall:
    """one batch in device memory, its verdict bitmap from verify_device, and sentinel-filled explain outputs"""

    def __init__(self, items, arena):
        self.n = len(items)
        self.items, self.arena, self.arena_len = to_dev(items), to_dev(arena), len(arena)
        self.bitmap = torch.zeros(max(1, (self.n + 31) // 32), dtype=torch.int32, device="cuda")
        self.reasons = torch.zeros(max(1, self.n), dtype=torch.uint8, device="cuda")
        self.rec = torch.zeros(max(1, self.n) * 20, dtype=torch.uint8, device="cuda")
        self.count = torch.zeros(1, dtype=torch.int32, device="cuda")
        self.stream = torch.cuda.Stream()
        torch.cuda.synchronize()

    def verify(self, eng):
        eng.verify_device(self.items.data_ptr(), self.n, self.arena.data_ptr(), self.arena_len, 0, self.n, self.bitmap.data_ptr(), 0,
                          self.stream.cuda_stream)
        self.stream.synchronize()
        return self.bitmap.cpu().numpy().view(np.uint32)[: (self.n + 31) // 32].copy()

    def fill(self):
        with torch.cuda.stream(self.stream):
            self.reasons.fill_(REASON_SENTINEL)
            self.rec.fill_(REC_SENTINEL)
            self.count.fill_(COUNT_SENTINEL)

    def explain(self, eng, lo, hi, recovered=True, count=True):
        """(reasons, recovered, count) after the call over [lo, hi), outputs sentinel-filled before it"""
        self.fill()
        eng.explain_device(self.items.data_ptr(), self.n, self.arena.data_ptr(), self.arena_len, lo, hi, self.bitmap.data_ptr(),
                           self.reasons.data_ptr(), self.rec.data_ptr() if recovered else 0, self.count.data_ptr() if count else 0,
                           self.stream.cuda_stream)
        return self.read()

    def read(self):
        self.stream.synchronize()
        return (self.reasons.cpu().numpy()[: self.n].copy(), self.rec.cpu().numpy()[: 20 * self.n].reshape(-1, 20).copy(),
                int(self.count.item()) & 0xFFFFFFFF)


def shards(n):
    """the whole range, empty shards (at 0 and at the last word boundary), aligned sub-shards, a trailing partial word and
    shard_hi == n"""
    w = n // 32
    out = [(0, n), (0, 0), (32 * w, 32 * w)]
    if w >= 3:
        out += [(32, 32 * (w // 2 + 1)), (32 * (w // 2), n)]
    if n % 32 and w >= 1:
        out.append((32 * w, n))
    return out


def check_shards(eng, dc, bitmap, want, want_rec, label):
    """every shard of shards(n): the host-path bytes inside [lo, hi), the sentinels outside, the count of zero bits"""
    bits = X.bits_of(bitmap, dc.n)
    for lo, hi in shards(dc.n):
        got, rec, cnt = dc.explain(eng, lo, hi)
        inside = np.zeros(dc.n, bool)
        inside[lo:hi] = True
        assert np.array_equal(got[inside], want[inside]), (label, lo, hi, np.nonzero(got[inside] != want[inside])[0][:8])
        assert np.array_equal(rec[inside], want_rec[inside]), (label, lo, hi)
        assert (got[~inside] == REASON_SENTINEL).all() and (rec[~inside] == REC_SENTINEL).all(), (label, lo, hi)
        assert cnt == int((~bits[lo:hi]).sum()), (label, lo, hi)


def parity(eng, label, items, arena, groups, oracle=None):
    """verify_device then explain_device over every shard; the host path's bytes for the same bitmap (and the oracle's on the
    zero bits, where given)"""
    eng.bind_groups(groups)
    dc = DeviceCall(items, arena)
    bm = dc.verify(eng)
    host_bm, _, _ = eng.verify_batch(items, arena, groups)
    assert np.array_equal(bm, host_bm), label
    want, want_rec = eng.explain_batch(items, arena, groups, bitmap=bm)
    if oracle is not None:
        zero = ~X.bits_of(bm, len(items))
        assert np.array_equal(want[zero], oracle[0][zero]) and np.array_equal(want_rec[zero], oracle[1][zero]), label
        assert not want[~zero].any() and not want_rec[~zero].any()
    check_shards(eng, dc, bm, want, want_rec, label)
    return dc, bm, want, want_rec


def test_parity_with_the_host_path_and_the_reference():
    eng = new_engine()
    try:
        for label, items, arena, tables, gt, want, want_rec in crafted_cases():
            parity(eng, label, items, arena or b"\x00", groups_for(eng, tables, gt), (want, want_rec))
        for name in ("config2", "config3"):
            items, arena, addrs, _, ng, want, want_rec = fixture_case(name)
            parity(eng, name, items, arena, set_fixture(eng, addrs, ng), (want, want_rec))
    finally:
        eng.close()


def test_without_recovered_or_count_and_a_shard_without_zero_bits():
    eng = new_engine()
    try:
        items, arena, addrs, _, ng, _, _ = fixture_case("config2")
        dc, bm, want, _ = parity(eng, "config2", items, arena, set_fixture(eng, addrs, ng))
        got, rec, cnt = dc.explain(eng, 0, dc.n, recovered=False, count=False)
        assert np.array_equal(got, want) and (rec == REC_SENTINEL).all() and cnt == COUNT_SENTINEL
        words = np.nonzero(bm == 0xFFFFFFFF)[0]
        assert len(words)
        lo = 32 * int(words[0])
        c0 = eng.launch_count()
        got, rec, cnt = dc.explain(eng, lo, lo + 32)
        assert eng.launch_count() - c0 == 2 and cnt == 0
        assert (got[lo: lo + 32] == X.OK).all() and not rec[lo: lo + 32].any()
        # an empty shard: no launch, count 0, nothing written
        c0 = eng.launch_count()
        got, rec, cnt = dc.explain(eng, 64, 64)
        assert eng.launch_count() == c0 and cnt == 0 and (got == REASON_SENTINEL).all() and (rec == REC_SENTINEL).all()
    finally:
        eng.close()


def test_needs_host_on_raw_frames():
    """exactly the items verify_batch_ex marks IBFT_ITEM_NEEDS_HOST are explained NEEDS_HOST on the device path"""
    items, arena, vs = edge_frame_batch()
    eng = new_engine()
    try:
        groups = groups_for(eng, [vs.addr_array()], [0, 0])
        _, _, status, _ = eng.verify_batch_ex(items, arena, groups)
        want = X.explain_batch(items, arena, [vs.addr_array()], [0, 0])
        dc, bm, got, _ = parity(eng, "frames", items, arena, groups, want)
        got, _, _ = dc.explain(eng, 0, dc.n)
        needs = status == ib.engine.ITEM_NEEDS_HOST
        assert needs.any() and np.array_equal(got == X.NEEDS_HOST, needs)
    finally:
        eng.close()


def test_bound_groups_slots_and_rules():
    """No groups bound: the bytes of explain_batch(groups=None).  Groups over two slots with DEFAULT / PREPARE / PREPREPARE rules,
    a second table without half the validators, and fewer groups than the items name: NOT_VALIDATOR and NO_GROUP where the host
    path puts them."""
    items, arena, addrs, _, ng, _, _ = fixture_case("config3")
    eng = new_engine()
    try:
        set_fixture(eng, addrs, ng)
        dc, _, want, _ = parity(eng, "no groups", items, arena, None)
        assert not np.isin(want, [X.NO_GROUP, X.NOT_VALIDATOR]).any()
        eng.set_validators(1, 7, addrs[::2], None)
        seen = set()
        for slots, rules in (([1, 0], [ib.engine.QUORUM_DEFAULT, ib.engine.QUORUM_PREPARE]),
                             ([0, 1], [ib.engine.QUORUM_PREPREPARE, ib.engine.QUORUM_DEFAULT]),
                             ([1], [ib.engine.QUORUM_PREPARE])):
            groups = eng.groups(len(slots), slot=slots, rule=rules, proposer=ib.engine.PROPOSER_NONE)
            _, _, want, _ = parity(eng, str(slots), items, arena, groups)
            seen |= set(int(x) for x in want)
        assert {X.NOT_VALIDATOR, X.NO_GROUP} <= seen
    finally:
        eng.close()


@pytest.mark.parametrize("budget", [None, 300], ids=["unbounded", "budget300"])
def test_key_registry_engines(budget):
    """reasons as on a plain engine; the registry's counts are not changed by the call (never consulted or taught)"""
    eng = new_engine(key_cache=True, key_table_budget=budget)
    try:
        for name in ("config2", "config3", "config2"):
            items, arena, addrs, _, ng, want, want_rec = fixture_case(name)
            groups = set_fixture(eng, addrs, ng)
            eng.bind_groups(groups)
            dc = DeviceCall(items, arena)
            for _ in range(2):                       # the second verify uses the keys the first one learned
                bm = dc.verify(eng)
                eng.refresh_key_tables()
            assert np.array_equal(X.bits_of(bm, dc.n), want == X.OK), name
            before = eng.key_registry()
            got, rec, cnt = dc.explain(eng, 0, dc.n)
            assert eng.key_registry() == before, name
            assert np.array_equal(got, want) and np.array_equal(rec, np.where((want == X.OK)[:, None], 0, want_rec)), name
            assert cnt == int((want != X.OK).sum())
    finally:
        eng.close()


@pytest.mark.parametrize("max_items", [20, 100, 1000])
def test_chunks_beyond_max_items(max_items):
    """an engine whose max_items is far below the shard: the same bytes in one call, two launches per chunk of max_items
    (rounded up to a multiple of 32 by the engine) items"""
    items, arena, addrs, _, ng, want, want_rec = fixture_case("config2")
    big, small = new_engine(), new_engine(max_items=max_items)
    try:
        for e in (big, small):
            groups = set_fixture(e, addrs, ng)
            e.bind_groups(groups)
        dc = DeviceCall(items, arena)
        bm = dc.verify(big)
        want, want_rec = big.explain_batch(items, arena, groups, bitmap=bm)
        chunk = -(-max_items // 32) * 32
        for lo, hi in ((0, dc.n), (32 * (chunk // 32 + 1), dc.n - dc.n % 32)):
            c0 = small.launch_count()
            got, rec, cnt = dc.explain(small, lo, hi)
            assert small.launch_count() - c0 == 2 * -(-(hi - lo) // chunk)
            assert np.array_equal(got[lo:hi], want[lo:hi]) and np.array_equal(rec[lo:hi], want_rec[lo:hi])
            assert (got[:lo] == REASON_SENTINEL).all() and (got[hi:] == REASON_SENTINEL).all()
            assert cnt == int((~X.bits_of(bm, dc.n)[lo:hi]).sum())
    finally:
        big.close()
        small.close()


def test_errors_launch_nothing_and_leave_the_outputs_untouched():
    items, arena, addrs, _, ng, _, _ = fixture_case("config2")
    eng, multi = new_engine(), new_engine(devices=[0, 0])
    try:
        eng.bind_groups(set_fixture(eng, addrs, ng))
        dc = DeviceCall(items, arena)
        dc.verify(eng)
        n, p = dc.n, dict(items=dc.items.data_ptr(), arena=dc.arena.data_ptr(), bitmap=dc.bitmap.data_ptr(), reasons=dc.reasons.data_ptr())
        lib = eng.lib

        def call(e, lo=0, hi=n, **kw):
            q = dict(p, **kw)
            return lib.ibft_explain_batch_device(e.handle, q["items"] or None, n, q["arena"] or None, dc.arena_len, lo, hi, q["bitmap"] or None,
                                                 q["reasons"] or None, dc.rec.data_ptr(), dc.count.data_ptr(), dc.stream.cuda_stream)
        cases = [dict(lo=16), dict(hi=48), dict(hi=n + 32), dict(lo=64, hi=32), dict(items=0), dict(bitmap=0), dict(reasons=0),
                 dict(arena=0), dict(e=multi), dict(e=multi.sub(1))]
        for kw in cases:
            e = kw.pop("e", eng)
            dc.fill()
            c0 = eng.launch_count() + multi.launch_count()
            assert call(e, **kw) == ib.engine.ERR_INVALID_ARG, kw
            got, rec, cnt = dc.read()
            assert eng.launch_count() + multi.launch_count() == c0, kw
            assert (got == REASON_SENTINEL).all() and (rec == REC_SENTINEL).all() and cnt == COUNT_SENTINEL, kw
        assert lib.ibft_explain_batch_device(None, None, 0, None, 0, 0, 0, None, None, None, None, None) == ib.engine.ERR_INVALID_ARG
    finally:
        eng.close()
        multi.close()


# ---- ShardedVerifier.explain, ranks as threads ------------------------------------------------------------------------------

def host_explain(c):
    """per batch: the whole-batch host explain on one engine against the host verify's bitmap"""
    e = c.engine()
    try:
        out = []
        for b in range(2):
            groups = c.groups(e)
            bm, _, _ = e.verify_batch(c.batches[b]["items"], c.arena, groups)
            out.append(e.explain_batch(c.batches[b]["items"], c.arena, groups, bitmap=bm))
        return out
    finally:
        e.close()


@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("exchange", ["nccl", "p2p"])
def test_sharded_verifier_explain(monkeypatch, world, exchange):
    """two rounds with different batches: each rank's local reasons are the whole-batch host explain of its slice, and the
    gather=True result is the whole-batch host explain on every rank"""
    c = case("config3.npz")
    ref = host_explain(c)
    assert not np.array_equal(ref[0][0], ref[1][0])
    fake = ThreadDist(world)
    monkeypatch.setattr(sharding, "dist", fake)
    registry, out = {}, [[] for _ in range(world)]

    def rank_main(r):
        fake.local.rank = r
        torch.cuda.set_device(0)
        e = c.engine()
        if exchange == "p2p":
            share_exchange_buffers(e, registry)
        lo, hi = sharding.shard_bounds(c.n, world, r)
        shards_ = [sharding.rebase_shard(c.batches[b]["items"], c.arena, lo, hi) for b in range(2)]
        sv = sharding.ShardedVerifier(e, c.n, c.groups(e), world, r, shards_[0][0], shards_[0][1], torch.cuda.Stream(), exchange=exchange)
        try:
            for b in (0, 1):
                if sv.h_items.numel():
                    sv.h_items.copy_(torch.from_numpy(shards_[b][0].view(np.uint8).reshape(-1)))
                fake.barrier()
                sv.run()
                local = sv.explain()
                full = sv.explain(gather=True)
                out[r].append((b, lo, hi, local, full))
        finally:
            sv.close()
            e.close()
    run_ranks(world, rank_main)
    for r in range(world):
        assert len(out[r]) == 2
        for b, lo, hi, (reasons, rec), (all_reasons, all_rec) in out[r]:
            assert reasons.shape == (hi - lo,) and rec.shape == (hi - lo, 20)
            assert np.array_equal(reasons, ref[b][0][lo:hi]) and np.array_equal(rec, ref[b][1][lo:hi]), (r, b)
            assert np.array_equal(all_reasons, ref[b][0]) and np.array_equal(all_rec, ref[b][1]), (r, b)
