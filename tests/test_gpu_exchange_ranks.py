"""The peer-memory exchange (k_quorum_exchange behind ShardedVerifier(exchange="p2p")) and the NCCL-style exchange at world sizes
2 to 8, on one device.

Ranks are simulated in one process: exchange buffers are plain device memory whose addresses go straight into the kernel's peer
list, and ShardedVerifier ranks are threads with their own Engine and stream over a thread-barrier stand-in for
torch.distributed.  This covers the kernel's per-rank bitmap assembly, the cross-rank OR of voted sets and sum of valid counts,
the parity alternation, the flag protocol (including the int32 wrap of flag - epoch and the bounded wait's timeout), the
rebased per-rank pointers of sharding.py and empty trailing shards.  It does not cover NVLink or two devices; the one
two-process test maps a real CUDA IPC handle on the same device."""
import functools
import importlib
import json
import multiprocessing as mp
import os
import sys
import threading
import time

import numpy as np
import pytest
import torch

import ibft_b200 as ib
import power_edges as pe
from oracle import coracle as co

pytestmark = pytest.mark.gpu
sharding = importlib.import_module("go-ibft_b200.sharding")
HERE = os.path.dirname(os.path.abspath(__file__))
HEIGHT = 1_000_000
ITEM_S_LAST = 63                      # last byte of s in an ibft_sig_item


class Case:
    """A fixture slice as two batches of the same shape: A (the fixture's items) and B (every third valid item with a flipped
    s byte, invalid to the oracle); the validator table carries a power-edge table."""

    def __init__(self, name, lo=0, n=None, pattern="limb-edge"):
        d, rows, votes = pe.load(name)
        n = len(rows) - lo if n is None else n
        self.addrs, self.n_groups = d["addrs"], len(d["groups"])
        self.arena = np.ascontiguousarray(d["arena"], dtype=np.uint8)
        self.pat = next(p for p in pe.patterns(votes, len(self.addrs)) if p.name == pattern)
        self.powers_be = pe.powers_be(self.pat.powers)
        rows = rows[lo: lo + n].copy()
        bits_a = pe.bits_of(d["bitmap"], lo + n)[lo:].copy()
        rows_b = rows.copy()
        flip = np.nonzero(bits_a)[0][::3]
        rows_b[flip, ITEM_S_LAST] ^= 1
        items_b = rows_b.view(ib.ITEM_DTYPE).reshape(-1)
        sub = co.verify_batch(items_b[flip].copy(), self.arena.tobytes(), tables=[self.addrs], group_table=[0] * self.n_groups,
                              n_threads=8)
        assert not pe.bits_of(sub, len(flip)).any(), "a flipped signature still verifies"
        bits_b = bits_a.copy()
        bits_b[flip] = 0
        self.n = n
        self.batches = []
        for r, bits in ((rows, bits_a), (rows_b, bits_b)):
            self.batches.append(dict(items=r.view(ib.ITEM_DTYPE).reshape(-1), bits=bits, words=pe.words_of(bits),
                                     votes=pe.votes_of(r, bits, self.addrs, self.n_groups)))
        self.rules = [pe.DEFAULT, pe.PREPARE, pe.PREPREPARE][: self.n_groups]

    def groups(self, eng):
        return eng.groups(self.n_groups, 0, rule=self.rules, proposer=[self.pat.proposer] * self.n_groups)

    def expected(self, b):
        v = self.batches[b]["votes"]
        return [pe.expected(self.pat, [v[g]], self.rules[g])[0] for g in range(self.n_groups)]

    def engine(self):
        e = ib.Engine(device=0, max_items=1 << 15, max_payload_bytes=1 << 22, max_groups=8, max_table_slots=4, max_validators=10_000)
        e.set_validators(0, HEIGHT, self.addrs, self.powers_be)
        return e


@functools.lru_cache(maxsize=None)
def case(name, lo=0, n=None, pattern="limb-edge"):
    return Case(name, lo, n, pattern)


def assert_results(res, want, what=""):
    got = [(int(r["n_valid"]), int(r["n_distinct"]), pe.value(r["power"]), bool(r["has_quorum"])) for r in res]
    assert got == [tuple(w) for w in want], what


def u32(x):
    return np.array([x & 0xFFFFFFFF], np.uint32).view(np.int32)[0].item()


class DeviceBatch:
    def __init__(self, items: np.ndarray, arena: np.ndarray):
        self.items = torch.from_numpy(items.view(np.uint8).reshape(-1).copy()).cuda()
        self.arena = torch.from_numpy(arena.copy()).cuda()
        self.arena_len = len(arena)


class World:
    """`world` ranks' exchange buffers on one device, laid out as ShardedVerifier lays them out: [2 parities][wpr] words, then
    the two flags."""

    def __init__(self, eng, n, world, n_groups):
        self.e, self.n, self.world = eng, n, world
        self.W = eng.quorum_partial_words()
        self.per = sharding.shard_words(n, world)
        self.wpr = (self.per + self.W + 63) // 64 * 64
        self.bufs = [torch.zeros(2 * self.wpr + 64, dtype=torch.int32, device="cuda") for _ in range(world)]
        self.ptrs = [b.data_ptr() for b in self.bufs]
        self.d_full = torch.zeros(world * self.per, dtype=torch.int32, device="cuda")
        self.d_res = torch.zeros(n_groups * ib.RESULT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
        self.d_timeout = torch.zeros(1, dtype=torch.int32, device="cuda")
        self.stream = torch.cuda.Stream()

    def fill(self, db: DeviceBatch, par: int):
        """every rank's parity-`par` region from a real verify + mark over its shard_bounds shard"""
        st = self.stream.cuda_stream
        with torch.cuda.stream(self.stream):
            for r in range(self.world):
                lo, hi = sharding.shard_bounds(self.n, self.world, r)
                self.bufs[r][par * self.wpr: (par + 1) * self.wpr].zero_()
                base = self.ptrs[r] + par * self.wpr * 4
                if hi > lo:
                    self.e.verify_device(db.items.data_ptr(), self.n, db.arena.data_ptr(), db.arena_len, lo, hi, base - (lo // 32) * 4, 0, st)
                self.e.quorum_mark_device(db.items.data_ptr(), self.n, lo, hi, base - (lo // 32) * 4, base + self.per * 4, st)

    def set_flag(self, r, par, epoch):
        with torch.cuda.stream(self.stream):
            self.bufs[r][2 * self.wpr + par] = u32(epoch)

    def flag(self, r, par):
        self.stream.synchronize()
        return int(self.bufs[r][2 * self.wpr + par].item()) & 0xFFFFFFFF

    def exchange(self, rank, epoch):
        with torch.cuda.stream(self.stream):
            self.d_full.fill_(-1)
            self.d_timeout.zero_()
            self.e.quorum_exchange_device(self.ptrs, rank, self.wpr, self.per, epoch, self.d_full.data_ptr(), self.d_res.data_ptr(),
                                          self.d_timeout.data_ptr(), self.stream.cuda_stream)
        self.stream.synchronize()
        return (self.d_res.cpu().numpy().view(ib.RESULT_DTYPE), self.d_full.cpu().numpy().view(np.uint32), int(self.d_timeout.item()))


def run_epochs(c: Case, world: int, epochs, ranks=None):
    """Kernel level: per epoch, the round's batch in its parity and the other batch in the other parity; the peers' flags read
    `epoch`, the calling rank's own flag is two epochs stale.  Every rank's exchange must return the round's batch."""
    eng = c.engine()
    try:
        eng.bind_groups(c.groups(eng))
        w = World(eng, c.n, world, c.n_groups)
        dbs = [DeviceBatch(c.batches[b]["items"], c.arena) for b in range(2)]
        assert not np.array_equal(c.batches[0]["words"], c.batches[1]["words"])
        for k, epoch in enumerate(epochs):
            par, b = epoch & 1, k % 2
            w.fill(dbs[b], par)
            w.fill(dbs[1 - b], 1 - par)
            full = np.zeros(world * w.per, np.uint32)
            full[: len(c.batches[b]["words"])] = c.batches[b]["words"]
            for rank in (range(world) if ranks is None else ranks):
                for r in range(world):
                    w.set_flag(r, par, epoch if r != rank else epoch - 2)
                    w.set_flag(r, 1 - par, epoch - 1)
                res, got_full, timeout = w.exchange(rank, epoch)
                assert timeout == 0, (world, epoch, rank)
                assert np.array_equal(got_full, full), (world, epoch, rank)
                assert_results(res, c.expected(b), (world, epoch, rank))
                assert w.flag(rank, par) == epoch & 0xFFFFFFFF
    finally:
        eng.close()


@pytest.mark.parametrize("world", [2, 3, 5, 8])
@pytest.mark.parametrize("shape", ["config3", "n100"])
def test_exchange_kernel_ranks_and_parities(world, shape):
    """k_quorum_exchange for every rank of `world`, epochs 1-4 alternating two batches.  n100: a 100-item slice across both
    groups of config 3 (not a multiple of 32; at world 8 ranks 4-7 have empty shards)."""
    c = case("config3.npz") if shape == "config3" else case("config3.npz", 9950, 100)
    if shape == "n100" and world == 8:
        assert [sharding.shard_bounds(100, 8, r) for r in range(4, 8)] == [(100, 100)] * 4
    run_epochs(c, world, [1, 2, 3, 4])


def test_exchange_kernel_epoch_wrap():
    """epochs around the int32 wrap of (flag - epoch)"""
    run_epochs(case("config3.npz", 9950, 100), 3, [0x7FFFFFFE, 0x7FFFFFFF, 0x80000000, 0x80000001, 0xFFFFFFFE, 0xFFFFFFFF])


def test_exchange_kernel_times_out_on_a_stale_peer():
    """One launch: a peer's flag two epochs stale.  The call returns after the kernel's bounded wait, reports through the
    timeout flag, and still publishes the caller's own flag."""
    c = case("config3.npz", 9950, 100)
    eng = c.engine()
    try:
        eng.bind_groups(c.groups(eng))
        w = World(eng, c.n, 3, c.n_groups)
        w.fill(DeviceBatch(c.batches[0]["items"], c.arena), 1)
        for r, f in ((1, 5), (2, 3)):
            w.set_flag(r, 1, f)
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record(w.stream)
        _, _, timeout = w.exchange(0, 5)
        t1.record(w.stream)
        t1.synchronize()
        print(f"stale-peer exchange returned after {t0.elapsed_time(t1):.1f} ms")
        assert timeout == 1
        assert w.flag(0, 1) == 5
    finally:
        eng.close()


# ---- ShardedVerifier ranks as threads -------------------------------------------------------------------------------------

class ThreadDist:
    """The parts of torch.distributed sharding.py uses, for ranks that are threads of one process."""

    def __init__(self, world):
        self.world = world
        self.bar = threading.Barrier(world, timeout=120)
        self.slots = [None] * world
        self.local = threading.local()

    def barrier(self):
        self.bar.wait()

    def all_gather_object(self, out, obj):
        self.slots[self.local.rank] = obj
        self.bar.wait()
        out[:] = list(self.slots)
        self.bar.wait()

    def all_gather_into_tensor(self, out, inp):
        torch.cuda.current_stream().synchronize()      # the caller's kernels that wrote `inp` have finished
        self.slots[self.local.rank] = inp
        self.bar.wait()
        out.copy_(torch.cat([s.reshape(-1) for s in self.slots]))
        torch.cuda.current_stream().synchronize()
        self.bar.wait()


def share_exchange_buffers(eng, registry):
    """CUDA IPC cannot open a handle in the process that exported it: peers of this process map a handle to the exporting
    rank's own pointer instead."""
    alloc = eng.exchange_alloc

    def exchange_alloc(words):
        p, h = alloc(words)
        registry[h] = p
        return p, h
    eng.exchange_alloc = exchange_alloc
    eng.exchange_open = lambda h: registry[h]
    eng.exchange_close = lambda p: None


def run_ranks(world, fn, timeout=300):
    errs, threads = [None] * world, []

    def main(r):
        try:
            fn(r)
        except BaseException as ex:       # noqa: BLE001  -- reported by the caller
            errs[r] = ex
    for r in range(world):
        threads.append(threading.Thread(target=main, args=(r,), daemon=True))
        threads[-1].start()
    for t in threads:
        t.join(timeout)
    assert not any(t.is_alive() for t in threads), "a rank did not finish"
    for r, ex in enumerate(errs):
        if ex is not None:
            raise AssertionError(f"rank {r}: {ex!r}") from ex


def host_reference(c: Case):
    """the single-call host-buffer result of each batch on a plain engine"""
    e = c.engine()
    try:
        out = []
        for b in range(2):
            bm, res, _ = e.verify_batch(c.batches[b]["items"], c.arena, c.groups(e))
            out.append((bm, res))
        return out
    finally:
        e.close()


@pytest.mark.parametrize("world", [2, 3, 8])
@pytest.mark.parametrize("exchange", ["nccl", "p2p"])
def test_sharded_verifier_ranks_as_threads(monkeypatch, world, exchange):
    """ShardedVerifier at world > 1: every rank its own Engine, tables and stream, 4 rounds alternating two batches; every
    rank's (results, bitmap) equals the single-call host-buffer result and the oracle."""
    c = case("config3.npz")
    ref = host_reference(c)
    for b in range(2):
        assert np.array_equal(ref[b][0], c.batches[b]["words"])
        assert_results(ref[b][1], c.expected(b))
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
        shards = [sharding.rebase_shard(c.batches[b]["items"], c.arena, lo, hi) for b in range(2)]
        assert np.array_equal(shards[0][1], shards[1][1])            # batch B differs in signatures only
        sv = sharding.ShardedVerifier(e, c.n, c.groups(e), world, r, shards[0][0], shards[0][1], torch.cuda.Stream(), exchange=exchange)
        try:
            for k in range(4):
                if sv.h_items.numel() and len(shards[k % 2][0]):
                    sv.h_items.copy_(torch.from_numpy(shards[k % 2][0].view(np.uint8).reshape(-1)))   # this round's batch
                fake.barrier()
                t0 = time.perf_counter()
                res, bm = sv.run()
                out[r].append((k % 2, res, bm, time.perf_counter() - t0))
        finally:
            sv.close()
            e.close()
    run_ranks(world, rank_main)
    for r in range(world):
        assert len(out[r]) == 4
        for b, res, bm, _ in out[r]:
            assert np.array_equal(bm, ref[b][0]), (r, b)
            assert res.tobytes() == ref[b][1].tobytes(), (r, b)
    print(f"{exchange} world {world}: slowest round {max(x[3] for o in out for x in o) * 1e3:.1f} ms")


class _DeviceWords:
    """a torch view of `n` int32 words at a raw device address"""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i4", "data": (ptr, False), "version": 3}


def test_sharded_verifier_timeout_raises_and_sticks(monkeypatch):
    """Rank 1 never runs its round: rank 0's finish() raises after the kernel's bounded wait.  The timeout flag is not cleared
    by later rounds (a timed-out verifier must be rebuilt, see ShardedVerifier): even with the peer's flags made current, the
    next round raises again."""
    c = case("config3.npz", 9950, 100)
    fake = ThreadDist(2)
    monkeypatch.setattr(sharding, "dist", fake)
    registry, svs, engines = {}, [None, None], [None, None]

    def build(r):
        fake.local.rank = r
        e = engines[r] = c.engine()
        share_exchange_buffers(e, registry)
        lo, hi = sharding.shard_bounds(c.n, 2, r)
        li, la = sharding.rebase_shard(c.batches[0]["items"], c.arena, lo, hi)
        svs[r] = sharding.ShardedVerifier(e, c.n, c.groups(e), 2, r, li, la, torch.cuda.Stream(), exchange="p2p")
    run_ranks(2, build)
    try:
        with pytest.raises(RuntimeError, match="did not publish"):
            svs[0].run()
        peer = torch.as_tensor(_DeviceWords(svs[1].xbuf_ptr, 2 * svs[1].wpr + 64), device="cuda")
        peer[2 * svs[1].wpr: 2 * svs[1].wpr + 2] = 1 << 20
        torch.cuda.synchronize()
        with pytest.raises(RuntimeError, match="did not publish"):
            svs[0].run()
    finally:
        def close(r):
            fake.local.rank = r
            svs[r].close()
            engines[r].close()
        run_ranks(2, close)


# ---- two processes, real CUDA IPC ------------------------------------------------------------------------------------------

def _ipc_worker(rank, store_path, payload, out_path):
    import torch.distributed as dist
    sys.path[:0] = [os.path.dirname(HERE), HERE]
    import ibft_b200 as ib2
    dist.init_process_group("gloo", store=dist.FileStore(store_path, 2), rank=rank, world_size=2)
    rep = {"rank": rank, "rounds": []}
    try:
        e = ib2.Engine(device=0, max_items=1 << 15, max_payload_bytes=1 << 22, max_groups=8, max_table_slots=4, max_validators=10_000)
        e.set_validators(0, HEIGHT, payload["addrs"], payload["powers_be"])
        groups = e.groups(payload["n_groups"], 0, rule=payload["rules"], proposer=[payload["proposer"]] * payload["n_groups"])
        lo, hi = sharding.shard_bounds(payload["n"], 2, rank)
        shards = [sharding.rebase_shard(items, payload["arena"], lo, hi) for items in payload["items"]]
        sv = sharding.ShardedVerifier(e, payload["n"], groups, 2, rank, shards[0][0], shards[0][1], torch.cuda.Stream(), exchange="p2p")
        for k in range(3):
            sv.h_items.copy_(torch.from_numpy(shards[k % 2][0].view(np.uint8).reshape(-1)))
            dist.barrier()
            t0 = time.perf_counter()
            try:
                res, bm = sv.run()
                ok = bool(np.array_equal(bm, payload["words"][k % 2]) and res.tobytes() == payload["results"][k % 2])
                rep["rounds"].append({"ok": ok, "ms": (time.perf_counter() - t0) * 1e3})
            except RuntimeError as ex:
                rep["rounds"].append({"ok": False, "error": str(ex), "ms": (time.perf_counter() - t0) * 1e3})
        sv.close()
        e.close()
    except Exception as ex:  # noqa: BLE001 -- reported to the parent
        rep["error"] = repr(ex)
    with open(out_path, "w") as f:
        json.dump(rep, f)
    dist.destroy_process_group()


def test_two_processes_real_ipc(tmp_path):
    """World 2 in two processes on the same device: exchange_alloc / exchange_open / exchange_close and open_peer_buffers for
    real, over a gloo group on a FileStore.  3 peer-memory rounds, alternating two batches."""
    c = case("config2.npz")
    ref = host_reference(c)
    payload = dict(addrs=c.addrs, powers_be=c.powers_be, n_groups=c.n_groups, rules=c.rules, proposer=c.pat.proposer, n=c.n,
                   arena=c.arena, items=[c.batches[b]["items"] for b in range(2)], words=[ref[b][0] for b in range(2)],
                   results=[ref[b][1].tobytes() for b in range(2)])
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=_ipc_worker, args=(r, str(tmp_path / "store"), payload, str(tmp_path / f"r{r}.json"))) for r in range(2)]
    for p in procs:
        p.start()
    deadline = time.time() + 240
    for p in procs:
        p.join(max(1, deadline - time.time()))
    alive = [p for p in procs if p.is_alive()]
    for p in alive:
        p.terminate()
        p.join(10)
        if p.is_alive():
            p.kill()
            p.join()
    assert not alive, "a worker did not finish"
    reps = [json.load(open(tmp_path / f"r{r}.json")) for r in range(2)]
    print("two-process rounds:", json.dumps([r["rounds"] for r in reps]))
    for r in reps:
        assert "error" not in r, r
        assert [x["ok"] for x in r["rounds"]] == [True] * 3, r
