"""Key sharing between the ranks of a sharded verifier (ShardedVerifier.share_keys, ibft_key_share_export_device /
ibft_key_share_adopt_device) at world sizes 2, 3 and 8, in both exchange modes, on one device.

Ranks are threads with their own key-registry engine and stream, as in test_gpu_exchange_ranks.py.  Every round permutes the
items with its own seed, so every validator moves across ranks; after one round and share_keys() every rank must know every
key any rank learned, checked against the oracle's public keys, and every round's results must stay those of a single engine's
host-buffer call.  Forged records are refused on the device; a bounded registry ends with the same known keys within its
budget; and one two-process run shares keys through real CUDA IPC mappings."""
import functools
import importlib
import json
import multiprocessing as mp
import os
import sys
import time

import numpy as np
import pytest
import torch

import adversarial as A
import ibft_b200 as ib
import power_edges as pe
import workloads as wl
from oracle import coracle as co
from oracle import secp256k1 as ec

pytestmark = pytest.mark.gpu
sharding = importlib.import_module("go-ibft_b200.sharding")
xr = importlib.import_module("test_gpu_exchange_ranks")
HERE = os.path.dirname(os.path.abspath(__file__))
HEIGHT = xr.HEIGHT
ROUNDS = 4
C = 1024
REC = 21
KEYTAB_BYTES = 17 * 128 * 64


def key_engine(c, budget=None):
    e = ib.Engine(device=0, max_items=1 << 15, max_payload_bytes=1 << 22, max_groups=8, max_table_slots=4, max_validators=10_000,
                  key_cache=True)
    if budget is not None:
        e.set_key_table_budget(budget)
    e.set_validators(0, HEIGHT, c.addrs, c.powers_be)
    return e


def words_of(v: int) -> list[int]:
    return [(v >> (32 * i)) & 0xFFFFFFFF for i in range(8)]


@functools.lru_cache(maxsize=None)
def config3_pubkeys() -> np.ndarray:
    """(10000, 16) u32: the oracle's public key of every config-3 validator, in the registry's little-endian word format"""
    c = xr.case("config3.npz")
    out = np.zeros((len(c.addrs), 16), np.uint32)
    for v in range(len(c.addrs)):
        q = co.pubkey_from_scalar(wl.privkey(2, v))
        out[v] = words_of(int.from_bytes(q[:32], "big")) + words_of(int.from_bytes(q[32:], "big"))
    return out


@functools.lru_cache(maxsize=None)
def rounds_of(c):
    """per round: (batch, permutation, bitmap words the oracle expects)"""
    out = []
    for k in range(ROUNDS):
        b = k % 2
        perm = np.random.default_rng(1000 + k).permutation(c.n)
        out.append((b, perm, pe.words_of(c.batches[b]["bits"][perm])))
    return tuple(out)


@functools.lru_cache(maxsize=None)
def host_reference(c):
    """every round's batch through one key-registry engine's host-buffer calls: per round (bitmap, results), the engine's
    ready keys after round 1 and every validator's known flag at the end"""
    e = key_engine(c)
    try:
        ref = []
        for k, (b, perm, words) in enumerate(rounds_of(c)):
            bm, res, _ = e.verify_batch(c.batches[b]["items"][perm], c.arena, c.groups(e))
            assert np.array_equal(bm, words)
            xr.assert_results(res, c.expected(b))
            ref.append((bm, res.tobytes()))
            if k == 0:
                ready1 = e.key_registry()[1]
        known = registry_view(e, range(len(c.addrs)))[0] != 0
        return ref, ready1, known
    finally:
        e.close()


def signers(c, b):
    """validators with a valid item in batch b"""
    return sorted(set().union(*[vs for _, vs in c.batches[b]["votes"]]))


def registry_view(e, validators):
    """(state, key) of each validator's registry entry"""
    st = np.zeros(len(validators), np.uint32)
    keys = np.zeros((len(validators), 16), np.uint32)
    for j, v in enumerate(validators):
        s, k, _ = e.key_table(0, int(v))
        st[j], keys[j] = s, k
    return st, keys


def run_sharded(monkeypatch, world, exchange, budget=None):
    """ROUNDS permuted rounds on `world` thread ranks; per rank: the rounds' (results, bitmap, adopted, refused, seconds) and the
    registry after round 1 and at the end"""
    c = xr.case("config3.npz")
    fake = xr.ThreadDist(world)
    monkeypatch.setattr(sharding, "dist", fake)
    registry, out = {}, [dict(rounds=[]) for _ in range(world)]
    v1, every = signers(c, 0), list(range(len(c.addrs)))

    def rank_main(r):
        fake.local.rank = r
        torch.cuda.set_device(0)
        e = key_engine(c, budget)
        if exchange == "p2p":
            xr.share_exchange_buffers(e, registry)
        lo, hi = sharding.shard_bounds(c.n, world, r)
        first = c.batches[0]["items"][rounds_of(c)[0][1]]
        # every rank keeps the whole arena: the items' payload offsets stay valid under any permutation
        sv = sharding.ShardedVerifier(e, c.n, c.groups(e), world, r, first[lo:hi], c.arena, torch.cuda.Stream(), exchange=exchange)
        try:
            for k, (b, perm, _) in enumerate(rounds_of(c)):
                sv.h_items.copy_(torch.from_numpy(c.batches[b]["items"][perm][lo:hi].view(np.uint8).reshape(-1)))
                fake.barrier()
                t0 = time.perf_counter()
                res, bm = sv.run()
                adopted, refused = sv.share_keys()
                out[r]["rounds"].append((res.tobytes(), bm, adopted, refused, time.perf_counter() - t0))
                if k == 0:
                    out[r]["registry1"] = e.key_registry()
                    out[r]["keys1"] = registry_view(e, v1)
                fake.barrier()
            out[r]["registry"] = e.key_registry()
            out[r]["states"] = registry_view(e, every)[0]
        finally:
            sv.close()
            e.close()
    xr.run_ranks(world, rank_main, timeout=900)
    return c, out


@pytest.mark.parametrize("world", [2, 3, 8])
@pytest.mark.parametrize("exchange", ["nccl", "p2p"])
def test_share_keys_ranks_as_threads(monkeypatch, world, exchange):
    c = xr.case("config3.npz")
    ref, ready1, known = host_reference(c)
    c, out = run_sharded(monkeypatch, world, exchange)
    v1 = signers(c, 0)
    assert ready1 == len(v1) and known.sum() == len(v1)
    want_keys = config3_pubkeys()[v1]
    for r in range(world):
        for k, (res, bm, adopted, refused, _) in enumerate(out[r]["rounds"]):
            assert np.array_equal(bm, ref[k][0]), (r, k)
            assert res == ref[k][1], (r, k)
            assert refused == 0, (r, k)
        # after round 1 every rank knows every key of round 1, with its table built
        assert out[r]["registry1"][1] == ready1, r
        st, keys = out[r]["keys1"]
        assert (st == 2).all(), (r, int((st != 2).sum()))
        assert np.array_equal(keys, want_keys), r
        assert out[r]["rounds"][0][2] > 0, r                       # every rank adopted keys it did not recover
    for r in range(world):
        assert np.array_equal(out[r]["states"] != 0, known), r
    print(f"{exchange} world {world}: adopted in round 1 {[o['rounds'][0][2] for o in out]}, slowest round with share_keys "
          f"{max(x[4] for o in out for x in o['rounds']) * 1e3:.1f} ms")


def test_share_keys_bounded_registry(monkeypatch):
    """Every rank under a 300-table budget (the set has 10,000): the same keys become known on every rank as without a budget,
    and no rank holds more tables than its budget."""
    budget = 300
    c = xr.case("config3.npz")
    ref, _, known = host_reference(c)
    c, out = run_sharded(monkeypatch, 3, "nccl", budget=budget)
    for r in range(3):
        for k, (res, bm, _, refused, _) in enumerate(out[r]["rounds"]):
            assert np.array_equal(bm, ref[k][0]) and res == ref[k][1] and refused == 0, (r, k)
        assert np.array_equal(out[r]["states"] != 0, known), r
        _, ready, nbytes = out[r]["registry"]
        assert ready <= budget and nbytes <= budget * KEYTAB_BYTES, (r, ready, nbytes)


def record(a: bytes, x: int, y: int) -> list[int]:
    return list(np.frombuffer(a, np.uint32)) + words_of(x) + words_of(y)


def block(records) -> np.ndarray:
    out = np.zeros(21568, np.uint32)
    out[0] = len(records)
    for i, rec in enumerate(records):
        out[1 + REC * i: 1 + REC * (i + 1)] = rec
    return out


def test_forged_records_are_refused():
    """Blocks written by the test: forged records (x >= p, y >= p, off the curve, another validator's key) are refused and
    their entries stay unknown; a block whose count exceeds the cap is refused whole; an address no resident table lists is
    dropped; the engine's own block is skipped; valid keys are adopted, from the first and the second resident table."""
    c = xr.case("config3.npz")
    edge = [(ec.pubkey_to_address(Q), Q) for Q in A.known_points()]
    sx = next(k for k in edge if k[1][0] + ec.P < 1 << 256)
    sy = next(k for k in edge if k[1][1] + ec.P < 1 << 256 and k is not sx)
    ok_edge = next(k for k in edge if k is not sx and k is not sy)
    edge_addrs = np.array([np.frombuffer(k[0], np.uint8) for k in (sx, sy, ok_edge)])
    pub = config3_pubkeys()

    def key(v):
        return (sum(int(w) << (32 * i) for i, w in enumerate(pub[v][:8])), sum(int(w) << (32 * i) for i, w in enumerate(pub[v][8:])))
    a = [bytes(x) for x in c.addrs]
    stranger = ec.privkey_to_pubkey(wl.privkey(99, 0))
    forged = [record(sx[0], sx[1][0] + ec.P, sx[1][1]),              # x >= p
              record(sy[0], sy[1][0], sy[1][1] + ec.P),              # y >= p
              record(a[2], key(2)[0], (key(2)[1] + 1) % ec.P),        # off the curve
              record(a[3], *key(4))]                                  # validator 4's key under validator 3's address
    over = block([record(a[5], *key(5))])
    over[0] = C + 1
    own = block([record(a[6], *key(6))])                               # the engine's own part: never read
    valid = block([record(ec.pubkey_to_address(stranger), *stranger),  # no resident table lists it: dropped
                   record(a[10], *key(10)), record(ok_edge[0], *ok_edge[1])])
    e = key_engine(c)
    try:
        e.set_validators(1, HEIGHT + 1, edge_addrs)
        blocks = torch.from_numpy(np.concatenate([own, block(forged), over, valid]).view(np.int32)).cuda()
        counts = torch.zeros(2, dtype=torch.int32, device="cuda")
        ptrs = [blocks.data_ptr() + 4 * 21568 * k for k in range(4)]
        e.key_share_adopt_device(ptrs, 0, counts.data_ptr())
        torch.cuda.synchronize()
        assert counts.tolist() == [2, len(forged) + 1]
        e.refresh_key_tables()
        for v in (2, 3, 5, 6):
            assert e.key_table(0, v)[0] == 0, v
        assert e.key_table(1, 0)[0] == 0 and e.key_table(1, 1)[0] == 0
        st, k10, _ = e.key_table(0, 10)
        assert st == 2 and np.array_equal(k10, pub[10])
        st, ke, _ = e.key_table(1, 2)
        assert st == 2 and np.array_equal(ke, np.array(words_of(ok_edge[1][0]) + words_of(ok_edge[1][1]), np.uint32))
        # adopted keys are not exported; nothing was learned by recovery
        out = torch.full((21568,), -1, dtype=torch.int32, device="cuda")
        e.key_share_export_device(out.data_ptr())
        torch.cuda.synchronize()
        assert int(out[0]) == 0
        # the same blocks again: the valid keys are known now, the forged ones still refused
        e.key_share_adopt_device(ptrs, 0, counts.data_ptr())
        torch.cuda.synchronize()
        assert counts.tolist() == [0, len(forged) + 1]
    finally:
        e.close()


def test_share_calls_refused_without_registry():
    c = xr.case("config3.npz", 9950, 100)
    e = c.engine()
    try:
        d = torch.zeros(21568, dtype=torch.int32, device="cuda")
        assert e.key_share_words() == 21568
        with pytest.raises(ib.EngineError, match="no key registry"):
            e.key_share_export_device(d.data_ptr())
        with pytest.raises(ib.EngineError, match="no key registry"):
            e.key_share_adopt_device([d.data_ptr(), d.data_ptr()], 0)
    finally:
        e.close()


# ---- two processes, real CUDA IPC ------------------------------------------------------------------------------------------

def _ipc_worker(rank, store_path, payload, out_path):
    import torch.distributed as dist
    sys.path[:0] = [os.path.dirname(HERE), HERE]
    import ibft_b200 as ib2
    dist.init_process_group("gloo", store=dist.FileStore(store_path, 2), rank=rank, world_size=2)
    rep = {"rank": rank, "rounds": []}
    try:
        e = ib2.Engine(device=0, max_items=1 << 15, max_payload_bytes=1 << 22, max_groups=8, max_table_slots=4, max_validators=10_000,
                       key_cache=True)
        e.set_validators(0, HEIGHT, payload["addrs"], payload["powers_be"])
        groups = e.groups(payload["n_groups"], 0, rule=payload["rules"], proposer=[payload["proposer"]] * payload["n_groups"])
        lo, hi = sharding.shard_bounds(payload["n"], 2, rank)
        sv = sharding.ShardedVerifier(e, payload["n"], groups, 2, rank, payload["items"][0][lo:hi], payload["arena"],
                                      torch.cuda.Stream(), exchange="p2p")
        for k in range(3):
            sv.h_items.copy_(torch.from_numpy(payload["items"][k][lo:hi].view(np.uint8).reshape(-1)))
            dist.barrier()
            try:
                res, bm = sv.run()
                adopted, refused = sv.share_keys()
                ok = bool(np.array_equal(bm, payload["words"][k]) and res.tobytes() == payload["results"][k])
                rep["rounds"].append({"ok": ok, "adopted": adopted, "refused": refused, "registry": list(e.key_registry())})
            except RuntimeError as ex:
                rep["rounds"].append({"ok": False, "error": str(ex)})
        sv.close()
        e.close()
    except Exception as ex:  # noqa: BLE001 -- reported to the parent
        rep["error"] = repr(ex)
    with open(out_path, "w") as f:
        json.dump(rep, f)
    dist.destroy_process_group()


def test_two_processes_share_keys_over_real_ipc(tmp_path):
    """World 2 in two processes on the same device, p2p exchange through real CUDA IPC mappings: 3 rounds of config 2, each
    permuted, with share_keys() after each.  After round 1 both ranks hold the same ready keys."""
    c = xr.case("config2.npz")
    e = c.engine()
    perms = [np.random.default_rng(2000 + k).permutation(c.n) for k in range(3)]
    items, words, results = [], [], []
    try:
        for k in range(3):
            it = c.batches[k % 2]["items"][perms[k]]
            bm, res, _ = e.verify_batch(it, c.arena, c.groups(e))
            assert np.array_equal(bm, pe.words_of(c.batches[k % 2]["bits"][perms[k]]))
            items.append(it)
            words.append(bm)
            results.append(res.tobytes())
    finally:
        e.close()
    payload = dict(addrs=c.addrs, powers_be=c.powers_be, n_groups=c.n_groups, rules=c.rules, proposer=c.pat.proposer, n=c.n,
                   arena=c.arena, items=items, words=words, results=results)
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=_ipc_worker, args=(r, str(tmp_path / "store"), payload, str(tmp_path / f"r{r}.json"))) for r in range(2)]
    for p in procs:
        p.start()
    deadline = time.time() + 300
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
    ready = reps[0]["rounds"][0]["registry"][1]
    assert ready > 0
    for r in reps:
        assert "error" not in r, r
        assert [x["ok"] for x in r["rounds"]] == [True] * 3, r
        assert r["rounds"][0]["adopted"] > 0 and all(x["refused"] == 0 for x in r["rounds"]), r
        assert r["rounds"][0]["registry"][1] == ready, r
