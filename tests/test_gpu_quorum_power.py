"""The device's 320-bit quorum arithmetic on the power-edge tables of tests/power_edges.py: ibft_set_validators' total and
quorum, k_quorum_reduce's per-thread and tree carries, and group_decision's proposer addition and limb compare, on every reduce
path (host-buffer call, device-resident reduce, shard marks + merge, peer-memory exchange) and under every quorum rule, against
the big-int restatement.  The fixtures' signatures and golden bitmaps are unchanged: only the powers differ."""
import functools
import importlib

import numpy as np
import pytest
import torch

import ibft_b200 as ib
import power_edges as pe
from test_gpu_exchange_ranks import DeviceBatch, World, assert_results

pytestmark = pytest.mark.gpu
host = importlib.import_module("go-ibft_b200.host")
sharding = importlib.import_module("go-ibft_b200.sharding")
HEIGHT = 1_000_000


class Fixture:
    def __init__(self, name):
        d, rows, self.votes = pe.load(name)
        self.addrs, self.n_groups, self.bitmap = d["addrs"], len(d["groups"]), d["bitmap"]
        self.items = rows.view(ib.ITEM_DTYPE).reshape(-1)
        self.arena = np.ascontiguousarray(d["arena"], dtype=np.uint8)
        self.n = len(rows)
        self.pats = pe.patterns(self.votes, len(self.addrs))
        self.plain_powers = d["powers"]
        vw = (len(self.addrs) + 31) // 32
        self.voted = np.zeros((self.n_groups, vw), np.uint32)
        for g, (_, vs) in enumerate(self.votes):
            bits = np.zeros(vw * 32, np.uint8)
            bits[sorted(vs)] = 1
            self.voted[g] = pe.words_of(bits)


@functools.lru_cache(maxsize=None)
def fixture(name):
    return Fixture(name)


@pytest.fixture(scope="module")
def eng():
    e = ib.Engine(device=0, max_items=1 << 15, max_payload_bytes=1 << 22, max_groups=8, max_table_slots=4, max_validators=10_000)
    yield e
    e.close()


def results_of(t_res):
    torch.cuda.synchronize()
    return t_res.cpu().numpy().view(ib.RESULT_DTYPE)


@pytest.mark.parametrize("name", ["config2.npz", "config3.npz"])
def test_power_edges_every_reduce_path(eng, name):
    f = fixture(name)
    st_obj = torch.cuda.Stream()
    st = st_obj.cuda_stream
    db = DeviceBatch(f.items, f.arena)
    t_bm = torch.zeros((f.n + 31) // 32, dtype=torch.int32, device="cuda")
    t_res = torch.zeros(f.n_groups * ib.RESULT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    # the voted sets of a plain table (the fixture's own powers): the power tables must not change them
    eng.set_validators(0, HEIGHT, f.addrs, f.plain_powers)
    _, _, _, plain_voted = eng.verify_batch_ex(f.items, f.arena, eng.groups(f.n_groups), voted_stride_words=f.voted.shape[1])
    assert np.array_equal(plain_voted, f.voted)
    for pat in f.pats:
        eng.set_validators(0, HEIGHT, f.addrs, pe.powers_be(pat.powers))
        q, _, nv = eng.get_quorum(0)
        assert (q, nv) == (pat.quorum, len(f.addrs)), pat.name
        ctx = host.HostContext("callback")
        assert ctx.set_validators(0, [bytes(a) for a in f.addrs], pat.powers) == 0
        for rule in pe.RULES:
            what = (pat.name, rule)
            want = pe.expected(pat, f.votes, rule)
            groups = eng.groups(f.n_groups, 0, rule=rule, proposer=pat.proposer)
            # host-buffer call
            bm, res, _, voted = eng.verify_batch_ex(f.items, f.arena, groups, voted_stride_words=f.voted.shape[1])
            assert np.array_equal(bm, f.bitmap), what
            assert np.array_equal(voted, f.voted), what
            assert_results(res, want, what)
            for g in range(f.n_groups):
                assert np.array_equal(eng.voted_bitmap(g, len(f.addrs)), f.voted[g]), what
                if rule == pe.DEFAULT:      # the C++ mirror's HasQuorumVoted on the device's voted set
                    assert ctx.has_quorum_voted(voted[g]) == want[g][3], what
            eng.bind_groups(groups)
            with torch.cuda.stream(st_obj):
                # device-resident verify + reduce
                t_bm.zero_()
                eng.verify_device(db.items.data_ptr(), f.n, db.arena.data_ptr(), db.arena_len, 0, f.n, t_bm.data_ptr(), 0, st)
                eng.quorum_reduce_device(db.items.data_ptr(), f.n, t_bm.data_ptr(), f.n_groups, t_res.data_ptr(), st)
            st_obj.synchronize()
            assert_results(results_of(t_res), want, what + ("device",))
            with torch.cuda.stream(st_obj):
                # three 32-aligned shards: marks, then the merge
                W = eng.quorum_partial_words()
                t_parts = torch.zeros((3, W), dtype=torch.int32, device="cuda")
                for r in range(3):
                    lo, hi = sharding.shard_bounds(f.n, 3, r)
                    eng.quorum_mark_device(db.items.data_ptr(), f.n, lo, hi, t_bm.data_ptr(), t_parts[r].data_ptr(), st)
                eng.quorum_merge_device(t_parts.data_ptr(), 3, W, t_res.data_ptr(), st)
            st_obj.synchronize()
            assert_results(results_of(t_res), want, what + ("merge",))
            # the peer-memory exchange at world 3 (rank 1 calls; the peers' flags read the epoch)
            w = World(eng, f.n, 3, f.n_groups)
            w.fill(db, 1)
            for r in range(3):
                w.set_flag(r, 1, 1)
            res_x, full, timeout = w.exchange(1, 1)
            assert timeout == 0 and np.array_equal(full[: len(f.bitmap)], f.bitmap), what
            assert_results(res_x, want, what + ("exchange",))
            eng.bind_groups(None)
        ctx.close()
