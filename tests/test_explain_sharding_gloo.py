"""ShardedVerifier.explain's assembly on CPU: a world-size-2 gloo run of the helpers it is built from (explain_shard's rebased
output pointers, the padded explain blocks, their all-gather in rank order and explain_rows), with a stand-in engine whose
explain_device writes the reasons and addresses of tests/explain_oracle.py where ibft_explain_batch_device would write them.
The GPU run of the same code is tests/test_gpu_explain_device.py::test_sharded_verifier_explain."""
import ctypes
import importlib
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

sharding = importlib.import_module("go-ibft_b200.sharding")
HERE = os.path.dirname(os.path.abspath(__file__))
ITEMS_BASE, BITMAP_BASE, ARENA = 0x10000, 0x20000, 0x30000      # stand-in device addresses: only passed through


class _FakeExplainEngine:
    """stands in for Engine.explain_device: writes rows [lo, hi) of the expected reasons / addresses at the pointers it is given,
    indexed by global item number as the device call does"""

    def __init__(self, reasons: np.ndarray, rec: np.ndarray):
        self.reasons, self.rec, self.calls = reasons, rec, []

    def explain_device(self, d_items, n, d_arena, arena_len, lo, hi, d_bitmap, d_reasons, d_recovered=0, d_count=0, stream=0):
        self.calls.append((d_items, n, d_arena, arena_len, lo, hi, d_bitmap, d_count, stream))
        r = np.ascontiguousarray(self.reasons[lo:hi])
        a = np.ascontiguousarray(self.rec[lo:hi])
        ctypes.memmove(d_reasons + lo, r.ctypes.data, r.nbytes)
        ctypes.memmove(d_recovered + 20 * lo, a.ctypes.data, a.nbytes)


def expected(n_items):
    """config 2's first n_items against its golden bitmap: OK and a zero address for a one bit, the reference's reason and
    address for a zero bit"""
    import sys
    sys.path.insert(0, HERE)
    import explain_oracle as X
    from test_explain_oracle import load_fixture
    items, arena, addrs, bitmap, _, ng = load_fixture("config2")
    items = items[:n_items]
    zero = np.nonzero(~X.bits_of(bitmap, len(items)))[0]
    reasons = np.zeros(n_items, np.uint8)
    rec = np.zeros((n_items, 20), np.uint8)
    reasons[zero], rec[zero] = X.explain_batch(items[zero], arena, [addrs], [0] * ng)
    assert np.isin(reasons[zero], [X.OK, X.INCONSISTENT], invert=True).all()
    return reasons, rec


def _worker(rank, world, port, n_items, out_dir, reasons, rec):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    eng = _FakeExplainEngine(reasons, rec)
    nb = sharding.explain_block_bytes(n_items, world)
    block = torch.zeros(nb, dtype=torch.uint8)
    sharding.explain_shard(eng, block, n_items, world, rank, ITEMS_BASE, ARENA, 77, BITMAP_BASE, 5)
    local = sharding.explain_rows(block.numpy(), n_items, world, rank)
    full = sharding.gather_explain_blocks(block, torch.zeros(world * nb, dtype=torch.uint8), world)
    whole = sharding.explain_rows(full.numpy(), n_items, world)
    np.savez(os.path.join(out_dir, f"explain_{rank}.npz"), reasons=local[0], rec=local[1], all_reasons=whole[0], all_rec=whole[1],
             block=block.numpy(), calls=np.array(eng.calls, dtype=np.int64).reshape(-1, 9))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("n_items", [3000, 1001])
def test_two_rank_gloo_explain_gather_matches_unsharded(tmp_path, n_items):
    reasons, rec = expected(n_items)
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    mp.spawn(_worker, args=(2, port, n_items, str(tmp_path), reasons, rec), nprocs=2, join=True)
    P = sharding.shard_words(n_items, 2) * 32
    for r in range(2):
        got = np.load(os.path.join(str(tmp_path), f"explain_{r}.npz"))
        lo, hi = sharding.shard_bounds(n_items, 2, r)
        # one call over the rank's shard, with the verify call's rebased tuple and bitmap pointers passed through
        assert got["calls"].tolist() == [[ITEMS_BASE, n_items, ARENA, 77, lo, hi, BITMAP_BASE, 0, 5]]
        assert np.array_equal(got["reasons"], reasons[lo:hi]) and np.array_equal(got["rec"], rec[lo:hi])
        # every rank holds the whole batch, in item order
        assert np.array_equal(got["all_reasons"], reasons) and np.array_equal(got["all_rec"], rec)
        # the padding of a short shard is never written
        blk = got["block"]
        assert not blk[hi - lo: P].any() and not blk[P + 20 * (hi - lo):].any()
    assert (reasons != 0).sum() > 0
