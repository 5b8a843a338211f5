"""Key sharing between the ranks of a sharded verifier: what ShardedVerifier.share_keys() costs and what it saves.

For W = 2 and 8 ranks (threads on one GPU, each with its own key-cache engine and stream, over a thread stand-in for
torch.distributed's all-gather; NCCL-mode exchange), each trial runs R rounds of config 3 (20,000 items, 10,000 validators),
each round in a fresh random order as go-ibft's map iteration hands them over, once without and once with share_keys() between
rounds.  Reported per W and mode:
  round_p50_ms        median over rounds 2..R and trials of the round's latency (the slowest rank's run(), wall time)
  share_keys_p50_ms   median of share_keys() itself (export, all-gather, adopt, refresh), slowest rank
  unknown_per_round   per round, per rank: items in the rank's shard whose signer's key the rank did not know before the round
                      (from key_table states on the host; first trial).  133 of config 3's items are signed by validators none
                      of whose items verifies, so no rank ever learns their key: with sharing the sum stays at 133
Every round's bitmap is checked against the oracle's before anything is reported.  All ranks share one GPU, so this is an
overhead figure, not a scaling figure.  The card's name and power limit are recorded beside the numbers.

    python tools/sharded_keys_bench.py [--worlds 2,8] [--rounds 6] [--trials 2] [--out FILE]
"""
from __future__ import annotations

import argparse
import importlib
import json
import os
import statistics
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from multi_device_bench import gpu_power_limit  # noqa: E402


class ThreadDist:
    """the all-gather sharding.py uses, for ranks that are threads of one process"""

    def __init__(self, world):
        self.bar = threading.Barrier(world, timeout=300)
        self.slots = [None] * world
        self.local = threading.local()

    def all_gather_into_tensor(self, out, inp):
        import torch
        torch.cuda.current_stream().synchronize()
        self.slots[self.local.rank] = inp
        self.bar.wait()
        out.copy_(torch.cat([s.reshape(-1) for s in self.slots]))
        torch.cuda.current_stream().synchronize()
        self.bar.wait()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--worlds", default="2,8")
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--trials", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import numpy as np
    import torch
    import ibft_b200 as ib
    sharding = importlib.import_module("go-ibft_b200.sharding")

    d = dict(np.load(os.path.join(ROOT, "tests", "golden", "config3.npz")))   # read once: the ranks' threads share it
    items = np.ascontiguousarray(d["items"]).view(ib.ITEM_DTYPE).reshape(-1)
    arena = np.ascontiguousarray(d["arena"], np.uint8)
    n = len(items)
    bits = np.unpackbits(np.asarray(d["bitmap"], np.uint32).view(np.uint8), bitorder="little")[:n].astype(bool)
    index = {bytes(a): i for i, a in enumerate(d["addrs"])}
    signer = np.array([index.get(bytes(s), -1) for s in items.view(np.uint8).reshape(n, 128)[:, 96:116]])
    orders = [np.random.default_rng(500 + r).permutation(n) for r in range(args.rounds)]
    kw = dict(device=0, max_items=1 << 15, max_payload_bytes=1 << 22, max_groups=8, max_table_slots=2, max_validators=10_000,
              key_cache=True)

    def trial(world, share):
        fake = ThreadDist(world)
        sharding.dist = fake
        run_s, share_s, unknown = ([[0.0] * world for _ in orders] for _ in range(3))
        bad = []

        def rank_main(r):
            fake.local.rank = r
            torch.cuda.set_device(0)
            e = ib.Engine(**kw)
            e.set_validators(0, int(d["meta"][2]), d["addrs"], d["powers"])
            groups = e.groups(len(d["groups"]), slot=0)
            lo, hi = sharding.shard_bounds(n, world, r)
            sv = sharding.ShardedVerifier(e, n, groups, world, r, items[orders[0]][lo:hi], arena, torch.cuda.Stream())
            try:
                for k, idx in enumerate(orders):
                    sv.h_items.copy_(torch.from_numpy(items[idx][lo:hi].view(np.uint8).reshape(-1)))
                    mine = signer[idx][lo:hi]
                    known = {v: e.key_table(0, int(v))[0] != 0 for v in set(mine[mine >= 0].tolist())}
                    unknown[k][r] = int(sum(1 for v in mine if v >= 0 and not known[v]))
                    fake.bar.wait()
                    t0 = time.perf_counter()
                    _, bm = sv.run()
                    t1 = time.perf_counter()
                    if share:
                        sv.share_keys()
                    t2 = time.perf_counter()
                    run_s[k][r], share_s[k][r] = t1 - t0, t2 - t1
                    got = np.unpackbits(bm.view(np.uint8), bitorder="little")[:n].astype(bool)
                    if not np.array_equal(got, bits[idx]):
                        bad.append((r, k))
                    fake.bar.wait()
            finally:
                sv.close()
                e.close()
        threads = [threading.Thread(target=rank_main, args=(r,), daemon=True) for r in range(world)]
        for t in threads:
            t.start()
        for t in threads:
            t.join(900)
        if any(t.is_alive() for t in threads) or bad:
            raise SystemExit(f"world {world}: a rank did not finish or a bitmap differs from the oracle: {bad}")
        return [max(x) for x in run_s], [max(x) for x in share_s], unknown

    report = {}
    for world in [int(x) for x in args.worlds.split(",")]:
        for share in (False, True):
            rounds, shares, unknown = [], [], None
            for _ in range(args.trials):
                rr, ss, uu = trial(world, share)
                rounds += rr[1:]
                shares += ss
                unknown = uu if unknown is None else unknown
            entry = {"round_p50_ms": round(statistics.median(rounds) * 1e3, 3), "unknown_per_round": unknown}
            if share:
                entry["share_keys_p50_ms"] = round(statistics.median(shares) * 1e3, 3)
            report[f"W={world} {'with' if share else 'without'} share_keys"] = entry
    text = json.dumps({"gpu_and_power_limit": gpu_power_limit(), "rounds": args.rounds, "trials": args.trials, "items": n,
                       "validators": int(len(d["addrs"])), "per_mode": report}, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
