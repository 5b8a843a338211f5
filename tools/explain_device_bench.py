"""The cost of ibft_explain_batch_device (CUDA events around the call on its stream, medians after warm-up).

Workloads (tests/golden/config3.npz: a 10,000-validator COMMIT round with 1 % adversarial items):
  round10k     the round's 10,000 committed seals, device-resident: ibft_explain_batch_device over the whole batch, beside the
               ibft_verify_batch_device it follows and the host-buffer ibft_explain_batch of the same items and bitmap
  sharded2     the same round as a 2-rank ShardedVerifier on one device (ranks are threads, the nccl exchange over a
               thread-barrier all-gather): the time one round's run() takes, and the time explain() and explain(gather=True) add
  tiled_2p20   2^20 tuples (config 3 tiled), device-resident: the explain call and its cost per explained item
Every row checks its reasons against the host path in the same run.  The card name, its power limit and its SM clock limit are
recorded beside the numbers.

    python tools/explain_device_bench.py [--steps 20] [--warmup 3] [--out FILE]
"""
from __future__ import annotations

import argparse
import importlib
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info() -> str:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return q.stdout.strip().replace("\n", "; ")
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def med_ms(ts):
    return round(statistics.median(ts) * 1e3, 4)


class DeviceBatch:
    def __init__(self, ib, torch, items, arena: bytes):
        import numpy as np
        self.n = len(items)
        self.items = torch.from_numpy(items.view(np.uint8).reshape(-1).copy()).cuda()
        self.arena = torch.from_numpy(np.frombuffer(arena, np.uint8).copy()).cuda()
        self.arena_len = len(arena)
        self.bitmap = torch.zeros((self.n + 31) // 32, dtype=torch.int32, device="cuda")
        self.reasons = torch.zeros(self.n, dtype=torch.uint8, device="cuda")
        self.rec = torch.zeros(self.n * 20, dtype=torch.uint8, device="cuda")
        self.count = torch.zeros(1, dtype=torch.int32, device="cuda")
        self.stream = torch.cuda.Stream()
        torch.cuda.synchronize()

    def verify(self, eng):
        eng.verify_device(self.items.data_ptr(), self.n, self.arena.data_ptr(), self.arena_len, 0, self.n, self.bitmap.data_ptr(), 0,
                          self.stream.cuda_stream)

    def explain(self, eng):
        eng.explain_device(self.items.data_ptr(), self.n, self.arena.data_ptr(), self.arena_len, 0, self.n, self.bitmap.data_ptr(),
                           self.reasons.data_ptr(), self.rec.data_ptr(), self.count.data_ptr(), self.stream.cuda_stream)


def timed(torch, stream, fn, steps, warmup):
    """median device time (CUDA events on `stream`) of fn()"""
    for _ in range(warmup):
        fn()
    stream.synchronize()
    ts = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        fn()
        b.record(stream)
        b.synchronize()
        ts.append(a.elapsed_time(b) / 1e3)
    return ts


def device_row(ib, torch, eng, groups, items, arena, steps, warmup, host_explain):
    import numpy as np
    db = DeviceBatch(ib, torch, items, arena)
    t_verify = timed(torch, db.stream, lambda: db.verify(eng), steps, warmup)
    bm = db.bitmap.cpu().numpy().view(np.uint32).copy()
    t_explain = timed(torch, db.stream, lambda: db.explain(eng), steps, warmup)
    db.stream.synchronize()
    reasons, rec = db.reasons.cpu().numpy(), db.rec.cpu().numpy().reshape(-1, 20)
    want, want_rec = eng.explain_batch(items, arena, groups, bitmap=bm)
    if not (np.array_equal(reasons, want) and np.array_equal(rec, want_rec)):
        raise SystemExit("the device path's reasons differ from the host path's")
    explained = int(db.count.item())
    row = {"items": db.n, "explained": explained, "verify_device_p50_ms": med_ms(t_verify), "explain_device_p50_ms": med_ms(t_explain),
           "explain_device_min_ms": round(min(t_explain) * 1e3, 4),
           "explain_device_ns_per_explained_item": round(statistics.median(t_explain) * 1e9 / max(1, explained), 1)}
    if host_explain:
        ts = []
        for k in range(warmup + steps):
            t0 = time.perf_counter()
            eng.explain_batch(items, arena, groups, bitmap=bm)
            if k >= warmup:
                ts.append(time.perf_counter() - t0)
        row["explain_batch_host_p50_ms"] = med_ms(ts)
    return row


class ThreadDist:
    """all_gather_into_tensor / barrier / all_gather_object for ranks that are threads of one process"""

    def __init__(self, torch, world):
        self.torch, self.bar, self.slots, self.local = torch, threading.Barrier(world, timeout=300), [None] * world, threading.local()

    def barrier(self):
        self.bar.wait()

    def all_gather_object(self, out, obj):
        self.slots[self.local.rank] = obj
        self.bar.wait()
        out[:] = list(self.slots)
        self.bar.wait()

    def all_gather_into_tensor(self, out, inp):
        self.torch.cuda.current_stream().synchronize()
        self.slots[self.local.rank] = inp
        self.bar.wait()
        out.copy_(self.torch.cat([s.reshape(-1) for s in self.slots]))
        self.torch.cuda.current_stream().synchronize()
        self.bar.wait()


def sharded_row(ib, torch, d, items, arena: bytes, steps, warmup, world=2):
    import numpy as np
    sharding = importlib.import_module("go-ibft_b200.sharding")
    fake = ThreadDist(torch, world)
    sharding.dist = fake
    out, errs = [None] * world, [None] * world

    def rank_main(r):
        try:
            fake.local.rank = r
            torch.cuda.set_device(0)
            e = ib.Engine(device=0, max_items=1 << 15, max_payload_bytes=1 << 22, max_groups=8, max_table_slots=4, max_validators=10_000)
            e.set_validators(0, 1_000_000, d["addrs"], d["powers"])
            lo, hi = sharding.shard_bounds(len(items), world, r)
            li, la = sharding.rebase_shard(items, np.frombuffer(arena, np.uint8), lo, hi)
            sv = sharding.ShardedVerifier(e, len(items), e.groups(len(d["groups"]), slot=0), world, r, li, la, torch.cuda.Stream())
            t = {"run": [], "explain": [], "explain_gather": []}
            for k in range(warmup + steps):
                fake.barrier()
                t0 = time.perf_counter()
                sv.run()
                t1 = time.perf_counter()
                local = sv.explain()
                t2 = time.perf_counter()
                full = sv.explain(gather=True)
                t3 = time.perf_counter()
                if k >= warmup:
                    for key, dt in (("run", t1 - t0), ("explain", t2 - t1), ("explain_gather", t3 - t2)):
                        t[key].append(dt)
            out[r] = (t, local, full, lo, hi)
            sv.close()
            e.close()
        except BaseException as ex:  # noqa: BLE001 -- reported below
            errs[r] = ex
            fake.bar.abort()
    threads = [threading.Thread(target=rank_main, args=(r,), daemon=True) for r in range(world)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    if any(errs):
        raise SystemExit(f"sharded run failed: {errs}")
    e = ib.Engine(device=0, max_items=1 << 15, max_payload_bytes=1 << 22, max_groups=8, max_table_slots=4, max_validators=10_000)
    e.set_validators(0, 1_000_000, d["addrs"], d["powers"])
    groups = e.groups(len(d["groups"]), slot=0)
    bm, _, _ = e.verify_batch(items, arena, groups)
    want = e.explain_batch(items, arena, groups, bitmap=bm)
    e.close()
    for t, local, full, lo, hi in out:
        if not (np.array_equal(local[0], want[0][lo:hi]) and np.array_equal(full[0], want[0]) and np.array_equal(full[1], want[1])):
            raise SystemExit("a rank's explain() differs from the host path's")
    t0 = out[0][0]
    return {"world": world, "items": len(items), "run_p50_ms": med_ms(t0["run"]), "explain_added_p50_ms": med_ms(t0["explain"]),
            "explain_gather_added_p50_ms": med_ms(t0["explain_gather"])}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import numpy as np
    import torch
    import ibft_b200 as ib

    d = dict(np.load(os.path.join(ROOT, "tests", "golden", "config3.npz")))     # read once: the ranks below are threads
    items3 = np.ascontiguousarray(d["items"]).view(ib.ITEM_DTYPE).reshape(-1)
    arena3 = d["arena"].tobytes()
    seals = np.ascontiguousarray(items3[items3["kind"] == ib.KIND_SEAL])
    big = np.ascontiguousarray(items3[np.arange(1 << 20) % len(items3)])
    eng = ib.Engine(device=0, max_items=1 << 20, max_payload_bytes=1 << 25, max_groups=8, max_table_slots=4, max_validators=10_000)
    eng.set_validators(0, 1_000_000, d["addrs"], d["powers"])
    groups = eng.groups(len(d["groups"]), slot=0)
    eng.bind_groups(groups)
    rows = {"round10k": device_row(ib, torch, eng, groups, seals, b"\x00", args.steps, args.warmup, True),
            "tiled_2p20": device_row(ib, torch, eng, groups, big, arena3, args.steps, args.warmup, False)}
    eng.close()
    rows["sharded2"] = sharded_row(ib, torch, d, seals, b"\x00", args.steps, args.warmup)
    text = json.dumps({"gpu_power_limit_sm_clock": gpu_info(), "steps": args.steps, "rows": rows}, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
