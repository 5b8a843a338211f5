"""Bounded key registry (ibft_set_key_table_budget): what a comb-table budget below the validator set costs.

On this tree's config-3 fixture (10,000 validators, 20,000 items), for each budget (unbounded = no budget set), in one engine per
budget: the fixture is verified once (keys learned, tables built into the budget on the way out, lowest addresses first), then
  known_verifies_s   known-key throughput, device-resident entry points, config 3 tiled to 120,000 items (CUDA events, 20 steps)
  round10k_p50_us    host-buffer round of the 10,000 COMMIT seals (wall clock, p50 of 50)
  set_next_ms        wall time of ibft_set_validators for the next height of the same set (a reclaim point in bounded mode)
  table_bytes        comb-table bytes the registry holds (ibft_debug_key_registry)
  tables             validators with a built table
The card name and its power limit are recorded beside the numbers.

    python tools/key_budget_bench.py [--budgets none,10000,7500,5000,2500,0] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def measure(budget: int | None) -> dict:
    import numpy as np
    import torch

    import ibft_b200 as ib

    d = np.load(os.path.join(ROOT, "tests", "golden", "config3.npz"))
    items = np.ascontiguousarray(d["items"]).view(ib.ITEM_DTYPE).reshape(-1)
    addrs, powers, h = d["addrs"], d["powers"], int(d["meta"][2])
    reps = 6
    big = np.tile(items, reps)
    eng = ib.Engine(device=0, max_items=len(big), max_payload_bytes=max(1 << 20, int(d["arena"].nbytes)), max_groups=8,
                    max_table_slots=2, max_validators=len(addrs), key_cache=True, key_table_budget=budget)
    out = {"budget": budget}
    try:
        eng.set_validators(0, h, addrs, powers)
        groups = eng.groups(len(d["groups"]), 0)
        eng.verify_batch(items, d["arena"], groups)
        out["keys_known"] = eng.refresh_key_tables()
        eng.bind_groups(groups)
        stream = torch.cuda.Stream()
        t_items = torch.from_numpy(big.view(np.uint8).reshape(-1, 128).copy()).cuda()
        t_arena = torch.from_numpy(np.ascontiguousarray(d["arena"]).copy()).cuda()
        n = len(big)
        t_bm = torch.zeros((n + 31) // 32, dtype=torch.int32, device="cuda")
        t_res = torch.zeros(len(groups) * ib.RESULT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")

        def step():
            eng.verify_device(t_items.data_ptr(), n, t_arena.data_ptr(), t_arena.numel(), 0, n, t_bm.data_ptr(), 0, stream.cuda_stream)
            eng.quorum_reduce_device(t_items.data_ptr(), n, t_bm.data_ptr(), len(groups), t_res.data_ptr(), stream.cuda_stream)

        for _ in range(3):
            step()
        torch.cuda.synchronize()
        gold = np.unpackbits(d["bitmap"].view(np.uint8), bitorder="little")[: len(items)]
        got = np.unpackbits(t_bm.cpu().numpy().view(np.uint8), bitorder="little")[:n]
        out["bitmap_matches_golden"] = bool(np.array_equal(got, np.tile(gold, reps)))
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        steps = 20
        a.record(stream)
        for _ in range(steps):
            step()
        b.record(stream)
        torch.cuda.synchronize()
        out["known_verifies_s"] = n / (a.elapsed_time(b) / steps * 1e-3)
        eng.bind_groups(None)
        seal_group = list(d["groups"]).index("COMMIT_SEAL")
        seals = np.ascontiguousarray(items[items["group"] == seal_group])
        lat = []
        for i in range(55):
            t0 = time.perf_counter()
            eng.verify_batch(seals, b"", groups)
            if i >= 5:
                lat.append((time.perf_counter() - t0) * 1e6)
        out["round10k_p50_us"] = statistics.median(lat)
        t0 = time.perf_counter()
        eng.set_validators(1, h + 1, addrs, powers)
        out["set_next_ms"] = (time.perf_counter() - t0) * 1e3
        _, out["tables"], out["table_bytes"] = eng.key_registry()
        out["device"] = eng.device_info()["name"]
    finally:
        eng.close()
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--budgets", default="none,10000,7500,5000,2500,0")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        card = q.stdout.strip().splitlines()[0]
    except Exception as ex:  # noqa: BLE001
        card = f"unknown ({ex})"
    rows = [measure(None if b == "none" else int(b)) for b in args.budgets.split(",")]
    text = json.dumps({"gpu_and_power_limit": card, "rows": rows}, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
