"""Key registry (IBFT_FLAG_KEY_CACHE) measurements, alternating between engine libraries in one run.

For each source tree (--tree NAME=DIR: a checkout whose go-ibft_b200/libibftverify.so is built, e.g. this one and an earlier
commit's), in a fresh process that imports that tree's package and loads its library, on this tree's config-3 fixture (10,000 validators, 20,000 items):
  set_next_ms        wall time of ibft_set_validators for the next height of the 10k set whose keys are known (15 heights:
                     slots 1..15 while slot 0 holds the height that learned the keys)
  registry_bytes     comb-table bytes held for the 16 resident heights (ibft_debug_key_registry where the library has it,
                     otherwise heights x validators x 136 KiB, the per-slot allocation)
  free_drop_bytes    drop of the device's free memory over the 15 calls (informational: the card may be shared)
  known_verifies_s   known-key throughput, device-resident entry points, config 3 tiled to 120,000 items (CUDA events)
  round10k_p50_us    host-buffer round of the 10,000 COMMIT seals on the known-key latency path (wall clock, p50 of 50)
Rounds alternate A B A B ...; the summary gives the median and the range of each figure per library.  The card name and its
power limit are recorded beside the numbers.

    python tools/key_registry_bench.py --tree new=. --tree old=/path/to/an/earlier/checkout
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


def child(tree: str, out_path: str) -> None:
    import numpy as np
    import torch

    sys.path.insert(0, tree)
    import ibft_b200 as ib

    d = np.load(os.path.join(ROOT, "tests", "golden", "config3.npz"))
    items = np.ascontiguousarray(d["items"]).view(ib.ITEM_DTYPE).reshape(-1)
    addrs, powers, h = d["addrs"], d["powers"], int(d["meta"][2])
    n_val = len(addrs)
    reps = 6
    big = np.tile(items, reps)
    eng = ib.Engine(device=0, max_items=len(big), max_payload_bytes=max(1 << 20, int(d["arena"].nbytes)), max_groups=8,
                    max_table_slots=16, max_validators=n_val, key_cache=True)
    out = {"lib": os.environ.get("IBFT_LIB", "")}
    try:
        eng.set_validators(0, h, addrs, powers)
        groups = eng.groups(len(d["groups"]), 0)
        eng.verify_batch(items, d["arena"], groups)            # keys learned, tables built on the way out
        out["keys_known"] = eng.refresh_key_tables()
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        times = []
        for k in range(1, 16):
            t0 = time.perf_counter()
            eng.set_validators(k, h + k, addrs, powers)
            times.append((time.perf_counter() - t0) * 1e3)
        out["free_drop_bytes"] = int(free0 - torch.cuda.mem_get_info()[0])
        out["set_next_ms"] = times[0]
        out["set_next_ms_p50_of_15"] = statistics.median(times)
        out["keys_known_16_heights"] = eng.refresh_key_tables()
        try:
            out["registry_bytes"] = eng.key_registry()[2]
            out["registry_bytes_source"] = "ibft_debug_key_registry"
        except (AttributeError, ib.EngineError):           # a library without ibft_debug_key_registry
            out["registry_bytes"] = 16 * n_val * 17 * 128 * 64
            out["registry_bytes_source"] = "16 heights x validators x 136 KiB (per-slot allocation)"
        # known-key throughput: device-resident entry points, as bench.py's key-registry leg
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
        # the 10,000-seal round on the known-key latency path, host buffers in / out
        seal_group = list(d["groups"]).index("COMMIT_SEAL")
        seals = np.ascontiguousarray(items[items["group"] == seal_group])
        lat = []
        for i in range(55):
            t0 = time.perf_counter()
            eng.verify_batch(seals, b"", groups)
            if i >= 5:
                lat.append((time.perf_counter() - t0) * 1e6)
        out["round10k_p50_us"] = statistics.median(lat)
        info = eng.device_info()
        out["device"] = info["name"]
    finally:
        eng.close()
    with open(out_path, "w") as f:
        json.dump(out, f)


def gpu_power_limit() -> str:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as ex:  # noqa: BLE001
        return f"unknown ({ex})"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--tree", action="append", default=[], help="NAME=DIR of a source tree with its library built (two or more)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="")
    ap.add_argument("--child", nargs=2, default=None, metavar=("TREE", "OUT"))
    args = ap.parse_args()
    if args.child:
        child(*args.child)
        return
    libs = [(name, os.path.abspath(path)) for name, path in (x.split("=", 1) for x in args.tree)]
    runs = {name: [] for name, _ in libs}
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        for r in range(args.rounds):
            for name, path in libs:
                res = os.path.join(tmp, f"{name}-{r}.json")
                env = dict(os.environ, IBFT_LIB=os.path.join(path, "go-ibft_b200", "libibftverify.so"))
                subprocess.run([sys.executable, os.path.abspath(__file__), "--child", path, res], env=env, check=True, cwd=tmp)
                with open(res) as f:
                    runs[name].append(json.load(f))
    keys = ["set_next_ms", "set_next_ms_p50_of_15", "registry_bytes", "free_drop_bytes", "known_verifies_s", "round10k_p50_us"]
    summary = {"gpu_and_power_limit": gpu_power_limit(), "rounds": args.rounds, "libs": {}}
    for name, rs in runs.items():
        s = {k: {"median": statistics.median(x[k] for x in rs), "min": min(x[k] for x in rs), "max": max(x[k] for x in rs)} for k in keys}
        s["bitmap_matches_golden"] = all(x["bitmap_matches_golden"] for x in rs)
        s["keys_known_16_heights"] = rs[0]["keys_known_16_heights"]
        s["registry_bytes_source"] = rs[0]["registry_bytes_source"]
        s["runs"] = rs
        summary["libs"][name] = s
    text = json.dumps(summary, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
