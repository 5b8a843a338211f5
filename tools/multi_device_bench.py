"""One engine over several devices (ibft_engine_create_multi) against one engine on the first of them, from host buffers.

Workloads, each timed alternately on the two engines (wall clock around the synchronous call, after warm-up):
  tuples_2p20     2^20 tuples (config 3 tiled) to verdicts and quorum; verdicts checked against the oracle's config-3 bitmap
  config5         the config-5 backlog (144,953 tuples, 16 validator tables); bitmap checked against tests/golden/config5_pin.npz
  round10k        the 10,000 committed seals of a config-3 round (p50 of the step times); bitmap checked against the oracle
On distinct GPUs (--devices 0,1,...) the ratio is the scaling; with a repeated ordinal (--devices 0,0) every shard runs on the
same GPU, so the ratio is the cost of the sharding, the per-device arena plans, the peer copies and the merge.  The card name
and its power limit are recorded beside the numbers.

    python tools/multi_device_bench.py --devices 0,0 [--steps 10] [--warmup 2] [--out FILE]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_power_limit() -> str:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return q.stdout.strip().replace("\n", "; ")
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def tiled_bitmap(bits_one, n_one, n):
    import numpy as np
    b = np.unpackbits(np.asarray(bits_one, np.uint32).view(np.uint8), bitorder="little")[:n_one]
    b = np.resize(b, n)
    return np.packbits(np.concatenate([b, np.zeros((-n) % 32, np.uint8)]), bitorder="little").view(np.uint32)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--devices", default="0,0")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import numpy as np
    import ibft_b200 as ib
    import workloads as wl

    devices = [int(x) for x in args.devices.split(",")]
    cap = dict(max_items=1 << 20, max_payload_bytes=1 << 25, max_groups=128, max_table_slots=17, max_validators=10_000)
    engines = {"single": ib.Engine(device=devices[0], **cap), "multi": ib.Engine(devices=devices, **cap)}
    if engines["multi"].device_count() != len(devices):
        raise SystemExit("multi-device engine did not take every listed device")

    w3 = wl.config3()
    want3 = wl.oracle_bitmap(w3)
    c5, pin5 = wl.load_full("config5")
    seals = np.ascontiguousarray(w3["items"][w3["items"]["kind"] == ib.KIND_SEAL])
    work = {}
    for name, e in engines.items():
        for k in range(16):
            e.set_validators(k, c5["heights"][k], c5["tables"][k], c5["powers"])
        e.set_validators(16, w3["height"], w3["addrs"], w3["powers"])
    g3 = engines["single"].groups(len(w3["groups"]), slot=16)
    work["config5"] = (c5["items"], c5["arena"], engines["single"].groups(c5["n_groups"], slot=c5["group_table"]), pin5["bitmap"])
    n = 1 << 20
    idx = np.arange(n) % len(w3["items"])
    big = np.ascontiguousarray(w3["items"][idx])
    work["tuples_2p20"] = (big, w3["arena"], g3, tiled_bitmap(want3, len(w3["items"]), n))
    work["round10k"] = (seals, b"", g3, None)

    rows = {}
    for wname in ("tuples_2p20", "round10k", "config5"):
        times = {"single": [], "multi": []}
        outs = {}
        for name, e in engines.items():
            items, arena, groups, want = work[wname]
            for _ in range(args.warmup):
                e.verify_batch(items, arena, groups)
        for step in range(args.steps):
            for name in (("single", "multi") if step % 2 == 0 else ("multi", "single")):
                e = engines[name]
                items, arena, groups, want = work[wname]
                t0 = time.perf_counter()
                bm, res, _ = e.verify_batch(items, arena, groups)
                times[name].append(time.perf_counter() - t0)
                outs[name] = (bm.tobytes(), res.tobytes())
        items, arena, groups, want = work[wname]
        if want is not None and outs["single"][0] != np.asarray(want, np.uint32).tobytes():
            raise SystemExit(f"{wname}: single-engine bitmap differs from the reference")
        if outs["single"] != outs["multi"]:
            raise SystemExit(f"{wname}: multi-device results differ from the single engine")
        if wname == "round10k":
            bits = np.unpackbits(np.asarray(want3, np.uint32).view(np.uint8), bitorder="little")[:len(w3["items"])]
            sb = bits[w3["items"]["kind"] == ib.KIND_SEAL]
            sb = np.packbits(np.concatenate([sb, np.zeros((-len(sb)) % 32, np.uint8)]), bitorder="little").view(np.uint32)
            if outs["single"][0] != sb.tobytes():
                raise SystemExit("round10k: bitmap differs from the oracle")
        p50 = {k: statistics.median(v) for k, v in times.items()}
        rows[wname] = {"items": int(len(items)), "single_p50_ms": round(p50["single"] * 1e3, 3), "multi_p50_ms": round(p50["multi"] * 1e3, 3),
                       "multi_over_single": round(p50["multi"] / p50["single"], 3),
                       "single_items_per_s": round(len(items) / p50["single"]), "multi_items_per_s": round(len(items) / p50["multi"])}
    for e in engines.values():
        e.close()
    text = json.dumps({"gpu_and_power_limit": gpu_power_limit(), "devices": devices, "steps": args.steps, "rows": rows}, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
