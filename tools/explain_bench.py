"""The cost of ibft_explain_batch alone, after a verify over the same inputs (wall clock around the synchronous call, after warm-up).

Workloads (tests/golden/config3.npz: a 10,000-validator COMMIT round with 1 % adversarial items):
  round10k   the round's 10,000 committed seals; the verify's ~100 rejected seals are explained
  tiled_2p20 2^20 tuples (config 3 tiled); the ~1 % rejected tuples are explained
Each row also times the verify call itself, for scale.  The explained reasons are checked in the same run: one non-OK reason per
zero bit, OK elsewhere, never IBFT_REASON_INCONSISTENT.  The card name and its power limit are recorded beside the numbers.

    python tools/explain_bench.py [--steps 20] [--warmup 3] [--out FILE]
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


def gpu_power_limit() -> str:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return q.stdout.strip().replace("\n", "; ")
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import numpy as np
    import ibft_b200 as ib

    d = np.load(os.path.join(ROOT, "tests", "golden", "config3.npz"))
    items3 = np.ascontiguousarray(d["items"]).view(ib.ITEM_DTYPE).reshape(-1)
    arena3 = d["arena"].tobytes()
    eng = ib.Engine(device=0, max_items=1 << 20, max_payload_bytes=1 << 25, max_groups=8, max_table_slots=4, max_validators=10_000)
    eng.set_validators(0, 1_000_000, d["addrs"], d["powers"])
    groups = eng.groups(len(d["groups"]), slot=0)
    seals = np.ascontiguousarray(items3[items3["kind"] == ib.KIND_SEAL])
    big = np.ascontiguousarray(items3[np.arange(1 << 20) % len(items3)])
    rows = {}
    for name, items, arena in (("round10k", seals, b"\x00"), ("tiled_2p20", big, arena3)):
        bm, _, _ = eng.verify_batch(items, arena, groups)
        bits = np.unpackbits(bm.view(np.uint8), bitorder="little")[: len(items)].astype(bool)
        for _ in range(args.warmup):
            eng.explain_batch(items, arena, groups, bitmap=bm)
            eng.verify_batch(items, arena, groups)
        t_explain, t_verify = [], []
        for _ in range(args.steps):
            t0 = time.perf_counter()
            reasons, _ = eng.explain_batch(items, arena, groups, bitmap=bm)
            t_explain.append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            eng.verify_batch(items, arena, groups)
            t_verify.append(time.perf_counter() - t0)
        if (reasons == ib.REASON_INCONSISTENT).any() or not np.array_equal(reasons != ib.REASON_OK, ~bits):
            raise SystemExit(f"{name}: the reasons do not match the verify's bitmap")
        counts = {int(r): int(c) for r, c in zip(*np.unique(reasons[~bits], return_counts=True))}
        rows[name] = {"items": int(len(items)), "explained": int((~bits).sum()), "reasons": counts,
                      "explain_p50_ms": round(statistics.median(t_explain) * 1e3, 3),
                      "explain_min_ms": round(min(t_explain) * 1e3, 3),
                      "verify_p50_ms": round(statistics.median(t_verify) * 1e3, 3)}
    eng.close()
    text = json.dumps({"gpu_and_power_limit": gpu_power_limit(), "steps": args.steps, "rows": rows}, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
