"""The cost of binding a COMMIT group to the accepted proposal's hash (ibft_verify_batch_hashed): the round's verify call from host
tuples to the group's decision, with and without the binding, alternated step by step (wall clock around the synchronous call,
after warm-up).

Workload (tests/golden/config3.npz): the 10,000 committed seals of a 10,000-validator COMMIT round (1 % adversarial), one group,
bound to the round's proposal hash.  Two engines: the recover path (no key registry) and the known-key path (IBFT_FLAG_KEY_CACHE,
every key learned during the warm-up).  Unbound, the recover kernels record the votes themselves; bound, they record none and one
k_quorum_mark_hashed launch marks the counted seals.  The decisions are checked in the same run: identical verdicts and results,
every valid seal counted.  The card name, power limit and SM clocks are recorded beside the numbers.

    python tools/group_hash_bench.py [--steps 30] [--warmup 5] [--out FILE]
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


def gpu_state() -> str:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip().replace("\n", "; ")
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import numpy as np
    import ibft_b200 as ib

    d = np.load(os.path.join(ROOT, "tests", "golden", "config3.npz"))
    items3 = np.ascontiguousarray(d["items"]).view(ib.ITEM_DTYPE).reshape(-1)
    seals = np.ascontiguousarray(items3[items3["kind"] == ib.KIND_SEAL]).copy()
    seals["group"] = 0
    accepted = bytes(np.asarray(d["proposal_hash"], dtype=np.uint8).reshape(-1))  # what every honest seal of the round names
    rows = {}
    for name, key_cache in (("recover", False), ("known_key", True)):
        eng = ib.Engine(device=0, max_items=1 << 15, max_payload_bytes=1 << 20, max_groups=4, max_table_slots=2, max_validators=10_000,
                        key_cache=key_cache)
        eng.set_validators(0, 1_000_000, d["addrs"], d["powers"])
        groups = eng.groups(1, slot=0)
        hashes = ib.group_hashes(1, {0: (ib.HASH_COMMIT, accepted)})
        for _ in range(args.warmup):
            eng.verify_batch_ex(seals, b"", groups)
            eng.verify_batch_ex(seals, b"", groups, group_hashes=hashes)
        t_plain, t_bound = [], []
        launches = {}
        for _ in range(args.steps):
            l0 = eng.launch_count()
            t0 = time.perf_counter()
            b0, r0, _, _ = eng.verify_batch_ex(seals, b"", groups)
            t_plain.append(time.perf_counter() - t0)
            l1 = eng.launch_count()
            t0 = time.perf_counter()
            b1, r1, _, _, c1 = eng.verify_batch_ex(seals, b"", groups, group_hashes=hashes)
            t_bound.append(time.perf_counter() - t0)
            launches = {"plain": l1 - l0, "bound": eng.launch_count() - l1}
        if not np.array_equal(b0, b1) or r0.tobytes() != r1.tobytes() or not np.array_equal(c1, b1):
            raise SystemExit(f"{name}: the bound call's verdicts or decision differ from the unbound call's")
        rows[name] = {"items": int(len(seals)), "valid": int(r1[0]["n_valid"]), "has_quorum": int(r1[0]["has_quorum"]),
                      "launches": launches,
                      "unbound_p50_ms": round(statistics.median(t_plain) * 1e3, 3),
                      "bound_p50_ms": round(statistics.median(t_bound) * 1e3, 3),
                      "unbound_min_ms": round(min(t_plain) * 1e3, 3), "bound_min_ms": round(min(t_bound) * 1e3, 3)}
        eng.close()
    text = json.dumps({"gpu_power_limit_clocks": gpu_state(), "steps": args.steps, "rows": rows}, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
