#!/usr/bin/env python3
"""Per-launch time split of bench.py's headline step, on the bench's own workload (config 3 tiled to 2^20 device-resident tuples,
one GPU): ibft_verify_batch_device (k_recover) and ibft_quorum_reduce_device (two memsets, k_quorum_mark, k_quorum_reduce).

Each build runs in a process of its own (the engine library is loaded once per process, IBFT_LIB selects it):
  1. timing: CUDA events around each of the two C-ABI calls of every step (median over --steps steps after --warmup);
  2. split:  a separate torch.profiler run over --prof-steps steps gives each kernel's and memset's device time per step.
The card's name, power limit and SM clock are read in the same process, around the timed steps.  Several --lib paths are run
alternately, --rounds times each, so that builds compare within one session on one card.  Needs a CUDA device.

  python tools/step_profile.py                                  # the in-tree build
  python tools/step_profile.py --lib A.so --lib B.so --rounds 3 --json split.json
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ITEMS = 1 << 20  # bench.py ITEMS_PER_GPU


def card() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0],
                              f"--query-gpu={q}", "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        name, plim, sm, smax = [p.strip() for p in out.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit_w": float(plim), "sm_mhz": int(float(sm)), "sm_max_mhz": int(float(smax))}
    except Exception as e:  # the split is still worth having without the card's clocks
        return {"error": str(e)}


def kernel_group(name: str) -> str:
    if name.startswith("k_recover") or "k_recover" in name:
        return "recover"
    if "k_quorum_mark" in name:
        return "mark"
    if "k_quorum_reduce" in name:
        return "reduce"
    if "memset" in name.lower():
        return "memset"
    return "other"


def child(args) -> dict:
    import numpy as np
    import torch
    sys.path.insert(0, ROOT)
    import ibft_b200 as ib
    if not torch.cuda.is_available():
        raise SystemExit("step_profile.py needs a CUDA device")
    d = np.load(os.path.join(ROOT, "tests", "golden", "config3.npz"))
    base = np.ascontiguousarray(d["items"]).view(ib.ITEM_DTYPE).reshape(-1)
    items = np.ascontiguousarray(np.tile(base, (ITEMS + len(base) - 1) // len(base))[:ITEMS])
    eng = ib.Engine(device=0, max_items=ITEMS, max_payload_bytes=max(1 << 22, len(d["arena"])), max_groups=8, max_table_slots=2,
                    max_validators=16384)
    eng.set_validators(0, int(d["meta"][2]), d["addrs"], d["powers"])
    groups = eng.groups(len(d["groups"]))
    eng.bind_groups(groups)
    t_items = torch.from_numpy(items.view(np.uint8).reshape(-1, 128)).cuda()
    t_arena = torch.from_numpy(np.ascontiguousarray(d["arena"])).cuda()
    t_bitmap = torch.zeros(ITEMS // 32, dtype=torch.int32, device="cuda")
    t_results = torch.zeros(len(groups) * ib.RESULT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)

    def recover():
        eng.verify_device(t_items.data_ptr(), ITEMS, t_arena.data_ptr(), t_arena.numel(), 0, ITEMS, t_bitmap.data_ptr(), 0,
                          stream.cuda_stream)

    def quorum():
        eng.quorum_reduce_device(t_items.data_ptr(), ITEMS, t_bitmap.data_ptr(), len(groups), t_results.data_ptr(), stream.cuda_stream)

    for _ in range(args.warmup):
        recover()
        quorum()
    torch.cuda.synchronize()
    golden = np.unpackbits(d["bitmap"].view(np.uint8), bitorder="little")[: len(base)]
    got = np.unpackbits(t_bitmap.cpu().numpy().view(np.uint8), bitorder="little")[:ITEMS]
    if not np.array_equal(got, np.tile(golden, (ITEMS + len(base) - 1) // len(base))[:ITEMS]):
        raise SystemExit("step_profile: verdict bitmap differs from the golden bitmap")

    info_before = card()
    ev = [[torch.cuda.Event(enable_timing=True) for _ in range(3)] for _ in range(args.steps)]
    for e in ev:
        e[0].record(stream)
        recover()
        e[1].record(stream)
        quorum()
        e[2].record(stream)
    torch.cuda.synchronize()
    info_after = card()
    rec = [e[0].elapsed_time(e[1]) for e in ev]
    quo = [e[1].elapsed_time(e[2]) for e in ev]
    step = [e[0].elapsed_time(e[2]) for e in ev]

    from torch.profiler import ProfilerActivity, profile
    split = {}
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.prof_steps):
            recover()
            quorum()
        torch.cuda.synchronize()
    for evt in prof.events():
        if not str(evt.device_type).endswith("CUDA"):
            continue
        g = kernel_group(evt.name)
        split.setdefault(g, []).append(evt.device_time_total / 1000.0 if hasattr(evt, "device_time_total") else evt.cuda_time_total / 1000.0)
    per_step = {g: sum(v) / args.prof_steps for g, v in split.items()}
    launches = {g: len(v) / args.prof_steps for g, v in split.items()}
    eng.close()
    return {"lib": os.environ.get("IBFT_LIB") or "in-tree", "card_before": info_before, "card_after": info_after,
            "steps": args.steps, "ms_recover_median": statistics.median(rec), "ms_quorum_median": statistics.median(quo),
            "ms_step_median": statistics.median(step), "ms_step_range": [min(step), max(step)],
            "verifies_per_s_median": ITEMS / (statistics.median(step) * 1e-3),
            "profiler_ms_per_step": per_step, "profiler_launches_per_step": launches}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--lib", action="append", default=[], help="engine library to time (repeatable; default: the in-tree build)")
    ap.add_argument("--rounds", type=int, default=1, help="runs per library, alternated")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--prof-steps", type=int, default=3)
    ap.add_argument("--json", default=None, help="also write every result to this file")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        print(json.dumps(child(args)), flush=True)
        return
    libs = args.lib or [None]
    results = []
    for r in range(args.rounds):
        for lib in libs:
            env = dict(os.environ)
            if lib:
                env["IBFT_LIB"] = os.path.abspath(lib)
            cmd = [sys.executable, os.path.abspath(__file__), "--child", "--steps", str(args.steps), "--warmup", str(args.warmup),
                   "--prof-steps", str(args.prof_steps)]
            with tempfile.TemporaryDirectory() as tmp:  # torch.profiler / caches write here, never into the tree
                env.setdefault("TMPDIR", tmp)
                out = subprocess.run(cmd, env=env, capture_output=True, text=True, cwd=tmp)
            if out.returncode != 0:
                sys.stderr.write(out.stderr)
                raise SystemExit(f"step_profile: run with {lib or 'the in-tree build'} failed")
            res = json.loads(out.stdout.strip().splitlines()[-1])
            res["round"] = r
            results.append(res)
            split = " ".join(f"{k}={v:.3f}" for k, v in sorted(res["profiler_ms_per_step"].items()))
            print(f"round {r} {res['lib']}: step {res['ms_step_median']:.3f} ms (recover {res['ms_recover_median']:.3f}, quorum "
                  f"{res['ms_quorum_median']:.3f}) = {res['verifies_per_s_median'] / 1e6:.2f} M/s | profiler ms/step: {split} | "
                  f"{res['card_before'].get('name')} {res['card_before'].get('power_limit_w')} W "
                  f"{res['card_before'].get('sm_mhz')}/{res['card_after'].get('sm_mhz')} MHz", flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
