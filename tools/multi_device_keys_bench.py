"""Key sharing on a multi-device engine: how fast a key-cache engine over several devices stops handing items back to recovery.

For each engine ([0] and the --devices list), each trial makes a fresh key-cache engine and runs R rounds of the 10,000
committed seals of config 3, each round in a fresh random order (as go-ibft's map iteration hands them over).  Per round:
  handed_back   items the known-key pass left to recovery, per device (ibft_debug_known_handed_back of each sub-engine)
  p50_ms        median over the trials of the round's wall time (a synchronous host-buffer call)
Then one more trial of round 1 on the multi-device engine runs under torch.profiler: the device time of k_adopt_peer_keys, of
the device-to-device / peer copies of that call (the share step's state and key copies, plus the quorum merge's small copies)
and of the comb-table builds.  Every round's bitmap is checked against the oracle's before anything is reported.  With a
repeated ordinal (--devices 0,0) this measures the overhead and the warm-up curve, not scaling.  The card's name and power
limit are recorded beside the numbers.

    python tools/multi_device_keys_bench.py --devices 0,0 [--rounds 6] [--trials 3] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from multi_device_bench import gpu_power_limit  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--devices", default="0,0")
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--trials", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import numpy as np
    import ibft_b200 as ib

    d = np.load(os.path.join(ROOT, "tests", "golden", "config3.npz"))
    items = np.ascontiguousarray(d["items"]).view(ib.ITEM_DTYPE).reshape(-1)
    bits = np.unpackbits(np.asarray(d["bitmap"], np.uint32).view(np.uint8), bitorder="little")[:len(items)].astype(bool)
    seal = items["kind"] == ib.KIND_SEAL
    seals, want = np.ascontiguousarray(items[seal]), bits[seal]
    kw = dict(max_items=1 << 15, max_payload_bytes=1 << 16, max_groups=4, max_table_slots=1, max_validators=10_000, key_cache=True)
    orders = [np.random.default_rng(100 + r).permutation(len(seals)) for r in range(args.rounds)]
    devices = [int(x) for x in args.devices.split(",")]

    def make(devs):
        e = ib.Engine(devices=devs, **kw)
        e.set_validators(0, int(d["meta"][2]), d["addrs"], d["powers"])
        return e, e.groups(len(d["groups"]), slot=0)

    def one_round(e, g, idx):
        t0 = time.perf_counter()
        bm, _, _ = e.verify_batch(seals[idx], b"", g)
        dt = time.perf_counter() - t0
        got = np.unpackbits(bm.view(np.uint8), bitorder="little")[:len(idx)].astype(bool)
        if not np.array_equal(got, want[idx]):
            raise SystemExit("bitmap differs from the oracle")
        return dt, [e.sub(k).known_handed_back() for k in range(e.device_count())]

    report = {}
    for devs in ([devices[0]], devices):
        times = [[] for _ in orders]
        handed = None
        for _ in range(args.trials):
            e, g = make(devs)
            try:
                run = [one_round(e, g, idx) for idx in orders]
            finally:
                e.close()
            for r, (dt, h) in enumerate(run):
                times[r].append(dt)
            handed = [h for _, h in run] if handed is None else handed
            if [h for _, h in run] != handed:
                raise SystemExit("handed-back counts differ between trials")
        report[",".join(map(str, devs))] = [{"round": r + 1, "handed_back_per_device": handed[r], "handed_back": sum(handed[r]),
                                             "p50_ms": round(statistics.median(times[r]) * 1e3, 3)} for r in range(len(orders))]

    # the share step of the learning round, from the device's own timeline
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    e, g = make(devices)
    try:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            one_round(e, g, orders[0])
        ev = prof.events()
    finally:
        e.close()

    def total_us(pred):
        sel = [x for x in ev if x.device_type == torch.autograd.DeviceType.CUDA and pred(x.name)]
        return round(sum(x.device_time for x in sel), 1), len(sel)
    adopt = total_us(lambda n: "k_adopt_peer_keys" in n)
    copies = total_us(lambda n: "Memcpy" in n and ("PtoP" in n or "DtoD" in n))
    build = total_us(lambda n: "k_build_keytabs" in n)
    share = {"k_adopt_peer_keys_us": adopt[0], "k_adopt_peer_keys_launches": adopt[1], "device_to_device_copies_us": copies[0],
             "device_to_device_copies": copies[1], "k_build_keytabs_us": build[0], "k_build_keytabs_launches": build[1]}
    text = json.dumps({"gpu_and_power_limit": gpu_power_limit(), "devices": devices, "rounds": args.rounds, "trials": args.trials,
                       "items": int(len(seals)), "rejects": int((~want).sum()), "per_round": report,
                       "learning_round_share_step": share}, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
