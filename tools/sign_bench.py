"""Batched signing: the Keccak-derived nonce (ibft_sign_batch, nonces = NULL) against libsecp256k1's RFC 6979 nonce
(ibft_sign_batch_rfc6979).

For each batch size, random keys in [1, n) and random digests; a call is timed on the host from the host buffers in to the
signatures back in host memory (the entry points synchronise the device before they return).  Each size is warmed up in both
modes, then the two modes alternate for --reps repetitions each; the medians are reported, with the rate and the RFC 6979
mode's time relative to the Keccak mode's.  The card name and its power limit are recorded beside the numbers.

    python tools/sign_bench.py [--sizes 16384,65536,1048576] [--reps 7] [--out FILE]
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


def card() -> str:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as ex:  # noqa: BLE001 -- the numbers stand without it, marked as such
        return f"unknown ({ex})"


def measure(eng, n: int, reps: int, seed: int) -> dict:
    import ctypes

    import numpy as np

    rng = np.random.default_rng(seed)
    D = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    D[:, 0] &= 0x7F                                   # < 2^255 < n: every key is valid in both modes
    D[:, 31] |= 1                                     # and not zero
    Z = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    out = np.zeros((n, 65), dtype=np.uint8)
    lib, h = eng.lib, eng.handle
    ptr = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731

    def keccak():
        eng._check(lib.ibft_sign_batch(h, ptr(D), ptr(Z), None, n, ptr(out)))

    def rfc6979():
        eng._check(lib.ibft_sign_batch_rfc6979(h, ptr(D), ptr(Z), n, ptr(out)))

    modes = {"keccak": keccak, "rfc6979": rfc6979}
    for f in modes.values():
        f()
        f()
    times = {m: [] for m in modes}
    for _ in range(reps):
        for m, f in modes.items():
            t0 = time.perf_counter()
            f()
            times[m].append(time.perf_counter() - t0)
    row = {"rows": n, "reps": reps}
    for m in modes:
        med = statistics.median(times[m])
        row[f"{m}_ms"] = round(med * 1e3, 3)
        row[f"{m}_min_ms"] = round(min(times[m]) * 1e3, 3)
        row[f"{m}_signs_per_s"] = round(n / med)
    row["rfc6979_over_keccak"] = round(row["rfc6979_ms"] / row["keccak_ms"], 4)
    return row


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--sizes", default="16384,65536,1048576")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import ibft_b200 as ib

    eng = ib.Engine(device=0, max_items=1 << 10, max_payload_bytes=1 << 20, max_groups=1, max_table_slots=1, max_validators=16)
    try:
        rows = [measure(eng, int(s), args.reps, seed=i) for i, s in enumerate(args.sizes.split(","))]
        device = eng.device_info()["name"]
    finally:
        eng.close()
    text = json.dumps({"gpu_and_power_limit": card(), "device": device, "rows": rows}, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
