"""Safegcd edge inputs (tests/golden/safegcd_edges.json) for tests/arith_edges.py.

    python tests/golden/make_safegcd_edges.py
Runs tests/arith_edges.py safegcd_model over CANDIDATES seeded random inputs below each modulus (p: fe_inv_safegcd, n:
sc_inv_safegcd) and keeps the inputs that take the most 30-divstep batches of modinv30_var, and some that end with f = -1
(the negating branch of normalize_30).  The search takes a few minutes, so its result is committed; the tests recompute the
model on the stored inputs.
"""
import json
import os
import random
import sys
from multiprocessing import Pool

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
import arith_edges as AE  # noqa: E402

CANDIDATES = 100_000
KEEP = 8


def scan(args):
    m, seed, count = args
    rnd = random.Random(seed)
    out = []
    for _ in range(count):
        x = rnd.randrange(1, m)
        b, s = AE.safegcd_model(x, m)
        out.append((b, s, x))
    return out


def main():
    res = {"candidates": CANDIDATES}
    with Pool() as pool:
        for tag, m, seed in (("p", AE.P, 1), ("n", AE.N, 2)):
            chunks = pool.map(scan, [(m, seed * 1000 + i, CANDIDATES // 50) for i in range(50)])
            found = [t for c in chunks for t in c]
            top = max(b for b, _, _ in found)
            most = [x for b, _, x in found if b == top][:KEEP]
            if len(most) < KEEP:  # fill up with the next batch count down
                most += [x for b, _, x in found if b == top - 1][: KEEP - len(most)]
            neg = [x for b, s, x in found if s < 0][:KEEP]
            res[tag] = {"batches": top, "most_batches": [hex(x) for x in most], "f_negative": [hex(x) for x in neg],
                        "histogram": {str(b): sum(1 for t in found if t[0] == b) for b in sorted({t[0] for t in found})}}
    with open(os.path.join(HERE, "safegcd_edges.json"), "w") as f:
        json.dump(res, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
