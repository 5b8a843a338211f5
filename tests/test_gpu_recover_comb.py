"""The one-thread recover kernels (k_recover<32> for one-wave batches, k_recover<128> beyond) forced with PATH_THREAD, on the
crafted vectors of tests/adversarial.py plus non-abscissa r with both recovery ids: their final addition A + B reaches A = B,
A = -B, u1 = 0 and a non-residue r^3 + 7 (tests/test_emul_recover_comb.py shows which vector takes which branch).  Verdicts and
recovered addresses against the oracle."""
import random

import numpy as np
import pytest

import ibft_b200 as ib
import workloads as wl
from oracle import coracle as co
from test_emul_recover_comb import non_abscissas
from test_gpu_adversarial import bits, crafted_batch, sm_count

pytestmark = pytest.mark.gpu


def batch():
    items, want, addrs = crafted_batch(seed=9)
    rnd = random.Random(10)
    rows, w, a = [items], [want], [addrs]
    for r in non_abscissas(8, 14):
        for v in (0, 1):
            sig = r.to_bytes(32, "big") + rnd.getrandbits(250).to_bytes(32, "big") + bytes([v])
            rows.append(wl.make_item(sig, bytes(20), 0, rnd.randbytes(32)))
            w.append(np.array([False]))
            a.append(np.zeros((1, 20), np.uint8))
    return np.concatenate(rows), np.concatenate(w), np.concatenate(a)


def test_thread_kernels_on_crafted_and_non_abscissa_vectors():
    items, want, addrs = batch()
    sms = sm_count()
    e = ib.Engine(device=0, max_items=1 << 16, max_payload_bytes=1 << 20, max_groups=4, max_table_slots=2, max_validators=1024)
    try:
        e.set_recover_path(ib.Engine.PATH_THREAD)
        # one wave of one-warp CTAs (k_recover<32>), then past SMs x 256 signatures (k_recover<128>)
        for n in (len(items), sms * 256 + 77):
            assert n <= 1 << 16
            reps = -(-n // len(items))
            it = np.ascontiguousarray(np.tile(items, reps)[:n])
            bm, _, rec = e.verify_batch(it, b"", None, want_results=False, want_recovered=True)
            assert np.array_equal(bits(bm, n), np.tile(want, reps)[:n]), n
            assert np.array_equal(rec, np.tile(addrs, (reps, 1))[:n]), n
            if n == len(items):
                assert np.array_equal(bm, co.verify_batch(items, b"", n_threads=8))
    finally:
        e.close()
