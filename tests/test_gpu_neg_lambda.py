"""The negated-lambda-digit vectors of tests/neg_lambda.py, with tests/adversarial.py's crafted set (P + P, P - P, infinity, Booth
edges, u1 = 0), on the device: the sign of every negated entry is folded into the mixed addition's r = -S2 - Y1.  Through
k_recover<32> (one wave), k_recover<128> (past SMs x 256 signatures), AUTO and the key registry's worklist pass, against the
oracle's verdicts and recovered addresses."""
import numpy as np
import pytest

import adversarial as A
import neg_lambda as NL
from oracle import coracle as co
from test_gpu_adversarial import sm_count
from test_gpu_wide_comb import bits, make_engine

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    e = make_engine()
    yield e
    e.close()


def vectors():
    vecs = list(NL.vectors()) + list(A.recover_vectors())
    items = A.recover_items(tuple(vecs))
    want = np.array([v.verdict for v in vecs], dtype=bool)
    addrs = np.array([np.frombuffer(v.addr or bytes(20), np.uint8) for v in vecs])
    return vecs, items, want, addrs


def test_negated_lambda_digits_through_every_kernel(eng):
    import ibft_b200 as ib
    vecs, items, want, addrs = vectors()
    n_big = sm_count() * 256 + 77
    for path in (ib.Engine.PATH_THREAD, ib.Engine.PATH_AUTO):
        eng.set_recover_path(path)
        for n in (len(NL.vectors()), len(items), n_big):
            reps = -(-n // len(items))
            it = np.ascontiguousarray(np.tile(items, reps)[:n])
            bm, _, rec = eng.verify_batch(it, b"", None, want_results=False, want_recovered=True)
            assert np.array_equal(bits(bm, n), np.tile(want, reps)[:n]), (path, n)
            assert np.array_equal(rec, np.tile(addrs, (reps, 1))[:n]), (path, n)
    eng.set_recover_path(ib.Engine.PATH_AUTO)
    assert np.array_equal(eng.verify_batch(items, b"", None, want_results=False)[0], co.verify_batch(items, b"", n_threads=8))
    # worklist pass: signers in the table, keys not known yet, so every member item goes to k_recover in worklist mode
    signers = sorted({v.addr for v in vecs if v.verdict})
    members = np.array([v.signer in signers for v in vecs])
    kc = make_engine(key_cache=True)
    try:
        kc.set_validators(0, 1, np.array([np.frombuffer(a, np.uint8) for a in signers]), None)
        reps = -(-n_big // len(items))
        it = np.ascontiguousarray(np.tile(items, reps)[:n_big])
        bm, _, _ = kc.verify_batch(it, b"", kc.groups(1))
        assert np.array_equal(bits(bm, n_big), np.tile(want, reps)[:n_big])
        assert kc.known_handed_back() == int(np.tile(members, reps)[:n_big].sum())
    finally:
        kc.close()
