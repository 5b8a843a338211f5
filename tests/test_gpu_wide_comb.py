"""The wide generator comb on the device (secp_ec.cuh ecmult_gen_wide; built by engine.cu k_build_wtable, one per process and
device): its entries against the oracle, the crafted u1 values of tests/wide_edges.py and the crafted recover vectors through
every kernel that reads it (k_recover<32>, k_recover<128>, the key registry's worklist pass, AUTO at throughput sizes), the
config-2 and config-3 fixtures bit-exact, the same bitmaps from a build without the table (-DIBFT_GEN_WIDE=0, in a subprocess),
and two engines sharing one table, closed in either order.

    python tests/test_gpu_wide_comb.py bitmaps OUT.npz   writes the bitmaps of the library named by IBFT_LIB (the fallback build)
    python tests/test_gpu_wide_comb.py share             the two-engine sharing check, in a process of its own"""
import os
import random
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import adversarial as A
import wide_edges as WE
from oracle import coracle as co
from oracle import secp256k1 as ec
from test_gpu_adversarial import sm_count

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
GIB = 1 << 30


def _need_gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def point(words) -> tuple:
    w = [int(x) for x in words]
    return sum(v << (32 * i) for i, v in enumerate(w[:8])), sum(v << (32 * i) for i, v in enumerate(w[8:16]))


def oracle_point(k: int) -> tuple:
    b = co.pubkey_from_scalar(k % ec.N)
    return int.from_bytes(b[:32], "big"), int.from_bytes(b[32:64], "big")


def crafted():
    """IBFT_KIND_DIGEST items of the wide-comb vectors and of tests/adversarial.py, with the expected verdicts and addresses"""
    vecs = WE.vectors() + list(A.recover_vectors())
    items = A.recover_items(vecs)
    want = np.array([v.verdict for v in vecs], dtype=bool)
    addrs = np.array([np.frombuffer(v.addr or bytes(20), np.uint8) for v in vecs])
    return vecs, items, want, addrs


def bits(bm, n):
    return np.unpackbits(np.asarray(bm, dtype="<u4").view(np.uint8), bitorder="little")[:n].astype(bool)


def fixture(name):
    d = np.load(os.path.join(HERE, "golden", name + ".npz"))
    items = np.ascontiguousarray(d["items"]).view(co.ITEM_DTYPE).reshape(-1)
    return d, items


def make_engine(**kw):
    import ibft_b200 as ib
    args = dict(device=0, max_items=1 << 16, max_payload_bytes=1 << 22, max_groups=4, max_table_slots=2, max_validators=16384)
    args.update(kw)
    return ib.Engine(**args)


def fixture_bitmaps(e):
    out = {}
    for name in ("config2", "config3"):
        d, items = fixture(name)
        e.set_validators(0, int(d["meta"][2]), d["addrs"], d["powers"])
        out[name] = e.verify_batch(items, d["arena"], e.groups(len(d["groups"])))[0]
    return out


def crafted_bitmaps(e, n):
    _, items, _, _ = crafted()
    reps = -(-n // len(items))
    it = np.ascontiguousarray(np.tile(items, reps)[:n])
    bm, _, rec = e.verify_batch(it, b"", None, want_results=False, want_recovered=True)
    return bm, rec


@pytest.fixture(scope="module")
def eng():
    _need_gpu()
    e = make_engine()
    yield e
    e.close()


def test_table_entries_against_oracle(eng):
    """all of the top position, the first and last 4,096 entries of every position, and 10^5 random entries: every contiguous
    block starts at an oracle point and steps by the position's base 2^(22 p) G; every random entry follows from its predecessor
    the same way, and 1,000 of them are compared with the oracle directly"""
    w, per, total = eng.wide_table_info()
    assert (w, per, total) == (WE.W, 1 << (WE.W - 1), (WE.POSITIONS - 1) * (1 << (WE.W - 1)) + (1 << WE.TOP_BITS) + 1)
    bases = [oracle_point(1 << (WE.W * p)) for p in range(WE.POSITIONS)]

    def check_block(p, m0, count):
        got = eng.wide_table_entries(p * per + m0 - 1, count)
        P = oracle_point(m0 << (WE.W * p))
        for i in range(count):
            assert point(got[i]) == P, (p, m0 + i)
            P = ec.point_add(P, bases[p])

    top = total - (WE.POSITIONS - 1) * per
    for p in range(WE.POSITIONS - 1):
        check_block(p, 1, 4096)
        check_block(p, per - 4095, 4096)
    check_block(WE.POSITIONS - 1, 1, top)
    rnd = random.Random(22)
    for i in range(100_000):
        p = rnd.randrange(WE.POSITIONS)
        m = rnd.randrange(2, (per if p < WE.POSITIONS - 1 else top) + 1)
        prev, cur = eng.wide_table_entries(p * per + m - 2, 2)
        assert point(cur) == ec.point_add(point(prev), bases[p]), (p, m)
        if i % 100 == 0:
            assert point(cur) == oracle_point(m << (WE.W * p)), (p, m)


def test_crafted_through_every_kernel(eng):
    """k_recover<32> (one wave), k_recover<128> and AUTO past SMs x 256 signatures, the key registry's worklist pass"""
    import ibft_b200 as ib
    vecs, items, want, addrs = crafted()
    sms = sm_count()
    for path in (ib.Engine.PATH_THREAD, ib.Engine.PATH_AUTO):
        eng.set_recover_path(path)
        for n in (len(items), sms * 256 + 77):
            reps = -(-n // len(items))
            it = np.ascontiguousarray(np.tile(items, reps)[:n])
            bm, _, rec = eng.verify_batch(it, b"", None, want_results=False, want_recovered=True)
            assert np.array_equal(bits(bm, n), np.tile(want, reps)[:n]), (path, n)
            assert np.array_equal(rec, np.tile(addrs, (reps, 1))[:n]), (path, n)
    eng.set_recover_path(ib.Engine.PATH_AUTO)
    assert np.array_equal(eng.verify_batch(items, b"", None, want_results=False)[0], co.verify_batch(items, b"", n_threads=8))
    # worklist pass: a key-registry engine, signers in the table, keys not known yet -- every member goes to k_recover in worklist mode
    signers = sorted({v.addr for v in vecs if v.verdict})
    members = np.array([v.signer in signers for v in vecs])
    kc = make_engine(key_cache=True)
    try:
        kc.set_validators(0, 1, np.array([np.frombuffer(a, np.uint8) for a in signers]), None)
        n = sms * 256 + 77
        reps = -(-n // len(items))
        it = np.ascontiguousarray(np.tile(items, reps)[:n])
        bm, _, _ = kc.verify_batch(it, b"", kc.groups(1))
        assert np.array_equal(bits(bm, n), np.tile(want, reps)[:n])
        assert kc.known_handed_back() == int(np.tile(members, reps)[:n].sum())
    finally:
        kc.close()


def test_fixtures_bit_exact(eng):
    for name, bm in fixture_bitmaps(eng).items():
        assert np.array_equal(bm, fixture(name)[0]["bitmap"]), name


def test_fallback_build_gives_identical_bitmaps(eng):
    """engine.cu built with -DIBFT_GEN_WIDE=0 (u1 G by the per-position comb), run in a subprocess of its own: the same bitmaps
    and recovered addresses"""
    import ibft_b200 as ib
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    with tempfile.TemporaryDirectory(prefix="ibft_nowide_") as tmp:
        so = os.path.join(tmp, "lib_nowide.so")
        p = subprocess.run([nvcc] + ib.build.NVCC_FLAGS + ["-DIBFT_GEN_WIDE=0", "-o", so, os.path.join(ib.build.CSRC, "engine.cu")],
                           cwd=ib.build.CSRC, capture_output=True, text=True)
        assert p.returncode == 0, p.stderr[-2000:]
        out = os.path.join(tmp, "bitmaps.npz")
        env = dict(os.environ, IBFT_LIB=so, PYTHONPATH=os.pathsep.join([ROOT, HERE, os.environ.get("PYTHONPATH", "")]))
        p = subprocess.run([sys.executable, os.path.abspath(__file__), "bitmaps", out], cwd=ROOT, env=env, capture_output=True,
                           text=True, timeout=900)
        assert p.returncode == 0, p.stdout[-4000:] + p.stderr[-4000:]
        got = dict(np.load(out))
    assert got.pop("wide") == 0
    eng.set_recover_path(ib.Engine.PATH_THREAD)
    n = sm_count() * 256 + 77
    bm, rec = crafted_bitmaps(eng, n)
    eng.set_recover_path(ib.Engine.PATH_AUTO)
    assert np.array_equal(got["crafted"], bm) and np.array_equal(got["crafted_recovered"], rec)
    for name, b in fixture_bitmaps(eng).items():
        assert np.array_equal(got[name], b), name


def test_engines_share_one_table_closed_in_either_order():
    """in a process of its own (no other engine holds the table): the first engine builds it, the second shares it, either can
    close first while the other keeps verifying, and the last close frees it"""
    _need_gpu()
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, HERE, os.environ.get("PYTHONPATH", "")]))
    p = subprocess.run([sys.executable, os.path.abspath(__file__), "share"], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=900)
    assert p.returncode == 0 and "share ok" in p.stdout, p.stdout[-4000:] + p.stderr[-4000:]


def _share_main():
    import torch
    _, items, want, _ = crafted()
    for first_closed in (0, 1):
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        es = [make_engine(max_items=4096)]
        free1 = torch.cuda.mem_get_info()[0]
        es.append(make_engine(max_items=4096))
        free2 = torch.cuda.mem_get_info()[0]
        try:
            assert es[0].wide_table_info()[0] == es[1].wide_table_info()[0] == WE.W
            assert free0 - free1 > GIB, (free0, free1)        # the first engine on the device builds the table
            assert free1 - free2 < GIB // 4, (free1, free2)   # the second one shares it
            es.pop(first_closed).close()
            bm, _, _ = es[0].verify_batch(items, b"", None, want_results=False)
            assert np.array_equal(bits(bm, len(items)), want)
        finally:
            for e in es:
                e.close()
        torch.cuda.synchronize()
        assert torch.cuda.mem_get_info()[0] - free2 > GIB, first_closed  # the last close frees it
    print("share ok")
    return 0


def _bitmaps_main(out):
    import ibft_b200 as ib
    e = make_engine()
    try:
        e.set_recover_path(ib.Engine.PATH_THREAD)
        bm, rec = crafted_bitmaps(e, sm_count() * 256 + 77)
        e.set_recover_path(ib.Engine.PATH_AUTO)
        np.savez(out, wide=e.wide_table_info()[0], crafted=bm, crafted_recovered=rec, **fixture_bitmaps(e))
    finally:
        e.close()
    return 0


if __name__ == "__main__" and sys.argv[1:2] == ["bitmaps"]:
    sys.exit(_bitmaps_main(sys.argv[2]))
if __name__ == "__main__" and sys.argv[1:] == ["share"]:
    sys.exit(_share_main())
