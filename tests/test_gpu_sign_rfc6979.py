"""The RFC 6979 signer on the device (ibft_sign_batch_rfc6979, k_sign's third nonce mode): the published vectors and the
committed fixtures byte for byte, random and ragged batches against rfc6979_rows.py's sign_libsecp, the DRBG's candidates
through IBFT_DBG_RFC6979, the re-signed config-3 round back through every recover kernel with its quorum, and the two older
nonce modes interleaved with it in one engine."""
import numpy as np
import pytest

import rfc6979_rows as R
import workloads as wl
from oracle import coracle as co
from oracle import secp256k1 as ec

pytestmark = pytest.mark.gpu
N = ec.N


@pytest.fixture(scope="module")
def dev():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import ibft_b200 as ib
    e = ib.Engine(device=0, max_items=1 << 16, max_validators=16384)
    yield e
    e.close()


def test_published_vectors(dev):
    vs = R.golden_vectors()
    got = dev.sign_batch_rfc6979([int(v["privkey"], 16) for v in vs], [bytes.fromhex(v["digest"]) for v in vs])
    for v, g in zip(vs, got):
        assert g == bytes.fromhex(v["r"] + v["s"]) + bytes([v["v"]]), v["message"]


def _fixture_rows(name: str):
    """the items of a committed config tagged '' (honest), with each signer's key and the digest it signed"""
    d = np.load(f"{wl._HERE}/golden/{name}.npz")
    items = np.ascontiguousarray(d["items"]).view(wl.ITEM).reshape(-1)
    vs = wl.ValidatorSet(int(d["meta"][0]), int(d["meta"][1]))
    key_of = dict(zip(vs.addrs, vs.keys))
    arena = d["arena"].tobytes()
    idx = np.flatnonzero(d["tags"] == "")
    keys, digests = [], []
    for i in idx:
        it = items[i]
        keys.append(key_of[it["signer"].tobytes()])
        if it["kind"] == wl.KIND_PAYLOAD:
            off, ln = int(it["payload_off"]), int(it["payload_len"])
            digests.append(co.keccak256(arena[off:off + ln]))
        else:
            assert it["kind"] == wl.KIND_SEAL
            digests.append(wl.seal_digest(it["digest"].tobytes()))
    want = [it["r"].tobytes() + it["s"].tobytes() + bytes([int(it["v"])]) for it in items[idx]]
    return d, items[idx].copy(), keys, digests, want


@pytest.fixture(scope="module")
def config3_resigned(dev):
    d, items, keys, digests, want = _fixture_rows("config3")
    return d, items, dev.sign_batch_rfc6979(keys, digests), want


@pytest.mark.parametrize("name,rows", [("config2", 2970), ("config3", 19800)])
def test_fixtures_resigned_byte_for_byte(dev, config3_resigned, name, rows):
    """the fixtures were signed with RFC 6979 nonces on the host; one device call re-signs every honest item identically"""
    if name == "config3":
        _, items, got, want = config3_resigned
    else:
        _, items, keys, digests, want = _fixture_rows(name)
        got = dev.sign_batch_rfc6979(keys, digests)
    assert len(got) == rows
    bad = [i for i in range(rows) if got[i] != want[i]]
    assert not bad, f"{name}: rows {bad[:20]} differ"


def test_random_rows(dev):
    """10,000 rows, among them keys 0, n and above n and digests at and above n"""
    ds, zs = R.random_rows(10_000, seed=1)
    assert sum(d == 0 for d in ds) and sum(d >= N for d in ds) >= 20 and sum(int.from_bytes(z, "big") >= N for z in zs) >= 20
    got = dev.sign_batch_rfc6979(ds, zs)
    want = R.want(ds, zs)
    bad = [i for i in range(len(ds)) if got[i] != want[i]]
    assert not bad, f"rows {bad[:20]} differ"
    refused = [i for i, d in enumerate(ds) if not 1 <= d < N]
    assert refused and all(got[i] == R.ZERO_SIG for i in refused)


def test_candidates_on_the_device(dev):
    """IBFT_DBG_RFC6979: candidates 0-3 of the edge rows and of random rows, before any range check"""
    rows = R.edge_rows()
    ds, zs = R.random_rows(500, seed=2)
    rows += list(zip(ds, zs))
    for c in range(4):
        got = dev.debug_op("RFC6979", [d for d, _ in rows], [int.from_bytes(z, "big") for _, z in rows],
                           [c.to_bytes(64, "big")] * len(rows))
        bad = [i for i, (d, z) in enumerate(rows) if int.from_bytes(got[i], "big") != R.rfc6979_candidate(d, z, c)]
        assert not bad, f"candidate {c}: rows {bad[:20]} differ"


@pytest.mark.parametrize("n", [1, 63, 64, 65, 4103, 100_000])
def test_batch_shapes(dev, n):
    ds, zs = R.random_rows(n, seed=n)
    got = dev.sign_batch_rfc6979(ds, zs)
    want = R.want(ds, zs)
    bad = [i for i in range(n) if got[i] != want[i]]
    assert not bad, f"n={n}: rows {bad[:20]} differ"
    for i in sorted({0, min(3, n - 1), min(63, n - 1), n - 1}):
        assert dev.sign_batch_rfc6979([ds[i]], [zs[i]]) == [got[i]], i


def _verify_resigned(e, config3_resigned):
    d, items, sigs, _ = config3_resigned
    items = items.copy()
    S = np.frombuffer(b"".join(sigs), np.uint8).reshape(-1, 65)
    items["r"], items["s"], items["v"] = S[:, :32], S[:, 32:64], S[:, 64]
    e.set_validators(0, int(d["meta"][2]), d["addrs"], d["powers"])
    bm, res, _ = e.verify_batch(items, d["arena"], e.groups(len(d["groups"])))
    n = len(items)
    bits = (bm[np.arange(n) >> 5] >> (np.arange(n) & 31).astype(np.uint32)) & 1
    assert bits.all(), f"rows {np.flatnonzero(bits == 0)[:20]} do not verify"
    assert all(int(r["has_quorum"]) == 1 for r in res)
    assert [int(r["n_valid"]) for r in res] == [int((items["group"] == g).sum()) for g in range(len(res))]


def test_resigned_round_verifies_on_every_kernel(engine, config3_resigned):
    _verify_resigned(engine, config3_resigned)


def test_resigned_round_verifies_through_auto(dev, config3_resigned):
    _verify_resigned(dev, config3_resigned)


def test_modes_interleaved(dev):
    """given, Keccak-derived and RFC 6979 calls alternate on one engine; every call returns what the same call returns alone"""
    ds, zs = R.random_rows(2000, seed=3)
    ds = [d % N or 1 for d in ds]                    # keys valid in all three modes
    ks = [R.rfc6979_candidate(d, z, 0) for d, z in zip(ds, zs)]
    rfc = R.want(ds, zs)
    D = np.frombuffer(b"".join(d.to_bytes(32, "big") for d in ds), np.uint8).reshape(-1, 32)
    Z = np.frombuffer(b"".join(zs), np.uint8).reshape(-1, 32)
    derived = [bytes(x) for x in co.sign_derived_batch(D, Z)]
    given = [co.sign_with_k(d, z, k, True) or R.ZERO_SIG for d, z, k in zip(ds, zs, ks)]
    assert given == rfc                              # candidate 0 is the nonce of every row here
    for _ in range(2):
        assert dev.sign_batch_rfc6979(ds, zs) == rfc
        assert dev.sign_batch(ds, zs) == derived
        assert dev.sign_batch_rfc6979(ds[:65], zs[:65]) == rfc[:65]
        assert dev.sign_batch(ds, zs, ks) == given
