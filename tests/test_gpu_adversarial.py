"""Crafted exceptional-case signatures (tests/adversarial.py) on every device kernel, the key registry read back entry by entry,
and the known-key pass made visible through the number of items it hands to the recover pass (ibft_debug_known_handed_back).

A known-key pass that rejects everything still produces the recover path's bitmap (the recover pass decides what it leaves);
only the handed-back count shows it.  Every count asserted here is derived from the oracle (see expected_handed_back)."""
import functools
import random

import numpy as np
import pytest

import adversarial as A
import ibft_b200 as ib
import workloads as wl
from oracle import coracle as co
from oracle import secp256k1 as ec
from test_gpu_verify import groups_for, load_fixture

pytestmark = pytest.mark.gpu
N = ec.N
POSITIONS, ENTRIES = 17, 128  # comb positions of the generator / key tables, entries per key-table position


def bits(bm, n):
    return np.unpackbits(np.ascontiguousarray(bm).view(np.uint8), bitorder="little")[:n].astype(bool)


def pack(b):
    b = np.asarray(b, dtype=np.uint8)
    out = np.packbits(np.concatenate([b, np.zeros((-len(b)) % 32, np.uint8)]), bitorder="little")
    return out.view(np.uint32)


def point_of(words):
    """16 little-endian words x || y -> affine point"""
    return (sum(int(words[i]) << (32 * i) for i in range(8)), sum(int(words[8 + i]) << (32 * i) for i in range(8)))


def in_range(it) -> bool:
    r, s = int.from_bytes(bytes(it["r"]), "big"), int.from_bytes(bytes(it["s"]), "big")
    return 0 < r < N and 0 < s < N and int(it["v"]) <= 1


def expected_handed_back(items, arena_len, members, valid_bits, known_signers, split=False) -> int:
    """What the known-key pass leaves to the recover pass (engine.cu k_verify_known / k_verify_split).  An item reaches it when
    resolve_item resolves it (digest / payload / seal kinds with the payload inside the arena) and group_member finds its signer
    in the group's table; it is accepted -- and settled -- exactly when the signature is valid and its signer's key is known.
    So: handed back = #{resolves, signer in table, not (valid and key known)}.  The chain + helper form (split) settles
    out-of-range (r, s, v) itself: those are not handed back there."""
    n = 0
    for i, it in enumerate(items):
        kind = int(it["kind"])
        if kind not in (wl.KIND_DIGEST, wl.KIND_PAYLOAD, wl.KIND_SEAL):
            continue
        if kind == wl.KIND_PAYLOAD and int(it["payload_off"]) + int(it["payload_len"]) > arena_len:
            continue
        signer = bytes(it["signer"])
        if signer not in members:
            continue
        if valid_bits[i] and signer in known_signers:
            continue
        if split and not in_range(it):
            continue
        n += 1
    return n


def sm_count():
    e = ib.Engine(device=0, max_items=64, max_payload_bytes=1 << 10, max_groups=1, max_table_slots=1, max_validators=16)
    try:
        return e.device_info()["sm_count"]
    finally:
        e.close()


# ------------------------------------------------------------------------------------- crafted recover vectors, every kernel
def crafted_batch(seed=5):
    """crafted vectors interleaved with ordinary signatures, so that exceptional and ordinary items share a warp, a quad and a CTA"""
    rnd = random.Random(seed)
    rows, want, addrs = [], [], []
    for i, v in enumerate(A.recover_vectors()):
        rows.append(A.recover_items([v]))
        want.append(v.verdict)
        addrs.append(v.addr or bytes(20))
        if i % 3 == 0:
            d = rnd.getrandbits(256) % (N - 1) + 1
            dig = rnd.getrandbits(256).to_bytes(32, "big")
            addr = wl.address_of(d)
            rows.append(wl.make_item(wl.sign(d, dig, low_s=bool(i & 1)), addr, 0, dig))
            want.append(True)
            addrs.append(addr)
    return np.concatenate(rows), np.array(want), np.frombuffer(b"".join(addrs), np.uint8).reshape(-1, 20)


def test_crafted_recover_vectors_on_every_kernel(engine):
    """P + P, P - P, Q = infinity, Booth-edge digits, u1 = 0 (z = 0 and z = n), high-s twins: verdicts and recovered addresses equal
    the oracle on the one-thread, four-lane, chain + helper and four-lane chain + helper kernels."""
    items, want, addrs = crafted_batch()
    bm, _, rec = engine.verify_batch(items, b"", None, want_results=False, want_recovered=True)
    assert np.array_equal(bits(bm, len(items)), want)
    assert np.array_equal(rec, addrs)
    assert np.array_equal(bm, co.verify_batch(items, b"", n_threads=8))


def test_crafted_recover_vectors_through_auto():
    """The same set, padded by replication, at one size in each AUTO range: <= SMs x 24 (four-lane chain + helper), the four-piece
    range (SMs x 48, SMs x 96] (chain + helper pieces), > SMs x 192 (one thread per signature)."""
    items, want, addrs = crafted_batch(seed=6)
    sms = sm_count()
    e = ib.Engine(device=0, max_items=1 << 16, max_payload_bytes=1 << 20, max_groups=4, max_table_slots=2, max_validators=1024)
    try:
        for n in (sms * 24 - 5, sms * 72 + 3, sms * 192 + 40):
            reps = -(-n // len(items))
            it = np.tile(items, reps)[:n]
            bm, _, rec = e.verify_batch(it, b"", None, want_results=False, want_recovered=True)
            assert np.array_equal(bits(bm, n), np.tile(want, reps)[:n]), n
            assert np.array_equal(rec, np.tile(addrs, (reps, 1))[:n]), n
    finally:
        e.close()


# ------------------------------------------------------------------------------------- key registry read back
KC = dict(device=0, max_items=1 << 16, max_payload_bytes=1 << 20, max_groups=4, max_table_slots=2, max_validators=1024)
PATHS = [ib.Engine.PATH_THREAD, ib.Engine.PATH_QUAD, ib.Engine.PATH_SPLIT, ib.Engine.PATH_QSPLIT]


def check_key_table(tab, Q, ms=(1, 2, 3, 4, 64, 127, 128)):
    base = Q
    for j in range(POSITIONS):
        for m in ms:
            assert point_of(tab[j * ENTRIES + m - 1]) == ec.point_mul(m, base), (j, m)
        base = ec.point_mul(256, base)


@functools.lru_cache(maxsize=None)
def key_table_reference(Q) -> tuple:
    """the whole comb table of Q by the big-int oracle: entry j * 128 + m - 1 = m * 2^(8j) * Q, affine"""
    out, base = [], Q
    for _ in range(POSITIONS):
        P = base
        for _ in range(ENTRIES):
            out.append(P)
            P = ec.point_add(P, base)
        base = ec.point_mul(256, base)
    return tuple(out)


def check_whole_key_table(tab, Q):
    ref = key_table_reference(Q)
    bad = [k for k in range(POSITIONS * ENTRIES) if point_of(tab[k]) != ref[k]]
    assert not bad, (hex(Q[0]), hex(Q[1]), [divmod(k, ENTRIES) for k in bad[:4]], len(bad))


def test_learned_keys_and_key_tables_on_every_recover_kernel():
    """Each recover kernel has its own learn_key call: one signature per validator through each forced kernel (recovered addresses
    requested, so the kernel itself runs), then the learned key must be Q exactly (canonical), entry m of position j of its comb
    table m * 2^(8j) * Q, whole tables of 2,176 entries must match, and the tables carried to the next height must be
    byte-identical to the donor's.  Besides four signing keys per kernel, each kernel learns its share of the coordinate-edge
    keys of tests/adversarial.py (coordinates below 2^256 - p or near p: learned, stored and tabled only if normalised) from
    signatures made without their private keys; every edge key's whole table is checked."""
    vs = wl.ValidatorSet(91, 4 * len(PATHS))
    edge = [Q for _, Q in A.key_edge_points()]
    keys = [ec.point_mul(d, ec.G) for d in vs.keys] + edge
    addrs = vs.addrs + [ec.pubkey_to_address(Q) for Q in edge]
    rnd = random.Random(92)
    eng = ib.Engine(**KC, key_cache=True)
    try:
        eng.set_validators(0, 5, np.frombuffer(b"".join(addrs), np.uint8).reshape(-1, 20).copy(), None)
        groups = groups_for(eng, 1)
        dig = co.keccak256(b"learn")

        def item(i):
            if i < vs.n:
                return wl.make_item(wl.sign(vs.keys[i], dig, low_s=bool(i & 1)), vs.addrs[i], 0, dig)
            v = A.signature_for("learn", keys[i], rnd)
            return wl.make_item(v.sig, addrs[i], 0, v.digest)

        for k, path in enumerate(PATHS):
            eng.set_recover_path(path)
            own = list(range(4 * k, 4 * k + 4)) + list(range(vs.n + k, len(keys), len(PATHS)))
            items = np.concatenate([item(i) for i in own])
            bm, _, _ = eng.verify_batch(items, b"", groups, want_recovered=True)
            assert bits(bm, len(own)).all(), path
            for i in own:
                state, key, _ = eng.key_table(0, i)
                assert state == 2, (path, i)                                 # learned, table built on the way out of the call
                assert point_of(key) == keys[i], (path, i)
        assert eng.refresh_key_tables() == len(keys)
        tables = []
        for i in range(len(keys)):
            _, _, tab = eng.key_table(0, i, 0, POSITIONS * ENTRIES)
            if i < vs.n:
                check_key_table(tab, keys[i])
            tables.append(tab)
        # whole tables, entry by entry: one signing key's and every edge key's
        for i in [5] + list(range(vs.n, len(keys))):
            check_whole_key_table(tables[i], keys[i])
        # next height in the other slot: every table carried over, byte for byte
        eng.set_validators(1, 6, np.frombuffer(b"".join(addrs), np.uint8).reshape(-1, 20).copy(), None)
        for i in range(len(keys)):
            state, key, tab = eng.key_table(1, i, 0, POSITIONS * ENTRIES)
            _, key0, _ = eng.key_table(0, i)
            assert state == 2 and np.array_equal(key, key0) and tab.tobytes() == tables[i].tobytes(), i
    finally:
        eng.close()


# ------------------------------------------------------------------------------------- crafted known-key vectors
def known_batch(group=0):
    """(items, number of items the known-key pass must hand back): the crafted valid set interleaved with its misattributed,
    recovery-id-flipped, cancelling and x = r + n forgery variants (all of them rejected by the verification, verdict 0)"""
    rows, handed = [], 0
    extra = A.known_cancelling() + A.known_r_plus_n()
    for n, v in enumerate(A.known_vectors()):
        rows.append(wl.make_item(v.sig, A.known_addr(v.key_index), 0, v.digest, group))
        sig, j = A.misattributed(v)
        rows.append(wl.make_item(sig, A.known_addr(j), 0, v.digest, group))
        rows.append(wl.make_item(A.flipped(v), A.known_addr(v.key_index), 0, v.digest, group))
        handed += 2
        if n < len(extra):
            c = extra[n]
            rows.append(wl.make_item(c.sig, A.known_addr(c.key_index), 0, c.digest, group))
            handed += 1
    assert len(A.known_vectors()) >= len(extra)
    items = np.concatenate(rows)
    return items, handed


def known_addrs():
    return np.frombuffer(b"".join(A.known_addr(i) for i in range(len(A.known_points()))), np.uint8).reshape(-1, 20).copy()


def valid_known_items(vectors=None):
    return np.concatenate([wl.make_item(v.sig, A.known_addr(v.key_index), 0, v.digest) for v in vectors or A.known_vectors()])


def test_crafted_known_key_vectors_on_every_known_key_kernel():
    """Learn the crafted keys (the six multiples, the coordinate-edge keys and the x = r + n forgery keys), then run the crafted
    set through k_verify_known<32> (THREAD, small batch), k_verify_known<128> (THREAD, replicated past SMs x 256), k_verify_split
    (SPLIT) and the AUTO four-piece path: bitmap = oracle, results = a plain engine's; the all-valid set hands back nothing, each
    rejected variant -- each x = r + n forgery, which plain ECDSA accepts for its key, among them -- exactly once."""
    addrs = known_addrs()
    sms = sm_count()
    eng = ib.Engine(**KC, key_cache=True)
    plain = ib.Engine(**KC)
    try:
        for e in (eng, plain):
            e.set_validators(0, 3, addrs, None)
        groups = groups_for(eng, 1)
        valid = valid_known_items()
        bm, _, _ = eng.verify_batch(valid, b"", groups)                      # pass 1: keys learned, tables built on the way out
        assert bits(bm, len(valid)).all()
        assert eng.refresh_key_tables() == len(A.known_points())
        bm, _, _ = eng.verify_batch(valid, b"", groups)
        assert bits(bm, len(valid)).all() and eng.known_handed_back() == 0
        items, handed = known_batch()
        want = co.verify_batch(items, b"", tables=[addrs], group_table=[0], n_threads=8)
        assert int(bits(want, len(items)).sum()) == len(A.known_vectors())
        cases = [(ib.Engine.PATH_THREAD, 1), (ib.Engine.PATH_THREAD, -(-(sms * 256 + 100) // len(items))), (ib.Engine.PATH_SPLIT, 1),
                 (ib.Engine.PATH_SPLIT, 7), (ib.Engine.PATH_AUTO, -(-(sms * 72) // len(items)))]
        assert sms * 48 < cases[-1][1] * len(items) <= sms * 96                # AUTO's four-piece range
        for path, reps in cases:
            eng.set_recover_path(path)
            it = np.tile(items, reps)
            bm, res, _ = eng.verify_batch(it, b"", groups)
            assert np.array_equal(bits(bm, len(it)), np.tile(bits(want, len(items)), reps)), (path, reps)
            assert eng.known_handed_back() == handed * reps, (path, reps)
            bp, rp, _ = plain.verify_batch(it, b"", groups)
            assert np.array_equal(bm, bp) and res.tobytes() == rp.tobytes(), (path, reps)
            bm, _, _ = eng.verify_batch(np.tile(valid, reps), b"", groups)
            assert bits(bm, len(valid) * reps).all() and eng.known_handed_back() == 0, (path, reps)
    finally:
        eng.close()
        plain.close()


# ------------------------------------------------------------------------------------- large key-registry calls
def test_large_key_registry_calls_across_chunks():
    """Config 3 (20,000 items, 10,000 validators) tiled to 140,000 items: two 2^17-item chunks on alternating streams and worklists,
    the first above SMs x 256 (k_verify_known<128>).  Pass 2 gives the tiled golden bitmap and a plain engine's results, and hands
    back 7 x the per-copy count; the same batch through the device-resident entry point gives the tiled bitmap too."""
    import torch
    d, items = load_fixture("config3.npz")
    reps = 7
    big = np.tile(items, reps)
    n = len(big)
    gold = bits(d["bitmap"], len(items))
    want = pack(np.tile(gold, reps))
    members = {bytes(a) for a in d["addrs"]}
    known = {bytes(items[i]["signer"]) for i in range(len(items)) if gold[i]}
    per_copy = expected_handed_back(items, len(d["arena"]), members, gold, known)
    kw = dict(device=0, max_items=n, max_payload_bytes=len(d["arena"]) + 1024, max_groups=4, max_table_slots=1, max_validators=10_000)
    eng = ib.Engine(**kw, key_cache=True)
    plain = ib.Engine(**kw)
    try:
        for e in (eng, plain):
            e.set_validators(0, int(d["meta"][2]), d["addrs"], d["powers"])
        groups = groups_for(eng, len(d["groups"]))
        bm1, res1, _ = eng.verify_batch(big, d["arena"], groups)             # pass 1: keys learned
        assert np.array_equal(bm1, want)
        assert eng.refresh_key_tables() == len(known)
        bp, rp, _ = plain.verify_batch(big, d["arena"], groups)
        for path in (ib.Engine.PATH_AUTO, ib.Engine.PATH_THREAD):
            eng.set_recover_path(path)
            bm2, res2, _ = eng.verify_batch(big, d["arena"], groups)
            assert np.array_equal(bm2, want), path
            assert res2.tobytes() == rp.tobytes() == res1.tobytes(), path
            assert eng.known_handed_back() == reps * per_copy, path
        eng.set_recover_path(ib.Engine.PATH_AUTO)
        eng.bind_groups(groups)
        t_items = torch.from_numpy(big.view(np.uint8).reshape(-1, 128).copy()).cuda()
        t_arena = torch.from_numpy(np.ascontiguousarray(d["arena"]).copy()).cuda()
        t_bm = torch.zeros((n + 31) // 32, dtype=torch.int32, device="cuda")
        st = torch.cuda.current_stream().cuda_stream
        eng.verify_device(t_items.data_ptr(), n, t_arena.data_ptr(), t_arena.numel(), 0, n, t_bm.data_ptr(), 0, st)
        torch.cuda.synchronize()
        got = t_bm.cpu().numpy().view(np.uint32)
        if n & 31:
            got[-1] &= (1 << (n & 31)) - 1
        assert np.array_equal(got, want)
        eng.bind_groups(None)
    finally:
        eng.close()
        plain.close()
