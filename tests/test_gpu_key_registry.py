"""One key registry per engine (IBFT_FLAG_KEY_CACHE): a key learned through any resident validator table serves every table that
lists the address, an entry is retired when no resident table lists it any more, and a retired entry that goes to a new
address never verifies against the old key.  Every bitmap, quorum result and voted set must equal a plain engine's and the
oracle's (which always recovers); the known-key pass is made visible through the launch count and the number of items it
hands back (ibft_debug_known_handed_back), the registry itself through ibft_debug_key_registry."""
import random
import threading

import numpy as np
import pytest

import ibft_b200 as ib
import workloads as wl
from oracle import coracle as co
from oracle import secp256k1 as ec
from test_gpu_adversarial import bits, expected_handed_back, point_of
from test_gpu_verify import expected_groups, groups_for, load_fixture

pytestmark = pytest.mark.gpu
CHUNK_BYTES = 256 * 17 * 128 * 64  # 256 comb tables of 136 KiB


def make_engine(slots=4, max_validators=16384, **kw):
    return ib.Engine(device=0, max_items=1 << 16, max_payload_bytes=1 << 22, max_groups=8, max_table_slots=slots,
                     max_validators=max_validators, **kw)


def addr_rows(addrs):
    return np.frombuffer(b"".join(addrs), np.uint8).reshape(-1, 20).copy()


def signers_ok(items, bm):
    return {bytes(items[i]["signer"]) for i in range(len(items)) if (int(bm[i >> 5]) >> (i & 31)) & 1}


def same_as_plain(eng, plain, items, arena, slot, n_groups, n_validators):
    """verify on both engines: bitmaps, results and voted sets equal; returns (bitmap, handed back)"""
    a, ra, _ = eng.verify_batch(items, arena, groups_for(eng, n_groups, slot=slot))
    handed = eng.known_handed_back()
    b, rb, _ = plain.verify_batch(items, arena, groups_for(plain, n_groups, slot=slot))
    assert np.array_equal(a, b) and ra.tobytes() == rb.tobytes()
    for g in range(n_groups):
        assert np.array_equal(eng.voted_bitmap(g, n_validators), plain.voted_bitmap(g, n_validators))
    return a, handed


# ------------------------------------------------------------------------------------- learned after the table was set
def test_key_learned_after_set_serves_the_next_height():
    """Slots 0 (H) and 1 (H+1) hold the same config-2 validators.  The keys learned while verifying H reach H+1's table: its batch
    takes exactly the known-key pass, an empty worklist pass and the quorum launch, and hands back only what a fully known set
    hands back."""
    d, items = load_fixture("config2.npz")
    h, addrs, powers, arena = int(d["meta"][2]), d["addrs"], d["powers"], d["arena"]
    ng = len(d["groups"])
    eng, plain = make_engine(key_cache=True), make_engine()
    try:
        for e in (eng, plain):
            e.set_validators(0, h, addrs, powers)
            e.set_validators(1, h + 1, addrs, powers)
        assert eng.refresh_key_tables() == 0
        bm0, _ = same_as_plain(eng, plain, items, arena, 0, ng, len(addrs))
        assert np.array_equal(bm0, d["bitmap"])
        known = signers_ok(items, bm0)
        assert eng.refresh_key_tables() == 2 * len(known) > 0
        assert eng.key_registry()[:2] == (len({bytes(a) for a in addrs}), len(known))
        launches = eng.launch_count()
        bm1, handed = same_as_plain(eng, plain, items, arena, 1, ng, len(addrs))
        assert eng.launch_count() - launches == 3           # known-key pass + worklist pass + quorum: nothing learned, nothing built
        assert np.array_equal(bm1, d["bitmap"])
        members = {bytes(a) for a in addrs}
        assert handed == expected_handed_back(items, len(arena), members, bits(bm1, len(items)), known) > 0
        want = co.verify_batch(items, arena.tobytes(), tables=[addrs], group_table=[0] * ng, n_threads=8)
        assert np.array_equal(bm1, want)
    finally:
        eng.close()
        plain.close()


def test_key_learned_at_h_reaches_a_table_set_later_for_h_plus_2():
    """H and H+1 are resident and only H has learned.  H+2, set in a third slot, is verified without a single recovery of a known
    signer (the greatest resident height, H+1, had learned nothing)."""
    d, items = load_fixture("config2.npz")
    h, addrs, powers, arena = int(d["meta"][2]), d["addrs"], d["powers"], d["arena"]
    ng = len(d["groups"])
    order = np.random.default_rng(3).permutation(len(addrs))
    addrs2, powers2 = np.ascontiguousarray(addrs[order]), np.ascontiguousarray(powers[order[::-1]])
    eng, plain = make_engine(key_cache=True), make_engine()
    try:
        for e in (eng, plain):
            e.set_validators(0, h, addrs, powers)
            e.set_validators(1, h + 1, addrs, powers)
        bm0, _, _ = eng.verify_batch(items, arena, groups_for(eng, ng, slot=0))
        known = signers_ok(items, bm0)
        assert eng.refresh_key_tables() == 2 * len(known)
        for e in (eng, plain):
            e.set_validators(2, h + 2, addrs2, powers2)
        assert eng.refresh_key_tables() == 3 * len(known)
        launches = eng.launch_count()
        bm2, handed = same_as_plain(eng, plain, items, arena, 2, ng, len(addrs))
        assert eng.launch_count() - launches == 3
        want = co.verify_batch(items, arena.tobytes(), tables=[addrs2], group_table=[0] * ng, n_threads=8)
        assert np.array_equal(bm2, want)
        assert handed == expected_handed_back(items, len(arena), {bytes(a) for a in addrs}, bits(want, len(items)), known) > 0
    finally:
        eng.close()
        plain.close()


# ------------------------------------------------------------------------------------- memory: one entry per address
def round_items(privs, addrs, digest, signer_of=None, group=0):
    """one digest item per private key, attributed to signer_of[i] (default: the key's own address)"""
    n = len(privs)
    sigs = co.sign_derived_batch(privs, np.tile(np.frombuffer(digest, np.uint8), (n, 1)))
    it = np.zeros(n, dtype=ib.ITEM_DTYPE)
    it["r"], it["s"], it["v"] = sigs[:, :32], sigs[:, 32:64], sigs[:, 64]
    it["digest"] = np.frombuffer(digest, np.uint8)
    it["signer"] = addrs if signer_of is None else signer_of
    it["kind"] = ib.KIND_DIGEST
    it["group"] = group
    return it


def test_registry_holds_one_entry_per_distinct_address():
    """The same 1,000 validators resident at 12 heights, some reordered, some with other powers: 1,000 entries and one set's worth
    of comb tables rounded up to a 256-entry chunk.  A key learned through one table is known in all 12.  100 new addresses grow
    the pool by one chunk; when they leave every table their entries are retired (the pool keeps its chunks)."""
    n, heights = 1000, 12
    privs = co.privkeys(731, n)
    addrs = co.addresses(privs)
    rng = np.random.default_rng(5)
    eng, plain = make_engine(slots=16, max_validators=1024, key_cache=True), make_engine(slots=16, max_validators=1024)
    try:
        tables = []
        for k in range(heights):
            order = np.arange(n) if k % 3 == 0 else (np.arange(n)[::-1] if k % 3 == 1 else rng.permutation(n))
            powers = np.zeros((n, 32), np.uint8)
            powers[:, 31] = 1 + (np.arange(n) + k) % (1 + k % 5)
            tables.append((np.ascontiguousarray(addrs[order]), powers))
            for e in (eng, plain):
                e.set_validators(k, 100 + k, *tables[-1])
        assert eng.key_registry() == (n, 0, 4 * CHUNK_BYTES)
        assert eng.refresh_key_tables() == 0
        dig = co.keccak256(b"registry-memory")
        items = round_items(privs, addrs, dig)
        bm, _ = same_as_plain(eng, plain, items, b"", 3, 1, n)
        assert bits(bm, n).all()
        assert eng.refresh_key_tables() == heights * n
        assert eng.key_registry() == (n, n, 4 * CHUNK_BYTES)
        for k in (0, 7, 11):                                  # every table verifies every signer against its key
            launches = eng.launch_count()
            bm, handed = same_as_plain(eng, plain, items, b"", k, 1, n)
            assert bits(bm, n).all() and handed == 0 and eng.launch_count() - launches == 3
        # 100 new addresses in one table: 1,100 entries need a fifth chunk; they are learned through that table only
        new_privs = co.privkeys(732, 100)
        mixed = np.concatenate([addrs[:900], co.addresses(new_privs)])
        for e in (eng, plain):
            e.set_validators(5, 200, mixed, None)
        assert eng.key_registry() == (1100, 1000, 5 * CHUNK_BYTES)
        assert eng.refresh_key_tables() == (heights - 1) * n + 900
        fresh = round_items(new_privs, co.addresses(new_privs), dig)
        bm, handed = same_as_plain(eng, plain, fresh, b"", 5, 1, 1000)
        assert bits(bm, 100).all() and handed == 100        # first signatures of new addresses are recovered
        assert eng.key_registry() == (1100, 1100, 5 * CHUNK_BYTES)
        # they leave every table: retired, the chunks stay
        for e in (eng, plain):
            e.set_validators(5, 201, *tables[5])
        assert eng.key_registry() == (n, n, 5 * CHUNK_BYTES)
        assert eng.refresh_key_tables() == heights * n
    finally:
        eng.close()
        plain.close()


# ------------------------------------------------------------------------------------- churn: retired entries, reused
def test_retired_entries_go_to_new_addresses_and_are_learned_again():
    """A[0:16] leave every table and B takes their retired entries, whose key words and comb tables still hold A's keys: B's
    first signatures are recovered, and a signature by the previous owner of B[i]'s entry attributed to B[i] is rejected, before
    and after B's keys are learned.  When B leaves and A[0:16] return (taking B's entries) they are learned again, and a
    signature by the previous owner of A[i]'s entry attributed to A[i] is rejected, before and after A is learned again.  The
    previous owner is read from the entry itself (the reset clears the state only, the stale key stays), so the pairing does
    not depend on the order in which the free list hands entries out."""
    A, B = wl.ValidatorSet(501, 32, weighted=True), wl.ValidatorSet(502, 16)
    A_pub = [ec.point_mul(k, ec.G) for k in A.keys[:16]]
    B_pub = [ec.point_mul(k, ec.G) for k in B.keys]
    eng, plain = make_engine(slots=2, max_validators=64, key_cache=True), make_engine(slots=2, max_validators=64)

    def previous_owners(n, pubs):
        """for validators 0..n-1 of slot 0: the index in `pubs` of the key their (reset) entry still holds -- one to one"""
        owners = []
        for v in range(n):
            state, key, _ = eng.key_table(0, v)
            assert state == 0, v                                   # reset to unknown on reuse
            owners.append(pubs.index(point_of(key)))
        assert sorted(owners) == list(range(n))                   # every new address took a retired entry of the other set
        return owners

    def check(batch, table, slot, known):
        members = {bytes(a) for a in table}
        bm, handed = same_as_plain(eng, plain, batch, b"", slot, 1, len(table))
        want = co.verify_batch(batch, b"", tables=[table], group_table=[0], n_threads=8)
        assert np.array_equal(bm, want)
        assert handed == expected_handed_back(batch, 0, members, bits(want, len(batch)), known)
        return bits(want, len(batch))

    try:
        for e in (eng, plain):
            e.set_validators(0, 1, A.addr_array(), A.power_array())
        d1 = co.keccak256(b"churn-1")
        warm = np.concatenate([wl.make_item(wl.sign(A.keys[i], d1), A.addrs[i], 0, d1) for i in range(32)])
        assert check(warm, A.addr_array(), 0, set()).all()
        assert eng.refresh_key_tables() == 32 and eng.key_registry()[:2] == (32, 32)
        # A[0:16] leave every table (retired), then B joins and takes their entries, reset to unknown
        for e in (eng, plain):
            e.set_validators(0, 2, addr_rows(A.addrs[16:]), None)
        assert eng.key_registry() == (16, 16, CHUNK_BYTES)
        t2 = addr_rows(B.addrs + A.addrs[16:])
        for e in (eng, plain):
            e.set_validators(0, 3, t2, None)
        assert eng.key_registry() == (32, 16, CHUNK_BYTES)
        assert eng.refresh_key_tables() == 16
        prev = previous_owners(16, A_pub)                          # B[i] holds A[prev[i]]'s former entry
        d2 = co.keccak256(b"churn-2")
        rows = []
        for i in range(16):
            rows.append(wl.make_item(wl.sign(B.keys[i], d2), B.addrs[i], 0, d2))             # new owner, first signature
            rows.append(wl.make_item(wl.sign(A.keys[prev[i]], d2), B.addrs[i], 0, d2))       # entry's previous owner's key
            rows.append(wl.make_item(wl.sign(A.keys[i], d2), A.addrs[i], 0, d2))             # left the set
            rows.append(wl.make_item(wl.sign(A.keys[16 + i], d2), A.addrs[16 + i], 0, d2))   # stayed, known
        batch = np.concatenate(rows)
        ok = check(batch, t2, 0, {bytes(a) for a in A.addrs[16:]})
        assert ok.sum() == 32 and not ok[1::4].any() and not ok[2::4].any()
        assert eng.refresh_key_tables() == 32
        ok = check(batch, t2, 0, {bytes(a) for a in A.addrs[16:]} | {bytes(a) for a in B.addrs})   # B known now
        assert ok.sum() == 32
        # B leaves, then A[0:16] return, take B's entries and are learned again
        for e in (eng, plain):
            e.set_validators(0, 4, addr_rows(A.addrs[16:]), None)
        assert eng.key_registry() == (16, 16, CHUNK_BYTES)
        for e in (eng, plain):
            e.set_validators(0, 5, A.addr_array(), A.power_array())
        assert eng.key_registry() == (32, 16, CHUNK_BYTES)
        assert eng.refresh_key_tables() == 16
        prev = previous_owners(16, B_pub)                          # A[i] holds B[prev[i]]'s former entry
        d3 = co.keccak256(b"churn-3")
        rows = []
        for i in range(16):
            rows.append(wl.make_item(wl.sign(B.keys[prev[i]], d3), A.addrs[i], 0, d3))       # entry's previous owner's key
            rows.append(wl.make_item(wl.sign(A.keys[i], d3), A.addrs[i], 0, d3))             # rejoined: recovered again
        batch = np.concatenate(rows)
        ok = check(batch, A.addr_array(), 0, {bytes(a) for a in A.addrs[16:]})
        assert not ok[0::2].any() and ok[1::2].all()
        assert eng.refresh_key_tables() == 32 and eng.key_registry() == (32, 32, CHUNK_BYTES)
        ok = check(batch, A.addr_array(), 0, {bytes(a) for a in A.addrs})                 # A[0:16] known again
        assert not ok[0::2].any() and ok[1::2].all()
    finally:
        eng.close()
        plain.close()


# ------------------------------------------------------------------------------------- two lanes at once
def test_two_lanes_learning_through_tables_that_share_entries():
    """Two host-buffer calls at once (one per lane) on slots that share 40 addresses, both learning new keys: verdicts equal the
    oracle's and a plain engine's, and after refresh_key_tables every learned key is ready."""
    V, W = wl.ValidatorSet(601, 48, weighted=True), wl.ValidatorSet(602, 8)
    t0, t1 = V.addr_array(), addr_rows(V.addrs[8:][::-1] + W.addrs)
    eng, plain = make_engine(key_cache=True), make_engine()
    try:
        for e in (eng, plain):
            e.set_validators(0, 10, t0, V.power_array())
            e.set_validators(1, 11, t1, None)
        d0 = co.keccak256(b"lanes-warm")
        warm = np.concatenate([wl.make_item(wl.sign(V.keys[i], d0), V.addrs[i], 0, d0) for i in range(24)])
        eng.verify_batch(warm, b"", groups_for(eng, 1, slot=0))
        assert eng.refresh_key_tables() == 24 + 16
        rnd = random.Random(4)
        batches = []
        for slot, keys, addrs in ((0, V.keys, V.addrs), (1, V.keys[8:] + W.keys, V.addrs[8:] + W.addrs)):
            dig = co.keccak256(b"lanes" + bytes([slot]))
            sigs = [wl.sign(k, dig) for k in keys]
            items = []
            for rep in range(40):
                for i, a in enumerate(addrs):
                    sig = sigs[i]
                    if rep % 7 == 3 and i % 5 == 1:
                        b = bytearray(sig); b[rnd.randrange(64)] ^= 1 << rnd.randrange(8); sig = bytes(b)
                    items.append(wl.make_item(sig, a, 0, dig))
            batches.append((slot, np.concatenate(items), addr_rows(addrs)))
        out = [None, None]

        def run(j):
            slot, items, _ = batches[j]
            out[j] = eng.verify_batch_ex(items, b"", groups_for(eng, 1, slot=slot), voted_stride_words=2)

        for _ in range(2):
            th = [threading.Thread(target=run, args=(j,)) for j in range(2)]
            for t in th:
                t.start()
            for t in th:
                t.join()
            for j, (slot, items, table) in enumerate(batches):
                bm, res, _, voted = out[j]
                want = co.verify_batch(items, b"", tables=[t0 if slot == 0 else t1], group_table=[0], n_threads=8)
                assert np.array_equal(bm, want), slot
                bp, rp, _ = plain.verify_batch(items, b"", groups_for(plain, 1, slot=slot))
                assert np.array_equal(bm, bp) and res.tobytes() == rp.tobytes(), slot
                assert np.array_equal(voted[0], plain.voted_bitmap(0, 48)), slot
        assert eng.refresh_key_tables() == 48 + 48
        assert eng.key_registry()[:2] == (56, 56)
        for slot in (0, 1):
            for v in range(48):
                assert eng.key_table(slot, v)[0] == 2
    finally:
        eng.close()
        plain.close()


# ------------------------------------------------------------------------------------- rejected verifications, shared entries
def test_rejected_and_misattributed_signatures_on_tables_that_share_entries():
    """test_gpu_keycache's mixed bag (corrupted, recovery-id-flipped, misattributed, high-s twins, seals) verified through a second
    table -- another height, another order -- whose keys were all learned through the first: bit-exact with the oracle."""
    rnd = random.Random(77)
    vs = wl.ValidatorSet(11, 64, weighted=True)
    order = list(range(64))[::-1]
    t1 = addr_rows([vs.addrs[i] for i in order])
    p1 = np.ascontiguousarray(vs.power_array()[order])
    eng, plain = make_engine(key_cache=True), make_engine()
    try:
        eng.set_recover_path(ib.Engine.PATH_THREAD)
        for e in (eng, plain):
            e.set_validators(0, 9, vs.addr_array(), vs.power_array())
            e.set_validators(1, 10, t1, p1)
        dig0 = co.keccak256(b"round-1")
        warm = np.concatenate([wl.make_item(wl.sign(vs.keys[i], dig0), vs.addrs[i], 0, dig0) for i in range(48)])
        bm, _, _ = eng.verify_batch(warm, b"", groups_for(eng, 1, slot=0))
        assert bits(bm, 48).all()
        assert eng.refresh_key_tables() == 2 * 48
        rows = []
        for i in range(64):
            dig = co.keccak256(bytes([i]) + b"round-2")
            sig = wl.sign(vs.keys[i], dig, low_s=bool(i & 1))
            kind = i % 6
            claimed = vs.addrs[i]
            if kind == 1:
                b = bytearray(sig); b[rnd.randrange(64)] ^= 1 << rnd.randrange(8); sig = bytes(b)
            elif kind == 2:
                sig = sig[:64] + bytes([sig[64] ^ 1])
            elif kind == 3:
                claimed = vs.addrs[(i + 1) % 48]
            elif kind == 4:
                s = int.from_bytes(sig[32:64], "big")
                sig = sig[:32] + (ec.N - s).to_bytes(32, "big") + bytes([sig[64] ^ 1])
            rows.append(wl.make_item(sig, claimed, 0, dig))
            ph = co.keccak256(bytes([i]) + b"seal")
            rows.append(wl.make_item(wl.sign(vs.keys[i], wl.seal_digest(ph)), vs.addrs[i], 2, ph))
        batch = np.concatenate(rows)
        bm2, handed = same_as_plain(eng, plain, batch, b"", 1, 1, 64)
        want = co.verify_batch(batch, b"", tables=[t1], group_table=[0], n_threads=4)
        assert np.array_equal(bm2, want)
        known = {bytes(a) for a in vs.addrs[:48]}
        assert handed == expected_handed_back(batch, 0, {bytes(a) for a in vs.addrs}, bits(want, len(batch)), known) > 0
        _, res2, _ = eng.verify_batch(batch, b"", groups_for(eng, 1, slot=1))
        exp, _ = expected_groups(batch, bm2, t1, p1)
        nv, nd, _, hq = exp.get(0, (0, 0, 0, False))
        assert (int(res2[0]["n_valid"]), int(res2[0]["n_distinct"]), bool(res2[0]["has_quorum"])) == (nv, nd, hq)
        assert eng.refresh_key_tables() == 2 * 64                   # the 16 late validators, learned through slot 1, serve slot 0 too
        for path in (ib.Engine.PATH_SPLIT, ib.Engine.PATH_AUTO):
            eng.set_recover_path(path)
            for slot, table in ((0, vs.addr_array()), (1, t1)):
                bm3, _ = same_as_plain(eng, plain, batch, b"", slot, 1, 64)
                assert np.array_equal(bm3, co.verify_batch(batch, b"", tables=[table], group_table=[0], n_threads=4)), (path, slot)
    finally:
        eng.close()
        plain.close()
