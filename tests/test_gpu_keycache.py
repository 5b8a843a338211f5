"""Key registry (IBFT_FLAG_KEY_CACHE): signatures of validators whose public key was learned from an earlier successful
recovery are VERIFIED against that key; every verdict must still be the recover path's verdict (include/ibft_verify.h)."""
import random

import numpy as np
import pytest

import ibft_b200 as ib
import workloads as wl
from oracle import coracle as co
from oracle import secp256k1 as ec
from test_gpu_adversarial import bits, expected_handed_back
from test_gpu_verify import expected_groups, groups_for, load_fixture

pytestmark = pytest.mark.gpu


def make_engine(**kw):
    return ib.Engine(device=0, max_items=1 << 16, max_payload_bytes=1 << 22, max_groups=8, max_table_slots=2, max_validators=16384, **kw)


@pytest.mark.parametrize("name", ["config2.npz", "config3.npz"])
def test_learn_then_verify_gives_the_golden_bitmap(name):
    d, items = load_fixture(name)
    eng = make_engine(key_cache=True)
    try:
        eng.set_recover_path(ib.Engine.PATH_THREAD)  # the kernel that holds the verify path
        eng.set_validators(0, int(d["meta"][2]), d["addrs"], d["powers"])
        groups = groups_for(eng, len(d["groups"]))
        assert eng.refresh_key_tables() == 0
        bm1, res1, _ = eng.verify_batch(items, d["arena"], groups)          # recover path, keys learned, tables built on the way out
        assert np.array_equal(bm1, d["bitmap"])
        known = eng.refresh_key_tables()
        signers_ok = {bytes(items[i]["signer"]) for i in range(len(items)) if (int(bm1[i >> 5]) >> (i & 31)) & 1}
        assert known == len(signers_ok) > 0
        launches = eng.launch_count()
        bm2, res2, _ = eng.verify_batch(items, d["arena"], groups)          # verify path for every known signer
        assert np.array_equal(bm2, d["bitmap"])
        assert res1.tobytes() == res2.tobytes()
        assert eng.launch_count() - launches == 3                           # k_verify_known + worklist k_recover + k_quorum_reduce: no table rebuild
        # every valid signer's key is known now: the known-key pass hands back exactly the member items it cannot accept
        members = {bytes(a) for a in d["addrs"]}
        handed = expected_handed_back(items, len(d["arena"]), members, bits(d["bitmap"], len(items)), signers_ok)
        assert eng.known_handed_back() == handed > 0
        # recovered addresses requested: the recover path must be taken (and give the same answers as a plain engine)
        bm3, _, rec3 = eng.verify_batch(items[:500], d["arena"], groups, want_recovered=True)
        plain = make_engine()
        plain.set_validators(0, int(d["meta"][2]), d["addrs"], d["powers"])
        bm4, _, rec4 = plain.verify_batch(items[:500], d["arena"], groups, want_recovered=True)
        plain.close()
        assert np.array_equal(bm3, bm4) and np.array_equal(rec3, rec4)
        # a validator set of OTHER addresses starts with an empty registry (keys are carried over by address only)
        strangers = np.frombuffer(b"".join(wl.address_of(wl.privkey(78, i)) for i in range(8)), np.uint8).reshape(8, 20)
        eng.set_validators(0, int(d["meta"][2]) + 1, strangers, None)
        assert eng.refresh_key_tables() == 0
        with pytest.raises(ib.EngineError):                                 # the old descriptors name the replaced height
            eng.verify_batch(items, d["arena"], groups)
        eng.set_validators(0, int(d["meta"][2]) + 2, d["addrs"], d["powers"])
        assert eng.refresh_key_tables() == 0                                # nothing to carry from the strangers' table
        groups = groups_for(eng, len(d["groups"]))
        bm5, _, _ = eng.verify_batch(items, d["arena"], groups)
        assert np.array_equal(bm5, d["bitmap"])
        assert eng.refresh_key_tables() == known                            # learned again
    finally:
        eng.close()


def test_rejected_verifications_fall_back_to_recovery_exactly():
    """Known validators, then a batch of valid / corrupted / recovery-id-flipped / misattributed signatures: bit-exact with the
    oracle (which always recovers)."""
    rnd = random.Random(77)
    vs = wl.ValidatorSet(11, 64, weighted=True)
    eng = make_engine(key_cache=True)
    try:
        eng.set_recover_path(ib.Engine.PATH_THREAD)
        eng.set_validators(0, 9, vs.addr_array(), vs.power_array())
        groups = groups_for(eng, 1)
        # round 1: everybody signs once -> all keys learned
        dig0 = co.keccak256(b"round-1")
        warm = np.concatenate([wl.make_item(wl.sign(vs.keys[i], dig0), vs.addrs[i], 0, dig0) for i in range(48)])  # 16 stay unknown
        bm, _, _ = eng.verify_batch(warm, b"", groups)
        assert all((int(bm[i >> 5]) >> (i & 31)) & 1 for i in range(48))
        assert eng.refresh_key_tables() == 48
        # round 2: a mixed bag
        rows = []
        for i in range(64):
            dig = co.keccak256(bytes([i]) + b"round-2")
            sig = wl.sign(vs.keys[i], dig, low_s=bool(i & 1))
            kind = i % 6
            claimed = vs.addrs[i]
            if kind == 1:      # corrupted r or s
                b = bytearray(sig); b[rnd.randrange(64)] ^= 1 << rnd.randrange(8); sig = bytes(b)
            elif kind == 2:    # flipped recovery id
                sig = sig[:64] + bytes([sig[64] ^ 1])
            elif kind == 3:    # signed by i, attributed to another (known) validator
                claimed = vs.addrs[(i + 1) % 48]
            elif kind == 4:    # high-s twin: same key, other recovery id -> still valid
                s = int.from_bytes(sig[32:64], "big")
                sig = sig[:32] + (ec.N - s).to_bytes(32, "big") + bytes([sig[64] ^ 1])
            rows.append(wl.make_item(sig, claimed, 0, dig))
            ph = co.keccak256(bytes([i]) + b"seal")
            rows.append(wl.make_item(wl.sign(vs.keys[i], wl.seal_digest(ph)), vs.addrs[i], 2, ph))
        batch = np.concatenate(rows)
        bm2, res2, _ = eng.verify_batch(batch, b"", groups)
        want = co.verify_batch(batch, b"", tables=[vs.addr_array()], group_table=[0], n_threads=4)
        assert np.array_equal(bm2, want)
        exp, _ = expected_groups(batch, bm2, vs.addr_array(), vs.power_array())
        nv, nd, power, hq = exp.get(0, (0, 0, 0, False))
        assert (int(res2[0]["n_valid"]), int(res2[0]["n_distinct"]), bool(res2[0]["has_quorum"])) == (nv, nd, hq)
        assert eng.refresh_key_tables() == 64      # the 16 late validators were learned in round 2
    finally:
        eng.close()


def test_known_key_latency_path_on_a_10k_round():
    """k_verify_known<32> (+ k_recover_qsplit on the worklist): one mid-size round of KNOWN validators on the latency path (and the
    same round through the chain + helper form k_verify_split, forced).  Round 1
    learns the keys through the recover kernels; round 2 -- same 10,000 seals incl. the 1 % adversarial ones, then fresh seals over
    another proposal hash -- is verified against the keys.  Bitmap, quorum results and voted sets bit-exact with the recover path."""
    d, items = load_fixture("config3.npz")
    seal_group = list(d["groups"]).index("COMMIT_SEAL")
    seals = np.ascontiguousarray(items[items["group"] == seal_group])
    gold_bits = np.unpackbits(d["bitmap"].view(np.uint8), bitorder="little")[: len(items)][items["group"] == seal_group]
    eng = make_engine(key_cache=True)
    plain = make_engine()
    try:
        for e in (eng, plain):
            e.set_validators(0, int(d["meta"][2]), d["addrs"], d["powers"])
        groups = groups_for(eng, len(d["groups"]))
        bm1, res1, _ = eng.verify_batch(seals, b"", groups)                 # recover path (k_recover_split pieces), keys learned
        assert np.array_equal(np.unpackbits(bm1.view(np.uint8), bitorder="little")[: len(seals)], gold_bits)
        assert eng.refresh_key_tables() == int(gold_bits.sum())
        launches = eng.launch_count()
        bm2, res2, _ = eng.verify_batch(seals, b"", groups)                 # known-key latency path
        assert np.array_equal(bm2, bm1) and res1.tobytes() == res2.tobytes()
        # four pieces x (k_verify_known + worklist k_recover_qsplit) + k_quorum_reduce; no table rebuild
        assert eng.launch_count() - launches == 9
        members = {bytes(a) for a in d["addrs"]}
        known = {bytes(seals[i]["signer"]) for i in range(len(seals)) if gold_bits[i]}
        gold = gold_bits.astype(bool)
        assert eng.known_handed_back() == expected_handed_back(seals, 0, members, gold, known) > 0
        for path in (ib.Engine.PATH_SPLIT, ib.Engine.PATH_THREAD):           # k_verify_split / one chunk of k_verify_known
            eng.set_recover_path(path)
            bm3, res3, _ = eng.verify_batch(seals, b"", groups)
            assert np.array_equal(bm3, bm1) and res1.tobytes() == res3.tobytes()
            split = path == ib.Engine.PATH_SPLIT                             # the chain + helper form settles out-of-range (r, s, v)
            assert eng.known_handed_back() == expected_handed_back(seals, 0, members, gold, known, split=split) > 0
        eng.set_recover_path(ib.Engine.PATH_AUTO)
        bmp, resp, _ = plain.verify_batch(seals, b"", groups)
        assert np.array_equal(bm2, bmp) and res2.tobytes() == resp.tobytes()
        for g in range(len(groups)):
            assert np.array_equal(eng.voted_bitmap(g, len(d["addrs"])), plain.voted_bitmap(g, len(d["addrs"])))
        # a fresh round: new proposal hash, every validator signs; one signature corrupted, one misattributed
        vs_keys = [wl.privkey(2, i) for i in range(0, 10_000, 97)]          # a subset is enough for the oracle-signed fresh items
        ph = co.keccak256(b"next block")
        fresh = []
        for j, k in enumerate(vs_keys):
            i = 97 * j
            sig = wl.sign(k, wl.seal_digest(ph))
            signer = bytes(d["addrs"][i])
            if j == 5:
                sig = sig[:40] + bytes([sig[40] ^ 2]) + sig[41:]           # verification rejects -> worklist -> recover says invalid
            if j == 9:
                signer = bytes(d["addrs"][i + 1])                           # valid signature of ANOTHER validator's key
            fresh.append(wl.make_item(sig, signer, 2, ph, seal_group))
        fresh = np.concatenate(fresh * 80)[:8000]                           # 8,000 tuples: the chain + helper kernel's range
        a, ra, _ = eng.verify_batch(fresh, b"", groups)
        handed = eng.known_handed_back()
        b, rb, _ = plain.verify_batch(fresh, b"", groups)
        assert np.array_equal(a, b) and ra.tobytes() == rb.tobytes()
        want = co.verify_batch(fresh, b"", tables=[d["addrs"]], group_table=[0] * len(groups), n_threads=8)
        assert np.array_equal(a, want)
        # the corrupted and the misattributed copies (and signers whose key round 1 could not learn) go to the recover pass
        assert handed == expected_handed_back(fresh, 0, members, bits(want, len(fresh)), known) >= 2 * 8000 // len(vs_keys)
    finally:
        eng.close()
        plain.close()


def test_keys_carry_over_to_the_next_height():
    """A key belongs to an address, not to a height: ibft_set_validators carries the finished comb tables over from the donor table
    (the previous height's slot, or the slot's own previous content) for every address that is still a validator.  Verdicts,
    quorum and voted sets stay those of a plain engine; the carried validators are verified without a single recovery."""
    d, items = load_fixture("config2.npz")
    h = int(d["meta"][2])
    addrs, powers = d["addrs"], d["powers"]
    eng = make_engine(key_cache=True)
    plain = make_engine()
    try:
        eng.set_validators(0, h, addrs, powers)
        bm1, _, _ = eng.verify_batch(items, d["arena"], groups_for(eng, len(d["groups"])))
        assert np.array_equal(bm1, d["bitmap"])
        known = eng.refresh_key_tables()
        assert 0 < known <= len(addrs)
        ok_signers = {bytes(items[i]["signer"]) for i in range(len(items)) if (int(bm1[i >> 5]) >> (i & 31)) & 1}
        # next height, ANOTHER slot: three validators gone, two new ones (never seen), order reversed, other voting powers
        newcomers = np.frombuffer(b"".join(wl.address_of(wl.privkey(77, i)) for i in range(2)), np.uint8).reshape(2, 20)
        addrs2 = np.ascontiguousarray(np.concatenate([addrs[3:][::-1], newcomers]))
        powers2 = np.ascontiguousarray(np.concatenate([powers[3:][::-1], powers[:2]]))
        carried = len({bytes(a) for a in addrs2} & ok_signers)
        for e in (eng, plain):
            e.set_validators(1, h + 1, addrs2, powers2)
        assert eng.refresh_key_tables() == known + carried
        g2 = groups_for(eng, len(d["groups"]), slot=1)
        launches = eng.launch_count()
        a, ra, _ = eng.verify_batch(items, d["arena"], g2)
        assert eng.launch_count() - launches == 3          # known-key pass + worklist pass + quorum: nothing to learn, nothing to build
        handed = eng.known_handed_back()
        b, rb, _ = plain.verify_batch(items, d["arena"], groups_for(plain, len(d["groups"]), slot=1))
        assert np.array_equal(a, b) and ra.tobytes() == rb.tobytes()
        want = co.verify_batch(items, d["arena"].tobytes(), tables=[addrs2], group_table=[0] * len(d["groups"]), n_threads=8)
        assert np.array_equal(a, want)
        # carried keys are verified: only the new table's member items that cannot be accepted reach the recover pass
        members2 = {bytes(x) for x in addrs2}
        assert handed == expected_handed_back(items, len(d["arena"]), members2, bits(want, len(items)), ok_signers & members2) > 0
        for g in range(len(g2)):
            assert np.array_equal(eng.voted_bitmap(g, len(addrs2)), plain.voted_bitmap(g, len(addrs2)))
        # the same slot re-used for the height after that: the donor is the slot's own previous content
        eng.set_validators(1, h + 2, addrs2, powers2)
        assert eng.refresh_key_tables() == known + carried
        c, rc, _ = eng.verify_batch(items, d["arena"], groups_for(eng, len(d["groups"]), slot=1))
        assert np.array_equal(c, a) and rc.tobytes() == ra.tobytes()
        # slot 0 still answers for its own height from its own registry
        z, _, _ = eng.verify_batch(items, d["arena"], groups_for(eng, len(d["groups"])))
        assert np.array_equal(z, d["bitmap"])
    finally:
        eng.close()
        plain.close()
