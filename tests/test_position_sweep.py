"""The position sweep's generator and expectations on the CPU (tests/position_sweep.py): every (class, position, geometry) cell is
built, each class item is what it claims to be by the big-integer oracle, and the expectations tiled from the distinct tuples equal
the references run directly on whole batches."""
import numpy as np
import pytest

import adversarial as A
import explain_oracle as X
import position_sweep as PS
from oracle import coracle as co
from oracle import secp256k1 as ec

N, P = ec.N, ec.P


@pytest.fixture(scope="module")
def S():
    return PS.sweep()


def int_of(b) -> int:
    return int.from_bytes(bytes(b), "big")


def test_every_cell_is_built(S):
    """each geometry's window: pattern (a) puts each class at each position exactly once (block p holds it at p, fillers around it),
    pattern (b) one valid filler at p among R_NOT_X items, pattern (c) ends the call right after the class item at p"""
    raw = lambda a: np.ascontiguousarray(a).view(np.uint8).reshape(len(a), 128)[:, :124]  # noqa: E731  (without group / offsets)
    cells = set()
    for geom, W in PS.WINDOWS.items():
        classes = S.known_classes if geom.startswith("verify") else S.classes
        for name, odd in classes.items():
            items = np.concatenate([S.block(W, p, W, odd, p, "a") for p in range(W)])
            assert len(items) == W * W
            for p in range(W):
                blk = items[p * W:(p + 1) * W]
                odd_at = [j for j in range(W) if (raw(blk[j:j + 1])[0][:116] == raw(odd)[0][:116]).all()]
                assert odd_at == [p], (geom, name, p)
                assert (blk["group"][[j for j in range(W) if j != p]] == [2 * p + j % 2 for j in range(W) if j != p]).all()
                cells.add((geom, name, p))
            if not geom.startswith("verify"):
                for p in (0, W // 2, W - 1):
                    tail = S.pattern_c(W, name, p)
                    assert len(tail) == p + 1 and (raw(tail[-1:])[0][:116] == raw(odd)[0][:116]).all()
        if not geom.startswith("verify"):
            b = S.pattern_b(W)
            for p in range(W):
                blk = b[p * W:(p + 1) * W]
                assert bytes(blk[p]["signer"]) == bytes(S.fillers[p]["signer"])
                assert all(int_of(blk[j]["r"]) == int_of(S.invalid[0]["r"]) for j in range(W) if j != p)
    want = sum(W * len(S.known_classes if g.startswith("verify") else S.classes) for g, W in PS.WINDOWS.items())
    assert len(cells) == want
    # neighbouring positions: different groups, on different table slots
    for W in (32, 96, 128):
        blk = S.block(W, 5, W, S.classes["valid_low_s"], 0, "a")
        slots = S.group_slots(W)
        g = blk["group"].astype(int)
        assert all(g[j] != g[j + 1] and slots[g[j]] != slots[g[j + 1]] for j in range(W - 1))


def test_each_class_is_what_it_claims(S):
    """by the big-integer oracle, not by the reference under test"""
    c = S.classes
    r = lambda name: int_of(c[name][0]["r"])  # noqa: E731
    s = lambda name: int_of(c[name][0]["s"])  # noqa: E731
    assert pow((r("r_not_x") ** 3 + 7) % P, (P - 1) // 2, P) == P - 1     # r^3 + 7 is a non-residue: no point has abscissa r
    assert r("r_zero") == 0 and r("r_eq_n") == N and s("s_eq_n") == N
    assert int(c["bad_v"][0]["v"]) > 1
    assert s("valid_low_s") <= N // 2 < s("valid_high_s")
    for name in ("u1_zero_z0", "u1_zero_zn"):
        z = int_of(c[name][0]["digest"])
        assert z % N == 0                                                   # u1 = -z / r = 0
        assert ec.recover_pubkey(z, r(name), s(name), int(c[name][0]["v"])) is not None
    assert int_of(c["u1_zero_zn"][0]["digest"]) == N
    # NO_KEY: Q = r^-1 (s R - z G) is the point at infinity
    it = c["no_key"][0]
    rr, ss, z = int_of(it["r"]), int_of(it["s"]), int_of(it["digest"])
    y2 = (rr ** 3 + 7) % P
    y = pow(y2, (P + 1) // 4, P)
    R = (rr, y if (y & 1) == int(it["v"]) else P - y)
    assert ec.point_add(ec.point_mul(ss, R), ec.point_mul((-z) % N, ec.G)) == ec.INF
    # SIGNER_MISMATCH / NOT_VALIDATOR: the recovered key is someone else's / no member's
    for name, member in (("signer_mismatch", True), ("not_validator", False), ("valid_low_s", True)):
        it = c[name][0]
        Q = ec.recover_pubkey(int_of(it["digest"]), int_of(it["r"]), int_of(it["s"]), int(it["v"]))
        addr = ec.pubkey_to_address(Q)
        assert (addr == bytes(it["signer"])) == (name != "signer_mismatch")
        assert (addr in S.members) == member
    assert int(c["no_group"][0]["group"]) >= 2 and int(c["no_table"][0]["group"]) == 1
    assert {int(c[k][0]["kind"]) for k in ("payload", "payload2", "wire", "wire_seal", "valid_low_s")} == \
        {X.KIND_PAYLOAD, X.KIND_PAYLOAD2, X.KIND_WIRE, X.KIND_WIRE_SEAL, X.KIND_DIGEST}
    assert int(c["malformed_span"][0]["payload_off"]) + int(c["malformed_span"][0]["payload_len"]) > len(S.arena)
    # known-key classes
    kc = S.known_classes
    # the x = r + n forgery: its nonce point has abscissa r + n < p (plain ECDSA accepts it for the key), while r itself lifts to
    # another point, so recovery does not yield the key
    it = kc["known_r_plus_n"][0]
    rr, ss, z = int_of(it["r"]), int_of(it["s"]), int_of(it["digest"])
    assert rr + N < P and pow(((rr + N) ** 3 + 7) % P, (P - 1) // 2, P) == 1
    Q = A.known_key(S.known_keys[1])
    w = pow(ss, -1, N)
    Rn = ec.point_add(ec.point_mul(z * w % N, ec.G), ec.point_mul(rr * w % N, Q))
    assert Rn[0] == rr + N                                              # u1 G + u2 Q has x = r + n: x mod n == r
    rec = ec.recover_pubkey(z, rr, ss, int(it["v"]))
    assert rec != Q
    # the cancelling signature: u1 G + u2 Q is the point at infinity for the claimed key Q = G
    it = kc["known_cancelling"][0]
    rr, ss, z = int_of(it["r"]), int_of(it["s"]), int_of(it["digest"])
    Q = A.known_key(S.known_keys[0])
    w = pow(ss, -1, N)
    assert ec.point_add(ec.point_mul(z * w % N, ec.G), ec.point_mul(rr * w % N, Q)) == ec.INF
    # the budget class: a valid signature of a member other than the fillers
    it = kc["known_no_table"][0]
    rec = ec.recover_pubkey(int_of(it["digest"]), int_of(it["r"]), int_of(it["s"]), int(it["v"]))
    assert ec.pubkey_to_address(rec) == bytes(it["signer"]) and bytes(it["signer"]) in S.members
    assert int_of(kc["known_flipped"][0]["r"]) == int_of(kc["known_valid"][0]["r"])
    assert int(kc["known_flipped"][0]["v"]) == 1 - int(kc["known_valid"][0]["v"])
    assert bytes(kc["unknown_signer"][0]["signer"]) not in {bytes(f["signer"]) for f in S.fillers}


def test_expectations_have_the_claimed_reasons(S):
    want = {"no_group": X.NO_GROUP, "malformed_span": X.MALFORMED, "malformed_frame": X.MALFORMED, "needs_host": X.NEEDS_HOST,
            "bad_v": X.BAD_V, "r_zero": X.R_RANGE, "r_eq_n": X.R_RANGE, "s_eq_n": X.S_RANGE, "r_not_x": X.R_NOT_X, "no_key": X.NO_KEY,
            "signer_mismatch": X.SIGNER_MISMATCH, "not_validator": X.NOT_VALIDATOR}
    for name in S.names:
        e = S.expect(S.pattern_c(32, name, 0), 1, 32)
        assert int(e["reason"][0]) == want.get(name, X.OK), name
        assert bool(e["bit"][0]) == (name not in want), name
        assert int(e["status"][0]) == (name == "needs_host"), name
    assert S.filler_gold.all()


@pytest.mark.parametrize("W,name", [(96, "u1_zero_zn"), (32, "signer_mismatch"), (96, "wire_seal"), (32, "payload2"), (96, None)])
def test_tiled_expectations_equal_the_direct_references(S, W, name):
    """the dedup-and-tile expectations against explain_batch and the C oracle run on the whole batch, item by item"""
    items = S.pattern_b(W) if name is None else S.pattern_a(W, name)
    e = S.expect(items, W, W)
    ng = S.n_groups(W)
    (a0, _), (a1, _) = S.tables(W)
    gt = [1 if s == 1 else (PS.NO_TABLE if s == PS.NO_TABLE else 0) for s in S.group_slots(W)]
    reasons, xrec = X.explain_batch(items, S.arena, [a0, a1], gt)
    assert np.array_equal(reasons, e["reason"]) and np.array_equal(xrec, e["xrec"])
    flat = ~np.isin(items["kind"], [X.KIND_WIRE, X.KIND_WIRE_SEAL])
    bm = co.verify_batch(items, S.arena, tables=[a0, a1], group_table=gt, n_threads=8)
    assert np.array_equal(PS.bits(bm, len(items))[flat], e["bit"][flat])
    for i in np.nonzero(flat)[0][:: 37]:
        why, got = X._signature_and_digest(items[i], S.arena)
        want = bytes(20) if why else (co.ecrecover_address(got[1], got[0]) or bytes(20))
        assert bytes(e["rec"][i]) == want
    assert len(e["groups"]) == ng
    assert sum(g[0] for g in e["groups"]) == int(e["bit"].sum())
