"""The reasons of ibft_explain_batch on the CPU: the reference of tests/explain_oracle.py against the oracle's verdicts, a
constructed item for every reason, config 2's adversarial items by kind, and explain_item of the csrc headers (the body of the
kernel k_explain, through the host emulation tests/emul/explain_driver.cpp) against the reference, byte for byte."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

import adversarial as A
import explain_oracle as X
import workloads as wl
from oracle import coracle as co
from oracle import ibft_proto as ip
from oracle import secp256k1 as ec
from test_emul import sample_frames, wire_item
from test_wire_edges import load_edges

HERE = os.path.dirname(os.path.abspath(__file__))
N, P = ec.N, ec.P


@pytest.fixture(scope="module")
def emul_explain(tmp_path_factory):
    """tests/emul/explain_driver.cpp: explain_item of the csrc headers on the host emulation"""
    emul = os.path.join(HERE, "emul")
    so = str(tmp_path_factory.mktemp("emul_explain") / "libibft_explain.so")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-fPIC", "-std=c++17", "-Wall", "-Wextra", "-Wno-unknown-pragmas",
                           '-DEMUL_DIR="%s"' % emul, "-shared", "-o", so, os.path.join(emul, "explain_driver.cpp"), "-lpthread"])
    return ctypes.CDLL(so)


def load_fixture(name):
    d = np.load(os.path.join(HERE, "golden", name + ".npz"))
    items = np.ascontiguousarray(d["items"]).view(co.ITEM_DTYPE).reshape(-1)
    return items, d["arena"].tobytes(), d["addrs"], d["bitmap"], [str(t) for t in d["tags"]], len(d["groups"])


def emul_batch(E, items, arena, tables=None, group_table=None):
    """explain_item of the csrc headers over every item (arguments of explain_oracle.explain_batch)"""
    items = np.ascontiguousarray(items)
    a = np.frombuffer(arena, np.uint8) if arena else np.zeros(1, np.uint8)
    tabs = [np.ascontiguousarray(t, dtype=np.uint8).reshape(-1, 20) for t in (tables or [])]
    reasons = np.zeros(len(items), np.uint8)
    rec = np.zeros((len(items), 20), np.uint8)
    out = (ctypes.c_uint8 * 20)()
    n_groups = 0 if group_table is None else len(group_table)
    for i in range(len(items)):
        g = int(items[i]["group"])
        t = None
        if group_table is not None and g < n_groups and group_table[g] != 0xFFFF:
            t = tabs[group_table[g]]
        reasons[i] = E.emul_explain_item(items[i:i + 1].ctypes.data_as(ctypes.c_void_p), a.ctypes.data_as(ctypes.c_void_p),
                                         ctypes.c_size_t(len(arena)), int(group_table is not None), ctypes.c_uint32(n_groups),
                                         None if t is None else t.ctypes.data_as(ctypes.c_void_p), ctypes.c_uint32(0 if t is None else len(t)), out)
        rec[i] = np.frombuffer(bytes(out), np.uint8)
    return reasons, rec


def check_against_verdicts(items, arena, tables, group_table, bits):
    reasons, rec = X.explain_batch(items, arena, tables, group_table)
    assert np.array_equal(reasons == X.OK, bits)
    assert not (reasons == X.INCONSISTENT).any()
    # the recovered address is there exactly for the items that got as far as recovery
    reached = np.isin(reasons, [X.OK, X.SIGNER_MISMATCH, X.NOT_VALIDATOR])
    assert (rec[reached].any(axis=1)).all() and not rec[~reached].any()
    return reasons, rec


# ---------------------------------------------------------------------------------------------------------- constructed items
def cancelling_signature(c: int, s: int):
    """(sig, z) with R = c G and z = s c: Q = r^-1 (s R - z G) is the point at infinity"""
    R = A.mul(c)
    assert R[0] < N
    z = s * c % N
    return R[0].to_bytes(32, "big") + s.to_bytes(32, "big") + bytes([R[1] & 1]), z.to_bytes(32, "big")


def non_abscissa(seed: int) -> int:
    rnd = random.Random(seed)
    while True:
        r = rnd.randrange(1, N)
        if pow((r ** 3 + 7) % P, (P - 1) // 2, P) == P - 1:
            return r


def every_reason_batch():
    """(items, arena, tables, group_table, want): at least one item per reason; group 0 has a table, group 1 has none"""
    vs = wl.ValidatorSet(5, 4)
    outsider = wl.privkey(99, 0)
    digest = co.keccak256(b"explain")
    good = wl.sign(vs.keys[0], digest)
    rows, arena = [], bytearray()

    def add(want, sig, signer, kind=X.KIND_DIGEST, dig=digest, group=0, off=0, ln=0):
        rows.append((wl.make_item(sig, signer, kind, dig, group, off, ln), want))

    add(X.OK, good, vs.addrs[0])
    add(X.OK, wl.sign(outsider, digest), wl.address_of(outsider), group=1)        # no table: no membership test
    add(X.NO_GROUP, good, vs.addrs[0], group=2)
    add(X.NO_GROUP, good[:64] + b"\x07", vs.addrs[0], group=7)                     # NO_GROUP comes first
    add(X.MALFORMED, b"", vs.addrs[0])                                              # KIND_INVALID
    it = wl.make_item(good, vs.addrs[0], 9, digest)                                 # unknown kind
    rows.append((it, X.MALFORMED))
    add(X.MALFORMED, good, vs.addrs[0], X.KIND_PAYLOAD, b"", 0, 0, 1 << 20)         # span outside the arena
    span2 = (1 << 30).to_bytes(8, "little") + (4).to_bytes(4, "little") + bytes(20)
    add(X.MALFORMED, good, vs.addrs[0], X.KIND_PAYLOAD2, span2, 0, 0, 0)           # second span outside the arena
    add(X.BAD_V, good[:64] + b"\x02", vs.addrs[0])
    add(X.BAD_V, bytes(64) + b"\xff", vs.addrs[0])                                  # BAD_V before R_RANGE
    for r in (0, N, 2**256 - 1):
        add(X.R_RANGE, r.to_bytes(32, "big") + good[32:], vs.addrs[0])
    add(X.R_RANGE, bytes(64) + b"\x00", vs.addrs[0])                                # R_RANGE before S_RANGE
    for s in (0, N, N + 1, 2**256 - 1):
        add(X.S_RANGE, good[:32] + s.to_bytes(32, "big") + good[64:], vs.addrs[0])
    for seed in range(3):
        r = non_abscissa(seed)
        add(X.R_NOT_X, r.to_bytes(32, "big") + good[32:], vs.addrs[0])
    add(X.R_NOT_X, (7).to_bytes(32, "big") + good[32:64] + b"\x01", vs.addrs[0])   # 7^3 + 7 is a non-residue
    for c, s in ((1, 1), (2, 5), (12345, N - 1)):
        sig, z = cancelling_signature(c, s)
        add(X.NO_KEY, sig, vs.addrs[0], dig=z)
    add(X.SIGNER_MISMATCH, good, vs.addrs[1])                                       # From != signer
    add(X.SIGNER_MISMATCH, wl.sign(vs.keys[2], digest), vs.addrs[0])                # signed with another key
    add(X.SIGNER_MISMATCH, good, vs.addrs[0], dig=co.keccak256(b"other"))           # another digest
    add(X.NOT_VALIDATOR, wl.sign(outsider, digest), wl.address_of(outsider))
    add(X.NOT_VALIDATOR, wl.sign(outsider, wl.seal_digest(digest)), wl.address_of(outsider), X.KIND_SEAL)
    # raw frames: canonical, a frame without From, a non-canonical frame, a PREPARE sent as a seal
    view = ip.View(3, 0)
    def frame(key, frm, t=ip.COMMIT, payload=None):
        payload = payload or ip.CommitMessage(digest, wl.sign(key, wl.seal_digest(digest)))
        m = ip.IbftMessage(view, frm, b"", t, payload)
        m.signature = wl.sign(key, co.keccak256(m.payload_no_sig()))
        return ip.encode_ibft_message(m)
    def add_frame(want, wire, kind):
        off = len(arena)
        arena.extend(wire)
        rows.append((wire_item(kind, off, len(wire), 0), want))
    f = frame(vs.keys[1], vs.addrs[1])
    add_frame(X.OK, f, X.KIND_WIRE)
    add_frame(X.OK, f, X.KIND_WIRE_SEAL)
    add_frame(X.SIGNER_MISMATCH, frame(vs.keys[1], vs.addrs[2]), X.KIND_WIRE)
    add_frame(X.NOT_VALIDATOR, frame(outsider, wl.address_of(outsider)), X.KIND_WIRE)
    add_frame(X.MALFORMED, frame(vs.keys[1], vs.addrs[1][:19]), X.KIND_WIRE)        # a 19-byte From
    add_frame(X.MALFORMED, frame(vs.keys[1], vs.addrs[1], ip.PREPARE, ip.PrepareMessage(digest)), X.KIND_WIRE_SEAL)
    add_frame(X.NEEDS_HOST, f + b"\x78\x01", X.KIND_WIRE)                           # unknown field 15: not canonical
    rows.append((wire_item(X.KIND_WIRE, 0, 1 << 20, 0), X.MALFORMED))               # frame span outside the arena
    items = np.concatenate([r[0] for r in rows])
    return items, bytes(arena), [vs.addr_array()], [0, 0xFFFF], np.array([r[1] for r in rows], np.uint8)


def test_every_reason_is_reached():
    items, arena, tables, gt, want = every_reason_batch()
    reasons, rec = X.explain_batch(items, arena, tables, gt)
    assert list(reasons) == list(want), [(i, X.NAMES[int(a)], X.NAMES[int(b)]) for i, (a, b) in enumerate(zip(reasons, want)) if a != b]
    assert set(int(r) for r in reasons) == set(range(11))
    bits = X.bits_of(co.verify_batch(items, arena, tables, gt), len(items))
    # the wire items are not the C oracle's (it has no frame walker): compare the others with its verdicts
    flat = ~np.isin(items["kind"], [X.KIND_WIRE, X.KIND_WIRE_SEAL])
    assert np.array_equal((reasons == X.OK)[flat], bits[flat])


def test_config2_adversarial_items_by_kind():
    """config 2's 1 % adversarial items (i % 100 == 7).  The "s_ge_n" items carry s + n reduced mod 2^256, which is s - (2^256 - n):
    an in-range s of another signature, so their reason is SIGNER_MISMATCH, not S_RANGE"""
    items, arena, addrs, bitmap, tags, ng = load_fixture("config2")
    reasons, rec = check_against_verdicts(items, arena, [addrs], [0] * ng, X.bits_of(bitmap, len(items)))
    want = dict(bad_v=X.BAD_V, r_zero=X.R_RANGE, s_ge_n=X.SIGNER_MISMATCH, flipped_digest=X.SIGNER_MISMATCH,
                non_member=X.NOT_VALIDATOR, from_ne_signer=X.SIGNER_MISMATCH)
    seen = set()
    for i, t in enumerate(tags):
        if t:
            assert reasons[i] == want[t], (i, t, X.NAMES[int(reasons[i])])
            seen.add(t)
            if t == "s_ge_n":
                assert 0 < int.from_bytes(bytes(items[i]["s"]), "big") < N
        else:
            assert reasons[i] == X.OK
    assert seen == set(want)


@pytest.mark.parametrize("name", ["config2", "config3"])
def test_fixture_reasons_match_verdicts(name):
    items, arena, addrs, bitmap, _, ng = load_fixture(name)
    check_against_verdicts(items, arena, [addrs], [0] * ng, X.bits_of(bitmap, len(items)))


def adversarial_sets():
    """(label, items): the crafted recover vectors, the coordinate-edge vectors with the x = r + n forgeries"""
    return [("recover", A.recover_items(A.recover_vectors())), ("coordinate-edges", A.recover_items(A.coordinate_edge_vectors()))]


def test_adversarial_vectors_match_verdicts():
    for label, items in adversarial_sets():
        bits = X.bits_of(co.verify_batch(items), len(items))
        reasons, _ = check_against_verdicts(items, b"", None, None, bits)
        for v, r in zip(A.coordinate_edge_vectors() if label == "coordinate-edges" else A.recover_vectors(), reasons):
            assert (r == X.OK) == v.verdict, (label, v.tag)
            if v.tag.startswith("r+n forgery"):
                assert r in (X.SIGNER_MISMATCH, X.R_NOT_X), v.tag  # x - n lifts to another key, or is no abscissa
        assert X.NO_KEY in reasons or label != "recover"


def edge_frame_batch():
    edges, vs = load_edges()
    arena, items = bytearray(), []
    for r in edges:
        off = len(arena)
        wire = bytes.fromhex(r["wire"])
        arena.extend(wire)
        for g, kind in enumerate((X.KIND_WIRE, X.KIND_WIRE_SEAL)):
            items.append(wire_item(kind, off, len(wire), g))
    _, frames = sample_frames()
    for wire in frames:
        off = len(arena)
        arena.extend(wire)
        items.append(wire_item(X.KIND_WIRE, off, len(wire), 0))
    return np.concatenate(items), bytes(arena), vs


def test_edge_frames_against_the_wire_expectations():
    """the raw frames of tests/golden/proto_wire.json "edges": NEEDS_HOST and MALFORMED exactly where the wire tests expect
    status NEEDS_HOST or a structural rejection, OK exactly where they expect verdict 1"""
    from test_wire_edges import edge_expectation
    edges, vs = load_edges()
    items, arena, _ = edge_frame_batch()
    reasons, rec = X.explain_batch(items, arena, [vs.addr_array()], [0, 0])
    for i, r in enumerate(edges):
        for k, kind in enumerate((X.KIND_WIRE, X.KIND_WIRE_SEAL)):
            st, ok, want_rec = edge_expectation(r, kind)
            got = int(reasons[2 * i + k])
            assert (got == X.NEEDS_HOST) == (st == 1), r["name"]
            assert (got == X.OK) == ok, (r["name"], X.NAMES[got])
            if want_rec is None:
                assert got in (X.NEEDS_HOST, X.MALFORMED), (r["name"], X.NAMES[got])
            elif got in (X.OK, X.SIGNER_MISMATCH, X.NOT_VALIDATOR):
                assert bytes(rec[2 * i + k]) == want_rec, r["name"]
    assert {X.OK, X.NEEDS_HOST, X.MALFORMED} <= set(int(x) for x in reasons)


def test_emulation_agrees_with_the_reference(emul_explain):
    """explain_item of the csrc headers, byte for byte (reasons and recovered addresses), on every set above"""
    sets = [every_reason_batch()[:4]]
    items, arena, vs = edge_frame_batch()
    sets.append((items, arena, [vs.addr_array()], [0, 0]))
    for _, its in adversarial_sets():
        sets.append((its, b"", None, None))
    items, arena, addrs, _, tags, ng = load_fixture("config2")
    sets.append((items, arena, [addrs], [0] * ng))
    # config 3: its rejected items and a stride of the accepted ones
    items, arena, addrs, bitmap, _, ng = load_fixture("config3")
    bits = X.bits_of(bitmap, len(items))
    pick = np.nonzero(~bits | (np.arange(len(items)) % 97 == 0))[0]
    sets.append((items[pick], arena, [addrs], [0] * ng))
    for items, arena, tables, gt in sets:
        want, want_rec = X.explain_batch(items, arena, tables, gt)
        got, got_rec = emul_batch(emul_explain, items, arena, tables, gt)
        bad = np.nonzero(got != want)[0]
        assert len(bad) == 0, [(int(i), X.NAMES[int(got[i])], X.NAMES[int(want[i])]) for i in bad[:10]]
        assert np.array_equal(got_rec, want_rec)
