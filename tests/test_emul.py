"""Host emulation of the DEVICE arithmetic (the very csrc/*.cuh headers, portable path) against the oracle.

Runs on a CPU-only box: it validates the algorithms the kernels use -- lazy-reduced field arithmetic, GLV split,
Booth digits, the group law with its exceptional cases, Keccak, address derivation -- before any GPU time is spent.
The PTX carry-chain multipliers themselves are covered on the GPU by test_gpu_primitives.py."""
import ctypes
import os
import random

import numpy as np
import pytest

from oracle import coracle as co
from oracle import secp256k1 as ec
from oracle.keccak import keccak256

import adversarial as A

P, N = ec.P, ec.N
LAM = 0x5363AD4CC05C30E0A5261C028812645A122E22EA20816678DF02967C1B23BD72
EDGE = [0, 1, 2, P - 1, P, P + 1, 2**256 - 1, 2**255, N, N - 1, 2**32, 2**32 + 977, 2**256 - 2**32 - 978, (1 << 224) - 1]


def B(b):
    return (ctypes.c_uint8 * len(b)).from_buffer_copy(b)


def dbg(E, op, a, b=0, c=None, outn=32):
    out = (ctypes.c_uint8 * 64)()
    rc = E.emul_debug_op(op, B(a.to_bytes(32, "big")), B(b.to_bytes(32, "big")), B(c) if c else None, out)
    return rc, bytes(out)[:outn]


def test_field_and_scalar_ops(emul):
    rnd = random.Random(3)
    vals = EDGE + [rnd.getrandbits(256) for _ in range(150)]
    for a in vals:
        for b in rnd.sample(vals, 4) + EDGE[:7]:
            assert int.from_bytes(dbg(emul, 1, a, b)[1], "big") == a * b % P
            assert int.from_bytes(dbg(emul, 8, a, b)[1], "big") == (a + b) % P
            assert int.from_bytes(dbg(emul, 9, a, b)[1], "big") == (a - b) % P
            assert int.from_bytes(dbg(emul, 5, a, b)[1], "big") == a * b % N
        assert int.from_bytes(dbg(emul, 2, a)[1], "big") == a * a % P
    for a in vals[:40]:
        assert int.from_bytes(dbg(emul, 3, a)[1], "big") == (pow(a % P, -1, P) if a % P else 0)
        assert int.from_bytes(dbg(emul, 6, a)[1], "big") == (pow(a % N, -1, N) if a % N else 0)
        assert int.from_bytes(dbg(emul, 4, a)[1], "big") == pow(a % P, (P + 1) // 4, P)


def test_glv_split(emul):
    rnd = random.Random(4)
    ks = [0, 1, 2, N - 1, N - 2, LAM, N - LAM, (N + 1) // 2, N // 2, 2**128, 2**128 - 1, 2**255] + [rnd.getrandbits(256) % N for _ in range(1500)]
    for k in ks:
        _, o = dbg(emul, 10, k, outn=64)
        k1 = int.from_bytes(o[0:20], "little") * (-1 if o[20] else 1)
        k2 = int.from_bytes(o[24:44], "little") * (-1 if o[44] else 1)
        assert (k1 + k2 * LAM) % N == k and abs(k1) < 2**129 and abs(k2) < 2**129


def ecm(E, a, b, pt):
    rc, o = dbg(E, 7, a, b, pt[0].to_bytes(32, "big") + pt[1].to_bytes(32, "big"), 64)
    return None if rc else (int.from_bytes(o[:32], "big"), int.from_bytes(o[32:], "big"))


def test_ecmult_including_exceptional_cases(emul):
    rnd = random.Random(5)
    G = ec.G
    pt = ec.point_mul(12345, G)
    cases = [(0, 0), (1, 0), (0, 1), (2, 0), (0, 2), (N - 1, 0), (0, N - 1), (1, N - 1), (5, 7), (N - 1, N - 1), (LAM, 0), (0, LAM), (N - LAM, LAM)]
    cases += [(rnd.getrandbits(256) % N, rnd.getrandbits(256) % N) for _ in range(12)]
    for a, b in cases:
        assert ecm(emul, a, b, pt) == ec.point_add(ec.point_mul(a, G), ec.point_mul(b, pt))
    # P chosen so that partial sums collide with table entries: doubling / cancellation branches of the adders
    for p2 in [G, ec.point_neg(G), ec.point_mul(2, G), ec.point_mul(LAM, G), ec.point_mul(N - LAM, G), ec.point_mul(8, G), ec.point_mul(N - 8, G)]:
        for a, b in [(1, 1), (1, N - 1), (2, N - 1), (N - 2, 1), (8, 1), (8, N - 1), (3, 5), (LAM, 1), (1, LAM), (N - 1, N - 1), (7, 1), (16, N - 2)]:
            assert ecm(emul, a, b, p2) == ec.point_add(ec.point_mul(a, G), ec.point_mul(b, p2)), (a, b)


def emul_item(E, item, arena=b""):
    out = (ctypes.c_uint8 * 20)()
    a = np.frombuffer(arena, np.uint8) if arena else np.zeros(1, np.uint8)
    ok = E.emul_verify_item(item.ctypes.data_as(ctypes.c_void_p), a.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(len(arena)), out)
    return bool(ok), bytes(out)


def test_recover_valid_highs_and_corrupted(emul):
    import workloads as wl
    rnd = random.Random(6)
    for i in range(60):
        d = rnd.getrandbits(256) % (N - 1) + 1
        dig = keccak256(bytes([i]) * 3)
        sig = wl.sign(d, dig, low_s=bool(i & 1))
        if i % 3 == 0:
            s = int.from_bytes(sig[32:64], "big")
            sig = sig[:32] + (N - s).to_bytes(32, "big") + bytes([sig[64] ^ 1])
        addr = co.ecrecover_address(dig, sig)
        assert emul_item(emul, wl.make_item(sig, addr, 0, dig)) == (True, addr)
        bad = bytearray(sig)
        bad[rnd.randrange(64)] ^= 1 << rnd.randrange(8)
        exp = co.ecrecover_address(dig, bytes(bad))
        assert emul_item(emul, wl.make_item(bytes(bad), addr, 0, dig)) == (exp == addr, exp or bytes(20))
        ph = keccak256(bytes([i, 1]))
        sg = wl.sign(d, wl.seal_digest(ph))
        assert emul_item(emul, wl.make_item(sg, addr, 2, ph)) == (True, addr)


def test_config2_fixture_bit_exact(emul):
    d = np.load(os.path.join(os.path.dirname(__file__), "golden", "config2.npz"))
    items = np.ascontiguousarray(d["items"]).view(co.ITEM_DTYPE).reshape(-1)
    arena = d["arena"].tobytes()
    members = {bytes(a) for a in d["addrs"]}
    bm = d["bitmap"]
    for i in range(len(items)):
        ok, _ = emul_item(emul, items[i:i + 1], arena)
        ok = ok and bytes(items[i]["signer"]) in members
        assert ok == bool((bm[i >> 5] >> (i & 31)) & 1), (i, d["tags"][i])


# ----------------------------------------------------------------------------------------------- raw gossip frames
WIRE_MAX_DEPTH = 12  # IBFT_WIRE_MAX_DEPTH of csrc/verify_core.cuh: nesting levels the device walks


def frame_shape(m, level: int = 1):
    """(nesting levels, [type of every IbftMessage]) of a decoded frame; the root is level 1, every present sub-message one more"""
    from oracle import ibft_proto as ip
    depth, types = level + (m.view is not None), [m.type]
    p = m.payload
    if p is None:
        return depth, types
    depth = max(depth, level + 1)
    inner = []
    if isinstance(p, ip.PrePrepareMessage):
        if p.proposal is not None:
            depth = max(depth, level + 2)
        if p.certificate is not None:
            depth = max(depth, level + 2)
            inner = p.certificate.round_change_messages
    elif isinstance(p, ip.RoundChangeMessage):
        if p.last_prepared_proposal is not None:
            depth = max(depth, level + 2)
        pc = p.latest_prepared_certificate
        if pc is not None:
            depth = max(depth, level + 2)
            inner = ([pc.proposal_message] if pc.proposal_message is not None else []) + list(pc.prepare_messages or [])
    for x in inner:
        d, t = frame_shape(x, level + 3)
        depth, types = max(depth, d), types + t
    return depth, types


def wire_expectation(wire: bytes, kind: int, members):
    """(status, verdict) the device must produce for a KIND_WIRE / KIND_WIRE_SEAL item, derived from the oracle codec, which
    decodes the way protobuf-go does (canonical <=> decode + encode reproduces the frame), and the oracle verifier.  A frame
    protobuf-go cannot decode, or one it would re-encode differently, comes back NEEDS_HOST.  So do exactly two kinds of
    canonical frames, which the device hands back on purpose: one nested deeper than IBFT_WIRE_MAX_DEPTH, and one with a
    negative `type` anywhere in it (the canonical 10-byte form of an int32 enum below zero)."""
    import workloads as wl
    from oracle import ibft_proto as ip
    try:
        m = ip.decode_ibft_message(wire)
    except (ip.DecodeError, RecursionError):
        return 1, False
    if ip.encode_ibft_message(m) != wire:
        return 1, False           # not canonical: the device hands the frame back, it never guesses
    levels, types = frame_shape(m)
    if levels > WIRE_MAX_DEPTH or min(types) < 0:
        return 1, False           # canonical, but one of the two allowed conservative hand-backs
    if len(m.from_) != 20:
        return 0, False
    if kind == 3:
        if m.view is None or len(m.signature) != 65:
            return 0, False
        addr = co.ecrecover_address(co.keccak256(m.payload_no_sig()), m.signature)
    else:
        if m.type != ip.COMMIT or not isinstance(m.payload, ip.CommitMessage) or len(m.payload.proposal_hash) != 32 or len(m.payload.committed_seal) != 65:
            return 0, False
        addr = co.ecrecover_address(wl.seal_digest(m.payload.proposal_hash), m.payload.committed_seal)
    return 0, addr == m.from_ and (members is None or m.from_ in members)


def wire_item(kind, off, ln, group=0):
    it = np.zeros(1, dtype=co.ITEM_DTYPE)
    it["kind"], it["payload_off"], it["payload_len"], it["group"] = kind, off, ln, group
    return it


def sample_frames():
    import workloads as wl
    from oracle import ibft_proto as ip
    vs = wl.ValidatorSet(77, 6)
    ph = co.keccak256(b"blk")
    frames = []
    for i in range(6):
        for t, payload in ((ip.PREPARE, ip.PrepareMessage(ph)), (ip.COMMIT, ip.CommitMessage(ph, wl.sign(vs.keys[i], wl.seal_digest(ph))))):
            for view in (ip.View(1_000_000, i), ip.View(0, 0), ip.View(5, 0)):
                m = ip.IbftMessage(view, vs.addrs[i], b"", t, payload)
                m.signature = wl.sign(vs.keys[i], co.keccak256(m.payload_no_sig()))
                frames.append(ip.encode_ibft_message(m))
    # nested frames (SURVEY.md §8f rank 2): the signed bytes of PREPREPARE / ROUND_CHANGE include their certificates
    def signed(m, k):
        m.signature = wl.sign(vs.keys[k], co.keccak256(m.payload_no_sig()))
        return m
    raw = bytes(range(200))
    v0, v1 = ip.View(7, 0), ip.View(7, 1)
    pp0 = signed(ip.IbftMessage(v0, vs.addrs[0], b"", ip.PREPREPARE, ip.PrePrepareMessage(ip.Proposal(raw, 0), ph, None)), 0)
    preps = [signed(ip.IbftMessage(v0, vs.addrs[i], b"", ip.PREPARE, ip.PrepareMessage(ph)), i) for i in range(1, 5)]
    pc = ip.PreparedCertificate(pp0, preps)
    rcs = [signed(ip.IbftMessage(v1, vs.addrs[i], b"", ip.ROUND_CHANGE, ip.RoundChangeMessage(ip.Proposal(raw, 0), pc if i % 2 else None)), i) for i in range(5)]
    rcs.append(signed(ip.IbftMessage(v1, vs.addrs[5], b"", ip.ROUND_CHANGE, ip.RoundChangeMessage(None, ip.PreparedCertificate(None, None))), 5))
    rcs.append(signed(ip.IbftMessage(v1, vs.addrs[2], b"", ip.ROUND_CHANGE, ip.RoundChangeMessage(None, ip.PreparedCertificate(ip.IbftMessage(), [ip.IbftMessage()]))), 2))
    pp1 = signed(ip.IbftMessage(v1, vs.addrs[1], b"", ip.PREPREPARE, ip.PrePrepareMessage(ip.Proposal(raw, 1), ph, ip.RoundChangeCertificate(rcs[:4]))), 1)
    pp1_forged = ip.IbftMessage(v1, vs.addrs[1], pp1.signature, ip.PREPREPARE, ip.PrePrepareMessage(ip.Proposal(raw, 1), ph, ip.RoundChangeCertificate(rcs[1:4])))
    frames += [ip.encode_ibft_message(x) for x in [pp0, pp1, pp1_forged] + rcs]
    m = ip.IbftMessage(ip.View(3, 1), vs.addrs[0], b"", ip.COMMIT, ip.CommitMessage(ph, wl.sign(vs.keys[1], wl.seal_digest(ph))))  # seal by someone else
    m.signature = wl.sign(vs.keys[0], co.keccak256(m.payload_no_sig()))
    frames.append(ip.encode_ibft_message(m))
    extra = [
        ip.IbftMessage(None, vs.addrs[0], b"\x01" * 65, ip.PREPARE, ip.PrepareMessage(ph)),                      # nil view
        ip.IbftMessage(ip.View(1, 1), vs.addrs[0], b"", ip.PREPARE, ip.PrepareMessage(ph)),                        # no signature
        ip.IbftMessage(ip.View(1, 1), b"short", b"\x01" * 65, ip.PREPARE, ip.PrepareMessage(ph)),                  # from != 20 bytes
        ip.IbftMessage(ip.View(1, 1), vs.addrs[0], b"\x01" * 64, ip.COMMIT, ip.CommitMessage(ph, b"\x02" * 64)),   # 64-byte sig / seal
        ip.IbftMessage(ip.View(1, 1), vs.addrs[0], b"\x01" * 65, ip.PREPARE, ip.CommitMessage(ph, b"\x02" * 65)),  # type/payload mismatch
        ip.IbftMessage(ip.View(1, 1), vs.addrs[0], b"\x01" * 65, ip.COMMIT, None),                                 # no payload
        ip.IbftMessage(ip.View(1, 1), vs.addrs[0], b"\x01" * 65, ip.PREPREPARE, ip.PrePrepareMessage(ip.Proposal(b"x", 1), ph, None)),  # nested payload, bad signature
        ip.IbftMessage(ip.View(1, 1), vs.addrs[0], b"\x01" * 65, ip.ROUND_CHANGE, ip.RoundChangeMessage(None, None)),
        ip.IbftMessage(ip.View(1, 1), vs.addrs[0], b"\x01" * 65, ip.PREPARE, ip.PrepareMessage()),                 # empty payload message
    ]
    frames += [ip.encode_ibft_message(m) for m in extra]
    # hand-made non-canonical encodings of a valid frame
    good = frames[0]
    frames += [good + b"\x48\x01",                      # unknown field 9
               good[:2] + b"\x80\x00"[:0] + good[2:],   # (identity) control
               b"\x12\x00" + good,                      # empty `from` ahead, fields out of order
               good.replace(b"\x20\x01", b"\x20\x81\x00", 1),  # non-minimal varint for `type`
               good[::-1], b"", b"\x0a"]
    return vs, frames


def test_raw_frame_kinds_canonical_and_mutated(emul):
    vs, frames = sample_frames()
    members = set(vs.addrs)
    rnd = random.Random(8)
    mutated = []
    for f in frames[:24] + frames[36:50]:
        for _ in range(12):
            b = bytearray(f)
            op = rnd.randrange(4)
            if op == 0 and b:
                b[rnd.randrange(len(b))] ^= 1 << rnd.randrange(8)
            elif op == 1 and b:
                del b[rnd.randrange(len(b))]
            elif op == 2:
                b.insert(rnd.randrange(len(b) + 1), rnd.randrange(256))
            else:
                i = rnd.randrange(len(b) + 1)
                b[i:i] = bytes([rnd.choice([0x0a, 0x12, 0x1a, 0x20, 0x32, 0x3a, 0x00, 0x80])])
            mutated.append(bytes(b))
    n_needs_host = n_true = 0
    for wire in frames + mutated:
        for kind in (3, 4):
            want_status, want_ok = wire_expectation(wire, kind, None)
            out = (ctypes.c_uint8 * 20)()
            arena = np.frombuffer(wire, np.uint8) if wire else np.zeros(1, np.uint8)
            rc = emul.emul_verify_item(wire_item(kind, 0, len(wire)).ctypes.data_as(ctypes.c_void_p), arena.ctypes.data_as(ctypes.c_void_p),
                                       ctypes.c_size_t(len(wire)), out)
            assert (1 if rc == -1 else 0, rc == 1) == (want_status, want_ok), (wire.hex(), kind, rc)
            n_needs_host += want_status
            n_true += want_ok
    assert n_true >= 40 and n_needs_host >= 40


# ------------------------------------------------------------------------ level-structured group law (four-lane kernel)
def ecm_levels(E, a, b, pt):
    out = (ctypes.c_uint8 * 64)()
    rc = E.emul_ecmult_levels(B(a.to_bytes(32, "big")), B(b.to_bytes(32, "big")), B(pt[0].to_bytes(32, "big") + pt[1].to_bytes(32, "big")), out)
    o = bytes(out)
    return None if rc else (int.from_bytes(o[:32], "big"), int.from_bytes(o[32:], "big"))


def test_level_structured_ecmult_matches_oracle(emul):
    """secp_ec.cuh jac_double_x / jac_add_affine_x (the product LEVELS exec_quad distributes over four lanes), run with the
    serial executor: same exceptional-case coverage as the one-thread routine."""
    rnd = random.Random(15)
    G = ec.G
    pt = ec.point_mul(54321, G)
    cases = [(0, 0), (1, 0), (0, 1), (2, 0), (0, 2), (N - 1, 0), (0, N - 1), (1, N - 1), (5, 7), (N - 1, N - 1), (LAM, 0), (0, LAM), (N - LAM, LAM)]
    cases += [(rnd.getrandbits(256) % N, rnd.getrandbits(256) % N) for _ in range(12)]
    for a, b in cases:
        assert ecm_levels(emul, a, b, pt) == ec.point_add(ec.point_mul(a, G), ec.point_mul(b, pt))
    for p2 in [G, ec.point_neg(G), ec.point_mul(2, G), ec.point_mul(LAM, G), ec.point_mul(N - LAM, G), ec.point_mul(8, G), ec.point_mul(N - 8, G)]:
        for a, b in [(1, 1), (1, N - 1), (2, N - 1), (N - 2, 1), (8, 1), (8, N - 1), (3, 5), (LAM, 1), (1, LAM), (N - 1, N - 1), (7, 1), (16, N - 2)]:
            assert ecm_levels(emul, a, b, p2) == ec.point_add(ec.point_mul(a, G), ec.point_mul(b, p2)), (a, b)


def test_level_structured_recover_config2(emul):
    d = np.load(os.path.join(os.path.dirname(__file__), "golden", "config2.npz"))
    items = np.ascontiguousarray(d["items"]).view(co.ITEM_DTYPE).reshape(-1)
    arena = d["arena"].tobytes()
    a = np.frombuffer(arena, np.uint8)
    for i in range(0, len(items), 3):
        o1, o2 = (ctypes.c_uint8 * 20)(), (ctypes.c_uint8 * 20)()
        it = items[i:i + 1]
        r1 = emul.emul_verify_item(it.ctypes.data_as(ctypes.c_void_p), a.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(len(arena)), o1)
        r2 = emul.emul_verify_item_levels(it.ctypes.data_as(ctypes.c_void_p), a.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(len(arena)), o2)
        assert (r1, bytes(o1)) == (r2, bytes(o2)), i


# ------------------------------------------------------------------ split pipeline (helper / chain warps of k_recover_split)
def both_paths(E, it, arena_np, arena_len):
    o1, o2 = (ctypes.c_uint8 * 20)(), (ctypes.c_uint8 * 20)()
    r1 = E.emul_verify_item(it.ctypes.data_as(ctypes.c_void_p), arena_np.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(arena_len), o1)
    r2 = E.emul_verify_item_split(it.ctypes.data_as(ctypes.c_void_p), arena_np.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(arena_len), o2)
    # ... and through the split pipeline with the level-structured (four-lane) chain: must agree with the one-lane chain
    o3 = (ctypes.c_uint8 * 20)()
    r3 = E.emul_verify_item_qsplit(it.ctypes.data_as(ctypes.c_void_p), arena_np.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(arena_len), o3)
    assert (r3, bytes(o3)) == (r2, bytes(o2))
    return (r1, bytes(o1)), (r2, bytes(o2))


def test_split_pipeline_isomorphic_curve_and_comb(emul):
    """k_recover_split's arithmetic: u2*R on the isomorphic curve E' (no square root on the chain), u1*G as a per-position comb,
    map back with Z' * y.  Must give the very same verdict and recovered address as the one-thread pipeline."""
    import workloads as wl
    rnd = random.Random(21)
    zero = np.zeros(1, np.uint8)
    for i in range(40):
        d = rnd.getrandbits(256) % (N - 1) + 1
        dig = keccak256(bytes([i, 7]))
        sig = wl.sign(d, dig, low_s=bool(i & 1))
        addr = co.ecrecover_address(dig, sig)
        a, b = both_paths(emul, wl.make_item(sig, addr, 0, dig), zero, 0)
        assert a == b == (1, addr)
        bad = bytearray(sig)
        bad[rnd.randrange(65)] ^= 1 << rnd.randrange(8)
        a, b = both_paths(emul, wl.make_item(bytes(bad), addr, 0, dig), zero, 0)
        assert a == b
    # z = 0 (u1 = 0: the generator part is the point at infinity) and high-s / v = 1 variants
    d = 0xC0FFEE
    sig = wl.sign(d, bytes(32))
    addr = co.ecrecover_address(bytes(32), sig)
    a, b = both_paths(emul, wl.make_item(sig, addr, 0, bytes(32)), zero, 0)
    assert a == b == (1, addr)
    # r that is not an abscissa, r = 0, s = 0, r >= n, v = 2
    for r, s, v in [(5, 1, 0), (0, 1, 0), (1, 0, 0), (N, 1, 0), (1, N, 1), (ec.G[0], 1, 2), (ec.G[0], 1, 0), (ec.G[0], N - 1, 1)]:
        sg = r.to_bytes(32, "big") + s.to_bytes(32, "big") + bytes([v])
        a, b = both_paths(emul, wl.make_item(sg, bytes(20), 0, keccak256(b"x")), zero, 0)
        assert a == b, (r, s, v)


def test_split_pipeline_config2_fixture(emul):
    d = np.load(os.path.join(os.path.dirname(__file__), "golden", "config2.npz"))
    items = np.ascontiguousarray(d["items"]).view(co.ITEM_DTYPE).reshape(-1)
    arena = d["arena"].tobytes()
    a_np = np.frombuffer(arena, np.uint8)
    for i in range(0, len(items), 5):
        a, b = both_paths(emul, items[i:i + 1], a_np, len(arena))
        assert a == b, i


# --------------------------------------------------------------- verification against a known (previously recovered) key
def test_verify_known_key_is_equivalent_to_recovering_that_key(emul):
    """ecdsa_verify_known(Q) accepts exactly when the recover path yields the key Q (not merely the same address): valid
    signatures (low and high s, both recovery ids), corrupted ones, a flipped recovery id, another signer's key."""
    import workloads as wl
    rnd = random.Random(31)
    zero = np.zeros(1, np.uint8)

    def run(item, key):
        rk = ctypes.c_int(0)
        key64 = key[0].to_bytes(32, "big") + key[1].to_bytes(32, "big")
        ok = emul.emul_verify_item_known(item.ctypes.data_as(ctypes.c_void_p), zero.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(0), B(key64),
                                         ctypes.byref(rk))
        return ok, rk.value

    accepted = 0
    for i in range(24):
        d = rnd.getrandbits(256) % (N - 1) + 1
        Q = ec.point_mul(d, ec.G)
        dig = keccak256(bytes([i, 9]))
        sig = wl.sign(d, dig, low_s=bool(i & 1))
        if i % 3 == 0:  # the high-s twin with the other recovery id is the same signature of the same key
            s = int.from_bytes(sig[32:64], "big")
            sig = sig[:32] + (N - s).to_bytes(32, "big") + bytes([sig[64] ^ 1])
        addr = co.ecrecover_address(dig, sig)
        assert run(wl.make_item(sig, addr, 0, dig), Q) == (1, 1)
        accepted += 1
        # committed-seal kind goes through the same digest resolution
        ph = keccak256(bytes([i, 3]))
        sg = wl.sign(d, wl.seal_digest(ph))
        assert run(wl.make_item(sg, addr, 2, ph), Q) == (1, 1)
        # flipped recovery id: recovery yields ANOTHER key -> reject
        flipped = sig[:64] + bytes([sig[64] ^ 1])
        ok, rk = run(wl.make_item(flipped, addr, 0, dig), Q)
        assert (ok, rk) == (0, 0)
        # random corruption: accept <=> recover yields Q
        bad = bytearray(sig)
        bad[rnd.randrange(64)] ^= 1 << rnd.randrange(8)
        ok, rk = run(wl.make_item(bytes(bad), addr, 0, dig), Q)
        assert ok == rk
        # somebody else's key
        Q2 = ec.point_mul(d + 1, ec.G)
        assert run(wl.make_item(sig, addr, 0, dig), Q2) == (0, 0)
    assert accepted == 24
    # out-of-range scalars
    for r, s, v in [(0, 1, 0), (1, 0, 0), (N, 1, 0), (1, N, 1), (ec.G[0], 1, 2)]:
        sg = r.to_bytes(32, "big") + s.to_bytes(32, "big") + bytes([v])
        assert run(wl.make_item(sg, bytes(20), 0, keccak256(b"x")), ec.G)[0] == 0


def run_known(E, item, key):
    """(verdict of ecdsa_verify_known against `key`, 1 when the recover path yields exactly that key); -2 = the chain / helper
    cut of k_verify_split disagreed with the one-thread verification"""
    zero = np.zeros(1, np.uint8)
    rk = ctypes.c_int(0)
    key64 = key[0].to_bytes(32, "big") + key[1].to_bytes(32, "big")
    ok = E.emul_verify_item_known(item.ctypes.data_as(ctypes.c_void_p), zero.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(0), B(key64),
                                  ctypes.byref(rk))
    return ok, rk.value


def test_verify_known_comb_edge_digits_and_colliding_points(emul):
    """The comb walk of ecdsa_verify_known on CONSTRUCTED scalars (tests/adversarial.py known_vectors): half-scalars whose 8-bit
    Booth digits sit on the window edges, u1 = 0 (zero digest), and keys that make the generator stream and the key stream meet
    in the adder (Q = G, -G, lambda*G, -lambda*G, 2G: P + P, P - P and a running sum at infinity).  Every signature is valid by
    construction, so the verification must accept and the recover path must yield exactly Q."""
    import workloads as wl
    built = 0
    for v in A.known_vectors():
        Q = A.known_key(v.key_index)
        item = wl.make_item(v.sig, A.known_addr(v.key_index), 0, v.digest)
        assert run_known(emul, item, Q) == (1, 1), v
        # the same signature against ANOTHER key never verifies, and agrees with "does recovery yield that key"
        assert run_known(emul, item, ec.point_mul(A.KNOWN_KEYS[v.key_index] + 7, ec.G)) == (0, 0), v
        built += 1
    assert built >= 60


def test_key_comb_table_entries_are_the_stated_multiples(emul):
    """build_keytab_pos (what k_build_keytabs runs per (validator, position)): entry m-1 of position j is m * 2^(8j) * Q, affine and
    canonical -- checked against the big-int oracle for the first, a middle and the last position."""
    assert emul.emul_keytab_positions() == 17
    d = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF % N
    Q = ec.point_mul(d, ec.G)
    key64 = Q[0].to_bytes(32, "big") + Q[1].to_bytes(32, "big")
    for pos in (0, 7, 16):
        out = ctypes.create_string_buffer(128 * 64)
        emul.emul_keytab_pos(B(key64), pos, out)
        base = ec.point_mul(pow(2, 8 * pos, N), Q)
        P = base
        for m in range(1, 129):
            e = out.raw[64 * (m - 1): 64 * m]
            assert (int.from_bytes(e[:32], "big"), int.from_bytes(e[32:], "big")) == P, (pos, m)
            P = ec.point_add(P, base)


# ------------------------------------------------- crafted exceptional-case vectors (tests/adversarial.py), every pipeline
BR = dict(ADD_DBL=0, ADD_NEG=1, ADD_INF=2, XADD_DBL=3, XADD_NEG=4, XADD_INF=5)  # IBFT_BR_* of secp_fe.cuh
FINAL = 6  # counters of the split pipelines' final "+ u1 G" follow the overall ones


def branch_counts(E):
    out = (ctypes.c_ulonglong * 12)()
    assert E.emul_branch_counts(out) == FINAL
    return list(out)


def test_crafted_vectors_agree_with_the_c_oracle():
    """the expected values of tests/adversarial.py (big-int oracle) against the C oracle, once"""
    for v in A.recover_vectors():
        assert co.ecrecover_address(v.digest, v.sig) == v.addr, v.tag
        if v.key is not None:  # the vector computes what it was built for: u1 G + u2 R
            R = ec.lift_x(int.from_bytes(v.sig[:32], "big"), v.sig[64] ^ 0)
            if int.from_bytes(v.digest, "big") < N and "high-s" not in v.tag:
                assert v.key == ec.point_add(ec.point_mul(v.u[0], ec.G), ec.point_mul(v.u[1], R)), v.tag
    for v in A.known_vectors():
        Q = A.known_key(v.key_index)
        assert co.ecrecover_pubkey(v.digest, v.sig) == Q[0].to_bytes(32, "big") + Q[1].to_bytes(32, "big")
    for v in A.known_cancelling():
        assert co.ecrecover_address(v.digest, v.sig) != A.known_addr(v.key_index)
    tags = [v.tag for v in A.recover_vectors()]
    assert sum(t.startswith("final-add inf") for t in tags) >= 10 and sum("z=n" in t for t in tags) >= 4


PIPELINES = {  # entry point -> (branch counters that must show the crafted collisions)
    "emul_verify_item": ("ADD_DBL", "ADD_NEG", "ADD_INF"),
    "emul_verify_item_levels": ("XADD_DBL", "XADD_NEG", "XADD_INF"),
    "emul_verify_item_split": ("ADD_DBL", "ADD_NEG", "ADD_INF"),
    "emul_verify_item_qsplit": ("XADD_DBL", "XADD_NEG", "XADD_INF"),
}


@pytest.mark.parametrize("fn", sorted(PIPELINES))
def test_crafted_recover_vectors_on_every_pipeline(emul, fn):
    """Every crafted recover vector gives the oracle's verdict and recovered address (zero when recovery fails, e.g. Q = infinity)
    on the one-thread, level-structured (four-lane), split and four-lane split pipelines -- and the branch counters prove that the
    set reaches P + P, P - P and the accumulator at infinity, in the split pipelines' final add too."""
    zero = np.zeros(1, np.uint8)
    emul.emul_branch_reset()
    vecs = A.recover_vectors()
    for v in vecs:
        item = A.recover_items([v])
        out = (ctypes.c_uint8 * 20)()
        rc = getattr(emul, fn)(item.ctypes.data_as(ctypes.c_void_p), zero.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(0), out)
        assert (rc, bytes(out)) == (int(v.key is not None), v.addr or bytes(20)), v.tag
    c = branch_counts(emul)
    for name in PIPELINES[fn]:
        assert c[BR[name]] >= 1, (name, c)
    if "split" in fn:  # (the accumulator u2 R of the final add is never at infinity: 0 < u2 < n)
        for name in PIPELINES[fn][:2]:
            assert c[FINAL + BR[name]] >= 1, ("final add", name, c)


def test_crafted_known_key_vectors_and_variants(emul):
    """ecdsa_verify_known and its chain / helper cut on the crafted known-key set: every valid vector accepted (recovery yields Q),
    a misattributed one (key i presented as validator i + 1), a flipped recovery id and a cancelling u1 G + u2 Q rejected; the
    counters show P + P and P - P in the walk and P + P / infinity in the cut's final add."""
    import workloads as wl
    emul.emul_branch_reset()
    for v in A.known_vectors():
        Q = A.known_key(v.key_index)
        assert run_known(emul, wl.make_item(v.sig, A.known_addr(v.key_index), 0, v.digest), Q) == (1, 1)
        sig, j = A.misattributed(v)
        assert run_known(emul, wl.make_item(sig, A.known_addr(j), 0, v.digest), A.known_key(j)) == (0, 0)
        assert run_known(emul, wl.make_item(A.flipped(v), A.known_addr(v.key_index), 0, v.digest), Q) == (0, 0)
    for v in A.known_cancelling():
        assert run_known(emul, wl.make_item(v.sig, A.known_addr(v.key_index), 0, v.digest), A.known_key(v.key_index)) == (0, 0)
    c = branch_counts(emul)
    assert c[BR["ADD_DBL"]] >= 1 and c[BR["ADD_NEG"]] >= 1 and c[BR["ADD_INF"]] >= 1, c
    assert c[FINAL + BR["ADD_DBL"]] >= 1 and c[FINAL + BR["ADD_NEG"]] >= 1, c
