"""Raw gossip frames on the device (IBFT_KIND_WIRE / IBFT_KIND_WIRE_SEAL, SURVEY.md §8f rank 2): the kernel parses the proto3
frame, cuts the signature TLV out to obtain PayloadNoSig, and verifies -- bit-exact against the oracle codec + verifier,
including non-canonical and mutated frames (which must come back as NEEDS_HOST, never as a guessed verdict)."""
import importlib
import random

import numpy as np
import pytest

import ibft_b200 as ib
from oracle import ibft_proto as ip
from test_emul import sample_frames, wire_expectation, wire_item
from test_wire_edges import edge_expectation, go_verdict, load_edges

pytestmark = pytest.mark.gpu


def test_raw_frames_batch(engine):
    vs, frames = sample_frames()
    members = set(vs.addrs[:5])                       # validator 5 signs correctly but is NOT in the table
    engine.set_validators(7, 1, np.frombuffer(b"".join(vs.addrs[:5]), np.uint8).reshape(5, 20), None)
    rnd = random.Random(9)
    for f in list(frames[:20]):
        for _ in range(6):
            b = bytearray(f)
            i = rnd.randrange(len(b))
            b[i] ^= 1 << rnd.randrange(8)
            frames.append(bytes(b))
    arena = bytearray()
    items, want = [], []
    for wire in frames:
        off = len(arena)
        arena.extend(wire)
        for kind in (ib.KIND_WIRE, ib.KIND_WIRE_SEAL):
            items.append(wire_item(kind, off, len(wire), 0 if kind == ib.KIND_WIRE else 1))
            want.append(wire_expectation(wire, kind, members))
    items = np.concatenate(items).view(ib.ITEM_DTYPE)
    groups = engine.groups(2, slot=7)
    bitmap, results, _ = engine.verify_batch(items, bytes(arena) or b"\x00", groups)
    status = engine.last_item_status(len(items))
    bits = np.unpackbits(bitmap.view(np.uint8), bitorder="little")[: len(items)]
    for i, (st, ok) in enumerate(want):
        assert (int(status[i]), bool(bits[i])) == (st, ok), (i, frames[i // 2].hex())
    # quorum kernels resolve the signer of a raw frame from the frame itself
    for g in (0, 1):
        voters = set()
        for i, (st, ok) in enumerate(want):
            if ok and int(items[i]["group"]) == g:
                from oracle import ibft_proto as ip
                voters.add(ip.decode_ibft_message(frames[i // 2]).from_)
        assert int(results[g]["n_distinct"]) == len(voters) and int(results[g]["n_valid"]) == sum(1 for i, (st, ok) in enumerate(want) if ok and int(items[i]["group"]) == g)
        assert bool(results[g]["has_quorum"]) == (len(voters) >= 2 * 5 // 3 + 1)
    assert sum(1 for st, _ in want if st == 1) > 20 and sum(1 for _, ok in want if ok) > 30


# ------------------------------------------------------------------------- edge frames (tests/golden/proto_wire.json "edges")
def edge_batch(edges):
    """every edge frame at arena offsets 0..7 mod 8, as a KIND_WIRE item (group 0) and a KIND_WIRE_SEAL item (group 1)"""
    arena = bytearray()
    items, want = [], []
    for shift in range(8):
        for r in edges:
            wire = bytes.fromhex(r["wire"])
            arena.extend(b"\xee" * ((shift - len(arena)) % 8))
            off = len(arena)
            arena.extend(wire)
            for g, kind in enumerate((ib.KIND_WIRE, ib.KIND_WIRE_SEAL)):
                items.append(wire_item(kind, off, len(wire), g))
                want.append(edge_expectation(r, kind))
    return np.concatenate(items).view(ib.ITEM_DTYPE), bytes(arena), want


def check_edge_batch(eng, vs, with_recovered=True):
    edges, _ = load_edges()
    items, arena, want = edge_batch(edges)
    eng.set_validators(8, 100, vs.addr_array(), None)
    groups = eng.groups(2, slot=8)
    bitmap, results, recovered = eng.verify_batch(items, arena, groups, want_recovered=with_recovered)
    status = eng.last_item_status(len(items))
    bits = np.unpackbits(bitmap.view(np.uint8), bitorder="little")[: len(items)]
    for i, (st, ok, rec) in enumerate(want):
        assert (int(status[i]), bool(bits[i])) == (st, ok), (i, edges[(i // 2) % len(edges)]["name"], int(items[i]["payload_off"]) % 8)
        if with_recovered and rec is not None:
            assert bytes(recovered[i]) == rec, (i, edges[(i // 2) % len(edges)]["name"])
    # k_quorum_mark resolves each frame's signer with the same walk (item_signer): every valid item counts, one distinct signer
    for g in (0, 1):
        n_ok = sum(1 for i, (_, ok, _) in enumerate(want) if ok and int(items[i]["group"]) == g)
        assert n_ok > 0 and int(results[g]["n_valid"]) == n_ok and int(results[g]["n_distinct"]) == 1
        assert not results[g]["has_quorum"]                 # 1 of 4 validators
    return items, arena, bitmap


def test_edge_frames_every_alignment(engine):
    """the edge frames at every arena offset mod 8 on all four recover kernels: status, verdict, recovered address, quorum"""
    _, vs = load_edges()
    check_edge_batch(engine, vs)


def test_edge_frames_auto_and_key_cache_engines():
    """the same frames through the AUTO kernel selection, and through a key-registry engine once the signer's key is known (the
    known-key pass sees the frames first)"""
    _, vs = load_edges()
    for key_cache in (False, True):
        eng = ib.Engine(device=0, max_items=1 << 14, max_payload_bytes=1 << 22, max_groups=8, max_table_slots=16, max_validators=64,
                        key_cache=key_cache)
        try:
            items, arena, bm1 = check_edge_batch(eng, vs, with_recovered=not key_cache)
            if key_cache:
                assert eng.refresh_key_tables() == 1
                bm2, _, _ = eng.verify_batch(items, arena, eng.groups(2, slot=8))
                assert np.array_equal(bm1, bm2)
                check_edge_batch(eng, vs, with_recovered=False)
        finally:
            eng.close()


def test_edge_frames_host_fallback_reaches_go_verdict():
    """GpuVerifier in raw-frame mode: every edge frame the device hands back (non-canonical, nested 13 or 14 levels, negative
    type) is decided on the host by the protobuf-go re-marshal, and every verdict is protobuf-go's"""
    host = importlib.import_module("go-ibft_b200.host")
    edges, vs = load_edges()
    params = host.EngineParams(0, 1 << 12, 1 << 22, 8, 8, 64, 0)
    c = host.HostContext("gpu", {"is_proposer": lambda a, h, r: False}, b"", params)
    try:
        c.set_wire_frames(True)
        assert c.set_validators(100, vs.addrs, vs.powers) == 0
        c.set_state(100, 3)
        handed = 0
        for r in edges:
            wire = bytes.fromhex(r["wire"])
            # IsValidValidator also asks for the validators at the frame's own height: the table is resident for height 100 only
            at_100 = r["go_parses"] and ip.decode_ibft_message(wire).view is not None and ip.decode_ibft_message(wire).view.height == 100
            assert c.is_valid_validator(wire) == (go_verdict(r, ib.KIND_WIRE) and at_100), r["name"]
            before, handed = handed, c.gpu_frames_handed_back()
            if r["go_parses"] and edge_expectation(r, ib.KIND_WIRE)[0] == 1 and len(ip.decode_ibft_message(wire).signature) == 65:
                assert handed == before + 1, r["name"]
        deep = [r for r in edges if r["name"].startswith("nesting_levels_14")]
        assert deep and all(c.is_valid_validator(bytes.fromhex(r["wire"])) for r in deep)
    finally:
        c.close()
