"""Raw gossip frames at protobuf's varint, enum, length and nesting edges (tests/edge_frames.py, with protobuf's answers in
tests/golden/proto_wire.json "edges"), on the CPU.

Every frame carries what protobuf-go answers for it: whether it decodes and is canonical, the Keccak-256 of its re-marshal and
of its PayloadNoSig, and whether a Go
node's IsValidValidator / IsValidCommittedSeal accept it.  Frames that decode come signed twice by a validator of the table:
over "frame minus the signature TLV" (the bytes the device hashes) and over protobuf-go's PayloadNoSig (the bytes go-ibft
hashes).  They differ exactly when the frame is not canonical, so a wrong "canonical" decision flips a verdict, not only a
status.  The oracle codec, the C++ host codec and the emulated device (the very csrc headers) must all give protobuf-go's
answers."""
import ctypes
import importlib
import json
import os

import numpy as np
import pytest

import workloads as wl
from oracle import coracle as co
from oracle import ibft_proto as ip
from edge_frames import EDGE_SEED, EDGE_VALIDATORS, EdgeFrames, signed_variants
from test_emul import WIRE_MAX_DEPTH, both_paths, frame_shape, wire_item

HERE = os.path.dirname(os.path.abspath(__file__))
KIND_WIRE, KIND_WIRE_SEAL = 3, 4
OK, NEEDS_HOST = 0, 1


def keccak_hex(b: bytes) -> str:
    return co.keccak256(b).hex()


def load_edges():
    """the fixture's rows, each with its frame rebuilt by tests/edge_frames.py (row["wire"], hex) and checked against the recorded
    Keccak-256; and the validator table"""
    d = json.load(open(os.path.join(HERE, "golden", "proto_wire.json")))
    assert d["edge_validators"] == [EDGE_SEED, EDGE_VALIDATORS]
    frames = EdgeFrames()
    bodies = dict(frames.bases())
    rows = []
    for r in d["edges"]:
        base, variant = r["name"].split("/")
        go_digest = bytes.fromhex(r["go_payload_no_sig_keccak"]) if r["go_parses"] else None
        wire = dict(signed_variants(bodies[base], frames.vs.keys[0], go_digest))[variant]
        assert keccak_hex(wire) == r["wire_keccak"], r["name"]
        rows.append(dict(r, wire=wire.hex()))
    return rows, frames.vs


def is_canonical(row) -> bool:
    return row["go_parses"] and row["go_canonical"]


def handed_back_on_purpose(row) -> bool:
    """the device's two allowed conservative hand-backs of a canonical frame: nested deeper than it walks, or a negative type"""
    return row["go_levels"] > WIRE_MAX_DEPTH or min(row["go_types"]) < 0


def go_verdict(row, kind) -> bool:
    """what a Go node decides for the frame (IsValidValidator for KIND_WIRE, IsValidCommittedSeal for KIND_WIRE_SEAL); every
    `from` in the fixture is a validator of the table"""
    if not row["go_parses"]:
        return False
    return row["go_sender_valid"] if kind == KIND_WIRE else row["go_seal_valid"]


def edge_expectation(row, kind):
    """(status, verdict, recovered address) the device must report for the frame as a KIND_WIRE / KIND_WIRE_SEAL item.  The
    recovered address is None where the device does no arithmetic (hand-back or structurally invalid item)."""
    if not is_canonical(row) or handed_back_on_purpose(row):
        return NEEDS_HOST, False, None
    m = ip.decode_ibft_message(bytes.fromhex(row["wire"]))
    if len(m.from_) != 20:
        return OK, False, None
    if kind == KIND_WIRE:
        if m.view is None or len(m.signature) != 65:
            return OK, False, None
        rec = co.ecrecover_address(bytes.fromhex(row["go_payload_no_sig_keccak"]), m.signature)
    else:
        p = m.payload
        if m.type != ip.COMMIT or not isinstance(p, ip.CommitMessage) or len(p.proposal_hash) != 32 or len(p.committed_seal) != 65:
            return OK, False, None
        rec = co.ecrecover_address(wl.seal_digest(p.proposal_hash), p.committed_seal)
    return OK, go_verdict(row, kind), rec or bytes(20)


def test_fixture_reaches_every_edge():
    edges, _ = load_edges()
    names = [r["name"] for r in edges]
    assert len(edges) >= 150
    # overflowing value varints: upb masks them, protobuf-go refuses them
    assert sum(1 for r in edges if r["upb_parses"] and not r["go_parses"]) >= 8
    # canonical frames that the device must hand back, and ones it must decide itself
    assert sum(1 for r in edges if is_canonical(r) and handed_back_on_purpose(r)) >= 8
    assert sum(1 for r in edges if is_canonical(r) and not handed_back_on_purpose(r)) >= 40
    # frames that are not canonical but decode are valid or invalid on a Go node depending on which bytes were signed
    sub = [r for r in edges if r["go_parses"] and not is_canonical(r)]
    assert any(r["go_sender_valid"] for r in sub) and any(not r["go_sender_valid"] for r in sub)
    assert any(r["go_seal_valid"] for r in edges if is_canonical(r) and not handed_back_on_purpose(r))
    assert {r["go_levels"] for r in edges if r["name"].startswith("nesting_")} == {8, 11, 12, 13, 14}
    for part in ("height_", "round_", "type_", "proposal_round_", "tag_", "len_", "trunc_", "type_depth3_", "type_depth6_"):
        assert any(n.startswith(part) for n in names), part


def test_oracle_codec_follows_protobuf_go():
    edges, _ = load_edges()
    for r in edges:
        wire = bytes.fromhex(r["wire"])
        if not r["go_parses"]:
            with pytest.raises(ip.DecodeError):
                ip.decode_ibft_message(wire)
            with pytest.raises(ip.DecodeError):
                ip.remarshal(wire)
            continue
        assert keccak_hex(ip.remarshal(wire)) == r["go_remarshal_keccak"], r["name"]
        assert keccak_hex(ip.payload_no_sig_from_wire(wire)) == r["go_payload_no_sig_keccak"], r["name"]
        m = ip.decode_ibft_message(wire)
        assert keccak_hex(m.payload_no_sig()) == r["go_payload_no_sig_keccak"], r["name"]
        # the typed model holds protobuf-go's int32 `type`, at every depth, and the nesting the device counts
        levels, types = frame_shape(m)
        assert (levels, types) == (r["go_levels"], r["go_types"]), r["name"]
        assert (ip.encode_ibft_message(m) == wire) == is_canonical(r), r["name"]


def test_cpp_codec_follows_protobuf_go():
    host = importlib.import_module("go-ibft_b200.host")
    edges, _ = load_edges()
    for r in edges:
        wire = bytes.fromhex(r["wire"])
        if not r["go_parses"]:
            assert host.remarshal(wire) is None and host.reencode(wire) is None, r["name"]
            continue
        assert keccak_hex(host.remarshal(wire)) == r["go_remarshal_keccak"], r["name"]
        assert keccak_hex(host.remarshal(wire, False)) == r["go_payload_no_sig_keccak"], r["name"]
        # typed model: the C++ one re-encodes to what the oracle's re-encodes to, so both hold the same `type` (and the rest)
        m = ip.decode_ibft_message(wire)
        assert host.reencode(wire) == ip.encode_ibft_message(m), r["name"]
        assert host.reencode(wire, False) == ip.encode_ibft_message(m, with_signature=False), r["name"]


@pytest.mark.parametrize("kind", [KIND_WIRE, KIND_WIRE_SEAL], ids=["wire", "wire_seal"])
def test_emulated_device_follows_protobuf_go(emul, kind):
    """the device's frame walk + sponge + recovery (csrc headers compiled for the host) on every edge frame, through the
    one-thread, split and four-lane split pipelines: status, verdict and recovered address"""
    edges, _ = load_edges()
    decided = 0
    for r in edges:
        wire = bytes.fromhex(r["wire"])
        arena = np.frombuffer(wire, np.uint8) if wire else np.zeros(1, np.uint8)
        status, verdict, rec = edge_expectation(r, kind)
        (r1, a1), (r2, a2) = both_paths(emul, wire_item(kind, 0, len(wire)), arena, len(wire))
        assert (r1, a1) == (r2, a2), r["name"]
        assert (1 if r1 == -1 else 0, r1 == 1) == (status, verdict), (r["name"], r1)
        if rec is not None:
            assert a1 == rec, r["name"]
            decided += 1
        # level-structured recovery of the four-lane kernel
        o = (ctypes.c_uint8 * 20)()
        it = wire_item(kind, 0, len(wire))
        r3 = emul.emul_verify_item_levels(it.ctypes.data_as(ctypes.c_void_p), arena.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(len(wire)), o)
        assert (r3, bytes(o)) == (r1, a1), r["name"]
    assert decided >= (40 if kind == KIND_WIRE else 20)
