"""Reference of ibft_explain_batch: why the recover path rejects an item, as an IBFT_REASON_* code, step by step in the order the
verify kernels decide.  Built on the oracle's primitives (the C oracle's recovery, Keccak and the protobuf codec), beside the
oracle's own verdict, which it must match: reason OK <=> verdict 1.

Raw frames (IBFT_KIND_WIRE / _WIRE_SEAL) take their canonical-encoding decision from oracle/ibft_proto.py, as the wire tests do:
a frame protobuf-go would not re-encode byte for byte, or one of the device's two conservative hand-backs, is NEEDS_HOST."""
from __future__ import annotations

import numpy as np

import workloads as wl
from oracle import coracle as co
from oracle import ibft_proto as ip
from oracle import secp256k1 as ec
from test_emul import WIRE_MAX_DEPTH, frame_shape

OK, NO_GROUP, MALFORMED, NEEDS_HOST, BAD_V, R_RANGE, S_RANGE, R_NOT_X, NO_KEY, SIGNER_MISMATCH, NOT_VALIDATOR = range(11)
INCONSISTENT = 255
NAMES = {OK: "OK", NO_GROUP: "NO_GROUP", MALFORMED: "MALFORMED", NEEDS_HOST: "NEEDS_HOST", BAD_V: "BAD_V", R_RANGE: "R_RANGE",
         S_RANGE: "S_RANGE", R_NOT_X: "R_NOT_X", NO_KEY: "NO_KEY", SIGNER_MISMATCH: "SIGNER_MISMATCH", NOT_VALIDATOR: "NOT_VALIDATOR",
         INCONSISTENT: "INCONSISTENT"}
KIND_DIGEST, KIND_PAYLOAD, KIND_SEAL, KIND_WIRE, KIND_WIRE_SEAL, KIND_PAYLOAD2 = 0, 1, 2, 3, 4, 5
P, N = ec.P, ec.N


def _signature_and_digest(it, arena: bytes):
    """(reason, None) when the item never reaches the arithmetic, else (None, (sig65, z, expected signer))"""
    kind, off, ln = int(it["kind"]), int(it["payload_off"]), int(it["payload_len"])
    if kind in (KIND_WIRE, KIND_WIRE_SEAL):
        if off + ln > len(arena):
            return MALFORMED, None
        frame = arena[off:off + ln]
        try:
            m = ip.decode_ibft_message(frame)
        except (ip.DecodeError, RecursionError):
            return NEEDS_HOST, None
        if ip.encode_ibft_message(m) != frame:
            return NEEDS_HOST, None
        levels, types = frame_shape(m)
        if levels > WIRE_MAX_DEPTH or min(types) < 0:
            return NEEDS_HOST, None
        if len(m.from_) != 20:
            return MALFORMED, None
        if kind == KIND_WIRE:
            if m.view is None or len(m.signature) != 65:
                return MALFORMED, None
            return None, (m.signature, co.keccak256(m.payload_no_sig()), m.from_)
        p = m.payload
        if m.type != ip.COMMIT or not isinstance(p, ip.CommitMessage) or len(p.proposal_hash) != 32 or len(p.committed_seal) != 65:
            return MALFORMED, None
        return None, (p.committed_seal, wl.seal_digest(p.proposal_hash), m.from_)
    sig = bytes(it["r"]) + bytes(it["s"]) + bytes([int(it["v"])])
    digest = bytes(it["digest"])
    if kind == KIND_DIGEST:
        z = digest
    elif kind == KIND_SEAL:
        z = wl.seal_digest(digest)
    elif kind == KIND_PAYLOAD:
        if off + ln > len(arena):
            return MALFORMED, None
        z = co.keccak256(arena[off:off + ln])
    elif kind == KIND_PAYLOAD2:
        off2, ln2 = int.from_bytes(digest[:8], "little"), int.from_bytes(digest[8:12], "little")
        if off + ln > len(arena) or off2 > len(arena) or ln2 > len(arena) - off2:
            return MALFORMED, None
        z = co.keccak256(arena[off:off + ln] + arena[off2:off2 + ln2])
    else:
        return MALFORMED, None
    return None, (sig, z, bytes(it["signer"]))


def explain_item(it, arena: bytes = b"", table=None, n_groups: int | None = None):
    """(reason, recovered address or 20 zero bytes) of one ITEM_DTYPE record.  table: the addresses of the item's group's validator
    table (None: a group without a table).  n_groups: groups of the call (None: a call without groups)."""
    if n_groups is not None and int(it["group"]) >= n_groups:
        return NO_GROUP, bytes(20)
    why, got = _signature_and_digest(it, arena)
    if why is not None:
        return why, bytes(20)
    sig, z, signer = got
    r, s, v = int.from_bytes(sig[:32], "big"), int.from_bytes(sig[32:64], "big"), sig[64]
    if v > 1:
        return BAD_V, bytes(20)
    if not 0 < r < N:
        return R_RANGE, bytes(20)
    if not 0 < s < N:
        return S_RANGE, bytes(20)
    if pow((r ** 3 + 7) % P, (P - 1) // 2, P) == P - 1:
        return R_NOT_X, bytes(20)
    addr = co.ecrecover_address(z, sig)
    if addr is None:
        return NO_KEY, bytes(20)
    if addr != signer:
        return SIGNER_MISMATCH, addr
    if table is not None and signer not in table:
        return NOT_VALIDATOR, addr
    return OK, addr


def explain_batch(items: np.ndarray, arena: bytes = b"", tables=None, group_table=None):
    """(reasons uint8[n], recovered uint8[n, 20]) with coracle.verify_batch's arguments: tables = list of (n x 20) address arrays,
    group_table = table index per group (0xFFFF = none), or None for a call without groups."""
    sets = [set(bytes(a) for a in np.asarray(t, dtype=np.uint8).reshape(-1, 20)) for t in (tables or [])]
    arena = bytes(arena)
    reasons = np.zeros(len(items), dtype=np.uint8)
    recovered = np.zeros((len(items), 20), dtype=np.uint8)
    n_groups = None if group_table is None else len(group_table)
    for i, it in enumerate(items):
        table = None
        if group_table is not None and int(it["group"]) < n_groups and group_table[int(it["group"])] != 0xFFFF:
            table = sets[group_table[int(it["group"])]]
        reasons[i], rec = explain_item(it, arena, table, n_groups)
        recovered[i] = np.frombuffer(rec, np.uint8)
    return reasons, recovered


def bits_of(bitmap: np.ndarray, n: int) -> np.ndarray:
    return np.unpackbits(np.ascontiguousarray(bitmap, dtype=np.uint32).view(np.uint8), bitorder="little")[:n].astype(bool)
