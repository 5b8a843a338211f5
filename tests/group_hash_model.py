"""Python model of groups bound to the accepted proposal's hash (ibft_group_hash, include/ibft_verify.h): which items count, and
the group results the engine must report for them.  Built on the oracle (oracle/ibft_proto.py decode, oracle/ibft_logic.py
extractors) and checked against oracle.ibft_logic's handle_prepare / handle_commit by tests/test_emul_group_hash.py; the GPU
tests compare the engine with it."""
from __future__ import annotations

from typing import Optional

import numpy as np

from oracle import ibft_logic as L
from oracle import ibft_proto as ip

HASH_UNBOUND, HASH_PREPARE, HASH_COMMIT = 0xFFFFFFFF, 1, 2
KIND_DIGEST, KIND_PAYLOAD, KIND_SEAL, KIND_WIRE, KIND_WIRE_SEAL = 0, 1, 2, 3, 4
NO_TABLE = 0xFFFF
QUORUM_DEFAULT, QUORUM_PREPARE = 0, 2
PROPOSER_NONE, PROPOSER_UNSET = 0xFFFFFFFF, 0xFFFFFFFE


def extract(buf: bytes, msg_type: int) -> Optional[bytes]:
    """ExtractPrepareHash (msg_type 1) / ExtractCommitHash (2) of the message protobuf-go decodes from buf; None for nil (a message
    protobuf-go refuses included)"""
    try:
        m = ip.decode_ibft_message(bytes(buf))
    except (ip.DecodeError, RecursionError):
        return None
    return (L.extract_prepare_hash if msg_type == HASH_PREPARE else L.extract_commit_hash)(m)


def item_hash(kind: int, msg_type: int, digest: bytes, span: bytes) -> Optional[bytes]:
    """the hash a bound group's extractor gets from an item (the table of include/ibft_verify.h), None when it has none"""
    if kind == KIND_SEAL:
        return bytes(digest) if msg_type == HASH_COMMIT else None
    if kind == KIND_WIRE_SEAL:
        return extract(span, HASH_COMMIT) if msg_type == HASH_COMMIT else None
    if kind in (KIND_WIRE, KIND_PAYLOAD):
        return extract(span, msg_type)
    return None


def _span(it, arena: bytes) -> bytes:
    off, ln = int(it["payload_off"]), int(it["payload_len"])
    return bytes(arena[off:off + ln]) if off + ln <= len(arena) else b""


def counted(items: np.ndarray, arena: bytes, bitmap: np.ndarray, n_groups: int, hashes: Optional[np.ndarray]) -> np.ndarray:
    """bool per item: its verdict bit is 1, its group is in range, and the group is unbound or the item names the bound hash"""
    arena = bytes(arena)
    out = np.zeros(len(items), dtype=bool)
    for i, it in enumerate(items):
        if not (int(bitmap[i // 32]) >> (i % 32)) & 1:
            continue
        g = int(it["group"])
        if g >= n_groups:
            continue
        mt = HASH_UNBOUND if hashes is None else int(hashes[g]["msg_type"])
        if mt == HASH_UNBOUND:
            out[i] = True
            continue
        h = item_hash(int(it["kind"]), mt, bytes(it["digest"]), _span(it, arena))
        out[i] = h is not None and len(h) == 32 and h == bytes(hashes[g]["hash"])
    return out


def pack_bits(flags: np.ndarray) -> np.ndarray:
    n = len(flags)
    words = np.zeros(max(1, (n + 31) // 32), dtype=np.uint32)
    for i in np.nonzero(flags)[0]:
        words[i // 32] |= np.uint32(1 << (int(i) % 32))
    return words[: (n + 31) // 32]


def signer(it, arena: bytes) -> Optional[bytes]:
    """the expected signer the quorum kernels resolve: From of a raw frame, else the tuple's signer"""
    if int(it["kind"]) in (KIND_WIRE, KIND_WIRE_SEAL):
        try:
            m = ip.decode_ibft_message(_span(it, bytes(arena)))
        except ip.DecodeError:
            return None
        return m.from_ if len(m.from_) == 20 else None
    return bytes(it["signer"])


class Table:
    """a validator table as the engine holds it: addresses in validator-index order and their voting power"""

    def __init__(self, addrs, powers):
        self.addrs = [bytes(a) for a in addrs]
        self.powers = [int(p) for p in powers]
        self.index = {a: i for i, a in enumerate(self.addrs)}
        self.quorum = 2 * sum(self.powers) // 3 + 1


def group_results(items: np.ndarray, arena: bytes, flags: np.ndarray, groups: np.ndarray, tables: dict):
    """(results, voted) of the engine's reduce over the items whose flag is set: results = RESULT_DTYPE-shaped dicts (power as an
    int, n_valid, n_distinct, has_quorum), voted = per group the set of validator indices (tables: slot -> Table)"""
    ng = len(groups)
    voted = [set() for _ in range(ng)]
    n_valid = [0] * ng
    for i in np.nonzero(flags)[0]:
        it = items[i]
        g = int(it["group"])
        n_valid[g] += 1
        slot = int(groups[g]["table_slot"])
        if slot == NO_TABLE or slot not in tables:
            continue
        a = signer(it, arena)
        v = tables[slot].index.get(a) if a is not None else None
        if v is not None:
            voted[g].add(v)
    res = []
    for g in range(ng):
        slot = int(groups[g]["table_slot"])
        t = tables.get(slot) if slot != NO_TABLE else None
        power = sum(t.powers[v] for v in voted[g]) if t else 0
        q = 0
        if t is not None:
            rule, prop = int(groups[g]["flags"]) & 3, int(groups[g]["reserved"])
            if rule == QUORUM_PREPARE:
                if prop == PROPOSER_UNSET or prop in voted[g]:
                    q = 0
                else:
                    if prop != PROPOSER_NONE:
                        power += t.powers[prop]
                    q = int(power >= t.quorum)
            elif rule == 1:
                q = int(n_valid[g] >= 1)
            else:
                q = int(power >= t.quorum)
        res.append(dict(power=power, n_valid=n_valid[g], n_distinct=len(voted[g]), has_quorum=q))
    return res, voted


def power_of(result_row) -> int:
    """the 320-bit little-endian power of an engine RESULT_DTYPE row as an int"""
    return sum(int(result_row["power"][k]) << (64 * k) for k in range(5))


def voted_set(words: np.ndarray) -> set:
    return {32 * w + b for w in range(len(words)) for b in range(32) if (int(words[w]) >> b) & 1}
