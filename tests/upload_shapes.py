"""Host-buffer batches shaped by how ibft_verify_batch / ibft_verify_submit move tuples onto the device (engine.cu submit_locked),
and the expectations of every item and group of such a call.

The upload path cuts a batch into chunks of CHUNK tuples.  Chunk c is staged (pageable input) or taken as it is (page-locked
input of a synchronous call), copied on the copy stream and verified on the kernel stream c & 1; with the key registry it fills
worklist c & 1, so chunk c + 2 reuses chunk c's list.  stage_copy moves a chunk of pageable tuples with one memcpy below
2 x STAGE_MIN bytes and with 2, 3 or 4 threads from there up, each part bytes / parts rounded up to 64 bytes -- so a part boundary
can fall inside a 128-byte tuple.  A slip in that bookkeeping loses, repeats or misplaces tuples at a chunk's or a part's edge,
or verifies bytes a previous call left in the staging.

So the shapes put the last chunk at one tuple, at exactly 4 MiB (two parts), at three parts whose boundaries cut tuples, and
reach five chunks (each worklist reused twice).  The fillers are config 3's distinct tuples, tiled from an offset that differs per
chunk and per call: no two chunks of a call and no chunk of two consecutive calls hold the same bytes, and since config 3 has
invalid items in several classes, bytes left over from another chunk or call change verdicts.  Class items (tests/position_sweep.py)
sit at the chunk's edges, its first and last CTAs' edges and on either side of every staging part boundary.

Expectations: the fillers' verdicts are config 3's golden bitmap; the class items' come from tests/explain_oracle.py and the C
oracle (position_sweep.item_expectation), once per distinct tuple, and are tiled.  Group results and voted sets are aggregated
from the tiled per-item arrays with numpy; no reference runs over the half million items of a batch."""
from __future__ import annotations

import functools
import os

import numpy as np

import explain_oracle as X
import group_hash_model as G
import position_sweep as PS
from oracle import coracle as co

HERE = os.path.dirname(os.path.abspath(__file__))
C = 1 << 17                # engine.cu submit_locked: CHUNK, tuples per upload chunk
ITEM_BYTES = 128           # sizeof(ibft_sig_item)
STAGE_MIN = 2 << 20        # engine.cu stage_copy: kMin; one memcpy below 2 x kMin bytes, else min(4, bytes / kMin) parts
NO_TABLE = 0xFFFF
SLOTS = [0, 0, NO_TABLE]   # group 0 (config 3's COMMIT payloads), group 1 (its seals), group 2 (no table)
BEYOND = 11                # the group of a no-group class item: beyond the call's groups
SPAN_BEYOND = 1 << 30      # where a class item's out-of-range span starts: past the largest arena a call uploads
SHAPES = {"C-1": C - 1, "C": C, "C+1": C + 1, "3chunks": 2 * C + 32768, "4chunks": 3 * C + 49153, "5chunks": 4 * C + 5}
KNOWN_NAMES = ["known_valid", "known_misattributed", "unknown_signer", "known_r_plus_n", "known_cancelling", "known_flipped"]


# ---------------------------------------------------------------------------------------------------------------- the upload model
def chunks(n: int) -> list[tuple[int, int]]:
    """[lo, hi) of each upload chunk of an n-tuple call"""
    return [(lo, min(n, lo + C)) for lo in range(0, n, C)]


def stage_parts(nbytes: int) -> list[tuple[int, int]]:
    """(offset, length) of each memcpy stage_copy makes of a chunk of nbytes"""
    if nbytes < 2 * STAGE_MIN:
        return [(0, nbytes)]
    parts = min(4, nbytes // STAGE_MIN)
    per = (nbytes // parts + 63) & ~63
    return [(k * per, per if k + 1 < parts else nbytes - k * per) for k in range(parts)]


def odd_slots(lo: int, hi: int) -> list[int]:
    """the chunk's class-item slots: its first tuples and first CTA edges, its last tuples and last CTA edges, and the last tuple of
    each staging part with the first tuple of the next"""
    rel = [0, 1, 31, 32, 127, 128]
    m = hi - lo
    rel += [m - 129, m - 128, m - 33, m - 32, m - 1]
    for off, _ in stage_parts(m * ITEM_BYTES)[1:]:
        rel += [(off - 1) // ITEM_BYTES, off // ITEM_BYTES]
    return sorted({lo + r for r in rel if 0 <= r < m})


# ---------------------------------------------------------------------------------------------------------------- batches
class Uploads:
    """config 3's fillers, the sweep's class items relocated behind config 3's arena, the slot-0 table and per-source expectations"""

    def __init__(self):
        S = self.S = PS.sweep()
        d = np.load(os.path.join(HERE, "golden", "config3.npz"))
        items = np.ascontiguousarray(d["items"]).view(co.ITEM_DTYPE).reshape(-1)
        gold = X.bits_of(d["bitmap"], len(items))
        raw = items.view(np.dtype((np.void, ITEM_BYTES)))
        _, first = np.unique(raw, return_index=True)
        keep = np.sort(first)                                # distinct tuples in fixture order
        self.fillers, self.filler_gold = items[keep].copy(), gold[keep]
        self.F = len(self.fillers)
        self.height = int(d["meta"][2])
        self.proposal_hash = bytes(d["proposal_hash"])
        base = len(d["arena"])
        self.arena = bytes(d["arena"]) + S.arena             # class spans move behind config 3's payloads
        # the slot-0 table: config 3's validators, then every class signer that is not one of them (power 1)
        c3 = [bytes(a) for a in d["addrs"]]
        skip = set(c3) | set(S.fresh.addrs)
        extra = [a for a in S.members if a not in skip]
        self.members = c3 + list(dict.fromkeys(extra))
        self.index = {a: i for i, a in enumerate(self.members)}
        self.addrs = np.frombuffer(b"".join(self.members), np.uint8).reshape(-1, 20).copy()
        self.powers = np.concatenate([np.ascontiguousarray(d["powers"], np.uint8).reshape(-1, 32),
                                      np.frombuffer(b"".join((1).to_bytes(32, "big") for _ in extra), np.uint8).reshape(-1, 32)])
        self.power_int = [int.from_bytes(bytes(p), "big") for p in self.powers]
        # class items: sweep code in the group field (0 member group, 1 no table, 2 no group), spans relocated
        self.names = list(S.names)
        cls = [self._relocate(S.classes[k], base) for k in self.names]
        cls += [self._relocate(S.known_classes[k], base) for k in KNOWN_NAMES]
        self.classes = np.concatenate(cls)
        self.class_of = {k: self.F + j for j, k in enumerate(self.names + KNOWN_NAMES)}
        self.sources = np.concatenate([self.fillers, self.classes])
        self._expect_sources()

    def _relocate(self, it: np.ndarray, base: int) -> np.ndarray:
        it = it.copy()
        if int(it["kind"][0]) in (X.KIND_PAYLOAD, X.KIND_PAYLOAD2, X.KIND_WIRE, X.KIND_WIRE_SEAL):
            if int(it["payload_off"][0]) + int(it["payload_len"][0]) > len(self.S.arena):
                it["payload_off"] = SPAN_BEYOND              # out of range in every arena the calls upload, up to 32 MiB
            else:
                it["payload_off"] += base
        if int(it["kind"][0]) == X.KIND_PAYLOAD2:              # the second span's offset: digest bytes 0..7
            off2 = int.from_bytes(bytes(it["digest"][0][:8]), "little") + base
            it["digest"][0][:8] = np.frombuffer(off2.to_bytes(8, "little"), np.uint8)
        return it

    def _expect_sources(self):
        """per source: verdict bit, status, recovered address, signer's table index (-1: none)"""
        n = len(self.sources)
        self.bit = np.zeros(n, bool)
        self.status = np.zeros(n, np.uint8)
        self.rec = np.zeros((n, 20), np.uint8)
        self.signer = np.full(n, -1, np.int64)
        for i in range(self.F):
            it = self.fillers[i]
            self.bit[i] = self.filler_gold[i]
            why, got = X._signature_and_digest(it, self.arena)
            rec = bytes(20) if why is not None else (co.ecrecover_address(got[1], got[0]) or bytes(20))
            self.rec[i] = np.frombuffer(rec, np.uint8)
            self.signer[i] = self.index.get(bytes(it["signer"]), -1)
        members = tuple(self.members)
        for j in range(len(self.classes)):
            b, st, rec, _, _, signer = PS.item_expectation(self.classes[j:j + 1].tobytes(), self.arena, members)
            k = self.F + j
            self.bit[k], self.status[k] = b, st
            self.rec[k] = np.frombuffer(rec, np.uint8)
            self.signer[k] = self.index.get(signer, -1)

    @staticmethod
    def rotation(c: int, call: int) -> int:
        return 7919 * c + 4099 * call + 1

    def batch(self, n: int, call: int, known: bool = False):
        """(items, src, groups of the items): call `call` of n tuples -- every chunk's fillers tiled from its own offset, its odd
        slots holding the class items (the key-registry classes when `known`), rotated per chunk and per call"""
        src = np.empty(n, np.int64)
        grp = np.empty(n, np.int64)
        names = KNOWN_NAMES if known else self.names
        for c, (lo, hi) in enumerate(chunks(n)):
            t = np.arange(hi - lo)
            src[lo:hi] = (t + self.rotation(c, call)) % self.F
            grp[lo:hi] = self.fillers["group"][src[lo:hi]]
            for j, i in enumerate(odd_slots(lo, hi)):
                k = self.class_of[names[(j + 5 * c + 3 * call) % len(names)]]
                src[i] = k
                code = int(self.sources[k]["group"])
                grp[i] = (j + c) % 2 if code == 0 else (2 if code == 1 else BEYOND)
        items = self.sources[src].copy()
        items["group"] = grp
        return items, src, grp

    def expect(self, src: np.ndarray, grp: np.ndarray, flags: np.ndarray | None = None):
        """per item: bit, status, rec (tiled); per group (n_valid, voted validator indices, power, has_quorum) over the items whose
        flag is set (default: the verdict bits), as the engine's default quorum rule decides it"""
        bit = self.bit[src]
        if flags is None:
            flags = bit
        groups = []
        for g, slot in enumerate(SLOTS):
            sel = flags & (grp == g)
            nv = int(sel.sum())
            if slot == NO_TABLE:
                groups.append((nv, set(), 0, False))
                continue
            voted = set(np.unique(self.signer[src[sel]]).tolist()) - {-1}
            power = sum(self.power_int[v] for v in voted)
            groups.append((nv, voted, power, power >= 2 * sum(self.power_int) // 3 + 1))
        return dict(bit=bit, status=self.status[src], rec=self.rec[src], groups=groups)

    # ------------------------------------------------------------------------------------------------------------ hashed groups
    def hashes(self) -> np.ndarray:
        """group 0 bound to config 3's proposal (its COMMIT payloads count), group 1 to another hash (its seals do not)"""
        h = np.zeros(len(SLOTS), dtype=G_HASH_DTYPE)
        h["msg_type"] = G.HASH_UNBOUND
        for g, digest in ((0, self.proposal_hash), (1, co.keccak256(b"another proposal"))):
            h[g]["msg_type"] = G.HASH_COMMIT
            h[g]["hash"] = np.frombuffer(digest, np.uint8)
        return h

    def counted(self, src: np.ndarray, grp: np.ndarray, hashes: np.ndarray) -> np.ndarray:
        """group_hash_model.counted once per distinct (source, group), tiled"""
        key = src * 16 + grp
        uk, inv = np.unique(key, return_inverse=True)
        us, ug = uk // 16, uk % 16
        items = self.sources[us].copy()
        items["group"] = ug
        flags = G.counted(items, self.arena, G.pack_bits(self.bit[us]), len(SLOTS), hashes)
        return flags[inv]


G_HASH_DTYPE = np.dtype([("hash", "u1", 32), ("msg_type", "<u4"), ("reserved", "<u4", 3)])   # ibft_group_hash


@functools.lru_cache(maxsize=None)
def uploads() -> Uploads:
    return Uploads()
