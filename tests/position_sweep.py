"""Position sweep of the verify kernels: one odd item (a rejection class, a crafted valid item, a valid item of each kind) at every
signature slot of a kernel's CTA, among valid fillers, and the expectations of every item and group of such a call.

The kernels differ in how a CTA maps signatures to lanes and where a verdict goes (engine.cu): one thread each and a ballot word
(k_recover<32 / 128>, k_verify_known<32 / 128>), four lanes each (k_recover_quad), three chain warps served by a helper warp
through named barriers (k_recover_split, k_verify_split: 96 per CTA), four-lane chains whose helper lane l serves signature l and
whose verdicts are OR-ed into words two CTAs share (k_recover_qsplit: 24 per CTA).  A slip in that bookkeeping moves one item's
verdict, status, recovered address or vote onto another item -- which only a sweep over every slot finds for certain.

Patterns of a window of W signatures (one block per position p in [0, W)):
  (a) fillers everywhere, the class item at p;
  (b) R_NOT_X everywhere, one valid filler at p;
  (c) fillers up to p, the class item at p, and the call ends there (the last CTA is partial).
Neighbouring positions use different groups on different table slots (group 2b + j % 2 of block b on slot j % 2; slot 1 holds the
table in reverse order with other powers), so a vote recorded for the wrong item or the wrong group shows in the quorum results.

Expectations come from tests/explain_oracle.py (the reason, hence the verdict bit) and the C oracle's recovery, computed once per
distinct (tuple, group kind) and tiled: a batch of 200,000 items has only a few hundred distinct tuples."""
from __future__ import annotations

import functools
import os

import numpy as np

import adversarial as A
import explain_oracle as X
import workloads as wl
from oracle import coracle as co
from oracle import secp256k1 as ec
from test_explain_oracle import every_reason_batch, non_abscissa

HERE = os.path.dirname(os.path.abspath(__file__))
N, P = ec.N, ec.P
NO_TABLE = 0xFFFF
# signatures per window of each kernel geometry: lcm(24, 32) = 96 for qsplit, so the odd item meets every (CTA slot, bit) pair
WINDOWS = {"thread32": 32, "thread128": 128, "quad": 32, "split": 96, "qsplit": 96, "verify_known32": 32, "verify_known128": 128,
           "verify_split": 96}
HEAVY = 1000  # slot-1 power of the fillers at odd positions (the others have power 1): group 2b + 1 can reach its quorum

# the rows of test_explain_oracle.every_reason_batch() the sweep takes, by the reason each must have
REASON_ROWS = {
    "no_group": (2, X.NO_GROUP), "malformed_span": (6, X.MALFORMED), "malformed_frame": (34, X.MALFORMED),
    "needs_host": (36, X.NEEDS_HOST), "bad_v": (8, X.BAD_V), "r_zero": (10, X.R_RANGE), "r_eq_n": (11, X.R_RANGE),
    "s_eq_n": (15, X.S_RANGE), "r_not_x": (18, X.R_NOT_X), "no_key": (22, X.NO_KEY), "signer_mismatch": (26, X.SIGNER_MISMATCH),
    "not_validator": (28, X.NOT_VALIDATOR), "wire": (30, X.OK), "wire_seal": (31, X.OK), "no_table": (1, X.OK),
}


class Sweep:
    """The fillers, the class items, the shared arena and the validator tables of the sweep."""

    def __init__(self):
        ritems, rarena, _, _, rwant = every_reason_batch()
        self.reason_vs = wl.ValidatorSet(5, 4)          # every_reason_batch's validators
        arena = bytearray(rarena)
        # fillers: config 3's committed seals of distinct validators whose golden bit is 1
        d = np.load(os.path.join(HERE, "golden", "config3.npz"))
        items = np.ascontiguousarray(d["items"]).view(co.ITEM_DTYPE).reshape(-1)
        gold = X.bits_of(d["bitmap"], len(items))
        fill, seen = [], set()
        for i in range(len(items) // 2, len(items)):
            s = bytes(items[i]["signer"])
            if gold[i] and items[i]["kind"] == X.KIND_SEAL and s not in seen:
                fill.append(i)
                seen.add(s)
            if len(fill) == 128:
                break
        self.fillers = items[fill].copy()
        self.fillers["group"] = 0                        # (config 3's seal group is 1; place() gives each its block's group)
        self.filler_gold = gold[fill]
        self.classes: dict[str, np.ndarray] = {}
        for name, (row, why) in REASON_ROWS.items():
            assert rwant[row] == why, name
            self.classes[name] = ritems[row:row + 1].copy()
        vs = self.reason_vs
        dig = co.keccak256(b"position sweep")
        self.classes["valid_low_s"] = wl.make_item(wl.sign(vs.keys[3], dig, low_s=True), vs.addrs[3], X.KIND_DIGEST, dig)
        self.classes["valid_high_s"] = wl.make_item(wl.sign(vs.keys[3], dig, low_s=False), vs.addrs[3], X.KIND_DIGEST, dig)
        # u1 = 0: z = 0 and z = n (the split helpers' u1*G is the point at infinity); no private key: the address joins the tables
        R = A.mul(12345)
        self.crafted = []
        for tag, z in (("u1_zero_z0", None), ("u1_zero_zn", N.to_bytes(32, "big"))):
            v = A.recover_vector(tag, R, 0, 7, z_override=z)
            self.classes[tag] = wl.make_item(v.sig, v.addr, X.KIND_DIGEST, v.digest)
            self.crafted.append(v)
        # one valid item of each hashed kind
        payload = bytes((7 * i + 3) & 0xFF for i in range(200))
        off = len(arena)
        arena.extend(payload)
        self.classes["payload"] = wl.make_item(wl.sign(vs.keys[2], co.keccak256(payload)), vs.addrs[2], X.KIND_PAYLOAD, b"", 0, off, 200)
        tail = b"second span"
        off2 = len(arena)
        arena.extend(tail)
        d2 = off2.to_bytes(8, "little") + len(tail).to_bytes(4, "little") + bytes(20)
        self.classes["payload2"] = wl.make_item(wl.sign(vs.keys[1], co.keccak256(payload[:150] + tail)), vs.addrs[1], X.KIND_PAYLOAD2,
                                                d2, 0, off, 150)
        self.arena = bytes(arena)
        self.names = sorted(self.classes)
        # r_not_x filler of pattern (b): signer = a validator, r not an abscissa
        r = non_abscissa(11)
        self.invalid = wl.make_item(r.to_bytes(32, "big") + wl.sign(vs.keys[0], dig)[32:], vs.addrs[0], X.KIND_DIGEST, dig)
        # known-key classes (tests/adversarial.py): a cancelling signature of Q = G and an x = r + n forgery of its key, with a
        # valid signature of each key to learn it from
        canc, fake = A.known_cancelling()[0], A.known_r_plus_n()[0]
        self.known_keys = [canc.key_index, fake.key_index]
        learn = {v.key_index: v for v in reversed(A.known_vectors())}
        self.known_warm = [wl.make_item(learn[k].sig, A.known_addr(k), X.KIND_DIGEST, learn[k].digest) for k in self.known_keys]
        sig_ok = wl.sign(vs.keys[3], dig)
        self.known_classes = {
            "known_valid": self.classes["valid_low_s"],
            "known_misattributed": wl.make_item(sig_ok, vs.addrs[2], X.KIND_DIGEST, dig),
            "known_flipped": wl.make_item(sig_ok[:64] + bytes([sig_ok[64] ^ 1]), vs.addrs[3], X.KIND_DIGEST, dig),
            "unknown_signer": wl.make_item(wl.sign(vs.keys[0], dig), vs.addrs[0], X.KIND_DIGEST, dig),
            "known_r_plus_n": wl.make_item(fake.sig, A.known_addr(fake.key_index), X.KIND_DIGEST, fake.digest),
            "known_cancelling": wl.make_item(canc.sig, A.known_addr(canc.key_index), X.KIND_DIGEST, canc.digest),
            # a member whose key is known but whose comb table a key-table budget has evicted
            "known_no_table": wl.make_item(wl.sign(vs.keys[1], dig), vs.addrs[1], X.KIND_DIGEST, dig),
        }
        # validators whose keys a known-key engine never learns before the call that hands their signatures back
        self.fresh = wl.ValidatorSet(77, 3 * 900)
        members = [bytes(f["signer"]) for f in self.fillers] + list(vs.addrs) + [v.addr for v in self.crafted]
        members += [A.known_addr(k) for k in self.known_keys] + list(self.fresh.addrs)
        self.members = list(dict.fromkeys(members))      # (z = 0 and z = n recover the same key)

    # ------------------------------------------------------------------------------------------------------------ tables
    def tables(self, W: int):
        """(addrs, powers) of slot 0 (member order, power 1) and slot 1 (reverse order; the fillers of odd positions of the window
        weigh HEAVY)"""
        n = len(self.members)
        p0 = [1] * n
        p1 = [HEAVY if (j < W and j % 2 == 1) else 1 for j in range(n)]
        a0 = np.frombuffer(b"".join(self.members), np.uint8).reshape(n, 20).copy()
        pw = lambda ps: np.frombuffer(b"".join(p.to_bytes(32, "big") for p in ps), np.uint8).reshape(n, 32).copy()  # noqa: E731
        return (a0, pw(p0)), (a0[::-1].copy(), pw(p1[::-1]))

    # ------------------------------------------------------------------------------------------------------------ batches
    def place(self, it: np.ndarray, b: int, j: int, n_blocks: int) -> np.ndarray:
        """item `it` at position j of block b: group 2b + j % 2 (slot j % 2), the no-table class in the no-table group, no-group beyond"""
        it = it.copy()
        g = int(it["group"][0])
        if g == 1:
            it["group"] = 2 * n_blocks                  # the call's no-table group
        elif g >= 2:
            it["group"] = 2 * n_blocks + 8             # beyond the call's groups
        else:
            it["group"] = 2 * b + j % 2
        return it

    def block(self, W: int, b: int, n_blocks: int, odd: np.ndarray | None, p: int, pattern: str) -> np.ndarray:
        rows = []
        for j in range(W if pattern != "c" else p + 1):
            if pattern == "b":
                it = self.fillers[j:j + 1] if j == p else self.invalid
            else:
                it = odd if j == p else self.fillers[j:j + 1]
            rows.append(self.place(it, b, j, n_blocks))
        return np.concatenate(rows)

    def pattern_a(self, W: int, name: str) -> np.ndarray:
        return np.concatenate([self.block(W, p, W, self.classes[name], p, "a") for p in range(W)])

    def pattern_b(self, W: int) -> np.ndarray:
        return np.concatenate([self.block(W, p, W, None, p, "b") for p in range(W)])

    def pattern_c(self, W: int, name: str, p: int) -> np.ndarray:
        return self.block(W, 0, 1, self.classes[name], p, "c")

    def pad(self, items: np.ndarray, n_blocks: int, total: int) -> np.ndarray:
        """fillers after the blocks, up to `total` items, in the call's pad group (slot 0)"""
        k = total - len(items)
        if k <= 0:
            return items
        extra = np.tile(self.fillers, -(-k // len(self.fillers)))[:k].copy()
        extra["group"] = 2 * n_blocks + 1
        return np.concatenate([items, extra])

    def prefix(self, items: np.ndarray, n_blocks: int, k: int) -> np.ndarray:
        """k fillers before the blocks (k a multiple of the CTA size, so the blocks keep their positions), in the pad group"""
        extra = np.tile(self.fillers, -(-k // len(self.fillers)))[:k].copy()
        extra["group"] = 2 * n_blocks + 1
        return np.concatenate([extra, items])

    @staticmethod
    def n_groups(n_blocks: int) -> int:
        return 2 * n_blocks + 2                          # block groups, the no-table group, the pad group

    def group_slots(self, n_blocks: int) -> list[int]:
        return [g % 2 for g in range(2 * n_blocks)] + [NO_TABLE, 0]

    # ------------------------------------------------------------------------------------------------------------ expectations
    def expect(self, items: np.ndarray, n_blocks: int, W: int):
        """per item: (bit, status, recovered address of the verify path, explain reason, explain address); per group: (n_valid,
        voted validator indices, power, has_quorum)"""
        ng = self.n_groups(n_blocks)
        g = items["group"].astype(np.int64)
        code = np.where(g >= ng, 2, np.where(g == 2 * n_blocks, 1, 0)).astype(np.uint16)
        canon = items.copy()
        canon["group"] = code
        v = np.ascontiguousarray(canon).view(np.uint8).reshape(len(items), 128).view(np.dtype((np.void, 128))).ravel()
        uniq, first, inv = np.unique(v, return_index=True, return_inverse=True)
        per = [item_expectation(bytes(u), self.arena, tuple(self.members)) for u in uniq]
        bit = np.array([e[0] for e in per], bool)[inv]
        status = np.array([e[1] for e in per], np.uint8)[inv]
        rec = np.array([np.frombuffer(e[2], np.uint8) for e in per])[inv]
        reason = np.array([e[3] for e in per], np.uint8)[inv]
        xrec = np.array([np.frombuffer(e[4], np.uint8) for e in per])[inv]
        signer = [per[k][5] for k in inv]
        (a0, p0), (a1, p1) = self.tables(W)
        idx = [{bytes(a): i for i, a in enumerate(a0)}, {bytes(a): i for i, a in enumerate(a1)}]
        pw = [[int.from_bytes(bytes(x), "big") for x in p0], [int.from_bytes(bytes(x), "big") for x in p1]]
        slots = self.group_slots(n_blocks)
        nv = np.zeros(ng, np.int64)
        voted = [set() for _ in range(ng)]
        for i in np.nonzero(bit)[0]:
            gi = int(g[i])
            nv[gi] += 1
            if slots[gi] != NO_TABLE:
                voted[gi].add(idx[slots[gi]][signer[i]])
        groups = []
        for gi in range(ng):
            if slots[gi] == NO_TABLE:
                groups.append((int(nv[gi]), set(), 0, False))
                continue
            ps = pw[slots[gi]]
            power = sum(ps[k] for k in voted[gi])
            groups.append((int(nv[gi]), voted[gi], power, power >= 2 * sum(ps) // 3 + 1))
        return dict(bit=bit, status=status, rec=rec, reason=reason, xrec=xrec, groups=groups)


@functools.lru_cache(maxsize=None)
def item_expectation(raw: bytes, arena: bytes, members: tuple):
    """(bit, status, recovered address, reason, explain address, signer) of one canonical item (group 0: a group with the table,
    1: a group without one, 2: no group)"""
    it = np.frombuffer(raw, co.ITEM_DTYPE)
    reasons, xrec = X.explain_batch(it, arena, [np.frombuffer(b"".join(members), np.uint8).reshape(-1, 20)], [0, NO_TABLE])
    why, got = X._signature_and_digest(it[0], arena)
    rec, signer = bytes(20), bytes(it[0]["signer"])
    if why is None:
        sig, z, signer = got
        rec = co.ecrecover_address(z, sig) or bytes(20)
    wire = int(it[0]["kind"]) in (X.KIND_WIRE, X.KIND_WIRE_SEAL)
    return bool(reasons[0] == X.OK), int(wire and why == X.NEEDS_HOST), rec, int(reasons[0]), bytes(xrec[0]), signer


@functools.lru_cache(maxsize=None)
def sweep() -> Sweep:
    return Sweep()


def bits(bm, n):
    return np.unpackbits(np.ascontiguousarray(bm, dtype=np.uint32).view(np.uint8), bitorder="little")[:n].astype(bool)
