"""Voting-power tables at the carry, borrow and compare edges of the 320-bit quorum arithmetic.

go-ibft keeps voting power as big.Int and decides quorum = floor(2 * total / 3) + 1 (core/validator_manager.go:130-135).  The
engine restates that in fixed 320-bit limbs: ibft_set_validators (total and quorum), k_quorum_reduce (a per-thread strided
add-with-carry, then a 1,024-way shared-memory tree that also carries), group_decision (the PREPARE rule's proposer addition and
the limb compare) and the host mirror's u320 (host/quorum.hpp).  Powers of 1 to 7 never carry, so each table here targets one
branch of that arithmetic.

Voting power does not enter a signature, so every table is a new `powers` array for a committed fixture (config2.npz /
config3.npz): same addresses, same items, same golden bitmap.  `patterns(fixture)` returns the tables; `expected()` is the
plain big-int answer per group and rule; `reduce_model()` replays the kernels limb by limb and records which branches a table
reaches, so that a coverage test can check every pattern reaches the branch it names."""
from __future__ import annotations

import os
import random
from dataclasses import dataclass, field

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
M64 = (1 << 64) - 1
MAX = (1 << 256) - 1                  # the largest voting power a 32-byte big-endian table entry holds
THREADS = 1024                        # IBFT_REDUCE_THREADS: validators t, t + 1024, ... are summed by reduce thread t
# quorum rules and proposer markers (include/ibft_verify.h; mirrored by engine.py)
DEFAULT, PREPREPARE, PREPARE = 0, 1, 2
PROPOSER_NONE, PROPOSER_UNSET = 0xFFFFFFFF, 0xFFFFFFFE
RULES = (DEFAULT, PREPREPARE, PREPARE)
ITEM_GROUP, ITEM_SIGNER = slice(118, 120), slice(96, 116)   # byte offsets in a 128-byte ibft_sig_item


def quorum(total: int) -> int:
    return 2 * total // 3 + 1


def load(name: str):
    """(fixture, items as raw 128-byte rows, votes) with votes[g] = (n_valid, set of voted validator indices) from the golden
    bitmap."""
    d = np.load(os.path.join(HERE, "golden", name))
    rows = np.ascontiguousarray(d["items"]).reshape(-1, 128)
    return d, rows, votes_of(rows, bits_of(d["bitmap"], len(rows)), d["addrs"], len(d["groups"]))


def bits_of(bitmap, n: int) -> np.ndarray:
    return np.unpackbits(np.ascontiguousarray(bitmap, dtype=np.uint32).view(np.uint8), bitorder="little")[:n]


def words_of(bits) -> np.ndarray:
    b = np.zeros((len(bits) + 31) // 32 * 32, np.uint8)
    b[: len(bits)] = bits
    return np.packbits(b, bitorder="little").view(np.uint32)


def votes_of(rows: np.ndarray, bits, addrs, n_groups: int):
    index = {bytes(a): i for i, a in enumerate(addrs)}
    groups = rows[:, ITEM_GROUP].copy().view("<u2").reshape(-1)
    out = [[0, set()] for _ in range(n_groups)]
    for i in np.nonzero(bits)[0]:
        g = int(groups[i])
        if g < n_groups:
            out[g][0] += 1
            v = index.get(bytes(rows[i, ITEM_SIGNER]))
            if v is not None:
                out[g][1].add(v)
    return [(nv, frozenset(vs)) for nv, vs in out]


def powers_be(powers) -> np.ndarray:
    return np.frombuffer(b"".join(int(p).to_bytes(32, "big") for p in powers), np.uint8).reshape(len(powers), 32).copy()


def limbs(x: int, k: int = 5) -> list[int]:
    return [(x >> (64 * i)) & M64 for i in range(k)]


def value(ls) -> int:
    return sum(int(x) << (64 * i) for i, x in enumerate(ls))


@dataclass
class Pattern:
    name: str
    powers: list                       # one int per validator, each in [0, 2^256 - 1]
    targets: set                       # branch events (reduce_model) the table exists to reach
    proposer: int = PROPOSER_NONE      # the PREPARE rule's proposer: a table index, PROPOSER_NONE or PROPOSER_UNSET
    rule: int = DEFAULT                # the rule under which `targets` are reached
    total: int = field(init=False)
    quorum: int = field(init=False)

    def __post_init__(self):
        assert all(0 <= p <= MAX for p in self.powers), self.name
        self.total = sum(self.powers)
        assert self.total > 0, self.name
        self.quorum = quorum(self.total)


def expected(pat: Pattern, votes, rule: int, proposer: int | None = None):
    """Per group: (n_valid, n_distinct, power, has_quorum) of hasQuorumByMsgType under `rule` (core/ibft.go:1273-1284,
    validator_manager.go:77-127), with `power` as the engine reports it: under the PREPARE rule the proposer's power joins the
    senders' sum when the proposer is a validator that did not send."""
    p = pat.proposer if proposer is None else proposer
    out = []
    for nv, vs in votes:
        s = sum(pat.powers[v] for v in vs)
        if rule == PREPREPARE:
            hq = nv >= 1
        elif rule == PREPARE:
            if p == PROPOSER_UNSET or (p != PROPOSER_NONE and p in vs):
                hq = False
            else:
                if p != PROPOSER_NONE:
                    s += pat.powers[p]
                hq = s >= pat.quorum
        else:
            hq = s >= pat.quorum
        out.append((nv, len(vs), s, hq))
    return out


def _add(a, b, tag, ev):
    """the kernels' 5-limb add-with-carry: t = a + b, c1 = t < b, t2 = t + c, c1 += t2 < c.  Returns the sum and whether the
    carry ran out of every one of limbs 0-3."""
    out, c, through = [], 0, True
    for k in range(5):
        t = (a[k] + b[k]) & M64
        c1 = int(t < b[k])
        t2 = (t + c) & M64
        c2 = int(t2 < c)
        if c1 and k < 4:
            ev.add(f"{tag}_carry_{k}")
        if c2:
            ev.add(f"{tag}_carry2")
        if (c1 or c2) and k == 4:
            ev.add(f"{tag}_overflow")             # would leave 320 bits: never reached by a table of 256-bit powers
        if k < 4 and not (c1 or c2):
            through = False
        out.append(t2)
        c = c1 + c2
    if through:
        ev.add(f"{tag}_through")
    return out, through


def reduce_model(pat: Pattern, voted, rule: int | None = None, proposer: int | None = None):
    """k_quorum_reduce + group_decision over one voted set, limb by limb.  Returns (power, has_quorum, events)."""
    rule = pat.rule if rule is None else rule
    p = pat.proposer if proposer is None else proposer
    n, ev = len(pat.powers), set()
    part = [[0] * 5 for _ in range(THREADS)]
    for t in range(THREADS):
        for v in range(t, n, THREADS):
            if v in voted:
                if pat.powers[v] == 0:
                    ev.add("zero_power_voter")
                part[t] = _add(part[t], limbs(pat.powers[v], 4) + [0], "thread", ev)[0]
    stride, first = THREADS // 2, None
    while stride:                                 # the shared-memory tree: thread t < stride adds thread t + stride
        for t in range(stride):
            before = len(ev)
            part[t], through = _add(part[t], part[t + stride], "tree", ev)
            if through:
                ev.add(f"tree_full_carry_{stride}")
            if len(ev) > before or through:
                first = first or stride
        stride //= 2
    if first:
        ev.add(f"tree_first_carry_{first}")
    power = part[0]
    q = limbs(pat.quorum)
    ev.add(f"total_mod3_{pat.total % 3}")
    if rule == PREPREPARE:
        return value(power), None, ev
    if rule == PREPARE:
        if p == PROPOSER_UNSET:
            return value(power), False, ev
        if p != PROPOSER_NONE:
            if p in voted:
                ev.add("proposer_among_senders")
                return value(power), False, ev
            power = _add(power, limbs(pat.powers[p], 4) + [0], "proposer", ev)[0]
        else:
            ev.add("proposer_none")
    for k in range(4, -1, -1):                    # group_decision's compare, from limb 4 down
        if power[k] != q[k]:
            ev.add(f"cmp_limb_{k}")
            return value(power), power[k] > q[k], ev
    ev.add("cmp_equal")
    return value(power), True, ev


def _spread(total: int, idx, rnd: random.Random) -> dict:
    """`total` over the validators `idx`, each share in [0, 2^256 - 1], unevenly"""
    idx = list(idx)
    k = len(idx)
    base, rem = divmod(total, k)
    assert base + 1 <= MAX or (base <= MAX and rem == 0), "total too large for the set"
    share = [base + (1 if i < rem else 0) for i in range(k)]
    room = min(base, MAX - base - 1)
    for i in range(0, k - 1, 2):                  # move a random amount between neighbours: sum unchanged
        if room > 0:
            m = rnd.randrange(room)
            share[i] -= m
            share[i + 1] += m
    assert sum(share) == total and all(0 <= s <= MAX for s in share)
    return dict(zip(idx, share))


def _table(n, *parts) -> list:
    pw = [0] * n
    for part in parts:
        for v, x in part.items():
            pw[v] = x
    return pw


def patterns(votes, n: int, seed: int = 1) -> list[Pattern]:
    """The power-edge tables for a fixture whose group 0 has the voted set votes[0][1] (n validators)."""
    rnd = random.Random(seed)
    voted = sorted(votes[0][1])
    absent = sorted(set(range(n)) - set(voted))
    assert len(voted) >= 32 and len(absent) >= 3, "the builder needs voters and non-voters"
    big = n > THREADS                              # several validators per reduce thread
    prop = absent[0]                               # default PREPARE proposer: a validator that did not send
    out = []

    def add(name, powers, targets, **kw):
        out.append(Pattern(name, powers, set(targets), **{"proposer": prop, **kw}))

    # every addition carries through limbs 0-3 into limb 4
    add("all-max", [MAX] * n, {"tree_carry_3"} | ({"thread_carry_3"} if big else set()))
    # 2^64 - 1, 2^128 - 1, 2^192 - 1 in turn: the partial sums carry out of each limb, and the carry-in term fires
    lvl = [(1 << 64) - 1, (1 << 128) - 1, (1 << 192) - 1]
    add("limb-edge", [lvl[i % 3] for i in range(n)],
        {f"{'thread' if big else 'tree'}_{e}" for e in ("carry_0", "carry_1", "carry_2", "carry2")})
    # the tree: two reduce threads a and a + s (a < s) hold 1 and 2^256 - 1, every other partial is 0; they meet at stride s,
    # and that step makes exactly 2^256 -- a carry out of every limb.  One absent validator brings the quorum to exactly 2^256.
    by_thread = {}
    for v in voted:
        by_thread.setdefault(v % THREADS, v)
    s = THREADS // 2
    while s:
        a = next(a for a in range(s) if a in by_thread and a + s in by_thread)
        add(f"tree-carry/s{s}", _table(n, {by_thread[a]: 1, by_thread[a + s]: MAX, absent[1]: (1 << 255) - 1}),
            {f"tree_full_carry_{s}", f"tree_first_carry_{s}", "cmp_equal"})
        s //= 2
    # exact threshold near 2^260 for every total mod 3: the voters hold exactly the quorum; in the twin table one voter holds
    # d less (d chosen so the twin's voters hold its quorum - 1)
    u = (1 << 259) + rnd.randrange(1 << 200)
    for r, dq in ((1, 1), (2, 2), (0, 3)):
        q = 2 * u + dq
        pw = _table(n, _spread(u, absent, rnd), _spread(q, voted, rnd))
        add(f"threshold/T%3={r}/at", pw, {f"total_mod3_{r}", "cmp_equal"})
        v0 = next(v for v in voted if pw[v] >= 3)
        for d in (1, 2, 3):
            if q - d == quorum(sum(pw) - d) - 1:
                break
        else:
            raise AssertionError("no twin table")
        twin = list(pw)
        twin[v0] -= d
        add(f"threshold/T%3={r}/short", twin, {f"total_mod3_{(sum(pw) - d) % 3}"})
    # quorum exactly 2^k: total 3 * 2^(k-1) - 1; voters 2^k - 1 (all lower limbs ones, decided at limb k/64) or 2^k
    for k in (64, 128, 192, 256):
        lo = _spread((1 << k) - 1, voted, rnd)
        add(f"limb-quorum/2^{k}/short", _table(n, _spread(1 << (k - 1), absent, rnd), lo), {f"cmp_limb_{k // 64}"})
        hi = dict(lo)
        hi[voted[0]] += 1
        assert hi[voted[0]] <= MAX
        add(f"limb-quorum/2^{k}/at", _table(n, _spread((1 << (k - 1)) - 1, absent, rnd), hi), {"cmp_equal"})
    # voters of power 0 count as distinct senders but add nothing
    half = {v: (0 if i % 2 == 0 else (1 << 250) + i) for i, v in enumerate(voted)}
    add("zero-power/some", _table(n, half, {v: 1 << 240 for v in absent}), {"zero_power_voter"})
    add("zero-power/all", _table(n, {v: 0 for v in voted}, {v: 5 for v in absent}), {"zero_power_voter", "cmp_limb_0"})
    # PREPARE: the absent proposer holds 2^256 - 1, the senders 2^256 + 1; its addition carries through every limb to 2^257,
    # which is the quorum, and one short of the twin table's quorum (one more unit of power outside the vote)
    senders = _spread((1 << 256) + 1, voted, rnd)
    for name, rest, tg in (("at", (1 << 256) - 1, "cmp_equal"), ("short", 1 << 256, "cmp_limb_0")):
        pw = _table(n, senders, _spread(rest, absent[1:], rnd), {absent[0]: MAX})
        add(f"prepare-carry/{name}", pw, {"proposer_carry_0", "proposer_carry2", "proposer_through", tg}, rule=PREPARE)
    pw = out[-2].powers
    add("prepare-carry/proposer-voted", pw, {"proposer_among_senders"}, rule=PREPARE, proposer=voted[len(voted) // 2])
    add("prepare-carry/proposer-none", pw, {"proposer_none"}, rule=PREPARE, proposer=PROPOSER_NONE)
    add("prepare-carry/proposer-unset", pw, set(), rule=PREPARE, proposer=PROPOSER_UNSET)
    return out


def coverage(pats, votes) -> dict:
    """name -> (targets reached?, missing targets, model agrees with the big-int sum?)"""
    rep = {}
    for p in pats:
        power, hq, ev = reduce_model(p, votes[0][1])
        want = expected(p, votes[:1], p.rule)[0]
        agrees = power == want[2] and (hq is None or hq == want[3]) and "thread_overflow" not in ev
        rep[p.name] = (p.targets <= ev, sorted(p.targets - ev), agrees)
    return rep
