"""Validator tables at the edges of the signer lookup, and a plain reference of what membership decides.

Between recovery and every verdict the engine finds the claimed signer in the group's validator table: ibft_set_validators sorts
the table and uploads each row as five big-endian words plus the validator index, and lookup_validator (engine.cu) binary-searches
those words.  The index it returns picks the voted bit, the power k_quorum_reduce adds, the PREPARE proposer rule's comparison and
the key registry entry a recovered key is learned into.  Addresses of independent random keys almost always differ in their first
word, so random tables never make the search decide on words 1-4.

This module builds tables whose members sit next to real signers: the 160-bit neighbours +-2^(8b), the signer with one byte set
to 0x00 or 0xFF, the zero and all-0xFF addresses.  Each signer sits at a chosen sorted rank with a chosen validator index; the
other signers are absent, and some are bracketed by the two addresses that differ from theirs in one word only, so that the
search must decide "not a member" on that word.  `reference()` decides membership with a dict from address to index, as
go-ibft's ValidatorManager does with its map (core/validator_manager.go), and `lookup_model()` replays lookup_validator's loop so
that a test can check that the lookups whose answer decides a verdict reach every branch of the compare."""
from __future__ import annotations

import functools
import random
from dataclasses import dataclass, field

import numpy as np

import adversarial as A
import workloads as wl
from oracle import coracle as co
from oracle import ibft_proto as ip
from oracle import secp256k1 as ec

MAX_VALIDATORS = 4096
SIZES = (1, 2, 3, 31, 32, 33, 63, 64, 65, 1023, 1024, 1025, 2047, 2048, 2049, MAX_VALIDATORS - 1, MAX_VALIDATORS)
RANKS = ("first", "second", "middle", "second_last", "last")
SEED = 0x6D656D62
SCAN = 4096
TOP = 1 << 160
HEIGHT = 77
DEFAULT, PREPREPARE, PREPARE = 0, 1, 2
# the signers: a real key whose address has byte `pos` equal to `val` -- a word's sign bit, and the two ends of the address space
SIGNER_BYTES = ((0, 0x00), (0, 0x7F), (0, 0x80), (0, 0xFF), (4, 0x7F), (4, 0x80), (8, 0x7F), (8, 0x80), (12, 0x7F), (12, 0x80),
                (16, 0x7F), (16, 0x80))


def a2i(a: bytes) -> int:
    return int.from_bytes(a, "big")


def i2a(x: int) -> bytes:
    return x.to_bytes(20, "big")


def words(a: bytes) -> tuple:
    return tuple(int.from_bytes(a[4 * i:4 * i + 4], "big") for i in range(5))


@functools.lru_cache(maxsize=None)
def signers() -> tuple:
    """((tag, private key, address), ...): the first of SCAN deterministic keys that matches each SIGNER_BYTES pattern"""
    privs = co.privkeys(SEED, SCAN)
    addrs = co.addresses(privs)
    out, used = [], set()
    for pos, val in SIGNER_BYTES:
        hit = next(i for i in range(SCAN) if addrs[i, pos] == val and i not in used)
        used.add(hit)
        d = int.from_bytes(bytes(privs[hit]), "big")
        assert wl.address_of(d) == bytes(addrs[hit])
        out.append((f"b{pos}={val:02x}", d, bytes(addrs[hit])))
    return tuple(out)


def decoys(a: bytes) -> list[bytes]:
    """addresses without a key next to `a`: +-2^(8b) for every byte b (+-1 and the +-2^32 word boundaries among them), `a` with one
    byte set to 0x00 or 0xFF, and the two ends of the address space"""
    x = a2i(a)
    out = set()
    for b in range(20):
        for y in (x + (1 << (8 * b)), x - (1 << (8 * b))):
            if 0 <= y < TOP:
                out.add(y)
        for val in (0x00, 0xFF):
            out.add(a2i(a[:b] + bytes([val]) + a[b + 1:]))
    out |= {0, TOP - 1}
    out.discard(x)
    return [i2a(y) for y in sorted(out)]


def rank_classes(r: int, n: int) -> set:
    return {name for name, want in zip(RANKS, (0, 1, n // 2, n - 2, n - 1)) if r == want}


@dataclass
class Table:
    n: int
    signer: int              # index into signers()
    brackets: dict           # index into signers() -> word k: a key whose address is not in the table while addr +- 2^(32 (4 - k)) are
    addrs: list              # validator index order
    powers: list
    zero_member: bool
    proposer: int            # the PREPARE rule's proposer for this table's group: 0, 31, 32 or n - 1
    index: dict = field(init=False)   # the reference: address -> validator index (go-ibft's map)

    def __post_init__(self):
        self.index = {a: v for v, a in enumerate(self.addrs)}
        assert len(self.index) == self.n, "a table lists an address twice"

    @property
    def signer_addr(self) -> bytes:
        return signers()[self.signer][2]

    @property
    def absent(self) -> list:
        """every other signer: its address is not in the table"""
        return [i for i in range(len(signers())) if i != self.signer]

    def sorted_rank(self, a: bytes) -> int:
        return sorted(self.addrs).index(a)

    def addr_array(self) -> np.ndarray:
        return np.frombuffer(b"".join(self.addrs), np.uint8).reshape(self.n, 20).copy()

    def power_array(self) -> np.ndarray:
        return np.frombuffer(b"".join(p.to_bytes(32, "big") for p in self.powers), np.uint8).reshape(self.n, 32).copy()


def bracket(a: bytes, k: int) -> tuple:
    """the two addresses that differ from `a` in word k alone, by one unit of that word"""
    d = 1 << (32 * (4 - k))
    lo, hi = i2a(a2i(a) - d), i2a(a2i(a) + d)
    for b in (lo, hi):
        assert [i for i in range(5) if words(b)[i] != words(a)[i]] == [k], (a.hex(), k)
    return lo, hi


def _filler(rnd, lo: int, hi: int, count: int, taken: set) -> list:
    out = []
    while len(out) < count:
        y = rnd.randrange(lo, hi)
        if y not in taken:
            taken.add(y)
            out.append(y)
    return out


BRACKET_WORDS = (4, 2, 0, 1, 3)   # the word of the +-1 neighbours first: the only bracket a table of 4 to 31 validators gets


def _table(j: int, n: int, rank: int, rnd: random.Random) -> Table:
    S = signers()
    si = j % len(S)
    s = a2i(S[si][2])
    # members that make a table interesting, most important first, each taken when it fits on its side of s: absent signers
    # bracketed by their neighbours in one word each (the search then decides on that word, both ways, to answer "not a
    # member"), then the zero address (the address a failed recovery leaves behind)
    cap = [rank, n - 1 - rank]
    must, brackets = [], {}
    for k in (BRACKET_WORDS if n >= 32 else BRACKET_WORDS[:1] if n >= 4 else ()):
        for step in range(1, len(S)):
            ti = (si + 4 + step) % len(S)
            if ti == si or ti in brackets:
                continue
            pair = [a2i(x) for x in bracket(S[ti][2], k)]
            if pair[0] < s < pair[1]:
                continue
            side = 0 if pair[1] < s else 1
            if cap[side] - (1 if side == 0 and n >= 5 else 0) >= 2:   # leave room below s for the zero address
                cap[side] -= 2
                must += pair
                brackets[ti] = k
                break
    if n >= 5 and cap[0] >= 1 and s > 0:
        must.append(0)
        cap[0] -= 1
    lo_m, hi_m = [m for m in must if m < s], [m for m in must if m > s]
    taken = {s} | {a2i(a) for _, _, a in S} | set(must)
    near = sorted((a2i(d) for d in decoys(S[si][2])), key=lambda y: abs(y - s))
    lo_d = [y for y in near if y < s and y not in taken][: rank - len(lo_m)]
    hi_d = [y for y in near if y > s and y not in taken][: n - 1 - rank - len(hi_m)]
    taken |= set(lo_d) | set(hi_d)
    lo_all = lo_m + lo_d + _filler(rnd, 0, s, rank - len(lo_m) - len(lo_d), taken)
    hi_all = hi_m + hi_d + _filler(rnd, s + 1, TOP, n - 1 - rank - len(hi_m) - len(hi_d), taken)
    assert len(lo_all) == rank and len(hi_all) == n - 1 - rank
    # the signer's validator index: 0, 31, 32 or n - 1 in turn, the others in shuffled order -- never the sorted order
    choices = sorted({v for v in (0, 31, 32, n - 1) if v < n})
    v_s = choices[j % len(choices)]
    others = lo_all + hi_all
    while True:
        rnd.shuffle(others)
        addrs = [i2a(y) for y in others]
        addrs.insert(v_s, S[si][2])
        if n < 3 or addrs != sorted(addrs):
            break
    # distinct powers below 2^256; every other table's signer outweighs everyone else, so that its vote alone reaches quorum
    powers = set()
    while len(powers) < n:
        powers.add(rnd.getrandbits(200) + 1)
    powers = sorted(powers)
    rnd.shuffle(powers)
    if j % 2 == 0:
        powers[v_s] = (1 << 255) + j
    assert len(set(powers)) == n and all(0 < p < 1 << 256 for p in powers)
    return Table(n, si, brackets, addrs, powers, zero_member=0 in must, proposer=choices[(j // 2) % len(choices)])


@functools.lru_cache(maxsize=None)
def tables() -> tuple:
    """one table per (size, rank) of SIZES x {0, 1, n // 2, n - 2, n - 1} (ranks that coincide at small n once), signers in turn"""
    rnd = random.Random(SEED)
    out = []
    for n in SIZES:
        ranks = sorted({r for r in (0, 1, n // 2, n - 2, n - 1) if 0 <= r < n})
        for rank in ranks:
            out.append(_table(len(out), n, rank, rnd))
    return tuple(out)


# ----------------------------------------------------------------------------------------------------------- items
DIGEST = co.keccak256(b"membership edges")


@functools.lru_cache(maxsize=None)
def signature(i: int) -> bytes:
    return wl.sign(signers()[i][1], DIGEST)


def failed_recoveries() -> list:
    """(tag, sig65, digest) whose recovery fails: r = 0, r not an abscissa (5^3 + 7 is not a square), and u1 G + u2 R = -G + G"""
    inf = A.recover_vector("infinity", ec.G, -1, 1)
    assert inf.key is None and 0 < int.from_bytes(inf.sig[:32], "big") < ec.N
    s1 = (1).to_bytes(32, "big")
    return [("r_zero", bytes(32) + s1 + b"\x00", DIGEST), ("r_not_x", (5).to_bytes(32, "big") + s1 + b"\x00", DIGEST),
            ("infinity", inf.sig, inf.digest)]


@dataclass
class Batch:
    items: np.ndarray        # ITEM_DTYPE, group g = table g
    tags: list               # per item: (case, claimed address)
    recovered: list          # per item: the address recovery yields, or None


def digest_batch() -> Batch:
    """per table: (a) the signer's signature claiming itself, (b) the same signature claiming each of its decoys, (c) every other
    signer's signature claiming itself (absent from the table; bracketed ones also claiming their two neighbours), (d) failed
    recoveries claiming the zero address"""
    S = signers()
    rows, tags, rec = [], [], []

    def add(case, sig, digest, claim, g, who):
        rows.append(wl.make_item(sig, claim, wl.KIND_DIGEST, digest, group=g))
        tags.append((case, claim))
        rec.append(who)

    for g, t in enumerate(tables()):
        sa = S[t.signer][2]
        add("a", signature(t.signer), DIGEST, sa, g, sa)
        for d in decoys(sa):
            add("b", signature(t.signer), DIGEST, d, g, sa)
        for ti in t.absent:
            ta = S[ti][2]
            add("c", signature(ti), DIGEST, ta, g, ta)
            if ti in t.brackets:
                for claim in bracket(ta, t.brackets[ti]):
                    add("c", signature(ti), DIGEST, claim, g, ta)
        for _, sig, dig in failed_recoveries():
            add("d", sig, dig, bytes(20), g, None)
    return Batch(np.concatenate(rows), tags, rec)


def wire_frame(d: int, claim: bytes, rnd: int = 0) -> bytes:
    m = ip.IbftMessage(view=ip.View(HEIGHT, rnd), from_=claim, type=ip.PREPARE, payload=ip.PrepareMessage(proposal_hash=DIGEST))
    m.signature = wl.sign(d, co.keccak256(m.payload_no_sig()))
    return ip.encode_ibft_message(m)


@functools.lru_cache(maxsize=None)
def wire_batch():
    """(items, arena): IBFT_KIND_WIRE PREPARE frames per table -- the signer claiming itself and its two nearest decoys, each
    bracketed absent signer claiming itself and its neighbours"""
    S = signers()
    arena = bytearray()
    rows, tags, rec = [], [], []
    for g, t in enumerate(tables()):
        sa = S[t.signer][2]
        near = sorted(decoys(sa), key=lambda a: abs(a2i(a) - a2i(sa)))[:2]
        frames = [(S[t.signer][1], c, sa) for c in [sa] + near]
        for ti, k in t.brackets.items():
            frames += [(S[ti][1], c, S[ti][2]) for c in (S[ti][2],) + bracket(S[ti][2], k)]
        for d, claim, who in frames:
            f = wire_frame(d, claim)
            it = np.zeros(1, dtype=co.ITEM_DTYPE)
            it["kind"], it["payload_off"], it["payload_len"], it["group"] = 3, len(arena), len(f), g
            arena.extend(f)
            rows.append(it)
            tags.append(("wire", claim))
            rec.append(who)
    return Batch(np.concatenate(rows), tags, rec), np.frombuffer(bytes(arena), np.uint8).copy()


def reference(batch: Batch, tabs=None, rule: int = DEFAULT, proposers=None, reps: int = 1):
    """go-ibft with a map: per item the verdict, per group (n_valid, n_distinct, power, has_quorum) and the voted index set.
    `reps`: the batch was tiled that many times.  proposers: per group, the PREPARE rule's proposer (validator index)."""
    tabs = tables() if tabs is None else tabs
    bits = np.zeros(len(batch.items), bool)
    votes = [[0, set()] for _ in tabs]
    for i, it in enumerate(batch.items):
        g, claim = int(it["group"]), batch.tags[i][1]
        v = tabs[g].index.get(claim)
        if batch.recovered[i] is not None and batch.recovered[i] == claim and v is not None:
            bits[i] = True
            votes[g][0] += reps
            votes[g][1].add(v)
    results = []
    for g, (nv, vs) in enumerate(votes):
        t = tabs[g]
        q = 2 * sum(t.powers) // 3 + 1
        s = sum(t.powers[v] for v in vs)
        if rule == PREPREPARE:
            hq = nv >= 1
        elif rule == PREPARE:
            p = t.proposer if proposers is None else proposers[g]
            hq = p not in vs and s + t.powers[p] >= q
            s += 0 if p in vs else t.powers[p]
        else:
            hq = s >= q
        results.append((nv, len(vs), s, hq))
    return bits, results, [frozenset(vs) for _, vs in votes]


def voted_words(voted, tabs=None):
    tabs = tables() if tabs is None else tabs
    stride = (max(t.n for t in tabs) + 31) // 32
    out = np.zeros((len(tabs), stride), np.uint32)
    for g, vs in enumerate(voted):
        for v in vs:
            out[g, v >> 5] |= np.uint32(1 << (v & 31))
    return out


# ---------------------------------------------------------------------------------------------------- coverage model
def lookup_model(sorted_rows, a: bytes, ev: set):
    """engine.cu lookup_validator line for line over [(5 words, validator index)] in sorted order: the index or -1.  Records
    ("word", i, -1 / +1) when word i decides a probe (table row below / above the address), ("hit", "first") / ("hit", "last") when
    the hit is the first probe / the probe at lo == hi, and ("miss", "low") / ("miss", "high") for a search that runs off an end."""
    aw = words(a)
    lo, hi = 0, len(sorted_rows) - 1
    first = True
    while lo <= hi:
        mid = (lo + hi) >> 1
        k, v = sorted_rows[mid]
        cmp = 0
        for i in range(5):
            if cmp == 0 and k[i] != aw[i]:
                cmp = -1 if k[i] < aw[i] else 1
                ev.add(("word", i, cmp))
        if cmp == 0:
            if first:
                ev.add(("hit", "first"))
            if lo == hi:
                ev.add(("hit", "last"))
            return v
        lo, hi = (mid + 1, hi) if cmp < 0 else (lo, mid - 1)
        first = False
    ev.add(("miss", "low" if hi < 0 else "high" if lo == len(sorted_rows) else "inner"))
    return -1


REQUIRED = {("word", i, c) for i in range(5) for c in (-1, 1)} | {("hit", "first"), ("hit", "last"), ("miss", "low"),
                                                                   ("miss", "high")}


def sorted_rows(t: Table):
    """ibft_set_validators' upload: rows sorted by address bytes (ties by index, which a refused duplicate never leaves)"""
    return [(words(t.addrs[v]), v) for v in sorted(range(t.n), key=lambda v: (t.addrs[v], v))]


def coverage(batch: Batch) -> set:
    """the lookup branches reached by the items whose verdict the lookup decides: those whose signature recovers the claimed
    address (for the others recovery already says no, whatever the search answers).  Asserts that the model answers as the dict."""
    ev = set()
    rows = [sorted_rows(t) for t in tables()]
    for i, it in enumerate(batch.items):
        g, claim = int(it["group"]), batch.tags[i][1]
        if batch.recovered[i] != claim:
            continue
        got = lookup_model(rows[g], claim, ev)
        assert got == tables()[g].index.get(claim, -1), (g, claim.hex())
    return ev
