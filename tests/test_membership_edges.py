"""The membership-edge tables of tests/membership_edges.py on the CPU: the generator builds what it promises, the tables reach
every branch of lookup_validator's compare (replayed line for line), the C oracle's own search agrees with the dict reference at
these edges, and the C++ host mirror refuses a table that lists an address twice."""
import importlib

import numpy as np
import pytest

import explain_oracle as eo
import membership_edges as me
from oracle import coracle as co

host = importlib.import_module("go-ibft_b200.host")


def test_signers_put_sign_bits_and_address_ends_under_test():
    S = me.signers()
    assert len({a for _, _, a in S}) == len(me.SIGNER_BYTES)
    for (pos, val), (_, d, a) in zip(me.SIGNER_BYTES, S):
        assert a[pos] == val and 0 < d < me.ec.N


def test_decoys_are_the_neighbours_and_byte_edges():
    for _, _, a in me.signers():
        x, ds = me.a2i(a), {me.a2i(d) for d in me.decoys(a)}
        assert x not in ds and {0, me.TOP - 1} <= ds
        assert {x + 1, x - 1, x + (1 << 32), x - (1 << 32), x + (1 << 128), x - (1 << 128)} <= ds
        for b in range(20):
            assert me.a2i(a[:b] + b"\x00" + a[b + 1:]) in ds | {x}
            assert me.a2i(a[:b] + b"\xff" + a[b + 1:]) in ds | {x}


def test_tables_sizes_ranks_indices_and_powers():
    T = me.tables()
    assert {t.n for t in T} == set(me.SIZES)
    reached = {}
    for j, t in enumerate(T):
        sa = t.signer_addr
        assert len(set(t.addrs)) == t.n and len(t.powers) == t.n and len(set(t.powers)) == t.n      # no duplicates
        assert all(0 < p < 1 << 256 for p in t.powers)
        assert all(me.signers()[i][2] not in t.index for i in t.absent)
        v = t.index[sa]
        assert v in (0, 31, 32, t.n - 1)
        assert t.proposer in (0, 31, 32, t.n - 1)
        r = t.sorted_rank(sa)
        classes = me.rank_classes(r, t.n)
        assert classes, (t.n, r)
        for c in classes:
            reached.setdefault(t.n, set()).add(c)
        if t.n >= 3:
            assert sorted(range(t.n), key=lambda i: t.addrs[i]) != list(range(t.n)), "index order must differ from sorted order"
        rows = sorted(t.addrs)
        for ti, k in t.brackets.items():
            # the bracket is the absent key's nearest pair of members: the search ends between them, on word k
            ta = me.signers()[ti][2]
            lo, hi = me.bracket(ta, k)
            i = next((i for i, a in enumerate(rows) if a > ta), len(rows))
            assert rows[i - 1] == lo and rows[i] == hi, (j, ti, k)
        assert t.zero_member == (bytes(20) in t.index)
    for n in me.SIZES:
        assert reached[n] == set(me.RANKS) if n >= 4 else reached[n] >= {"first", "last"}, n
    # every signer index and proposer choice; from 31 validators on, brackets and a member zero address at every size, and from
    # 32 on a bracket in each of the five words
    assert {t.index[t.signer_addr] for t in T if t.n >= 64} >= {0, 31, 32} and any(t.index[t.signer_addr] == t.n - 1 for t in T)
    for n in me.SIZES[3:]:
        assert any(t.brackets for t in T if t.n == n) and any(t.zero_member for t in T if t.n == n), n
        if n >= 32:
            assert set().union(*(t.brackets.values() for t in T if t.n == n)) == set(range(5)), n
    # every signer is used at three ranks or more; the signer's vote alone reaches quorum in half the tables
    for i in range(len(me.signers())):
        ranks = set().union(*(me.rank_classes(t.sorted_rank(t.signer_addr), t.n) for t in T if t.signer == i))
        assert len(ranks) >= 3, (i, ranks)
    assert sum(t.powers[t.index[t.signer_addr]] >= 2 * sum(t.powers) // 3 + 1 for t in T) >= len(T) // 2


def test_lookup_model_reaches_every_branch():
    batch = me.digest_batch()
    ev = me.coverage(batch)
    missing = me.REQUIRED - ev
    print("lookup branches reached:", sorted(ev))
    assert not missing, sorted(missing)
    # the wire frames (k_quorum_mark's own lookup): every word decides, both ways, and hits on the first and the last probe
    wb, _ = me.wire_batch()
    assert me.coverage(wb) >= me.REQUIRED - {("miss", "low"), ("miss", "high")}


def mutant_lookup(sorted_rows, a: bytes, skip=None, signed=False):
    """lookup_validator with one word left out of the compare, or with the words compared as signed integers"""
    aw = me.words(a)
    lo, hi = 0, len(sorted_rows) - 1
    while lo <= hi:
        mid = (lo + hi) >> 1
        k, v = sorted_rows[mid]
        cmp = 0
        for i in range(5):
            x, y = (k[i] ^ 0x80000000, aw[i] ^ 0x80000000) if signed else (k[i], aw[i])
            if i != skip and cmp == 0 and x != y:
                cmp = -1 if x < y else 1
        if cmp == 0:
            return v
        lo, hi = (mid + 1, hi) if cmp < 0 else (lo, mid - 1)
    return -1


@pytest.mark.parametrize("mutant", ["skip0", "skip1", "skip2", "skip3", "skip4", "signed"])
def test_a_wrong_compare_changes_a_verdict(mutant):
    """a search that leaves any one word out of the compare, or compares signed, answers differently from the dict on items whose
    verdict the lookup decides (their signature recovers the claimed address), in both the digest and the frame batches"""
    skip, signed = (None, True) if mutant == "signed" else (int(mutant[-1]), False)
    rows = [me.sorted_rows(t) for t in me.tables()]
    for batch in (me.digest_batch(), me.wire_batch()[0]):
        wrong = 0
        for i, it in enumerate(batch.items):
            g, claim = int(it["group"]), batch.tags[i][1]
            if batch.recovered[i] == claim:
                wrong += mutant_lookup(rows[g], claim, skip, signed) != me.tables()[g].index.get(claim, -1)
        assert wrong > 0, mutant


def test_items_cover_the_four_cases():
    batch = me.digest_batch()
    bits, res, voted = me.reference(batch)
    cases = {}
    for i, (case, _) in enumerate(batch.tags):
        cases.setdefault(case, []).append(bool(bits[i]))
    assert all(cases["a"]) and not any(cases["b"]) and not any(cases["c"]) and not any(cases["d"])
    assert [len(v) for v in voted] == [1] * len(me.tables())
    assert any(r[3] for r in res) and not all(r[3] for r in res)


def test_c_oracle_search_matches_the_dict():
    batch = me.digest_batch()
    want, _, _ = me.reference(batch)
    tabs = [t.addr_array() for t in me.tables()]
    got = co.verify_batch(batch.items, b"", tables=tabs, group_table=list(range(len(tabs))), n_threads=8)
    bits = np.unpackbits(got.view(np.uint8), bitorder="little")[: len(batch.items)].astype(bool)
    assert np.array_equal(bits, want)


def test_explain_oracle_matches_the_dict_on_frames():
    """the wire frames, through tests/explain_oracle.py's codec and recovery: reason OK exactly where the dict says valid"""
    wb, arena = me.wire_batch()
    want, _, _ = me.reference(wb)
    tabs = [t.addr_array() for t in me.tables()]
    reasons, rec = eo.explain_batch(wb.items, arena.tobytes(), tabs, list(range(len(tabs))))
    assert np.array_equal(reasons == eo.OK, want)
    assert [bytes(r) for r in rec] == wb.recovered
    assert set(reasons.tolist()) == {eo.OK, eo.SIGNER_MISMATCH, eo.NOT_VALIDATOR}


@pytest.mark.parametrize("where", ["adjacent", "far"])
def test_host_mirror_refuses_a_table_that_lists_an_address_twice(where):
    """ValidatorManager's input is a map: the mirror refuses a duplicate (IBFT_ERR_INVALID_ARG) and keeps its previous table"""
    ctx = host.HostContext("callback")
    names = [b"v%03d" % i for i in range(40)]
    assert ctx.set_validators(0, names, [1] * 40) == 0
    dup = list(names)
    dup[1 if where == "adjacent" else 39] = dup[0]
    assert ctx.set_validators(0, dup, [1000] + [1] * 39) == 1
    assert ctx.set_validators(0, dup, None) == 1
    # the previous table still decides: 27 of 40 unit powers is a quorum, 26 is not
    assert ctx.has_quorum_senders(names[:27]) and not ctx.has_quorum_senders(names[:26])
    ctx.close()
