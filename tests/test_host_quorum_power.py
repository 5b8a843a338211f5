"""The C++ host mirror's 320-bit voting-power arithmetic (host/quorum.hpp u320: add, sub, quorum, cmp) on the power-edge tables
of tests/power_edges.py, against the big-int restatement and oracle/ibft_logic.py.  CPU only."""
import functools
import importlib
import random

import numpy as np
import pytest

import power_edges as pe
from oracle import ibft_logic as L
from oracle import ibft_proto as ip
from test_host_logic import Dual
from test_oracle_logic import HASH

host = importlib.import_module("go-ibft_b200.host")
FIXTURES = ["config2.npz", "config3.npz"]
FAMILIES = {"all-max", "limb-edge", "tree-carry", "threshold", "limb-quorum", "zero-power", "prepare-carry"}


@functools.lru_cache(maxsize=None)
def fixture(name):
    d, _, votes = pe.load(name)
    return [bytes(a) for a in d["addrs"]], votes, pe.patterns(votes, len(d["addrs"]))


@pytest.mark.parametrize("name", FIXTURES)
def test_power_edge_patterns_reach_their_branches(name):
    """Every table reaches the branch it is named for in the limb-by-limb model of k_quorum_reduce / group_decision, and the
    model's sum and decision equal the big-int ones."""
    _, votes, pats = fixture(name)
    rep = pe.coverage(pats, votes)
    assert {p.name.split("/")[0] for p in pats} == FAMILIES
    assert {k for k in rep if k.startswith("tree-carry/")} == {f"tree-carry/s{1 << i}" for i in range(10)}
    assert not {k: v for k, v in rep.items() if not (v[0] and v[2])}
    by_name = {p.name: p for p in pats}
    assert by_name["all-max"].total.bit_length() >= 266
    for k in (64, 128, 192, 256):
        assert by_name[f"limb-quorum/2^{k}/short"].quorum == by_name[f"limb-quorum/2^{k}/at"].quorum == 1 << k
    for r in (0, 1, 2):
        at, short = by_name[f"threshold/T%3={r}/at"], by_name[f"threshold/T%3={r}/short"]
        assert at.total % 3 == r and at.total.bit_length() in (260, 261)
        assert sum(a != b for a, b in zip(at.powers, short.powers)) == 1         # the twins differ in one voter's power
        s_at, s_short = (sum(p.powers[v] for v in votes[0][1]) for p in (at, short))
        assert (s_at, s_short) == (at.quorum, short.quorum - 1)


@pytest.mark.parametrize("name", FIXTURES)
def test_host_mirror_decides_power_edges(name):
    """HasQuorum over the address set and over the voted-set words (HasQuorumVoted), and HasPrepareQuorum's sender set (the
    senders plus the proposer), for every group of every table: the C++ u320 against Python's big ints and the oracle."""
    addrs, votes, pats = fixture(name)
    for p in pats:
        ctx = host.HostContext("callback")
        assert ctx.set_validators(0, addrs, p.powers) == 0
        vm = L.ValidatorManager(lambda h, p=p: dict(zip(addrs, p.powers)))
        vm.init(0)
        assert vm.quorum_size == p.quorum
        for nv, vs in votes:
            senders = [addrs[v] for v in sorted(vs)]
            want = pe.expected(p, [(nv, vs)], pe.DEFAULT)[0][3]
            bits = np.zeros(len(addrs), np.uint8)
            bits[sorted(vs)] = 1
            got = (vm.has_quorum(senders), ctx.has_quorum_senders(senders), ctx.has_quorum_voted(pe.words_of(bits)))
            assert got == (want,) * 3, (p.name, got, want)
            if p.proposer < len(addrs) and p.proposer not in vs:
                want_p = pe.expected(p, [(nv, vs)], pe.PREPARE)[0][3]
                assert ctx.has_quorum_senders(senders + [addrs[p.proposer]]) == want_p, p.name
        ctx.close()


LEVELS = [(1 << 64) - 1, (1 << 128) - 1, (1 << 192) - 1, (1 << 256) - 1]


def test_incremental_accumulators_carry_and_borrow_at_huge_powers():
    """The store's per-view power accumulators (u320 add on insert, sub when GetValidMessages prunes) at powers just below a
    limb boundary, where almost every add carries and almost every prune borrows: AddMessage must signal exactly when the
    reference's recompute-everything path does -- with zero-power validators, pruning, unknown senders and table swaps
    mid-round."""
    rnd = random.Random(2026)
    for trial in range(32):
        lvl = LEVELS[trial % 4]
        n = rnd.randint(4, 10)

        def table():
            pw = {b"node %d" % i: rnd.choice([lvl, lvl, lvl - 1, lvl - rnd.randrange(1 << 32), 1, 0]) for i in range(n)}
            pw[b"node 1"] = lvl
            return pw
        powers = table()
        d = Dual(n, powers=powers, is_valid_proposal_hash=lambda p, h: h == HASH)
        d.c.set_incremental_quorum(True)
        proposal = ip.IbftMessage(ip.View(3, 0), b"node 0", b"", ip.PREPREPARE, ip.PrePrepareMessage(ip.Proposal(b"b", 0), HASH))
        d.set_state(3, 0, L.PREPARE_STATE if rnd.random() < 0.7 else L.NEW_ROUND, proposal if rnd.random() < 0.8 else None)
        for step in range(40):
            who = b"node %d" % rnd.randint(0, n + 1)                  # includes two non-validators
            t = rnd.choice([ip.PREPARE, ip.PREPARE, ip.COMMIT, ip.ROUND_CHANGE, ip.PREPREPARE])
            view = ip.View(3, rnd.choice([0, 0, 0, 1]))
            payload = {ip.PREPARE: ip.PrepareMessage(HASH if rnd.random() < 0.7 else b"x"), ip.COMMIT: ip.CommitMessage(HASH, b"s"),
                       ip.ROUND_CHANGE: ip.RoundChangeMessage(), ip.PREPREPARE: ip.PrePrepareMessage(ip.Proposal(b"b", 0), HASH)}[t]
            d.add_message(ip.IbftMessage(view, who, bytes([step]), t, payload))
            assert d.c.signal_count() == len(d.o.messages.signals), (trial, step)
            if rnd.random() < 0.25:
                d.handle_prepare(3, 0)                                   # prunes bad-hash PREPAREs: the accumulators subtract
                d.set_state(3, 0, L.PREPARE_STATE, proposal)
            if step == 20 or rnd.random() < 0.05:                        # the validator table is swapped mid-round
                powers = table()
                d.vm.set_current_voting_power(powers)
                names = sorted(powers)
                assert d.c.set_validators(3, names, [powers[k] for k in names]) == 0
