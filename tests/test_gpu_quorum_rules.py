"""Quorum rules per message type (ibft_group_desc.flags bits 0-1, proposer in ibft_group_desc.reserved): a PREPARE group's
has_quorum is HasPrepareQuorum and a PREPREPARE group's is "at least one valid message" (hasQuorumByMsgType, reference
core/ibft.go:1273-1284) on every reduce path -- host-buffer calls on all four recover kernels, the key registry, the
device-resident reduce, the shard-local marks + merge and both ShardedVerifier exchanges.  Expected values come from the oracle
(oracle/ibft_logic.py) fed with the messages whose verdict the oracle itself computed."""
import functools
import importlib

import numpy as np
import pytest
import torch

import ibft_b200 as ib
from oracle import coracle as co
from oracle import ibft_logic as L
from oracle import ibft_proto as ip

pytestmark = pytest.mark.gpu
sharding = importlib.import_module("go-ibft_b200.sharding")

SLOT_BIG, SLOT_UNIT = 12, 13
HEIGHT_BIG, HEIGHT_UNIT = 7_000_001, 7_000_002
N_BIG = 10_000
RULE_TYPE = {ib.QUORUM_DEFAULT: ip.COMMIT, ib.QUORUM_PREPREPARE: ip.PREPREPARE, ib.QUORUM_PREPARE: ip.PREPARE}


class Table:
    def __init__(self, seed, n, weighted, height):
        self.privs = co.privkeys(seed, n)
        self.addrs = co.addresses(self.privs)
        self.powers = [1 + (i % 7) if weighted else 1 for i in range(n)]   # config 3's weights
        self.powers_be = np.frombuffer(b"".join(p.to_bytes(32, "big") for p in self.powers), np.uint8).reshape(n, 32).copy()
        self.quorum = 2 * sum(self.powers) // 3 + 1
        self.height, self.n = height, n
        self.digest = co.keccak256(b"quorum-rules" + height.to_bytes(8, "big"))
        self.sigs = co.sign_derived_batch(self.privs, np.tile(np.frombuffer(self.digest, np.uint8), (n, 1)))

    def addr(self, i):
        return bytes(self.addrs[i])

    def senders(self, target, exclude=()):
        """validators (none of `exclude`) whose powers sum to exactly `target`"""
        out, acc = [], 0
        for i in sorted(range(self.n), key=lambda i: -self.powers[i]):
            if i in exclude or acc + self.powers[i] > target:
                continue
            out.append(i)
            acc += self.powers[i]
            if acc == target:
                return out
        raise AssertionError("no sender set of that power")


def item(tab, sig, signer, group):
    it = np.zeros(1, dtype=ib.ITEM_DTYPE)
    it["r"][0] = np.frombuffer(bytes(sig[:32]), np.uint8)
    it["s"][0] = np.frombuffer(bytes(sig[32:64]), np.uint8)
    it["v"][0] = sig[64]
    it["digest"][0] = np.frombuffer(tab.digest, np.uint8)
    it["signer"][0] = np.frombuffer(signer, np.uint8)
    it["kind"][0] = ib.KIND_DIGEST
    it["group"][0] = group
    return it


@functools.lru_cache(maxsize=None)
def scenario():
    """Groups of a 10k weighted table and a 4-validator unit table.  Each: (table, rule, proposer, proposer address for the
    oracle or None, items).  Returns the groups' specs, the items, and the oracle's verdict bitmap and expected results."""
    big, unit = Table(41, N_BIG, True, HEIGHT_BIG), Table(42, 4, False, HEIGHT_UNIT)
    outsider_priv = co.privkeys(9998, 1)
    outsider = bytes(co.addresses(outsider_priv)[0])
    outsider_sig = co.sign_derived_batch(outsider_priv, np.frombuffer(unit.digest, np.uint8).reshape(1, 32))[0]
    Q, p = big.quorum, 3
    specs = []   # (table, rule, proposer, [(validator index or None, kind)])

    def valid(idx):
        return [(i, "ok") for i in idx]
    P = ib.QUORUM_PREPARE
    # PREPARE, proposer absent: the senders reach the quorum only together with the proposer -- exactly, and one unit short
    specs.append((big, P, p, valid(big.senders(Q - big.powers[p], {p}))))
    specs.append((big, P, p, valid(big.senders(Q - big.powers[p] - 1, {p}))))
    # the proposer's own PREPARE is valid, every validator signs: false
    specs.append((big, P, p, valid(range(N_BIG))))
    # the proposer's PREPARE is present but invalid (bad signature / From != signer): treated as absent
    specs.append((big, P, p, valid(big.senders(Q - big.powers[p], {p})) + [(p, "bad_sig")]))
    specs.append((big, P, p, valid(big.senders(Q - big.powers[p], {p})) + [(p, "from_ne_signer")]))
    # the proposer is not a validator of the table / there is no proposal message
    specs.append((big, P, ib.PROPOSER_NONE, valid(big.senders(Q))))
    specs.append((big, P, ib.PROPOSER_UNSET, valid(big.senders(Q))))
    # proposers at the table's first and last index
    specs.append((big, P, 0, valid(big.senders(Q - big.powers[0], {0}))))
    specs.append((big, P, N_BIG - 1, valid(big.senders(Q - big.powers[N_BIG - 1], {N_BIG - 1}))))
    # rule 0 groups in the same call: the first group's senders without the proposer rule (false), and a plain quorum (true)
    specs.append((big, ib.QUORUM_DEFAULT, 0, valid(big.senders(Q - big.powers[p], {p}))))
    specs.append((big, ib.QUORUM_DEFAULT, 0, valid(big.senders(Q))))
    # PREPREPARE: no items, one valid item, only invalid items, one valid item from a non-member
    PP = ib.QUORUM_PREPREPARE
    specs.append((unit, PP, 0, []))
    specs.append((unit, PP, 0, [(2, "ok")]))
    specs.append((unit, PP, 0, [(1, "bad_sig"), (2, "from_ne_signer")]))
    specs.append((unit, PP, 0, [(None, "outsider")]))
    # the unit table: PREPARE with the proposer absent (2 senders + proposer = quorum 3) and present; rule 0 at 3 and 2
    specs.append((unit, P, 1, valid([0, 2])))
    specs.append((unit, P, 1, valid([0, 1, 2, 3])))
    specs.append((unit, ib.QUORUM_DEFAULT, 0, valid([0, 2, 3])))
    specs.append((unit, ib.QUORUM_DEFAULT, 0, valid([0, 2])))

    items = []
    for g, (tab, rule, prop, its) in enumerate(specs):
        for i, kind in its:
            if kind == "ok":
                items.append(item(tab, tab.sigs[i], tab.addr(i), g))
            elif kind == "bad_sig":
                sig = tab.sigs[i].copy()
                sig[5] ^= 1
                items.append(item(tab, sig, tab.addr(i), g))
            elif kind == "from_ne_signer":                      # From = validator i, signed by another validator
                items.append(item(tab, tab.sigs[(i + 1) % tab.n], tab.addr(i), g))
            else:
                items.append(item(tab, outsider_sig, outsider, g))
    items = np.concatenate(items)
    group_table = [0 if s[0] is big else 1 for s in specs]
    bitmap = co.verify_batch(items, b"", tables=[big.addrs, unit.addrs], group_table=group_table, n_threads=16)
    ok = [(int(bitmap[i >> 5]) >> (i & 31)) & 1 == 1 for i in range(len(items))]
    # the oracle's decisions over the messages the oracle found valid
    view = ip.View(0, 0)
    vms = {}
    for tab in (big, unit):
        vm = L.ValidatorManager(lambda h, t=tab: {t.addr(i): t.powers[i] for i in range(t.n)})
        vm.init(tab.height)
        vms[id(tab)] = vm
    expected = np.zeros(len(specs), dtype=ib.RESULT_DTYPE)
    for g, (tab, rule, prop, _) in enumerate(specs):
        froms = [bytes(items[i]["signer"]) for i in range(len(items)) if ok[i] and int(items[i]["group"]) == g]
        index = {tab.addr(i): i for i in range(tab.n)}
        o = L.IBFT(L.Backend(), vms[id(tab)])
        if rule == ib.QUORUM_PREPARE and prop != ib.PROPOSER_UNSET:
            o.state.proposal_message = ip.IbftMessage(view, outsider if prop == ib.PROPOSER_NONE else tab.addr(prop), b"", ip.PREPREPARE)
        msgs = [ip.IbftMessage(view, f, b"", RULE_TYPE[rule]) for f in froms]
        voted = {index[f] for f in froms}
        power = sum(tab.powers[v] for v in voted)
        if rule == ib.QUORUM_PREPARE and prop < tab.n and prop not in voted:
            power += tab.powers[prop]                       # the proposer joins the sender set
        expected[g]["power"][0] = power                     # every sum here fits one limb
        expected[g]["n_valid"] = len(froms)
        expected[g]["n_distinct"] = len(voted)
        expected[g]["has_quorum"] = int(o.has_quorum_by_msg_type(msgs, RULE_TYPE[rule]))
    return dict(big=big, unit=unit, specs=specs, items=items, bitmap=bitmap, expected=expected, ok=ok)


def set_tables(eng, sc):
    for slot, tab in ((SLOT_BIG, sc["big"]), (SLOT_UNIT, sc["unit"])):
        eng.set_validators(slot, tab.height, tab.addrs, tab.powers_be)


def ruled_groups(eng, sc):
    specs = sc["specs"]
    return eng.groups(len(specs), slot=[SLOT_BIG if s[0] is sc["big"] else SLOT_UNIT for s in specs], rule=[s[1] for s in specs],
                      proposer=[s[2] for s in specs])


def assert_results(results, sc):
    exp = sc["expected"]
    for g in range(len(exp)):
        got = (int(results[g]["n_valid"]), int(results[g]["n_distinct"]), [int(x) for x in results[g]["power"]], int(results[g]["has_quorum"]))
        want = (int(exp[g]["n_valid"]), int(exp[g]["n_distinct"]), [int(x) for x in exp[g]["power"]], int(exp[g]["has_quorum"]))
        assert got == want, (g, sc["specs"][g][1:3], got, want)


def test_scenario_is_meaningful():
    """The cases the groups stand for: the rule decides differently from HasQuorum where it should, and every invalid item the
    scenario plants is invalid to the oracle."""
    sc = scenario()
    hq = [int(x) for x in sc["expected"]["has_quorum"]]
    assert hq == [1, 0, 0, 1, 1, 1, 0, 1, 1, 0, 1, 0, 1, 0, 0, 1, 0, 1, 0]
    assert sum(sc["ok"]) == len(sc["items"]) - 5                    # bad_sig x 2, from_ne_signer x 2, the outsider
    exp, big = sc["expected"], sc["big"]
    assert int(exp[0]["power"][0]) == big.quorum and int(exp[1]["power"][0]) == big.quorum - 1


def run_host(eng, sc, groups):
    bitmap, results, _, voted = eng.verify_batch_ex(sc["items"], b"", groups, voted_stride_words=(N_BIG + 31) // 32)
    assert np.array_equal(bitmap, sc["bitmap"]), "verdict bitmap differs from the oracle"
    return results, voted


def test_rules_on_every_recover_kernel(engine):
    """ibft_verify_batch_ex on each recover kernel.  Rule-0 groups of the call, and every group's voted set and counts, are
    byte-identical to the same call with every flags / reserved field 0."""
    sc = scenario()
    set_tables(engine, sc)
    groups = ruled_groups(engine, sc)
    results, voted = run_host(engine, sc, groups)
    assert_results(results, sc)
    plain = groups.copy()
    plain["flags"] = 0
    plain["reserved"] = 0
    results0, voted0 = run_host(engine, sc, plain)
    assert voted.tobytes() == voted0.tobytes()
    for g, spec in enumerate(sc["specs"]):
        if spec[1] == ib.QUORUM_DEFAULT:
            assert results[g].tobytes() == results0[g].tobytes(), g
        assert (results[g]["n_valid"], results[g]["n_distinct"]) == (results0[g]["n_valid"], results0[g]["n_distinct"])


@pytest.fixture(scope="module")
def eng():
    e = ib.Engine(device=0, max_items=1 << 16, max_payload_bytes=1 << 20, max_groups=64, max_table_slots=16, max_validators=N_BIG)
    set_tables(e, scenario())
    yield e
    e.close()


def test_rules_key_registry_after_keys_learned():
    sc = scenario()
    e = ib.Engine(device=0, max_items=1 << 16, max_payload_bytes=1 << 20, max_groups=64, max_table_slots=16, max_validators=N_BIG,
                  key_cache=True)
    try:
        e.set_recover_path(ib.Engine.PATH_THREAD)   # the kernel that holds the known-key pass
        set_tables(e, sc)
        groups = ruled_groups(e, sc)
        run_host(e, sc, groups)                     # keys learned, tables built on the way out
        assert e.refresh_key_tables() > 0
        results, _ = run_host(e, sc, groups)        # known signers verified against their keys
        assert_results(results, sc)
    finally:
        e.close()


def device_inputs(sc):
    items = sc["items"]
    t_items = torch.from_numpy(items.view(np.uint8).reshape(-1, 128).copy()).cuda()
    t_arena = torch.zeros(16, dtype=torch.uint8, device="cuda")
    t_bm = torch.zeros((len(items) + 31) // 32, dtype=torch.int32, device="cuda")
    t_res = torch.zeros(len(sc["specs"]) * ib.RESULT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    return t_items, t_arena, t_bm, t_res


def test_rules_device_resident_reduce(eng):
    """ibft_bind_groups + ibft_verify_batch_device + ibft_quorum_reduce_device: no return to the host in between."""
    sc = scenario()
    n = len(sc["items"])
    eng.bind_groups(ruled_groups(eng, sc))
    t_items, t_arena, t_bm, t_res = device_inputs(sc)
    st = torch.cuda.current_stream().cuda_stream
    eng.verify_device(t_items.data_ptr(), n, t_arena.data_ptr(), 0, 0, n, t_bm.data_ptr(), 0, st)
    eng.quorum_reduce_device(t_items.data_ptr(), n, t_bm.data_ptr(), len(sc["specs"]), t_res.data_ptr(), st)
    torch.cuda.synchronize()
    assert np.array_equal(t_bm.cpu().numpy().view(np.uint32), sc["bitmap"])
    assert_results(t_res.cpu().numpy().view(ib.RESULT_DTYPE), sc)
    eng.bind_groups(None)


def test_rules_shard_marks_and_merge(eng):
    """ibft_quorum_mark_device over three 32-aligned shards on one GPU, then ibft_quorum_merge_device with n_parts = 3."""
    sc = scenario()
    n = len(sc["items"])
    eng.bind_groups(ruled_groups(eng, sc))
    t_items, t_arena, t_bm, t_res = device_inputs(sc)
    W = eng.quorum_partial_words()
    t_parts = torch.zeros((3, W), dtype=torch.int32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    for r in range(3):
        lo, hi = sharding.shard_bounds(n, 3, r)
        assert lo % 32 == 0 and hi > lo
        eng.verify_device(t_items.data_ptr(), n, t_arena.data_ptr(), 0, lo, hi, t_bm.data_ptr(), 0, st)
        eng.quorum_mark_device(t_items.data_ptr(), n, lo, hi, t_bm.data_ptr(), t_parts[r].data_ptr(), st)
    eng.quorum_merge_device(t_parts.data_ptr(), 3, W, t_res.data_ptr(), st)
    torch.cuda.synchronize()
    assert np.array_equal(t_bm.cpu().numpy().view(np.uint32), sc["bitmap"])
    assert_results(t_res.cpu().numpy().view(ib.RESULT_DTYPE), sc)
    eng.bind_groups(None)


@pytest.mark.parametrize("exchange", ["nccl", "p2p"])
def test_rules_sharded_verifier(eng, exchange):
    """ShardedVerifier at world size 1 (as tests/test_gpu_configs.py runs it): the descriptors pass through to the exchange."""
    sc = scenario()
    items, n = sc["items"], len(sc["items"])
    li, la = sharding.rebase_shard(items, np.zeros(0, np.uint8), 0, n)
    sv = sharding.ShardedVerifier(eng, n, ruled_groups(eng, sc), 1, 0, li, la, torch.cuda.current_stream(), exchange=exchange)
    try:
        for _ in range(2):
            res, bm = sv.run()
            assert np.array_equal(bm, sc["bitmap"])
            assert_results(res, sc)
    finally:
        sv.close()
    eng.bind_groups(None)


@pytest.mark.parametrize("case", ["rule3", "proposer_out_of_range", "rule_without_table"])
def test_rule_argument_errors(eng, case):
    """Each bad descriptor fails the host-buffer call and ibft_bind_groups with IBFT_ERR_INVALID_ARG; the next valid call is
    answered correctly."""
    sc = scenario()
    good = ruled_groups(eng, sc)
    bad = good.copy()
    if case == "rule3":
        bad[0]["flags"] = 3
    elif case == "proposer_out_of_range":
        g = next(i for i, s in enumerate(sc["specs"]) if s[0] is sc["unit"] and s[1] == ib.QUORUM_PREPARE)
        bad[g]["reserved"] = 4                                       # the unit table has 4 validators
    else:
        g = next(i for i, s in enumerate(sc["specs"]) if s[1] == ib.QUORUM_PREPREPARE)
        bad[g]["table_slot"] = ib.NO_TABLE
        bad[g]["height"] = 0
    for call in (lambda: eng.verify_batch_ex(sc["items"], b"", bad), lambda: eng.bind_groups(bad)):
        with pytest.raises(ib.EngineError) as ei:
            call()
        assert ei.value.code == 1
    results, _ = run_host(eng, sc, good)
    assert_results(results, sc)
