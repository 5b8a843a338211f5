"""ibft_explain_batch on the H100: the reasons and recovered addresses of every item against the reference of
tests/explain_oracle.py, after a verify on every recover path and on key-registry engines, only the zero bits explained (launch
counts), a multi-device engine, the errors with untouched outputs, and GpuVerifier's reject hook through the round handlers."""
import collections
import ctypes
import functools
import importlib

import numpy as np
import pytest

import explain_oracle as X
import ibft_b200 as ib
import workloads as wl
from oracle import coracle as co
from oracle import ibft_logic as L
from oracle import ibft_proto as ip
from oracle import secp256k1 as ec
from test_explain_oracle import adversarial_sets, edge_frame_batch, every_reason_batch, load_fixture, non_abscissa

pytestmark = pytest.mark.gpu
host = importlib.import_module("go-ibft_b200.host")
N = ec.N
HEIGHT = 1_000_000
PATHS = {"thread": ib.Engine.PATH_THREAD, "quad": ib.Engine.PATH_QUAD, "split": ib.Engine.PATH_SPLIT, "qsplit": ib.Engine.PATH_QSPLIT,
         "auto": ib.Engine.PATH_AUTO}


def new_engine(**kw):
    args = dict(device=0, max_items=1 << 16, max_payload_bytes=1 << 24, max_groups=64, max_table_slots=16, max_validators=16384)
    args.update(kw)
    return ib.Engine(**args)


@functools.lru_cache(maxsize=None)
def fixture_case(name):
    """(items, arena, addrs, golden bitmap, n_groups, oracle reasons, oracle recovered)"""
    items, arena, addrs, bitmap, _, ng = load_fixture(name)
    reasons, rec = X.explain_batch(items, arena, [addrs], [0] * ng)
    return items, arena, addrs, bitmap, ng, reasons, rec


@functools.lru_cache(maxsize=None)
def crafted_cases():
    """(label, items, arena, tables, group_table, reasons, recovered) of the constructed, adversarial and raw-frame sets"""
    out = []
    items, arena, tables, gt, _ = every_reason_batch()
    out.append(("every-reason", items, arena, tables, gt))
    items, arena, vs = edge_frame_batch()
    out.append(("frames", items, arena, [vs.addr_array()], [0, 0]))
    for label, its in adversarial_sets():
        out.append((label, its, b"", None, None))
    return [c + X.explain_batch(c[1], c[2], c[3], c[4]) for c in out]


def groups_for(eng, tables, gt):
    """set the tables into slots 0.. and return the call's groups (None for a call without groups)"""
    if gt is None:
        return None
    for k, t in enumerate(tables):
        eng.set_validators(k, HEIGHT + k, np.asarray(t, np.uint8).reshape(-1, 20), None)
    return eng.groups(len(gt), slot=list(gt))


def set_fixture(eng, addrs, ng):
    eng.set_validators(0, HEIGHT, addrs, None)
    return eng.groups(ng, slot=0)


def test_every_item_against_the_reference():
    eng = new_engine()
    try:
        for label, items, arena, tables, gt, want, want_rec in crafted_cases():
            groups = groups_for(eng, tables, gt)
            got, rec = eng.explain_batch(items, arena or b"\x00", groups)
            bad = np.nonzero(got != want)[0]
            assert len(bad) == 0, (label, [(int(i), X.NAMES[int(got[i])], X.NAMES[int(want[i])]) for i in bad[:10]])
            assert np.array_equal(rec, want_rec), label
            bm, _, _ = eng.verify_batch(items, arena or b"\x00", groups)
            assert np.array_equal(got == X.OK, X.bits_of(bm, len(items))), label
        for name in ("config2", "config3"):
            items, arena, addrs, bitmap, ng, want, want_rec = fixture_case(name)
            got, rec = eng.explain_batch(items, arena, set_fixture(eng, addrs, ng))
            assert np.array_equal(got, want) and np.array_equal(rec, want_rec), name
            assert np.array_equal(got == X.OK, X.bits_of(bitmap, len(items))), name
    finally:
        eng.close()


def check_after_verify(eng, name, with_recovered=True):
    items, arena, addrs, _, ng, want, want_rec = fixture_case(name)
    groups = set_fixture(eng, addrs, ng)
    bm, _, _ = eng.verify_batch(items, arena, groups)
    bits = X.bits_of(bm, len(items))
    got, rec = eng.explain_batch(items, arena, groups, bitmap=bm)
    assert not (got == X.INCONSISTENT).any()
    assert np.array_equal(got[bits], np.zeros(bits.sum(), np.uint8)) and not rec[bits].any()
    assert np.array_equal(got[~bits], want[~bits]) and np.array_equal(rec[~bits], want_rec[~bits])
    assert np.array_equal(bits, want == X.OK)
    return bm


@pytest.mark.parametrize("path", list(PATHS))
def test_after_verify_on_every_path(path):
    eng = new_engine()
    try:
        eng.set_recover_path(PATHS[path])
        for name in ("config2", "config3"):
            check_after_verify(eng, name)
    finally:
        eng.close()


@pytest.mark.parametrize("budget", [None, 300], ids=["unbounded", "budget300"])
def test_after_verify_on_a_warm_key_registry(budget):
    eng = new_engine(key_cache=True, key_table_budget=budget)
    try:
        for _ in range(2):              # the second pass verifies against the learned keys
            check_after_verify(eng, "config2")
            assert eng.refresh_key_tables() > 0
        check_after_verify(eng, "config3")
        check_after_verify(eng, "config3")
    finally:
        eng.close()


def test_only_the_zero_bits_are_explained():
    eng = new_engine()
    try:
        items, arena, addrs, bitmap, ng, want, _ = fixture_case("config2")
        groups = set_fixture(eng, addrs, ng)
        c0 = eng.launch_count()
        got, _ = eng.explain_batch(items, arena, groups, bitmap=bitmap)
        assert eng.launch_count() - c0 == 1
        assert np.array_equal(got, np.where(X.bits_of(bitmap, len(items)), 0, want))
        # every bit set: nothing is staged or launched, every reason is OK
        ones = np.full_like(bitmap, 0xFFFFFFFF)
        c0 = eng.launch_count()
        got, rec = eng.explain_batch(items, arena, groups, bitmap=ones)
        assert eng.launch_count() == c0 and not got.any() and not rec.any()
        # one zero bit: one item explained
        one = ones.copy()
        k = int(np.nonzero(want != X.OK)[0][0])
        one[k >> 5] &= ~np.uint32(1 << (k & 31))
        got, _ = eng.explain_batch(items, arena, groups, bitmap=one)
        assert eng.launch_count() - c0 == 1 and got[k] == want[k] and np.count_nonzero(got) == 1
        # an accepted item handed in with bit 0 is decided again (not INCONSISTENT without a bitmap, but with one it is)
        j = int(np.nonzero(want == X.OK)[0][0])
        one = ones.copy()
        one[j >> 5] &= ~np.uint32(1 << (j & 31))
        got, _ = eng.explain_batch(items, arena, groups, bitmap=one)
        assert got[j] == X.INCONSISTENT and np.count_nonzero(got) == 1
    finally:
        eng.close()


def test_multi_device_engine_gives_the_single_engines_bytes():
    single, multi = new_engine(), new_engine(devices=[0, 0])
    try:
        for name in ("config2", "config3"):
            items, arena, addrs, bitmap, ng, _, _ = fixture_case(name)
            outs = []
            for eng in (single, multi):
                groups = set_fixture(eng, addrs, ng)
                outs.append(eng.explain_batch(items, arena, groups) + eng.explain_batch(items, arena, groups, bitmap=bitmap))
            for a, b in zip(*outs):
                assert np.array_equal(a, b), name
    finally:
        single.close()
        multi.close()


def raw_explain(eng, items, arena, groups, bitmap=None):
    """the C call with sentinel-filled outputs: (status, reasons, recovered)"""
    n = len(items)
    reasons = np.full(n, 0xAB, np.uint8)
    rec = np.full((n, 20), 0xCD, np.uint8)
    a = np.frombuffer(arena, np.uint8)
    rc = eng.lib.ibft_explain_batch(eng.handle, items.ctypes.data_as(ctypes.c_void_p), n, a.ctypes.data_as(ctypes.c_void_p), len(a),
                                    None if groups is None else groups.ctypes.data_as(ctypes.c_void_p), 0 if groups is None else len(groups),
                                    None if bitmap is None else bitmap.ctypes.data_as(ctypes.c_void_p), reasons.ctypes.data_as(ctypes.c_void_p),
                                    rec.ctypes.data_as(ctypes.c_void_p))
    return rc, reasons, rec


def test_errors_leave_the_outputs_untouched():
    items, arena, addrs, bitmap, ng, _, _ = fixture_case("config2")
    eng = new_engine(max_items=4096, max_payload_bytes=1 << 20)
    try:
        groups = set_fixture(eng, addrs, ng)
        wrong = groups.copy()
        wrong["height"][1] += 1
        bad_rule = groups.copy()
        bad_rule["flags"][0] = 3
        cases = [(ib.engine.ERR_NO_TABLE, items, arena, wrong), (ib.engine.ERR_INVALID_ARG, items, arena, bad_rule),
                 (ib.engine.ERR_CAPACITY, np.concatenate([items, items]), arena, groups),
                 (ib.engine.ERR_CAPACITY, items, arena + bytes((1 << 20) - len(arena) + 1), groups)]
        for code, its, ar, gr in cases:
            for bm in (None, np.zeros((len(its) + 31) // 32, np.uint32)):
                rc, reasons, rec = raw_explain(eng, its, ar, gr, bm)
                assert rc == code and (reasons == 0xAB).all() and (rec == 0xCD).all(), code
        rc = eng.lib.ibft_explain_batch(eng.handle, items.ctypes.data_as(ctypes.c_void_p), len(items), None, 0, None, 0, None, None, None)
        assert rc == ib.engine.ERR_INVALID_ARG
        rc, reasons, rec = raw_explain(eng, items, arena, groups)
        assert rc == 0 and not (reasons == X.INCONSISTENT).any()
    finally:
        eng.close()


# ---------------------------------------------------------------------------------------------- GpuVerifier's reject hook
def hook_round(n=40, seed=33):
    """a PREPARE + COMMIT round with adversarial messages of every kind the handlers can meet"""
    vs = wl.ValidatorSet(seed, n)
    raw = bytes(range(100)) * 2
    ph = wl.proposal_hash(raw, 0)
    view = ip.View(HEIGHT, 0)
    outsider = wl.privkey(seed + 1000, 0)
    out_addr = wl.address_of(outsider)

    def signed(m, key):
        m.signature = wl.sign(key, co.keccak256(m.payload_no_sig()))
        return m
    pp = signed(ip.IbftMessage(view, vs.addrs[0], b"", ip.PREPREPARE, ip.PrePrepareMessage(ip.Proposal(raw, 0), ph, None)), vs.keys[0])
    prepares = [signed(ip.IbftMessage(view, vs.addrs[i], b"", ip.PREPARE, ip.PrepareMessage(ph)), vs.keys[i]) for i in range(1, n)]
    commits = [signed(ip.IbftMessage(view, vs.addrs[i], b"", ip.COMMIT, ip.CommitMessage(ph, wl.sign(vs.keys[i], wl.seal_digest(ph)))), vs.keys[i])
               for i in range(n)]
    s = prepares[1].signature
    prepares[1].signature = s[:64] + bytes([s[64] + 2])                              # BAD_V
    prepares[2].signature = bytes(32) + prepares[2].signature[32:]                   # R_RANGE
    prepares[3].signature = s[:32] + N.to_bytes(32, "big") + s[64:]                  # S_RANGE
    prepares[4].signature = non_abscissa(4).to_bytes(32, "big") + s[32:]             # R_NOT_X
    signed(prepares[5], vs.keys[9])                                                  # SIGNER_MISMATCH
    prepares.append(signed(ip.IbftMessage(view, out_addr, b"", ip.PREPARE, ip.PrepareMessage(ph)), outsider))  # NOT_VALIDATOR
    commits[3].payload.committed_seal = wl.sign(vs.keys[4], wl.seal_digest(ph))     # seal: SIGNER_MISMATCH
    commits[5].payload.committed_seal = commits[5].payload.committed_seal[:64] + b"\x05"  # seal: BAD_V
    signed(commits[6], vs.keys[6])
    commits[6].signature = bytes(32) + commits[6].signature[32:]                     # sender: R_RANGE
    commits.append(signed(ip.IbftMessage(view, out_addr, b"", ip.COMMIT, ip.CommitMessage(ph, wl.sign(outsider, wl.seal_digest(ph)))), outsider))
    return vs, pp, prepares, commits, ph


def run_hook_round(with_hook):
    vs, pp, prepares, commits, ph = hook_round()
    c = host.HostContext("gpu", {"is_proposer": lambda a, h, r: a == vs.addrs[0]}, b"", host.EngineParams(0, 1 << 14, 1 << 24, 32, 8, 4096, 0))
    calls = []
    if with_hook:
        c.set_reject_hook(lambda *a: calls.append(a))
    assert c.set_validators(HEIGHT, vs.addrs, vs.powers) == 0
    c.set_state(HEIGHT, 0, L.PREPARE_STATE, ip.encode_ibft_message(pp))
    for m in prepares:
        c.store_add(ip.encode_ibft_message(m))
    c.handle_prepare(HEIGHT, 0)
    c.set_state(HEIGHT, 0, L.COMMIT_STATE, ip.encode_ibft_message(pp))
    for m in commits:
        c.store_add(ip.encode_ibft_message(m))
    c.handle_commit(HEIGHT, 0)
    # every message's verdict, from the verifier itself (cached verdicts, or a device call of their own)
    verdicts = {}
    for m in prepares + commits:
        verdicts[(ib.KIND_PAYLOAD, m.payload_no_sig(), m.from_)] = (c.is_valid_validator(ip.encode_ibft_message(m)), m)
    for m in commits:
        verdicts[(ib.KIND_SEAL, ph, m.from_)] = (c.is_valid_committed_seal(ph, m.from_, m.payload.committed_seal), m)
    return c, calls, verdicts, vs


def test_reject_hook_once_per_rejected_message_with_the_reference_reason():
    c, calls, verdicts, vs = run_hook_round(True)
    try:
        table = set(vs.addrs)
        got = collections.Counter((k, bytes(m), f) for k, _, m, f, _, _ in calls)
        assert all(v == 1 for v in got.values()), "a message was reported twice"
        rejected = {key for key, (ok, _) in verdicts.items() if not ok}
        assert set(got) == rejected and len(rejected) >= 10
        counts = collections.Counter()
        for kind, height, message, frm, reason, rec in calls:
            _, m = verdicts[(kind, message, frm)]
            if kind == ib.KIND_SEAL:
                it = wl.make_item(m.payload.committed_seal, frm, X.KIND_SEAL, message)
                want, want_rec = X.explain_item(it[0], b"", table)
            else:
                it = wl.make_item(m.signature, frm, X.KIND_PAYLOAD, b"", 0, 0, len(message))
                want, want_rec = X.explain_item(it[0], message, table)
            assert height == HEIGHT and (reason, rec) == (want, want_rec), (kind, X.NAMES[reason], X.NAMES[want])
            counts[reason] += 1
        assert {X.BAD_V, X.R_RANGE, X.S_RANGE, X.R_NOT_X, X.SIGNER_MISMATCH, X.NOT_VALIDATOR} <= set(counts)
        for r in range(256):
            assert c.gpu_rejects(r) == counts.get(r, 0)
        assert c.gpu_explain_calls() >= 1
        # without a hook: the same device calls, and no explain call
        c2, calls2, verdicts2, _ = run_hook_round(False)
        try:
            assert calls2 == [] and c2.gpu_explain_calls() == 0
            assert c2.gpu_device_calls() == c.gpu_device_calls()
            assert {k: v[0] for k, v in verdicts2.items()} == {k: v[0] for k, v in verdicts.items()}
        finally:
            c2.close()
    finally:
        c.close()
