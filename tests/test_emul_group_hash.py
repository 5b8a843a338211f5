"""The proposal-hash extraction of groups bound to the accepted proposal (go-ibft_b200/csrc/group_hash.cuh, the function the
hashed mark kernel runs) on the host, against ExtractPrepareHash / ExtractCommitHash of oracle.ibft_logic over oracle.ibft_proto's
protobuf-go decode; and the Python model of counted items and group results (tests/group_hash_model.py) against the decisions of
oracle.ibft_logic's handle_prepare / handle_commit on the same message stores."""
import ctypes
import json
import os
import random
import subprocess

import numpy as np
import pytest

import group_hash_model as M
from oracle import ibft_logic as L
from oracle import ibft_proto as ip

HERE = os.path.dirname(os.path.abspath(__file__))
ITEM_DTYPE = np.dtype([
    ("r", "u1", 32), ("s", "u1", 32), ("digest", "u1", 32), ("signer", "u1", 20),
    ("v", "u1"), ("kind", "u1"), ("group", "<u2"), ("payload_off", "<u4"), ("payload_len", "<u4"),
])
GROUP_DTYPE = np.dtype([("table_slot", "<u2"), ("flags", "<u2"), ("reserved", "<u4"), ("height", "<u8")])
GROUP_HASH_DTYPE = np.dtype([("hash", "u1", 32), ("msg_type", "<u4"), ("reserved", "<u4", 3)])


@pytest.fixture(scope="module")
def gh(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_group_hash") / "libibft_group_hash.so")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-fPIC", "-std=c++17", "-Wall", "-Wextra", "-Wno-unknown-pragmas",
                           "-shared", "-o", so, os.path.join(HERE, "emul", "group_hash_driver.cpp")])
    lib = ctypes.CDLL(so)
    lib.gh_extract.argtypes = [ctypes.c_char_p, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_char_p, ctypes.c_uint32,
                               ctypes.POINTER(ctypes.c_uint32)]
    lib.gh_item_names_hash.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_size_t, ctypes.c_uint32, ctypes.c_char_p]
    return lib


def device_extract(lib, buf: bytes, msg_type: int):
    out = ctypes.create_string_buffer(max(1, len(buf)))
    n = ctypes.c_uint32(0)
    if not lib.gh_extract(bytes(buf), len(buf), msg_type, out, len(out), ctypes.byref(n)):
        return None
    return out.raw[: n.value]


def check(lib, buf: bytes, name: str):
    for mt in (M.HASH_PREPARE, M.HASH_COMMIT):
        want = M.extract(buf, mt)
        got = device_extract(lib, buf, mt)
        # nil and an absent proposalHash: the oracle gives b"" for a present member without the field, as the device does
        assert got == want, (name, mt, buf.hex(), got, want)


# ----------------------------------------------------------------------------- hand-built frames
v, fb, fm = ip._varint, ip._f_bytes, ip._f_msg
H1, H2 = bytes([0x11]) * 32, bytes([0x22]) * 32
VIEW = fm(1, ip.encode_view(ip.View(5, 1)))
FROM = fb(2, bytes(range(0xA0, 0xB4)))
SIG = fb(3, b"\x01" * 65)


def typ(t):
    return v(4 << 3) + v(t & ((1 << 64) - 1))


def prep(*fields):
    return fm(6, b"".join(fields))


def comm(*fields):
    return fm(7, b"".join(fields))


def ph(h):
    return v((1 << 3) | 2) + v(len(h)) + h


def group(num, body=b""):
    return v((num << 3) | 3) + body + v((num << 3) | 4)


CONSTRUCTED = {
    "prepare": VIEW + FROM + typ(1) + prep(ph(H1)),
    "commit": VIEW + FROM + SIG + typ(2) + comm(ph(H1), fb(2, b"\x05" * 65)),
    "prepare_twice_merged_hash_kept": VIEW + typ(1) + prep(ph(H1)) + prep(),
    "prepare_twice_merged_hash_replaced": VIEW + typ(1) + prep(ph(H1)) + prep(ph(H2)),
    "commit_twice_merged_seal_only": typ(2) + comm(ph(H2)) + comm(fb(2, b"\x07" * 65)),
    "oneof_prepare_then_commit": typ(2) + prep(ph(H1)) + comm(ph(H2)),
    "oneof_commit_then_prepare": typ(1) + comm(ph(H2)) + prep(ph(H1)),
    "oneof_prepare_commit_prepare_no_hash": typ(1) + prep(ph(H1)) + comm(ph(H2)) + prep(),
    "oneof_roundchange_replaces": typ(1) + prep(ph(H1)) + fm(8, b""),
    "type_disagrees_prepare_member": typ(2) + prep(ph(H1)),
    "type_disagrees_commit_member": typ(1) + comm(ph(H1)),
    "type_twice_last_wins": typ(2) + typ(1) + prep(ph(H1)),
    "type_after_member": prep(ph(H1)) + typ(1),
    "type_int32_wraps": typ(1 + (1 << 32)) + prep(ph(H1)),
    "type_negative": typ(-1) + prep(ph(H1)),
    "type_missing": prep(ph(H1)),
    "hash_empty": typ(1) + prep(ph(b"")),
    "hash_absent": typ(1) + prep(),
    "hash_31": typ(1) + prep(ph(H1[:31])),
    "hash_33": typ(1) + prep(ph(H1 + b"\x00")),
    "hash_twice_last_wins": typ(1) + prep(ph(H2), ph(H1)),
    "hash_twice_last_empty": typ(1) + prep(ph(H1), ph(b"")),
    "hash_wrong_wiretype": typ(1) + prep(ph(H1), v(1 << 3) + v(7)),
    "member_wrong_wiretype": typ(1) + v(6 << 3) + v(3) + prep(ph(H1)),
    "member_as_varint_after": typ(1) + prep(ph(H1)) + v(6 << 3) + v(3),
    "type_as_bytes_ignored": typ(1) + fb(4, b"\x02") + prep(ph(H1)),
    "unknown_fields": v((9 << 3) | 0) + v(300) + typ(1) + fb(15, b"zz") + prep(fb(9, b"u"), ph(H1), v((3 << 3) | 5) + b"abcd"),
    "unknown_fixed64": v((20 << 3) | 1) + b"12345678" + typ(1) + prep(ph(H1)),
    "group_top": group(9, v((1 << 3) | 0) + v(5) + fb(2, b"g")) + typ(1) + prep(ph(H1)),
    "group_nested": group(9, group(10, group(11)) + v((2 << 3) | 5) + b"wxyz") + typ(1) + prep(ph(H1)),
    "group_in_member": typ(1) + prep(group(3, fb(1, H2)), ph(H1)),
    "group_hides_hash": typ(1) + prep(ph(H1), group(4, ph(H2))),
    "group_unterminated": typ(1) + prep(ph(H1)) + v((9 << 3) | 3) + v(8) + v(1),
    "group_mismatched_end": typ(1) + prep(ph(H1)) + v((9 << 3) | 3) + v((10 << 3) | 4),
    "end_group_alone": typ(1) + prep(ph(H1)) + v((9 << 3) | 4),
    "wiretype_6": typ(1) + prep(ph(H1)) + v((9 << 3) | 6),
    "wiretype_7_in_member": typ(1) + prep(ph(H1), v((9 << 3) | 7)),
    "field_zero": typ(1) + prep(ph(H1)) + v(0) + v(1),
    "field_too_large": typ(1) + prep(ph(H1)) + v((1 << 32) | 0) + v(1),
    "overlong_varint": typ(1) + prep(ph(H1)) + v(9 << 3) + b"\xff" * 10 + b"\x01",
    "tenth_byte_two": typ(1) + prep(ph(H1)) + v(9 << 3) + b"\xff" * 9 + b"\x02",
    "tenth_byte_one": typ(1) + prep(ph(H1)) + v(9 << 3) + b"\xff" * 9 + b"\x01",
    "nonminimal_varints": v(4 << 3) + b"\x81\x80\x80\x00" + v(6 << 3 | 2) + b"\xa2\x80\x00" + ph(H1),
    "length_past_end": typ(1) + prep(ph(H1)) + v((9 << 3) | 2) + v(5) + b"ab",
    "length_past_member_end": typ(1) + v((6 << 3) | 2) + v(34) + v((1 << 3) | 2) + v(40) + H1,
    "truncated_fixed32": typ(1) + prep(ph(H1)) + v((9 << 3) | 5) + b"ab",
    "truncated_key": typ(1) + prep(ph(H1)) + b"\x80",
    "bad_nested_view": fm(1, b"\x08") + typ(1) + prep(ph(H1)),
    "bad_nested_certificate": typ(1) + fm(5, fm(3, fm(1, b"\x22\x05ab"))) + prep(ph(H1)),
    "good_nested_certificate": typ(1) + fm(5, fm(3, fm(1, VIEW + typ(3)))) + prep(ph(H1)),
    "preprepare_certificate_then_prepare": typ(1) + fm(5, fm(2, H2) + fm(3, fm(1, fm(8, fm(2, fm(2, VIEW + prep(ph(H2)))))))) + prep(ph(H1)),
    "empty": b"",
}


def golden():
    d = json.load(open(os.path.join(HERE, "golden", "proto_wire.json")))
    for c in d["cases"]:
        yield c["name"] + "/wire", bytes.fromhex(c["wire"])
        yield c["name"] + "/payload_no_sig", bytes.fromhex(c["payload_no_sig"])
    for c in d["noncanonical"]:
        yield c["name"] + "/wire", bytes.fromhex(c["wire"])
        if c.get("payload_no_sig"):
            yield c["name"] + "/payload_no_sig", bytes.fromhex(c["payload_no_sig"])


def test_golden_frames_and_payloads(gh):
    n = 0
    for name, buf in golden():
        check(gh, buf, name)
        n += 1
    assert n > 100


def test_constructed_frames(gh):
    # the cases are meaningful only if the oracle sees what their names say
    assert M.extract(CONSTRUCTED["prepare_twice_merged_hash_kept"], 1) == H1
    assert M.extract(CONSTRUCTED["prepare_twice_merged_hash_replaced"], 1) == H2
    assert M.extract(CONSTRUCTED["commit_twice_merged_seal_only"], 2) == H2
    assert M.extract(CONSTRUCTED["oneof_prepare_then_commit"], 2) == H2
    assert M.extract(CONSTRUCTED["oneof_prepare_commit_prepare_no_hash"], 1) == b""
    assert M.extract(CONSTRUCTED["oneof_roundchange_replaces"], 1) is None
    assert M.extract(CONSTRUCTED["type_disagrees_prepare_member"], 1) is None
    assert M.extract(CONSTRUCTED["type_int32_wraps"], 1) == H1
    assert M.extract(CONSTRUCTED["hash_twice_last_wins"], 1) == H1
    assert M.extract(CONSTRUCTED["hash_twice_last_empty"], 1) == b""
    assert M.extract(CONSTRUCTED["group_hides_hash"], 1) == H1
    assert M.extract(CONSTRUCTED["tenth_byte_one"], 1) == H1
    for bad in ("group_unterminated", "group_mismatched_end", "end_group_alone", "wiretype_6", "field_zero", "overlong_varint",
                "tenth_byte_two", "length_past_end", "length_past_member_end", "bad_nested_view", "bad_nested_certificate"):
        assert M.extract(CONSTRUCTED[bad], 1) is None, bad
    assert M.extract(CONSTRUCTED["good_nested_certificate"], 1) == H1
    for name, buf in CONSTRUCTED.items():
        check(gh, buf, name)


def mutants(buf: bytes, rng: random.Random, k: int):
    for _ in range(k):
        b = bytearray(buf)
        for _ in range(rng.randint(1, 3)):
            op = rng.randrange(5)
            if op == 0 and b:
                b[rng.randrange(len(b))] ^= 1 << rng.randrange(8)
            elif op == 1 and b:
                b[rng.randrange(len(b))] = rng.randrange(256)
            elif op == 2:
                b.insert(rng.randrange(len(b) + 1), rng.randrange(256))
            elif op == 3 and b:
                del b[rng.randrange(len(b))]
            elif b:
                b = b[: rng.randrange(len(b))]
        yield bytes(b)


def test_seeded_byte_mutants(gh):
    rng = random.Random(20261018)
    bases = [buf for _, buf in golden()][:60] + list(CONSTRUCTED.values())
    n = 0
    for buf in bases:
        for m in mutants(buf, rng, 60):
            check(gh, m, "mutant")
            n += 1
    assert n > 5000


def one_item(kind, group=0, digest=b"", off=0, ln=0):
    it = np.zeros(1, dtype=ITEM_DTYPE)
    it["kind"], it["group"], it["payload_off"], it["payload_len"] = kind, group, off, ln
    if digest:
        it["digest"][0] = np.frombuffer(digest, np.uint8)
    return it


def test_item_kinds_against_the_model(gh):
    commit = CONSTRUCTED["commit"]
    prepare = CONSTRUCTED["prepare"]
    arena = b"\x00" * 7 + commit + prepare
    oc, op_ = 7, 7 + len(commit)
    cases = [
        one_item(M.KIND_SEAL, digest=H1), one_item(M.KIND_SEAL, digest=H2), one_item(0, digest=H1), one_item(5, digest=H1),
        one_item(255, digest=H1), one_item(M.KIND_WIRE_SEAL, off=oc, ln=len(commit)), one_item(M.KIND_WIRE, off=oc, ln=len(commit)),
        one_item(M.KIND_WIRE, off=op_, ln=len(prepare)), one_item(M.KIND_PAYLOAD, off=op_, ln=len(prepare)),
        one_item(M.KIND_PAYLOAD, off=op_, ln=len(prepare) - 1), one_item(M.KIND_WIRE_SEAL, off=op_, ln=len(prepare)),
        one_item(M.KIND_PAYLOAD, off=len(arena) - 3, ln=4),  # span past the arena: never
    ]
    seen = set()
    for it in cases:
        for mt in (M.HASH_PREPARE, M.HASH_COMMIT):
            for bound in (H1, H2):
                h = np.zeros(1, dtype=GROUP_HASH_DTYPE)
                h["msg_type"], h["hash"][0] = mt, np.frombuffer(bound, np.uint8)
                want = bool(M.counted(it, arena, np.array([1], np.uint32), 1, h)[0])
                got = bool(gh.gh_item_names_hash(it.ctypes.data_as(ctypes.c_void_p), arena, len(arena), mt, bound))
                assert got == want, (int(it["kind"][0]), mt, bound[:1])
                seen.add((int(it["kind"][0]), mt, want))
    assert (M.KIND_SEAL, M.HASH_COMMIT, True) in seen and (M.KIND_SEAL, M.HASH_PREPARE, True) not in seen
    assert (M.KIND_WIRE_SEAL, M.HASH_COMMIT, True) in seen and (M.KIND_WIRE, M.HASH_PREPARE, True) in seen
    assert (M.KIND_PAYLOAD, M.HASH_PREPARE, True) in seen
    assert not any(w for k, _, w in seen if k in (0, 5, 255))


# ----------------------------------------------------------------------------- the model against handle_prepare / handle_commit
def addr(i):
    return bytes([0x40 + i % 200]) + i.to_bytes(4, "big") + bytes(15)


def run_round(rng: random.Random, msg_type: int, n_val: int, weighted: bool):
    """One store of PREPAREs or COMMITs for a round: senders naming the accepted hash, a competing proposal, a stale round's hash,
    nil hashes and undecodable bytes, each as a PAYLOAD or raw-frame item; items with verdict 0 are never in the store.  Returns
    the oracle's decision and valid senders, and the model's."""
    powers = [1 + (i % 7) if weighted else 1 for i in range(n_val)]
    tab = M.Table([addr(i) for i in range(n_val)], powers)
    accepted = ip.Proposal(b"block-%d" % rng.randrange(1 << 30), 3)
    acc_hash = bytes(rng.randrange(256) for _ in range(32))
    others = [bytes(rng.randrange(256) for _ in range(32)) for _ in range(2)]
    proposer = rng.randrange(n_val)
    view = ip.View(9, 3)
    store, items, arena = [], [], bytearray()
    bits = []
    for i in range(n_val):
        r = rng.random()
        if r < 0.25:
            continue
        h = acc_hash if r < 0.75 else (others[0] if r < 0.85 else (others[1] if r < 0.93 else b""))
        payload = ip.PrepareMessage(h) if msg_type == ip.PREPARE else ip.CommitMessage(h, b"\x09" * 65)
        m = ip.IbftMessage(view, tab.addrs[i], b"\x01" * 65, msg_type, payload)
        if rng.random() < 0.05:  # a type that disagrees with the member
            m.type = ip.COMMIT if msg_type == ip.PREPARE else ip.PREPARE
        kind = rng.choice([M.KIND_PAYLOAD, M.KIND_WIRE] + ([M.KIND_SEAL, M.KIND_WIRE_SEAL] if msg_type == ip.COMMIT else []))
        buf = ip.encode_ibft_message(m, with_signature=kind != M.KIND_PAYLOAD)
        if kind == M.KIND_PAYLOAD and rng.random() < 0.2:  # a re-marshalled non-canonical message keeps unknown fields
            buf += v((12 << 3) | 2) + v(3) + b"xyz"
            m = ip.decode_ibft_message(buf)
        it = one_item(kind, 0, digest=h if (kind == M.KIND_SEAL and len(h) == 32) else b"", off=len(arena), ln=len(buf))
        if kind == M.KIND_SEAL and m.type != ip.COMMIT:
            continue  # a seal tuple comes from a COMMIT the host parsed
        it["signer"][0] = np.frombuffer(tab.addrs[i], np.uint8)
        arena += buf
        verdict = rng.random() < 0.9
        items.append(it)
        bits.append(verdict)
        if verdict:
            store.append(m)
    items = np.concatenate(items)
    bitmap = M.pack_bits(np.array(bits))
    groups = np.zeros(1, dtype=GROUP_DTYPE)
    groups["table_slot"] = 0
    groups["flags"] = M.QUORUM_PREPARE if msg_type == ip.PREPARE else M.QUORUM_DEFAULT
    groups["reserved"] = proposer if msg_type == ip.PREPARE else 0
    hashes = np.zeros(1, dtype=GROUP_HASH_DTYPE)
    hashes["msg_type"] = M.HASH_PREPARE if msg_type == ip.PREPARE else M.HASH_COMMIT
    hashes["hash"][0] = np.frombuffer(acc_hash, np.uint8)
    flags = M.counted(items, bytes(arena), bitmap, 1, hashes)
    res, voted = M.group_results(items, bytes(arena), flags, groups, {0: tab})

    # the oracle: the same store, the node's accepted proposal, IsValidProposalHash against its hash
    vm = L.ValidatorManager(lambda h: dict(zip(tab.addrs, tab.powers)))
    vm.init(view.height)
    backend = L.Backend(is_valid_proposal_hash=lambda p, h: p == accepted and h == acc_hash)
    node = L.IBFT(backend, vm)
    node.state.view = view
    node.state.name = L.PREPARE_STATE if msg_type == ip.PREPARE else L.COMMIT_STATE
    node.state.proposal_message = ip.IbftMessage(view, tab.addrs[proposer], b"", ip.PREPREPARE, ip.PrePrepareMessage(accepted, acc_hash))
    for m in store:
        node.messages.add_message(m)
    decided = node.handle_prepare(view) if msg_type == ip.PREPARE else node.handle_commit(view)
    valid_senders = {tab.index[m.from_] for m in node.messages.maps[msg_type].get(view.height, {}).get(view.round, {}).values()}
    return decided, valid_senders, res[0], voted[0], flags, items


@pytest.mark.parametrize("msg_type", [ip.PREPARE, ip.COMMIT])
@pytest.mark.parametrize("weighted", [False, True])
def test_model_matches_handle_prepare_and_commit(msg_type, weighted):
    rng = random.Random(7 * msg_type + weighted)
    outcomes = set()
    for trial in range(40):
        n_val = rng.choice([4, 7, 10, 31, 64])
        decided, senders, res, voted, flags, items = run_round(rng, msg_type, n_val, weighted)
        assert voted == senders, trial  # GetValidMessages keeps exactly the items that count
        assert bool(res["has_quorum"]) == decided, trial
        assert res["n_valid"] == int(flags.sum())
        outcomes.add(decided)
    assert outcomes == {False, True}
