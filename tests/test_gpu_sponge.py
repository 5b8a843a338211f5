"""Sponge sweep: Keccak-256 of payload spans at every alignment and around every rate-block boundary, on the device.

On the device keccak256_bytes / keccak256_two_spans read unaligned 8-byte lanes as three aligned words and two funnel shifts
(load_le64_any); the host emulation builds the same lane byte by byte, so only the GPU runs that code.  Every item carries a real
signature over the correct digest, so a wrong digest flips the verdict, and the recovered address is compared with the
oracle's.  The same items also go through the emulation: a failure on both says the sponge algorithm is wrong, a failure on
the GPU only says the device's load path is."""
import ctypes

import numpy as np
import pytest

import workloads as wl
from oracle import coracle as co
from oracle import ibft_proto as ip
from test_emul import wire_item

RATE = 136
KIND_WIRE = 3  # IBFT_KIND_WIRE
PAYLOAD_LENS = sorted(set(range(281)) | {RATE * k + d for k in range(1, 9) for d in (-1, 0, 1)})
PAYLOAD2_N2 = (0, 1, 135, 136, 137, 300)
N_VALIDATORS = 8


def validators():
    privs = co.privkeys(4242, N_VALIDATORS)
    return privs, co.addresses(privs)


def signed_items(kind, spans, arena, privs, addrs):
    """one item per entry of spans: (off, len[, off2, len2]); signed by validator i % N over Keccak-256 of its bytes"""
    cat = bytearray()
    offs, lens = [], []
    for sp in spans:
        offs.append(len(cat))
        cat += arena[sp[0]:sp[0] + sp[1]] + (arena[sp[2]:sp[2] + sp[3]] if len(sp) == 4 else b"")
        lens.append(len(cat) - offs[-1])
    digests = co.keccak256_batch(bytes(cat), offs, lens)
    who = np.arange(len(spans)) % N_VALIDATORS
    sigs = co.sign_derived_batch(privs[who], digests)
    items = []
    for i, sp in enumerate(spans):
        it = wl.make_item(bytes(sigs[i]), bytes(addrs[who[i]]), kind, b"", 0, sp[0], sp[1])
        if len(sp) == 4:
            it["digest"][0][:8] = np.frombuffer(sp[2].to_bytes(8, "little"), np.uint8)
            it["digest"][0][8:12] = np.frombuffer(sp[3].to_bytes(4, "little"), np.uint8)
        items.append(it)
    return np.concatenate(items), [bytes(addrs[w]) for w in who]


def pad_to(arena: bytearray, residue: int, rng):
    arena += rng.integers(0, 256, (residue - len(arena)) % 8, dtype=np.uint8).tobytes()


def payload_sweep():
    """IBFT_KIND_PAYLOAD: every payload_off mod 8, lengths 0..280 and 136k - 1, 136k, 136k + 1 for k <= 8"""
    privs, addrs = validators()
    rng = np.random.default_rng(11)
    arena, spans = bytearray(), []
    for res in range(8):
        for n in PAYLOAD_LENS:
            pad_to(arena, res, rng)
            spans.append((len(arena), n))
            arena += rng.integers(0, 256, n, dtype=np.uint8).tobytes()
    items, want = signed_items(wl.KIND_PAYLOAD, spans, arena, privs, addrs)
    return items, bytes(arena), want


def payload2_sweep():
    """IBFT_KIND_PAYLOAD2: first span n1 = 0..272 (the stream's block boundary at every position relative to the split), the
    second span at every offset mod 8, n2 in {0, 1, 135, 136, 137, 300}"""
    privs, addrs = validators()
    rng = np.random.default_rng(12)
    arena, spans = bytearray(), []
    for n1 in range(2 * RATE + 1):
        for res in range(8):
            for n2 in PAYLOAD2_N2:
                pad_to(arena, (res + n1) % 8, rng)
                off1 = len(arena)
                arena += rng.integers(0, 256, n1, dtype=np.uint8).tobytes()
                pad_to(arena, res, rng)
                off2 = len(arena)
                arena += rng.integers(0, 256, n2, dtype=np.uint8).tobytes()
                spans.append((off1, n1, off2, n2))
    items, want = signed_items(wl.KIND_PAYLOAD2, spans, arena, privs, addrs)
    return items, bytes(arena), want


def wire_sweep():
    """IBFT_KIND_WIRE: multi-block PREPREPARE / ROUND_CHANGE frames whose hashed bytes (frame minus the signature TLV) are
    136k - 1, 136k or 136k + 1 long, with view heights of 1..10 varint bytes (the cut point moves), at offsets 0..7"""
    privs, addrs = validators()
    keys = [int.from_bytes(bytes(p), "big") for p in privs]
    rng = np.random.default_rng(13)
    ph = co.keccak256(b"sponge sweep")
    frames, want = [], []
    for k in range(1, 7):
        for width in range(1, 11):
            height = 1 << (7 * (width - 1))
            for d in (-1, 0, 1):
                for t in (ip.PREPREPARE, ip.ROUND_CHANGE):
                    v = len(frames) % N_VALIDATORS

                    def build(raw_len):
                        raw = bytes(rng.integers(0, 256, raw_len, dtype=np.uint8)) if raw_len else b""
                        payload = ip.PrePrepareMessage(ip.Proposal(raw, 0), ph, None) if t == ip.PREPREPARE else \
                            ip.RoundChangeMessage(ip.Proposal(raw, 0), None)
                        return ip.IbftMessage(ip.View(height, t), bytes(addrs[v]), b"", t, payload)
                    target = RATE * k + d
                    raw_len = max(0, target - len(build(0).payload_no_sig()))
                    while len(build(raw_len).payload_no_sig()) > target:   # a longer length prefix
                        raw_len -= 1
                    m = build(raw_len)
                    if len(m.payload_no_sig()) != target:
                        continue
                    m.signature = wl.sign(keys[v], co.keccak256(m.payload_no_sig()))
                    frames.append(ip.encode_ibft_message(m))
                    want.append(bytes(addrs[v]))
    arena, items, addr_want = bytearray(), [], []
    for res in range(8):
        for f, a in zip(frames, want):
            pad_to(arena, res, rng)
            items.append(wire_item(KIND_WIRE, len(arena), len(f)))
            arena += f
            addr_want.append(a)
    return np.concatenate(items).view(co.ITEM_DTYPE), bytes(arena), addr_want


SWEEPS = {"payload": payload_sweep, "payload2": payload2_sweep, "wire": wire_sweep}


@pytest.fixture(scope="module")
def sweeps():
    return {name: f() for name, f in SWEEPS.items()}


def test_sweeps_cover_the_boundaries(sweeps):
    items, arena, _ = sweeps["payload"]
    assert {(int(o) % 8, int(n)) for o, n in zip(items["payload_off"], items["payload_len"])} == \
        {(r, n) for r in range(8) for n in PAYLOAD_LENS}
    items, _, _ = sweeps["payload2"]
    n1 = items["payload_len"].astype(int)
    off2 = items["digest"][:, :8].copy().view("<u8")[:, 0].astype(int)
    assert set(n1 % RATE) == set(range(RATE)) and {int(o) % 8 for o in off2} == set(range(8))
    items, arena, _ = sweeps["wire"]
    assert len(items) >= 8 * 6 * 10 * 2 * 2 and {int(o) % 8 for o in items["payload_off"]} == set(range(8))


@pytest.mark.parametrize("name", sorted(SWEEPS))
def test_sweep_on_the_emulation(emul, sweeps, name):
    """the same items through the host emulation of the device headers (byte-wise lane loads)"""
    items, arena, want = sweeps[name]
    a = np.frombuffer(arena, np.uint8)
    for i in range(len(items)):
        out = (ctypes.c_uint8 * 20)()
        rc = emul.emul_verify_item(items[i:i + 1].ctypes.data_as(ctypes.c_void_p), a.ctypes.data_as(ctypes.c_void_p),
                                   ctypes.c_size_t(len(arena)), out)
        assert (rc, bytes(out)) == (1, want[i]), (name, i, int(items[i]["payload_off"]) % 8, int(items[i]["payload_len"]))


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(SWEEPS))
def test_sweep_on_the_device(engine, sweeps, name):
    """every item valid with the oracle's recovered address, on all four recover kernels"""
    import ibft_b200 as ib
    items, arena, want = sweeps[name]
    items = np.ascontiguousarray(items).view(ib.ITEM_DTYPE)
    _, addrs = validators()
    engine.set_validators(9, 1, addrs, None)
    bitmap, results, recovered = engine.verify_batch(items, arena, engine.groups(1, slot=9), want_recovered=True)
    bits = np.unpackbits(bitmap.view(np.uint8), bitorder="little")[: len(items)]
    bad = [i for i in range(len(items)) if not bits[i] or bytes(recovered[i]) != want[i]]
    assert not bad, [(i, int(items[i]["payload_off"]) % 8, int(items[i]["payload_len"])) for i in bad[:10]]
    assert int(results[0]["n_valid"]) == len(items) and int(results[0]["n_distinct"]) == N_VALIDATORS


@pytest.mark.gpu
def test_keccak_and_proposal_hash_batches_with_fillers(engine):
    """ibft_keccak256_batch and ibft_proposal_hash_batch pack their messages contiguously: 1..7-byte fillers between the measured
    messages cycle the alignment of every length of the sweep"""
    rng = np.random.default_rng(14)
    msgs, measured = [], []
    for j, n in enumerate(PAYLOAD_LENS * 2):
        msgs.append(rng.integers(0, 256, 1 + j % 7, dtype=np.uint8).tobytes())
        measured.append(len(msgs))
        msgs.append(rng.integers(0, 256, n, dtype=np.uint8).tobytes())
    got = engine.keccak256_batch(msgs)
    offs = np.cumsum([0] + [len(m) for m in msgs[:-1]])
    assert {int(offs[i]) % 8 for i in measured} == set(range(8))
    want = co.keccak256_batch(b"".join(msgs), offs, [len(m) for m in msgs])
    assert [got[i] for i in measured] == [bytes(want[i]) for i in measured]
    rounds = [j * 977 for j in range(len(msgs))]
    ph = engine.proposal_hash_batch(msgs, rounds)
    assert [ph[i] for i in measured] == [wl.proposal_hash(msgs[i], rounds[i]) for i in measured]
