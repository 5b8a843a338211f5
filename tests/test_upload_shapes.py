"""The upload shapes on the CPU (tests/upload_shapes.py): the sizes reach every chunk count and staging split the upload path has,
every odd slot holds a class item, no two chunks and no two consecutive calls upload the same bytes, and the tiled expectations
equal the references run on a whole batch."""
import numpy as np
import pytest

import explain_oracle as X
import group_hash_model as G
import upload_shapes as U
from oracle import coracle as co

C = U.C


@pytest.fixture(scope="module")
def up():
    return U.uploads()


def last_parts(n):
    lo, hi = U.chunks(n)[-1]
    return U.stage_parts((hi - lo) * U.ITEM_BYTES)


def test_shapes_reach_every_chunk_count_and_staging_split():
    """1 to 5 chunks; the last chunk staged in 1, 2, 3 and 4 parts; parts that tile the chunk; a part boundary inside a tuple"""
    sizes = U.SHAPES
    assert {len(U.chunks(n)) for n in sizes.values()} == {1, 2, 3, 4, 5}
    assert {len(last_parts(n)) for n in sizes.values()} == {1, 2, 3, 4}
    for n in sizes.values():
        ch = U.chunks(n)
        assert ch[0][0] == 0 and ch[-1][1] == n and all(a[1] == b[0] for a, b in zip(ch, ch[1:]))
        assert all(hi - lo == C for lo, hi in ch[:-1])
        for lo, hi in ch:
            parts = U.stage_parts((hi - lo) * U.ITEM_BYTES)
            assert parts[0][0] == 0 and sum(p[1] for p in parts) == (hi - lo) * U.ITEM_BYTES
            assert all(a[0] + a[1] == b[0] for a, b in zip(parts, parts[1:]))
            assert all(off % 64 == 0 for off, _ in parts)
    assert U.chunks(sizes["C+1"])[-1] == (C, C + 1)                                              # one item in the last chunk
    assert last_parts(sizes["3chunks"]) == [(0, 2 << 20), (2 << 20, 2 << 20)]                     # exactly 4 MiB: two parts
    p = last_parts(sizes["4chunks"])
    assert [q[1] for q in p[:2]] == [2_097_216, 2_097_216] and p[1][0] % U.ITEM_BYTES == 64
    # tuple 16,384 of that chunk: its first 64 bytes in part 0, its last 64 in part 1
    assert 16384 * U.ITEM_BYTES < p[1][0] < 16385 * U.ITEM_BYTES
    assert len(U.chunks(sizes["5chunks"])) == 5       # worklists 0 and 1 each filled by three and two chunks


def test_odd_slots_hold_class_items(up):
    """every odd slot of every chunk holds a class item, byte for byte but the group, and every other slot a filler; the classes
    differ between chunks"""
    cls = up.classes.view(np.uint8).reshape(-1, U.ITEM_BYTES)
    for name, n in U.SHAPES.items():
        for call in (0, 1):
            items, src, grp = up.batch(n, call)
            raw = items.view(np.uint8).reshape(n, U.ITEM_BYTES)
            slots = np.zeros(n, bool)
            per_chunk = []
            for lo, hi in U.chunks(n):
                s = U.odd_slots(lo, hi)
                assert lo in s and hi - 1 in s
                slots[s] = True
                per_chunk.append(tuple(src[s]))
                for i in s:
                    assert src[i] >= up.F, (name, i)
                    mask = np.ones(U.ITEM_BYTES, bool)
                    mask[118:120] = False                                      # ibft_sig_item.group
                    assert (raw[i][mask] == cls[src[i] - up.F][mask]).all(), (name, i)
            assert (src[~slots] < up.F).all() and (src[slots] >= up.F).all(), name
            assert len(set(per_chunk)) == len(per_chunk), name
    # part boundaries: the tuples on both sides of each one are odd slots
    n = U.SHAPES["4chunks"]
    lo, hi = U.chunks(n)[-1]
    s = set(U.odd_slots(lo, hi))
    for off, _ in U.stage_parts((hi - lo) * U.ITEM_BYTES)[1:]:
        assert {lo + (off - 1) // U.ITEM_BYTES, lo + off // U.ITEM_BYTES} <= s
    assert lo + 16384 in s


def test_no_two_chunks_or_consecutive_calls_alike(up):
    """within a call no two chunks upload the same bytes; from one call to the next every tuple of every chunk changes"""
    for name, n in U.SHAPES.items():
        prev = None
        for call in range(4):
            items, _, _ = up.batch(n, call)
            raw = items.view(np.uint8).reshape(n, U.ITEM_BYTES)
            ch = [raw[lo:hi].tobytes() for lo, hi in U.chunks(n)]
            assert len(set(ch)) == len(ch), (name, call)
            if prev is not None:
                assert (raw != prev).any(axis=1).all(), (name, call)
            prev = raw


def test_tiled_expectations_equal_the_whole_references(up):
    """the smallest shape, whole: the C oracle's bitmap, its recovered addresses (every 61st item), the group model's results and
    voted sets over the oracle's bitmap, and the group model's counted bits for bound groups"""
    n = U.SHAPES["C-1"]
    items, src, grp = up.batch(n, 0)
    e = up.expect(src, grp)
    gt = [0 if s == 0 else U.NO_TABLE for s in U.SLOTS]
    flat = ~np.isin(items["kind"], [X.KIND_WIRE, X.KIND_WIRE_SEAL])
    bm = co.verify_batch(items, up.arena, tables=[up.addrs], group_table=gt, n_threads=8)
    got = X.bits_of(bm, n)
    assert np.array_equal(got[flat], e["bit"][flat])
    wire = np.nonzero(~flat)[0]
    assert len(wire) > 0
    for i in wire:                                      # (the C oracle does not decode frames: the explain oracle, per item)
        reasons, _ = X.explain_batch(items[i:i + 1], up.arena, [up.addrs], gt)
        assert bool(reasons[0] == X.OK) == bool(e["bit"][i]), i
    assert int(e["status"].sum()) == int(sum(e["status"][i] for i in wire)) > 0
    for i in list(np.nonzero(flat)[0][::61]) + list(np.nonzero(src >= up.F)[0]):
        why, sig = X._signature_and_digest(items[i], up.arena)
        want = bytes(20) if why is not None else (co.ecrecover_address(sig[1], sig[0]) or bytes(20))
        assert bytes(e["rec"][i]) == want, i
    groups = np.zeros(len(U.SLOTS), dtype=[("table_slot", "<u2"), ("flags", "<u2"), ("reserved", "<u4"), ("height", "<u8")])
    groups["table_slot"] = U.SLOTS
    tables = {0: G.Table(up.addrs, up.power_int)}
    bits_all = e["bit"]
    res, voted = G.group_results(items, up.arena, bits_all & (grp < len(U.SLOTS)), groups, tables)
    for g, (nv, vs, power, hq) in enumerate(e["groups"]):
        assert (res[g]["n_valid"], voted[g], res[g]["power"], bool(res[g]["has_quorum"])) == (nv, vs, power, hq), g
    assert e["groups"][0][3] and e["groups"][1][3] and e["groups"][2][0] > 0
    h = up.hashes()
    want = G.counted(items, up.arena, G.pack_bits(bits_all), len(U.SLOTS), h)
    cnt = up.counted(src, grp, h)
    assert np.array_equal(cnt, want)
    assert cnt[grp == 0].any() and not cnt[grp == 1].any() and (cnt != bits_all).any()


def test_class_expectations_hold_in_the_largest_arena(up):
    """the GPU calls pad the arena up to 32 MiB: no class item's expectation may depend on where the arena ends"""
    padded = up.arena + bytes((32 << 20) - len(up.arena))
    members = tuple(up.members)
    for j in range(len(up.classes)):
        raw = up.classes[j:j + 1].tobytes()
        assert U.PS.item_expectation(raw, padded, members) == U.PS.item_expectation(raw, up.arena, members), j
