"""Multi-GPU sharding of the signature batch (SURVEY.md §8e): contiguous 32-aligned index ranges per rank, validator tables
replicated, ONE all-gather of the pass/fail bitmap words (NCCL over NVLink on GPUs; gloo in the CPU tests), after which
every rank reduces quorum on the complete bitmap.  Works with any torch.distributed backend."""
from __future__ import annotations

import torch
import torch.distributed as dist


def shard_bounds(n: int, world: int, rank: int) -> tuple[int, int]:
    """[lo, hi) of `rank`: contiguous, disjoint, covering [0, n), every boundary except n a multiple of 32 (one bitmap word
    never straddles two ranks).  Trailing ranks may get an EMPTY shard (lo == hi == n): skip the verify call for those."""
    words = (n + 31) // 32
    per = (words + world - 1) // world
    lo = min(rank * per * 32, n)
    hi = min((rank + 1) * per * 32, n)
    return lo, hi


def shard_words(n: int, world: int) -> int:
    """bitmap words every rank contributes to the all-gather (equal on all ranks; trailing ranks pad with zeros)."""
    return ((n + 31) // 32 + world - 1) // world


def all_gather_bitmap(local_words: torch.Tensor, n: int, world: int) -> torch.Tensor:
    """local_words: int32 tensor of shard_words(n, world) words (this rank's slice, zero padded).  Returns the complete
    bitmap of (n+31)//32 words on every rank.  One collective."""
    per = shard_words(n, world)
    assert local_words.numel() == per
    if world == 1:
        return local_words[: (n + 31) // 32]
    full = torch.empty(per * world, dtype=local_words.dtype, device=local_words.device)
    dist.all_gather_into_tensor(full, local_words.contiguous())
    return full[: (n + 31) // 32]


# ---------------------------------------------------------------------------------------------------------------------
# One round / one backlog split over N ranks (strong scaling): every rank HOLDS ONLY ITS SHARD of the tuples and of the
# payload bytes; per call: H2D of the shard -> recover kernel over the shard -> shard-local quorum marks -> ONE all-gather of
# (bitmap words | partial voted sets | valid counts) -> merge + weighted reduce on every rank.  No signature is looked at twice.
# ---------------------------------------------------------------------------------------------------------------------
import numpy as np  # noqa: E402

_KINDS_WITH_PAYLOAD = (1, 3, 4, 5)  # IBFT_KIND_PAYLOAD, _WIRE, _WIRE_SEAL, _PAYLOAD2 (include/ibft_verify.h)
_KEY_RECORDS, _KEY_MAX_PARTS = 1024, 256  # IBFT_KEY_SHARE_RECORDS, IBFT_KEY_SHARE_MAX_PARTS (include/ibft_verify.h)


def rebase_shard(items: np.ndarray, arena: np.ndarray, lo: int, hi: int):
    """items[lo:hi] as a rank-local batch: a copy of the tuples whose payload offsets point into a PRIVATE arena that holds only
    the bytes this shard references (second spans of IBFT_KIND_PAYLOAD2 tuples -- shared certificates -- once each)."""
    local = items[lo:hi].copy()
    arena = np.ascontiguousarray(arena, dtype=np.uint8).reshape(-1)
    parts, pos, seen2 = [], 0, {}
    kinds = local["kind"]
    for i in np.nonzero(np.isin(kinds, _KINDS_WITH_PAYLOAD))[0]:
        off, ln = int(local["payload_off"][i]), int(local["payload_len"][i])
        if off + ln > arena.size:
            continue  # out-of-range payloads stay out of range (verdict 0 either way)
        parts.append(arena[off:off + ln])
        local["payload_off"][i] = pos
        pos += ln
        if kinds[i] == 5:
            off2 = int.from_bytes(bytes(local["digest"][i][:8]), "little")
            len2 = int.from_bytes(bytes(local["digest"][i][8:12]), "little")
            if (off2, len2) not in seen2 and off2 + len2 <= arena.size:
                seen2[(off2, len2)] = pos
                parts.append(arena[off2:off2 + len2])
                pos += len2
            if (off2, len2) in seen2:
                local["digest"][i][:8] = np.frombuffer(int(seen2[(off2, len2)]).to_bytes(8, "little"), np.uint8)
    local_arena = np.concatenate(parts) if parts else np.zeros(0, np.uint8)
    return local, local_arena


def explain_block_bytes(n: int, world: int) -> int:
    """bytes of one rank's explain block: P = shard_words(n, world) * 32 reason bytes, then P x 20 recovered-address bytes (a
    rank's shard padded to P items, so that the blocks of ranks 0.. all-gathered in rank order list items 0.. in order)"""
    return shard_words(n, world) * 32 * 21


def explain_shard(engine, block: torch.Tensor, n: int, world: int, rank: int, d_items: int, d_arena: int, arena_len: int,
                  d_bitmap: int, stream: int = 0):
    """Enqueue engine.explain_device over this rank's shard with its outputs in `block` (explain_block_bytes(n, world) bytes):
    the reason and address pointers are rebased by the shard's first item, as the device calls index by global item number.
    d_items and d_bitmap are the rebased pointers the rank's verify call took.  Bytes of the padding are never written."""
    lo, hi = shard_bounds(n, world, rank)
    if hi > lo:
        P = shard_words(n, world) * 32
        base = block.data_ptr()
        engine.explain_device(d_items, n, d_arena, arena_len, lo, hi, d_bitmap, base - lo, base + P - 20 * lo, 0, stream)


def gather_explain_blocks(block: torch.Tensor, out: torch.Tensor, world: int) -> torch.Tensor:
    """Collective: every rank's explain block in rank order, in `out` (world blocks); the block itself at world 1."""
    if world == 1:
        return block
    dist.all_gather_into_tensor(out, block)
    return out


def explain_rows(blocks: np.ndarray, n: int, world: int, rank: int | None = None):
    """(reasons uint8[m], recovered uint8[m, 20]) out of explain blocks: with rank, `blocks` is that rank's block and m its
    shard's length; without, `blocks` is every rank's block in rank order (the all-gather) and m = n."""
    P = shard_words(n, world) * 32
    b = np.asarray(blocks, dtype=np.uint8).reshape(-1, 21 * P)
    reasons, rec = b[:, :P].reshape(-1), b[:, P:].reshape(-1, 20)
    m = n
    if rank is not None:
        lo, hi = shard_bounds(n, world, rank)
        m = hi - lo
    return reasons[:m].copy(), rec[:m].copy()


def open_peer_buffers(engine, world: int, rank: int, own_ptr: int, own_handle: bytes) -> list:
    """Collective: exchange the CUDA IPC handles of the ranks' exchange buffers and map every peer's buffer on this rank's device
    (engine.exchange_open).  Returns the per-rank device addresses (own_ptr at `rank`).  Either every rank succeeds or every rank
    raises RuntimeError -- a rank that failed alone would leave the others waiting in their next collective; on failure the
    mappings made so far are closed and the rank's own buffer is freed."""
    handles = [None] * world
    dist.all_gather_object(handles, own_handle)
    opened, err = [], None
    try:
        for r in range(world):
            opened.append(own_ptr if r == rank else engine.exchange_open(handles[r]))
    except RuntimeError as ex:      # e.g. no peer access between two devices of this node
        err = str(ex)
    errs = [None] * world
    dist.all_gather_object(errs, err)
    if any(errs):
        for r, p in enumerate(opened):
            if r != rank:
                engine.exchange_close(p)
        engine.exchange_free(own_ptr)
        raise RuntimeError("peer-memory exchange unavailable: " + "; ".join(f"rank {r}: {e}" for r, e in enumerate(errs) if e))
    return opened


class ShardedVerifier:
    """Device-side pipeline of one rank.  `engine` must hold the validator tables and have `groups` bound by this object.

        sv = ShardedVerifier(engine, n_global, groups, world, rank, local_items, local_arena)
        results, bitmap = sv.run()        # host arrays, identical on every rank

    The descriptors are bound as given, quorum rule and proposer included (Engine.groups(..., rule=, proposer=)): both exchanges
    return go-ibft's per-message-type decision (HasPrepareQuorum for PREPARE groups, one valid message for PREPREPARE groups).

    group_hashes (ibft_b200.group_hashes(...), one record per group): every rank binds the PREPARE and COMMIT groups to the accepted
    proposal's hash (Engine.bind_group_hashes), so each rank marks only the items of its shard that name it and the merged or
    exchanged decision is go-ibft's handlePrepare / handleCommit decision.  After finish(), `counted` holds the shard's counted
    bits ((hi - lo + 31) // 32 words, bit i = item lo + i counted): the messages GetValidMessages keeps.

    Key registry (engine flag key_cache): a rank only recovers the signers whose items land in its shard.  Call share_keys()
    between rounds and every rank also knows the keys the other ranks learned, so from the next round on no rank recovers a
    validator any rank already knows.  A caller that never calls it sees no change, except that a p2p-mode rank with a key
    registry exports its new keys into its exchange buffer every round (see share_keys).

    Peer-memory exchange: when a peer does not publish its round within the kernel's bounded wait, finish() raises RuntimeError,
    and so does every later round of this verifier -- the timeout flag is never cleared.  Rebuild the verifiers of all ranks
    after a timeout: the parity alternation only guarantees that a peer has finished reading this rank's buffer of round e when
    this rank has seen the peer's flag of round e + 1, and a timed-out round skipped that check.
    """

    def __init__(self, engine, n_global: int, groups: np.ndarray, world: int, rank: int, local_items: np.ndarray,
                 local_arena: np.ndarray, stream=None, exchange: str = "nccl", group_hashes: np.ndarray | None = None):
        """exchange = "nccl": one all_gather_into_tensor + merge kernel (any backend / any topology);
        exchange = "p2p": every rank's words live in a buffer its peers map over NVLink (CUDA IPC, one node, <= 8 ranks) and ONE
        kernel publishes, waits for the peers and merges straight out of peer memory (ibft_quorum_exchange_device)."""
        from . import engine as _e
        self.e, self.n, self.world, self.rank = engine, n_global, world, rank
        self.lo, self.hi = shard_bounds(n_global, world, rank)
        assert len(local_items) == self.hi - self.lo
        self.groups = groups
        engine.bind_groups(groups)
        self.hashed = group_hashes is not None
        if self.hashed:
            engine.bind_group_hashes(group_hashes)
        self.W = engine.quorum_partial_words()
        self.per = shard_words(n_global, world)
        dev = torch.device("cuda", torch.cuda.current_device())
        self.stream = stream or torch.cuda.current_stream()
        if self.stream.cuda_stream == 0:
            # the C ABI reads a NULL stream as "the engine's own stream": the legacy default stream cannot be named through it, and
            # the engine's kernels would then run unordered with torch's copies -- use a real stream
            self.stream = torch.cuda.Stream()
        pin = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).pin_memory()  # noqa: E731
        self.h_items = pin(local_items) if len(local_items) else torch.zeros(0, dtype=torch.uint8).pin_memory()
        self.h_arena = pin(local_arena) if len(local_arena) else torch.zeros(0, dtype=torch.uint8).pin_memory()
        self.d_items = torch.zeros(max(1, self.h_items.numel()), dtype=torch.uint8, device=dev)
        self.d_arena = torch.zeros(max(16, self.h_arena.numel()), dtype=torch.uint8, device=dev)
        self.d_local = torch.zeros(self.per + self.W, dtype=torch.int32, device=dev)
        self.d_gather = torch.zeros(world * (self.per + self.W), dtype=torch.int32, device=dev)
        self.d_results = torch.zeros(len(groups) * _e.RESULT_DTYPE.itemsize, dtype=torch.uint8, device=dev)
        self.h_out = torch.zeros(self.d_results.numel() + 4 * world * self.per, dtype=torch.uint8).pin_memory()
        self.result_dtype = _e.RESULT_DTYPE
        # the kernels index tuples and bitmap words by GLOBAL item number: hand them rebased pointers
        self.items_base = self.d_items.data_ptr() - self.lo * 128
        self.bitmap_base = self.d_local.data_ptr() - (self.lo // 32) * 4
        self.counted = None
        if self.hashed:  # the shard's counted bits, by global item number as the mark call indexes them
            self.d_counted = torch.zeros(max(1, self.per), dtype=torch.int32, device=dev)
            self.h_counted = torch.zeros(max(1, self.per), dtype=torch.int32).pin_memory()
            self.counted_base = self.d_counted.data_ptr() - (self.lo // 32) * 4
        self.exchange = exchange
        # key sharing (share_keys): each rank sends key_blocks blocks of key_words words per step, enough for a whole validator
        # table (a rank that learned more keys sends the rest at the next step); key_words = 0 when the engine has no key registry
        self.key_words = engine.key_share_words() if engine.params.flags & 1 else 0
        self.key_blocks = -(-engine.params.max_validators // _KEY_RECORDS)
        kw = self.key_blocks * self.key_words                             # words per rank and step
        if self.key_words:
            n_calls = -(-(world - 1) * self.key_blocks // (_KEY_MAX_PARTS - 1)) if world > 1 else 1
            self.d_key_counts = torch.zeros(2 * n_calls, dtype=torch.int32, device=dev)
            self.h_key_counts = torch.zeros(2 * n_calls, dtype=torch.int32).pin_memory()
            if exchange != "p2p":
                self.d_keys = torch.zeros(kw, dtype=torch.int32, device=dev)
                self.d_keys_all = torch.zeros(world * kw, dtype=torch.int32, device=dev)
        if exchange == "p2p":
            self.wpr = (self.per + self.W + 63) // 64 * 64                   # words per rank and parity
            # [2][wpr] words, then the two flags (64 words), then with a key registry [2][kw] words of key blocks: an engine-owned
            # cudaMalloc block whose IPC handle the peers open on THEIR device
            self.xbuf_ptr, handle = engine.exchange_alloc(2 * self.wpr + 64 + 2 * kw)
            self.epoch = 0
            self.d_full = torch.zeros(world * self.per, dtype=torch.int32, device=dev)
            self.d_timeout = torch.zeros(1, dtype=torch.int32, device=dev)
            self.h_out = torch.zeros(self.d_results.numel() + 4 * world * self.per + 4, dtype=torch.uint8).pin_memory()
            self.peer_ptrs = [self.xbuf_ptr]
            if world > 1:
                try:
                    self.peer_ptrs = open_peer_buffers(engine, world, rank, self.xbuf_ptr, handle)
                except RuntimeError:
                    self.xbuf_ptr = 0
                    raise

    def close(self):
        """unmap the peers' exchange buffers and free this rank's (p2p only; collective: every rank calls it)"""
        if self.exchange == "p2p" and getattr(self, "xbuf_ptr", 0):
            self.stream.synchronize()
            if self.world > 1:
                dist.barrier()
            for r, p in enumerate(self.peer_ptrs):
                if r != self.rank:
                    self.e.exchange_close(p)
            if self.world > 1:
                dist.barrier()
            self.e.exchange_free(self.xbuf_ptr)
            self.xbuf_ptr = 0

    def _enqueue_p2p(self):
        st = self.stream.cuda_stream
        self.epoch += 1
        par = self.epoch & 1
        with torch.cuda.stream(self.stream):
            if self.h_items.numel():
                self.d_items[: self.h_items.numel()].copy_(self.h_items, non_blocking=True)
            if self.h_arena.numel():
                self.d_arena[: self.h_arena.numel()].copy_(self.h_arena, non_blocking=True)
            self.e.exchange_clear(self.xbuf_ptr, par * self.wpr, self.wpr, st)
            base = self.xbuf_ptr + par * self.wpr * 4
            if self.hi > self.lo:
                self.e.verify_device(self.items_base, self.n, self.d_arena.data_ptr(), self.h_arena.numel(), self.lo, self.hi,
                                     base - (self.lo // 32) * 4, 0, st)
            self.e.quorum_mark_device(self.items_base, self.n, self.lo, self.hi, base - (self.lo // 32) * 4, base + self.per * 4, st,
                                      self.counted_base if self.hashed else 0)
            if self.hashed:
                self.h_counted.copy_(self.d_counted, non_blocking=True)
            if self.key_words:
                self._export_keys(self._key_region(self.xbuf_ptr, par), st)
            self.e.quorum_exchange_device(self.peer_ptrs, self.rank, self.wpr, self.per, self.epoch, self.d_full.data_ptr(),
                                          self.d_results.data_ptr(), self.d_timeout.data_ptr(), st)
            nres = self.d_results.numel()
            self.h_out[:nres].copy_(self.d_results, non_blocking=True)
            self.h_out[nres: nres + 4 * self.world * self.per].copy_(self.d_full.view(torch.uint8), non_blocking=True)
            self.h_out[nres + 4 * self.world * self.per:].copy_(self.d_timeout.view(torch.uint8), non_blocking=True)

    def enqueue(self):
        """H2D of the shard, kernels and the collective on self.stream; returns nothing (call finish() for the host copies)."""
        if self.exchange == "p2p":
            return self._enqueue_p2p()
        st = self.stream.cuda_stream
        with torch.cuda.stream(self.stream):
            if self.h_items.numel():
                self.d_items[: self.h_items.numel()].copy_(self.h_items, non_blocking=True)
            if self.h_arena.numel():
                self.d_arena[: self.h_arena.numel()].copy_(self.h_arena, non_blocking=True)
            self.d_local.zero_()
            if self.hi > self.lo:
                self.e.verify_device(self.items_base, self.n, self.d_arena.data_ptr(), self.h_arena.numel(), self.lo, self.hi,
                                     self.bitmap_base, 0, st)
            self.e.quorum_mark_device(self.items_base, self.n, self.lo, self.hi, self.bitmap_base,
                                      self.d_local.data_ptr() + self.per * 4, st, self.counted_base if self.hashed else 0)
            if self.hashed:
                self.h_counted.copy_(self.d_counted, non_blocking=True)
            if self.world > 1:
                dist.all_gather_into_tensor(self.d_gather, self.d_local)
            else:
                self.d_gather.copy_(self.d_local)
            self.e.quorum_merge_device(self.d_gather.data_ptr() + self.per * 4, self.world, self.per + self.W,
                                       self.d_results.data_ptr(), st)
            nres = self.d_results.numel()
            self.h_out[:nres].copy_(self.d_results, non_blocking=True)
            words = self.d_gather.view(self.world, self.per + self.W)[:, : self.per].contiguous().view(torch.uint8).reshape(-1)
            self.h_out[nres:].copy_(words, non_blocking=True)

    def finish(self):
        self.stream.synchronize()
        if self.hashed:
            self.counted = self.h_counted.numpy().view(np.uint32)[: (self.hi - self.lo + 31) // 32].copy()
        nres = self.d_results.numel()
        res = self.h_out[:nres].numpy().view(self.result_dtype).copy()
        if self.exchange == "p2p":
            nb = 4 * self.world * self.per
            if int(self.h_out[nres + nb:].numpy().view(np.uint32)[0]):
                raise RuntimeError("peer-memory exchange: a peer did not publish its round in time")
            bm = self.h_out[nres: nres + nb].numpy().view(np.uint32)[: (self.n + 31) // 32].copy()
            return res, bm
        bm = self.h_out[nres:].numpy().view(np.uint32)[: (self.n + 31) // 32].copy()
        return res, bm

    def run(self):
        self.enqueue()
        return self.finish()

    def explain(self, gather: bool = False):
        """After finish(): why this rank's items of the round were rejected, decided again on the device (Engine.explain_device
        on self.stream, against the round's own verdict words: the local words in nccl mode, the rank's words of the assembled
        bitmap in p2p mode).  Returns host arrays (reasons uint8[hi - lo], recovered uint8[hi - lo, 20]) of the shard -- REASON_OK
        for an accepted item, REASON_NEEDS_HOST for a non-canonical raw frame to re-submit through the host path.
        gather=True is collective (every rank calls it): one all-gather of the ranks' reasons and addresses, and every rank
        returns all n items, what Engine.explain_batch returns for the whole batch and its bitmap."""
        if not hasattr(self, "d_explain"):                 # allocated on the first call, reused by every later round
            nb = explain_block_bytes(self.n, self.world)
            dev = self.d_items.device
            self.d_explain = torch.zeros(nb, dtype=torch.uint8, device=dev)
            self.d_explain_all = torch.zeros(self.world * nb, dtype=torch.uint8, device=dev) if self.world > 1 else self.d_explain
            self.h_explain = torch.zeros(self.world * nb, dtype=torch.uint8).pin_memory()
        bitmap = self.d_full.data_ptr() if self.exchange == "p2p" else self.bitmap_base
        with torch.cuda.stream(self.stream):
            explain_shard(self.e, self.d_explain, self.n, self.world, self.rank, self.items_base, self.d_arena.data_ptr(),
                          self.h_arena.numel(), bitmap, self.stream.cuda_stream)
            src = gather_explain_blocks(self.d_explain, self.d_explain_all, self.world) if gather else self.d_explain
            self.h_explain[: src.numel()].copy_(src, non_blocking=True)
        self.stream.synchronize()
        return explain_rows(self.h_explain[: src.numel()].numpy(), self.n, self.world, None if gather else self.rank)

    def _key_region(self, xbuf_ptr: int, par: int) -> int:
        """device address of a rank's key blocks of parity `par` in its exchange buffer"""
        return xbuf_ptr + (2 * self.wpr + 64 + par * self.key_blocks * self.key_words) * 4

    def _export_keys(self, region: int, st: int):
        for j in range(self.key_blocks):             # each export takes the next (up to) 1,024 keys not yet exported
            self.e.key_share_export_device(region + 4 * j * self.key_words, st)

    def share_keys(self) -> tuple[int, int]:
        """Between rounds, after finish(): every rank takes the validator keys the other ranks learned by recovery, each checked on
        its device (the key must hash to the address it claims), then builds their comb tables.  Collective: every rank calls it.
        Returns (keys adopted, records refused) of this rank.

        Each rank sends key_blocks key blocks per step, enough for every validator of a full table; keys beyond that go at the
        next step.  nccl: export this rank's new keys into its blocks, one all_gather_into_tensor of every rank's blocks, adopt,
        on self.stream.  p2p: each round's enqueue() exports into this rank's key blocks of the round's parity, before the
        exchange kernel publishes the round's flag; here the rank adopts from the peers' blocks of that parity, which its
        exchange kernel has seen published.
        The read is safe for the same reason the exchange's is: a peer rewrites parity p only in round e + 2, after it has seen
        this rank's flag of round e + 1, which this rank publishes after the adoption (same stream).  Keys a rank exported in a
        round that was not followed by share_keys() are not sent again; the peers learn them by recovery."""
        if not self.key_words:
            raise RuntimeError("share_keys needs an engine with the key registry (key_cache=True)")
        st = self.stream.cuda_stream
        if self.exchange == "p2p":
            self.stream.synchronize()
            nres = self.d_results.numel() + 4 * self.world * self.per
            if self.epoch and int(self.h_out[nres:].numpy().view(np.uint32)[0]):
                raise RuntimeError("peer-memory exchange: a peer did not publish its round in time")
            regions = [self._key_region(p, self.epoch & 1) for p in self.peer_ptrs]
        else:
            regions = [self.d_keys_all.data_ptr() + 4 * k * self.key_blocks * self.key_words for k in range(self.world)]
        blocks = [[reg + 4 * j * self.key_words for j in range(self.key_blocks)] for reg in regions]
        peers = [b for k in range(self.world) if k != self.rank for b in blocks[k]]
        own = blocks[self.rank][0]
        with torch.cuda.stream(self.stream):
            if self.exchange != "p2p":
                self._export_keys(self.d_keys.data_ptr(), st)
                if self.world > 1:
                    dist.all_gather_into_tensor(self.d_keys_all, self.d_keys)
                else:
                    self.d_keys_all.copy_(self.d_keys)
            # own block first, as the skipped part: at most IBFT_KEY_SHARE_MAX_PARTS - 1 peer blocks per call
            per_call = _KEY_MAX_PARTS - 1
            for j, i in enumerate(range(0, max(len(peers), 1), per_call)):
                self.e.key_share_adopt_device([own] + peers[i: i + per_call], 0, self.d_key_counts.data_ptr() + 8 * j, st)
            self.h_key_counts.copy_(self.d_key_counts, non_blocking=True)
        self.stream.synchronize()        # the adopted keys are in the registry before the refresh reads its learn counter
        self.e.refresh_key_tables()
        c = self.h_key_counts.numpy().reshape(-1, 2).sum(axis=0)
        return int(c[0]), int(c[1])
