// engine.cu -- CUDA kernels (sm_90a, H100) and the C ABI (include/ibft_verify.h) of the batched verification engine.
//
// Kernels (SURVEY.md §2.2 checklist):
//   k_recover        K1+K2 fused: Keccak-256 of the payload / seal wrap, secp256k1 public-key recovery, address
//                    derivation + compare with msg.From / seal.Signer, validator-set membership, warp-ballot of the
//                    32 verdicts of a warp into one word of the pass/fail bitmap.
//   k_quorum_mark /  K3: resolve every passing item's signer to its validator index and OR it into the group's voted
//   k_quorum_reduce  set; then per group: distinct count, 320-bit weighted voting-power sum, and the decision of the group's
//                    quorum rule: HasQuorum, HasPrepareQuorum or "one valid PREPREPARE" (reference core/ibft.go:1273-1284,
//                    core/validator_manager.go:77-135).
//   k_keccak_batch   hash-only batch for IsValidProposalHash (reference core/backend.go:50-51).
// There is no CPU fallback anywhere in this file: without a CUDA device ibft_engine_create fails.
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <functional>
#include <mutex>
#include <shared_mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "../../include/ibft_verify.h"
#include "verify_core.cuh"
#include "group_hash.cuh"
#include "debug_arith.cuh"
#include "key_share.cuh"
#include "key_budget.hpp"
#include "shard_plan.hpp"
#include "recover_plan.hpp"

#include "secp_gtable.inc"

using namespace ibft;

static_assert(sizeof(ibft_sig_item) == 128, "packed item must be 128 bytes");
static_assert(sizeof(ibft_group_desc) == 16, "group descriptor must be 16 bytes");
static_assert(sizeof(ibft_group_hash) == 48, "group hash binding must be 48 bytes");
static_assert(IBFT_GTABLE_WG == IBFT_WG, "regenerate secp_gtable.inc (tools/gen_tables.py) for this IBFT_WG");

#ifndef IBFT_GTAB_SMEM
#define IBFT_GTAB_SMEM (IBFT_WG <= 8 && IBFT_WC == 0)  // with a combined table the recover kernel never reads the small one
#endif
#define IBFT_ITEM_ROW_WORDS 33  // 128-byte item + 1 pad word: conflict-free per-thread reads from shared memory

// ------------------------------------------------------------------------------------------------------------
// device-side tables
// ------------------------------------------------------------------------------------------------------------
__device__ uint32_t g_gtable[IBFT_GTAB_ENTRY_WORDS * IBFT_GTAB_ENTRIES];  // filled from IBFT_GTABLE at engine creation

struct slot_dev {
  const uint32_t* keys;    // n x 6 words: address as 5 big-endian words (sorted ascending) + validator index
  const uint64_t* powers;  // n x 4 little-endian limbs, validator-index order
  uint64_t quorum[5];      // floor(2*total/3) + 1
  uint32_t n;
  uint32_t valid;
  // key registry (engine flag IBFT_FLAG_KEY_CACHE; all nullptr otherwise).  One registry per ENGINE, one entry per distinct
  // address of the resident tables: a key belongs to an address, not to a height, so every slot that lists the address reads
  // the same entry.  key_ref maps this table's validator index to its entry; the other pointers are the engine's registry
  // (the same in every slot).
  const uint32_t* key_ref;     // n words, validator-index order: registry entry of the validator's address
  uint32_t* key_state;         // per entry: 0 = unknown, 1 = key learned from a successful recovery, 3 = table being built,
                               // 2 = comb table built
  uint32_t* key_xy;            // 16 words per entry: affine public key
  uint32_t* const* key_chunks; // comb tables, IBFT_KEY_CHUNK entries per chunk of IBFT_KEY_CHUNK x IBFT_KEYTAB_WORDS words; per
                               // entry 17 comb positions x 128 entries x 16 words, affine (build_keytab_pos)
  uint32_t* learn_count;       // number of keys learned so far, engine-wide (the host compares it with the number it built)
  // bounded registry (ibft_set_key_table_budget; both nullptr otherwise): key_chunks is then a pool of table slots
  const uint32_t* key_tab;     // per entry: its table slot, or IBFT_KEY_NO_TAB (nullptr: entry r's table is slot r)
  uint8_t* key_used;           // per entry: set by the known-key pass on every lookup; read and cleared at reclaim points
};
// entry states IBFT_KEY_UNKNOWN / _LEARNED / _READY / _BUILDING / _EVICTED: key_share.cuh
#define IBFT_KEY_NO_TAB 0xFFFFFFFFu
#define IBFT_KEY_CHUNK 256u   // registry entries per comb-table chunk (34 MiB): the pool grows by whole chunks, never by copying
#define IBFT_KEY_REF_FRESH 0x80000000u  // key_ref mark of an entry new to its address (k_adopt_entries); entries are < 2^31

// comb table in slot t
__device__ __forceinline__ uint32_t* key_table_of(uint32_t* const* __restrict__ chunks, uint32_t t) {
  return chunks[t / IBFT_KEY_CHUNK] + (size_t)(t % IBFT_KEY_CHUNK) * IBFT_KEYTAB_WORDS;
}
// known-key pass: the table slot of registry entry r, and whether the table can be used.  The state and the slot depend only on
// r and are loaded side by side; a bounded registry also records the use.
__device__ __forceinline__ uint32_t key_lookup(const slot_dev& s, uint32_t r, bool* ready) {
  const uint32_t st = s.key_state[r];
  const uint32_t t = s.key_tab != nullptr ? s.key_tab[r] : r;
  if (s.key_used != nullptr) s.key_used[r] = 1;
  *ready = st == IBFT_KEY_READY && t != IBFT_KEY_NO_TAB;
  return t;
}

__device__ __forceinline__ uint32_t bswap32(uint32_t x) { return __byte_perm(x, 0, 0x0123); }

// binary search of an address, as five big-endian words, in a slot's sorted key table; returns validator index or -1
__device__ int lookup_validator_words(const slot_dev& s, const uint32_t* a) {
  int lo = 0, hi = (int)s.n - 1;
  while (lo <= hi) {
    int mid = (lo + hi) >> 1;
    const uint32_t* k = s.keys + 6 * (size_t)mid;
    int cmp = 0;
#pragma unroll
    for (int i = 0; i < 5; i++) {
      uint32_t kv = __ldg(k + i);
      if (cmp == 0 && kv != a[i]) cmp = kv < a[i] ? -1 : 1;
    }
    if (cmp == 0) return (int)__ldg(k + 5);
    if (cmp < 0) lo = mid + 1; else hi = mid - 1;
  }
  return -1;
}
// the same for a 20-byte address
__device__ int lookup_validator(const slot_dev& s, const uint8_t* addr) {
  uint32_t a[5];
#pragma unroll
  for (int i = 0; i < 5; i++)
    a[i] = ((uint32_t)addr[4 * i] << 24) | ((uint32_t)addr[4 * i + 1] << 16) | ((uint32_t)addr[4 * i + 2] << 8) | addr[4 * i + 3];
  return lookup_validator_words(s, a);
}

// The last 32 bytes of a tuple, all that the quorum marking reads of it: the signer (words 0..4, as loaded), v | kind << 8 |
// group << 16, payload_off, payload_len.  Two 16-byte loads instead of a copy of the whole tuple.
struct item_tail {
  uint32_t w[8];
  __device__ __forceinline__ uint32_t group() const { return w[5] >> 16; }
  __device__ __forceinline__ uint32_t kind() const { return (w[5] >> 8) & 0xFFu; }
};
__device__ __forceinline__ item_tail load_item_tail(const ibft_sig_item* it) {
  const uint4* p = reinterpret_cast<const uint4*>(it) + 6;
  const uint4 a = __ldg(p), b = __ldg(p + 1);
  return item_tail{{a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w}};
}
// the expected signer of a tuple as five big-endian words (raw frames: the frame's From); false when it has none
__device__ bool item_signer_words(const item_tail& t, const uint8_t* arena, size_t arena_len, uint32_t* a) {
  const uint32_t kind = t.kind();
  if (kind == IBFT_KIND_WIRE || kind == IBFT_KIND_WIRE_SEAL) {
    const uint32_t off = t.w[6], len = t.w[7];
    if ((size_t)off + len > arena_len) return false;
    const uint8_t* w = arena + off;
    wire_frame f;
    if (!parse_wire_frame(w, len, f) || f.from_len != 20) return false;
    w += f.from_off;
#pragma unroll
    for (int i = 0; i < 5; i++)
      a[i] = ((uint32_t)w[4 * i] << 24) | ((uint32_t)w[4 * i + 1] << 16) | ((uint32_t)w[4 * i + 2] << 8) | w[4 * i + 3];
    return true;
  }
#pragma unroll
  for (int i = 0; i < 5; i++) a[i] = bswap32(t.w[i]);
  return true;
}

// One atomicAdd of the count per group and warp instead of one per valid item: the items of a warp mostly share one group,
// and atomics on one address serialise at L2.  Every lane of the warp calls it (valid: the lane's item counts in group g).
__device__ __forceinline__ void count_valid_warp(uint32_t* n_valid, bool valid, uint32_t g) {
  const uint32_t m = __ballot_sync(0xFFFFFFFFu, valid);
  if (!valid) return;
  const uint32_t peers = __match_any_sync(m, g);
  if ((threadIdx.x & 31u) == (uint32_t)(__ffs(peers) - 1)) atomicAdd(&n_valid[g], (uint32_t)__popc(peers));
}
// The same for the vote bits: the lanes that set bits of one voted word OR them together and one of them does the atomicOr.  A
// warp's items mostly come from consecutive validators of one group, so most warps touch one or two words.  bit == 0: no vote.
__device__ __forceinline__ void or_votes_warp(uint32_t* voted, uint32_t word, uint32_t bit) {
  const uint32_t m = __ballot_sync(0xFFFFFFFFu, bit != 0);
  if (bit == 0) return;
  const uint32_t peers = __match_any_sync(m, word);
  const uint32_t bits = __reduce_or_sync(peers, bit);
  if ((threadIdx.x & 31u) == (uint32_t)(__ffs(peers) - 1)) atomicOr(&voted[word], bits);
}

struct group_dev {
  uint32_t voted_off;  // word offset of the group's voted set
  uint32_t n_words;
};

// Where a recover kernel may record a VALID item's vote right away (K2 + the marking half of K3 fused): the group's voted
// set and valid count.  voted == nullptr: no fused marking (device-resident / sharded callers run k_quorum_mark themselves).
struct vote_sink {
  uint32_t* voted;
  uint32_t* n_valid;
  const group_dev* gdev;
};

// validator-set membership at the message's height (reference core/backend.go:44).  Returns false when the item can never
// get verdict 1 (unknown group, unset table, signer not in the set); *v_out = validator index, or -1 when the group has no
// table (IBFT_NO_TABLE) or no groups were given.
__device__ __forceinline__ bool group_member(const ibft_group_desc* __restrict__ groups, uint32_t n_groups,
                                             const slot_dev* __restrict__ slots, uint32_t n_slots, uint32_t group,
                                             const uint8_t* signer, int* v_out, uint32_t* slot_out) {
  *v_out = -1;
  *slot_out = IBFT_NO_TABLE;
  if (groups == nullptr) return true;
  if (group >= n_groups) return false;
  uint32_t slot = groups[group].table_slot;
  if (slot == IBFT_NO_TABLE) return true;
  if (slot >= n_slots || !slots[slot].valid) return false;
  int v = lookup_validator(slots[slot], signer);
  if (v < 0) return false;
  *v_out = v;
  *slot_out = slot;
  return true;
}
// the vote of a valid item: same effect as k_quorum_mark on this item
__device__ __forceinline__ void record_vote(const vote_sink& sink, const ibft_group_desc* __restrict__ groups, uint32_t group, int v) {
  if (groups == nullptr || sink.voted == nullptr) return;
  atomicAdd(&sink.n_valid[group], 1u);
  if (v >= 0) atomicOr(&sink.voted[sink.gdev[group].voted_off + ((uint32_t)v >> 5)], 1u << (v & 31));
}
// the same for the valid items of a whole warp: counts and vote bits go per warp (count_valid_warp, or_votes_warp).  Every lane
// of the warp calls it.
__device__ __forceinline__ void record_votes_warp(const vote_sink& sink, const ibft_group_desc* __restrict__ groups, uint32_t group,
                                                  bool ok, int v) {
  if (groups == nullptr || sink.voted == nullptr) return;
  count_valid_warp(sink.n_valid, ok, group);
  const bool vote = ok && v >= 0;
  or_votes_warp(sink.voted, vote ? sink.gdev[group].voted_off + ((uint32_t)v >> 5) : 0u, vote ? 1u << (v & 31) : 0u);
}
// membership + vote for an item whose signature verified (the latency kernels look the signer up at the end)
__device__ __forceinline__ bool member_and_vote(const ibft_group_desc* __restrict__ groups, uint32_t n_groups,
                                                const slot_dev* __restrict__ slots, uint32_t n_slots, uint32_t group,
                                                const uint8_t* signer, const vote_sink& sink, bool record, int* v_out = nullptr,
                                                uint32_t* slot_out = nullptr) {
  int v;
  uint32_t slot;
  bool ok = group_member(groups, n_groups, slots, n_slots, group, signer, &v, &slot);
  if (v_out) *v_out = v;
  if (slot_out) *slot_out = slot;
  if (ok && record) record_vote(sink, groups, group, v);
  return ok;
}
// key registry: remember the public key a successful recovery produced for validator v of `slot`, in the registry entry of
// its address -- every other resident table that lists the address sees it too (first writer wins; concurrent writers store
// the same key)
__device__ __forceinline__ void learn_key(const slot_dev* __restrict__ slots, uint32_t slot, int v, const aff& K) {
  if (slot == IBFT_NO_TABLE || v < 0) return;
  const slot_dev& s = slots[slot];
  if (s.key_ref == nullptr) return;
  const uint32_t r = s.key_ref[v];
  if (s.key_state[r] != IBFT_KEY_UNKNOWN) return;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    s.key_xy[16 * (size_t)r + i] = K.x.v[i];
    s.key_xy[16 * (size_t)r + 8 + i] = K.y.v[i];
  }
  __threadfence();
  if (atomicCAS(&s.key_state[r], IBFT_KEY_UNKNOWN, IBFT_KEY_LEARNED) == IBFT_KEY_UNKNOWN) atomicAdd(s.learn_count, 1u);
}

// stage the packed tuples [base, min(base + ROWS, hi)) into 33-word shared rows, THREADS threads with coalesced 16-byte loads
template <int ROWS, int THREADS>
__device__ __forceinline__ void stage_items(uint32_t* s_items, const ibft_sig_item* __restrict__ items, uint32_t base, uint32_t hi,
                                            uint32_t tid) {
  static_assert((ROWS * 8) % THREADS == 0, "every thread stages the same number of 16-byte pieces");
  const uint4* src = reinterpret_cast<const uint4*>(items + base);
  uint32_t avail = base < hi ? min((uint32_t)ROWS, hi - base) : 0u;
#pragma unroll
  for (int k = 0; k < (ROWS * 8) / THREADS; k++) {
    uint32_t q = tid + k * THREADS;  // uint4 index within the staged block
    uint32_t row = q >> 3, col = q & 7;
    if (row < avail) {
      uint4 v = __ldg(src + q);
      uint32_t* d = s_items + row * IBFT_ITEM_ROW_WORDS + col * 4;
      d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
    }
  }
}
// the tuple staged in shared row `row`
__device__ __forceinline__ void load_item(ibft_sig_item& it, const uint32_t* s_items, uint32_t row) {
  uint32_t* w = reinterpret_cast<uint32_t*>(&it);
  const uint32_t* s = s_items + row * IBFT_ITEM_ROW_WORDS;
#pragma unroll
  for (int i = 0; i < 32; i++) w[i] = s[i];
}

// ------------------------------------------------------------------------------------------------------------
// K1 + K2: recover kernel.  One thread per signature; a warp's 32 verdicts become one bitmap word.
// ------------------------------------------------------------------------------------------------------------
#ifndef IBFT_MIN_BLOCKS
#define IBFT_MIN_BLOCKS 3
#endif
// BLOCK = 128 for throughput (12 resident warps/SM at 166 registers); BLOCK = 32 for latency-critical small batches (a
// 10k-validator COMMIT round is only 313 warps: one-warp CTAs spread them over all 132 SMs of an H100 instead of 79).
// WIDE: u1*G from the wide generator comb `wtable` (an engine that holds it launches these); else from the per-position comb.
template <int BLOCK, bool WIDE>
__global__ void __launch_bounds__(BLOCK, (IBFT_MIN_BLOCKS * IBFT_BLOCK) / BLOCK)
k_recover(const ibft_sig_item* __restrict__ items, uint32_t n, const uint8_t* __restrict__ arena, size_t arena_len,
          uint32_t shard_lo, uint32_t shard_hi, const ibft_group_desc* __restrict__ groups, uint32_t n_groups,
          const slot_dev* __restrict__ slots, uint32_t n_slots, uint32_t* __restrict__ bitmap,
          uint8_t* __restrict__ recovered, uint8_t* __restrict__ status, const uint32_t* __restrict__ ctable, vote_sink sink,
          const uint32_t* __restrict__ list, const uint32_t* __restrict__ wtable) {
  // list != nullptr: WORKLIST mode (second pass of the key-registry path): list[0] = count, list[1..] = item indices that the
  // verify pass could not decide; the items are gathered, verdict bits are OR-ed into the bitmap the first pass wrote.
#if IBFT_GTAB_SMEM
  __shared__ uint32_t s_gtab[IBFT_GTAB_ENTRY_WORDS * IBFT_GTAB_ENTRIES];
#else
  const uint32_t* s_gtab = g_gtable;  // the table stays in global memory (L1/L2 resident)
#endif
  // Dynamic shared memory, BLOCK x 128 words, used twice: first as the staging area of the CTA's packed tuples (33-word
  // rows), then -- once every thread holds its tuple in registers -- as the per-signature tables {1..8}*R (thread-interleaved).
  extern __shared__ uint32_t s_rtab[];
  uint32_t* s_items = s_rtab;
  const uint32_t tid = threadIdx.x;
#if IBFT_GTAB_SMEM
  // stage the generator window table (shared by every signature of the CTA)
  for (uint32_t i = tid; i < IBFT_GTAB_ENTRY_WORDS * IBFT_GTAB_ENTRIES; i += BLOCK) s_gtab[i] = g_gtable[i];
#endif
  // stage this CTA's 128 packed tuples with coalesced 16-byte loads
  const uint32_t base = shard_lo + blockIdx.x * BLOCK;
  if (list == nullptr) stage_items<BLOCK, BLOCK>(s_items, items, base, shard_hi, tid);
  __syncthreads();
  uint32_t idx = base + tid;
  bool active = idx < shard_hi;
  bool ok = false;
  ibft_sig_item it;
  if (list == nullptr) {
    load_item(it, s_items, tid);
  } else {
    const uint32_t t = blockIdx.x * BLOCK + tid;
    active = t < list[0];
    idx = active ? list[1 + t] : 0u;
    const uint4* src = reinterpret_cast<const uint4*>(items + idx);
    uint4* w = reinterpret_cast<uint4*>(&it);
#pragma unroll
    for (int i = 0; i < 8; i++) w[i] = __ldg(src + i);
  }
  __syncthreads();  // the staging area becomes the R tables from here on
  int v = -1;  // the signer's validator index
  if (active) {
    uint8_t addr[20];
#pragma unroll
    for (int i = 0; i < 20; i++) addr[i] = 0;
    resolved_item ri;
    bool have = false;
    IBFT_STAGE(0);
    int st = resolve_item(it, arena, arena_len, ri, &have);  // raw frames are parsed here (IBFT_KIND_WIRE*)
    if (status != nullptr && list == nullptr) status[idx] = (uint8_t)st;
    gtab_view G{s_gtab};
    G.comb = ctable;
    G.wide = WIDE ? wtable : nullptr;
    rtab_view T{s_rtab + tid, (uint32_t)BLOCK};
    // the signer is looked up FIRST: an item of an unknown group / a non-member can never get verdict 1 (its signature is
    // still recovered when the caller asked for the recovered addresses)
    uint32_t slot = IBFT_NO_TABLE;
    const bool member = have && group_member(groups, n_groups, slots, n_slots, it.group, ri.signer, &v, &slot);
    if (have && (member || recovered != nullptr)) {
      aff K;
#if IBFT_GEN_WIDE > 0
      const bool rec = WIDE ? ecrecover_address_x(exec_serial_wide{}, ri.r, ri.s, ri.v, ri.z, G, T, addr, &K)
                            : ecrecover_address(ri.r, ri.s, ri.v, ri.z, G, T, addr, &K);
#else
      const bool rec = ecrecover_address(ri.r, ri.s, ri.v, ri.z, G, T, addr, &K);
#endif
      if (!rec) {
#pragma unroll
        for (int i = 0; i < 20; i++) addr[i] = 0;
      }
      ok = rec && member;
#pragma unroll
      for (int i = 0; i < 20; i++) ok = ok && (addr[i] == ri.signer[i]);
      if (ok) learn_key(slots, slot, v, K);
    }
    if (recovered != nullptr) {
#pragma unroll
      for (int i = 0; i < 20; i++) recovered[(size_t)idx * 20 + i] = addr[i];
    }
    if (list != nullptr && ok) atomicOr(&bitmap[idx >> 5], 1u << (idx & 31u));
  }
  record_votes_warp(sink, groups, ok ? (uint32_t)it.group : 0u, ok, v);
  if (list != nullptr) return;
  // warp-ballot reduction of the 32 verdicts into one bitmap word (shard bounds are multiples of 32)
  uint32_t word = __ballot_sync(0xFFFFFFFFu, ok);
  if ((tid & 31) == 0 && idx < shard_hi) bitmap[idx >> 5] = word;
}

#if IBFT_WC > 0
// ------------------------------------------------------------------------------------------------------------
// Key-registry path, first pass (engine flag IBFT_FLAG_KEY_CACHE, throughput regime): one thread per signature; a signature
// whose signer's key table is ready is VERIFIED against the key (verify_core.cuh ecdsa_verify_known).  Whatever this pass
// cannot accept -- key not known yet, or the verification rejected -- goes to the worklist and is decided by the recover
// path in a second, dense launch of k_recover (so a warp never walks both window loops, and every verdict is the recover
// path's verdict).  Items that can never be valid (malformed, unknown group, signer not in the set) are settled here.
// ------------------------------------------------------------------------------------------------------------
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK, (IBFT_MIN_BLOCKS * IBFT_BLOCK) / BLOCK)
k_verify_known(const ibft_sig_item* __restrict__ items, uint32_t n, const uint8_t* __restrict__ arena, size_t arena_len,
               uint32_t shard_lo, uint32_t shard_hi, const ibft_group_desc* __restrict__ groups, uint32_t n_groups,
               const slot_dev* __restrict__ slots, uint32_t n_slots, uint32_t* __restrict__ bitmap,
               uint8_t* __restrict__ status, const uint32_t* __restrict__ ctable, vote_sink sink, uint32_t* __restrict__ worklist) {
  __shared__ uint32_t s_items[BLOCK * IBFT_ITEM_ROW_WORDS];
  const uint32_t tid = threadIdx.x;
  const uint32_t base = shard_lo + blockIdx.x * BLOCK;
  stage_items<BLOCK, BLOCK>(s_items, items, base, shard_hi, tid);
  __syncthreads();
  const uint32_t idx = base + tid;
  bool ok = false;
  if (idx < shard_hi) {
    ibft_sig_item it;
    load_item(it, s_items, tid);
    resolved_item ri;
    bool have = false;
    int st = resolve_item(it, arena, arena_len, ri, &have);
    if (status != nullptr) status[idx] = (uint8_t)st;
    int v = -1;
    uint32_t slot = IBFT_NO_TABLE;
    const bool member = have && group_member(groups, n_groups, slots, n_slots, it.group, ri.signer, &v, &slot);
    if (member) {
      uint32_t t = 0;  // table slot of the signer's registry entry
      bool ready = false;
      if (v >= 0 && slots[slot].key_ref != nullptr) t = key_lookup(slots[slot], slots[slot].key_ref[v], &ready);
      if (ready) {
        gtab_view G{g_gtable};
        G.comb = ctable;
        gtab_view Qt{key_table_of(slots[slot].key_chunks, t)};
        ok = ecdsa_verify_known(ri, G, Qt);
      }
      if (ok) record_vote(sink, groups, it.group, v);
      else worklist[1 + atomicAdd(&worklist[0], 1u)] = idx;  // key unknown, or rejected: the recover pass decides (the host
                                                             // only takes this path when the shard fits the worklist)
    }
  }
  uint32_t word = __ballot_sync(0xFFFFFFFFu, ok);
  if ((tid & 31) == 0 && idx < shard_hi) bitmap[idx >> 5] = word;
}
#endif

// ------------------------------------------------------------------------------------------------------------
// K1 + K2, latency variant: FOUR LANES PER SIGNATURE.  A 10k-validator COMMIT round is one wave of independent serial
// chains on the throughput kernel (~5.4k dependent field multiplications each); here the quad's lanes share each chain --
// every lane holds the full state, the up-to-four independent products of a group-law level go one per lane and come back
// through shared memory (secp_ec.cuh, exec_quad).  Everything outside the double-scalar multiplication (Keccak, sqrt,
// inversions) is simply replicated: the kernel does ~4x the work of k_recover and is only used when the batch is too small
// to fill the machine anyway.  CTA = 128 threads = 32 signatures = one bitmap word.
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(4 * IBFT_QUAD_SIGS, 2)
k_recover_quad(const ibft_sig_item* __restrict__ items, uint32_t n, const uint8_t* __restrict__ arena, size_t arena_len,
               uint32_t shard_lo, uint32_t shard_hi, const ibft_group_desc* __restrict__ groups, uint32_t n_groups,
               const slot_dev* __restrict__ slots, uint32_t n_slots, uint32_t* __restrict__ bitmap,
               uint8_t* __restrict__ recovered, uint8_t* __restrict__ status, const uint32_t* __restrict__ ctable, vote_sink sink) {
  __shared__ uint32_t s_items[IBFT_QUAD_SIGS * IBFT_ITEM_ROW_WORDS];
  __shared__ uint32_t s_rtab[IBFT_QUAD_SIGS * IBFT_QTAB_WORDS];  // projective (XYZZ) tables {1..8}*R
  __shared__ uint4 s_xb[4 * 4 * IBFT_QUAD_SIGS];  // exec_quad's product exchange buffer (2 parities x 2 halves per thread)
  __shared__ uint32_t s_word;
  const uint32_t tid = threadIdx.x;
  const uint32_t q = tid >> 2;  // signature within the CTA
  const uint32_t base = shard_lo + blockIdx.x * IBFT_QUAD_SIGS;
  stage_items<IBFT_QUAD_SIGS, 4 * IBFT_QUAD_SIGS>(s_items, items, base, shard_hi, tid);
  if (tid == 0) s_word = 0;
  __syncthreads();
  const uint32_t idx = base + q;
  bool ok = false;
  if (idx < shard_hi) {  // uniform over the quad
    ibft_sig_item it;
    load_item(it, s_items, q);
    exec_quad ex;
    ex.role = (int)(tid & 3u);
    ex.mask = 0xFu << (tid & 28u);
    ex.xb = s_xb;
    ex.par = 0;
    uint8_t addr[20];
    resolved_item ri;
    bool have = false;
    IBFT_STAGE(0);
    int st = resolve_item(it, arena, arena_len, ri, &have);
    gtab_view G{g_gtable};
    G.comb = ctable;
    rtab_view T{s_rtab + q, (uint32_t)IBFT_QUAD_SIGS};
    aff K;
    bool rec = have && ecrecover_address_x(ex, ri.r, ri.s, ri.v, ri.z, G, T, addr, &K);
    if (!rec) {
#pragma unroll
      for (int i = 0; i < 20; i++) addr[i] = 0;
    }
    ok = rec;
#pragma unroll
    for (int i = 0; i < 20; i++) ok = ok && (addr[i] == ri.signer[i]);
    int vi = -1;
    uint32_t vslot = IBFT_NO_TABLE;
    if (ok) ok = member_and_vote(groups, n_groups, slots, n_slots, it.group, ri.signer, sink, ex.leader(), &vi, &vslot);
    if (ok && ex.leader()) learn_key(slots, vslot, vi, K);
    if (ex.leader()) {
      if (status != nullptr) status[idx] = (uint8_t)st;
      if (recovered != nullptr) {
#pragma unroll
        for (int i = 0; i < 20; i++) recovered[(size_t)idx * 20 + i] = addr[i];
      }
      if (ok) atomicOr(&s_word, 1u << q);
    }
  }
  __syncthreads();
  if (tid == 0 && base < shard_hi) bitmap[base >> 5] = s_word;
}

#if IBFT_WC > 0
// ------------------------------------------------------------------------------------------------------------
// K1 + K2, mid-size latency variant: CHAIN warps + one HELPER warp per CTA, one CTA per SM, one warp per scheduler.
// A 10k-validator COMMIT round is 313 warps on the one-thread kernel -- 279 of the 592 schedulers idle while every busy one
// walks the whole serial chain.  Here CTA = 3 chain warps (96 signatures, one per lane) + 1 helper warp that serves all
// three: the helper takes the digest, r^-1, the GLV splits, the square root and u1*G (a comb without doublings) off the
// chain, which only computes u2*R -- on an isomorphic curve, so that it does not have to wait for the root (verify_core.cuh,
// "Split pipeline").  Hand-off through shared memory and named barriers (bar.arrive by the helper, bar.sync by the chain).
// Capacity of one wave: SMs x 96 signatures (12,672 on an H100).
// ------------------------------------------------------------------------------------------------------------
// Hand-off slot of the split kernels (k_recover_split, k_verify_split, k_recover_qsplit): word w of signature i at
// s_slot[w * S + i], S = signatures per CTA.  The two phases have their own flag words: the helper may post phase 2 before a
// chain warp has read phase 1 -- same bits either way, but two words keep the hand-off free of unordered accesses.
#define IBFT_SLOT_K1 0     // [0..4] |k1| of u2
#define IBFT_SLOT_K2 5     // [5..9] |k2| of u2
#define IBFT_SLOT_F1 10    // phase-1 flags
#define IBFT_SLOT_A 11     // [11..18] the helper's parked operand (r or s, then its inverse), then u1*G's x
#define IBFT_SLOT_B 19     // [19..26] the other parked operand (s or r), then u1*G's y
#define IBFT_SLOT_F2 27    // phase-2 flags of the recovering kernels
#define IBFT_SLOT_WORDS (IBFT_SLOT_F2 + 1)
#define IBFT_VSLOT_SIGNER 27  // k_verify_split, in place of IBFT_SLOT_F2: validator index | table slot << 16 of the signer
#define IBFT_VSLOT_F2 28      // k_verify_split: phase-2 flags
#define IBFT_VSLOT_TAB 29     // k_verify_split: table slot of the signer's key
#define IBFT_VSLOT_WORDS (IBFT_VSLOT_TAB + 1)
#define IBFT_SPLIT_SMEM ((IBFT_SPLIT_SIGS * (IBFT_ITEM_ROW_WORDS + IBFT_RTAB_WORDS + IBFT_SLOT_WORDS + 8)) * 4)
#define IBFT_VSPLIT_SMEM ((IBFT_SPLIT_SIGS * (IBFT_ITEM_ROW_WORDS + IBFT_VSLOT_WORDS)) * 4)
#define IBFT_SF_VALID 1u   // phase 1: digits of u2 posted, the chain runs
#define IBFT_SF_NEG0 2u
#define IBFT_SF_NEG1 4u
#define IBFT_SF_ROOT 8u    // recover phase 2: r is an abscissa, y posted
#define IBFT_SF_GINF 16u   // phase 2: u1*G is the point at infinity
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }
__device__ __forceinline__ void named_bar_arrive(uint32_t id, uint32_t count) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory"); }

// the 8-word operands at IBFT_SLOT_A and (b != nullptr) IBFT_SLOT_B of signature i's slot
__device__ __forceinline__ void slot_get8(const uint32_t* s_slot, uint32_t S, uint32_t i, uint32_t* a, uint32_t* b = nullptr) {
#pragma unroll
  for (int k = 0; k < 8; k++) {
    a[k] = s_slot[(IBFT_SLOT_A + k) * S + i];
    if (b != nullptr) b[k] = s_slot[(IBFT_SLOT_B + k) * S + i];
  }
}
__device__ __forceinline__ void slot_put8(uint32_t* s_slot, uint32_t S, uint32_t i, const uint32_t* a, const uint32_t* b = nullptr) {
#pragma unroll
  for (int k = 0; k < 8; k++) {
    s_slot[(IBFT_SLOT_A + k) * S + i] = a[k];
    if (b != nullptr) s_slot[(IBFT_SLOT_B + k) * S + i] = b[k];
  }
}
// helper: the phase-1 flags of the digits of u2, and their posting (two calls: each kernel keeps its own order of the two)
__device__ __forceinline__ uint32_t u2_flags(const ecmult_digits& dg) {
  return IBFT_SF_VALID | (dg.kneg[0] ? IBFT_SF_NEG0 : 0u) | (dg.kneg[1] ? IBFT_SF_NEG1 : 0u);
}
__device__ __forceinline__ void post_u2_digits(uint32_t* s_slot, uint32_t S, uint32_t i, const ecmult_digits& dg) {
#pragma unroll
  for (int k = 0; k < 5; k++) {
    s_slot[(IBFT_SLOT_K1 + k) * S + i] = dg.ks[0][k];
    s_slot[(IBFT_SLOT_K2 + k) * S + i] = dg.ks[1][k];
  }
}
// chain: the posted digits of u2 (flags: phase-1 flags), the other two streams zero
__device__ __forceinline__ void take_u2_digits(const uint32_t* s_slot, uint32_t S, uint32_t i, uint32_t flags, ecmult_digits& dg) {
#pragma unroll
  for (int k = 0; k < 5; k++) {
    dg.ks[0][k] = s_slot[(IBFT_SLOT_K1 + k) * S + i];
    dg.ks[1][k] = s_slot[(IBFT_SLOT_K2 + k) * S + i];
    dg.ks[2][k] = dg.ks[3][k] = 0;
  }
  dg.ks[0][5] = dg.ks[1][5] = dg.ks[2][5] = dg.ks[3][5] = 0;
  dg.kneg[0] = flags & IBFT_SF_NEG0; dg.kneg[1] = flags & IBFT_SF_NEG1;
  dg.kneg[2] = dg.kneg[3] = false;
}
// chain: the root y and the affine u1*G the helper posted in phase 2 for signature i
__device__ __forceinline__ void take_root_u1g(const uint32_t* s_slot, const uint32_t* s_y, uint32_t S, uint32_t i, fe& y, fe& gx, fe& gy) {
#pragma unroll
  for (int k = 0; k < 8; k++) {
    y.v[k] = s_y[k * S + i];
    gx.v[k] = s_slot[(IBFT_SLOT_A + k) * S + i];
    gy.v[k] = s_slot[(IBFT_SLOT_B + k) * S + i];
  }
}

__global__ void __launch_bounds__(32 * (IBFT_SPLIT_CHAINS + 1), 1)
k_recover_split(const ibft_sig_item* __restrict__ items, uint32_t n, const uint8_t* __restrict__ arena, size_t arena_len,
                uint32_t shard_lo, uint32_t shard_hi, const ibft_group_desc* __restrict__ groups, uint32_t n_groups,
                const slot_dev* __restrict__ slots, uint32_t n_slots, uint32_t* __restrict__ bitmap,
                uint8_t* __restrict__ recovered, uint8_t* __restrict__ status, const uint32_t* __restrict__ ctable, vote_sink sink) {
  extern __shared__ uint32_t s_dyn[];
  uint32_t* s_items = s_dyn;                                              // 96 packed tuples, 33-word rows
  uint32_t* s_rtab = s_items + IBFT_SPLIT_SIGS * IBFT_ITEM_ROW_WORDS;     // 96 tables {1..8}*phi(R), signature-interleaved
  uint32_t* s_slot = s_rtab + IBFT_SPLIT_SIGS * IBFT_RTAB_WORDS;          // hand-off slots, word w of signature i at [w*96 + i]
  uint32_t* s_y = s_slot + IBFT_SPLIT_SIGS * IBFT_SLOT_WORDS;             // the root y, 8 words per signature, same interleave
  const uint32_t tid = threadIdx.x, warp = tid >> 5, lane = tid & 31u;
  const uint32_t base = shard_lo + blockIdx.x * IBFT_SPLIT_SIGS;
  stage_items<IBFT_SPLIT_SIGS, 32 * (IBFT_SPLIT_CHAINS + 1)>(s_items, items, base, shard_hi, tid);
  __syncthreads();
  gtab_view G{g_gtable};
  G.comb = ctable;
  if (warp == IBFT_SPLIT_CHAINS) {
    // ------------------------------------------------------------------ helper warp: lane l serves signature 32p + l of
    // every chain warp p.  Order of work = order in which the chains need it:
    //   1a  range checks, ONE scalar inversion for the lane's three signatures (Montgomery's trick), digits of u2 -> posted
    //       while the chains are still building their tables;
    //   1b/2 per pass: digest, digits of u1, square root, u1*G comb, affine -> posted long before the chain's loop ends.
    // Between the steps the lane's per-signature state (r, s, then r^-1) is parked in the result area of the hand-off slot,
    // which phase 2 overwrites only after reading it -- nothing big is carried in registers across the passes.
    uint32_t okmask = 0;
    IBFT_ROLLED
    for (uint32_t p = 0; p < IBFT_SPLIT_CHAINS; p++) {
      const uint32_t i = 32 * p + lane, idx = base + i;
      bool have = false;
      if (idx < shard_hi) {
        ibft_sig_item it;
        load_item(it, s_items, i);
        resolved_item ri;
        resolve_item(it, arena, arena_len, ri, &have, false);
        have = have && split_sig_in_range(ri);
        if (have) {
          sc r = sc_from_be(ri.r), sv = sc_from_be(ri.s);
          slot_put8(s_slot, IBFT_SPLIT_SIGS, i, r.v, sv.v);
        }
      }
      if (have) okmask |= 1u << p;
    }
    {
      // prefix products of the valid r's (an invalid one contributes 1), one inversion, peel backwards
      sc one;
#pragma unroll
      for (int k = 0; k < 8; k++) one.v[k] = k == 0;
      sc rr[IBFT_SPLIT_CHAINS], pre[IBFT_SPLIT_CHAINS];
#pragma unroll
      for (uint32_t p = 0; p < IBFT_SPLIT_CHAINS; p++) {
        rr[p] = one;
        if ((okmask >> p) & 1u) {
#pragma unroll
          for (int k = 0; k < 8; k++) rr[p].v[k] = s_slot[(IBFT_SLOT_A + k) * IBFT_SPLIT_SIGS + 32 * p + lane];
        }
        pre[p] = p ? sc_mul(pre[p - 1], rr[p]) : rr[p];
      }
      sc inv = IBFT_SC_INV(pre[IBFT_SPLIT_CHAINS - 1]);
#pragma unroll
      for (int p = IBFT_SPLIT_CHAINS - 1; p >= 0; p--) {
        sc ri = p ? sc_mul(inv, pre[p - 1]) : inv;
        if (p) inv = sc_mul(inv, rr[p]);
#pragma unroll
        for (int k = 0; k < 8; k++) s_slot[(IBFT_SLOT_A + k) * IBFT_SPLIT_SIGS + 32 * p + lane] = ri.v[k];  // r^-1 replaces r
      }
    }
    IBFT_ROLLED
    for (uint32_t p = 0; p < IBFT_SPLIT_CHAINS; p++) {
      const uint32_t i = 32 * p + lane;
      uint32_t flags = 0;
      if ((okmask >> p) & 1u) {
        sc sv, rinv;
        slot_get8(s_slot, IBFT_SPLIT_SIGS, i, rinv.v, sv.v);
        ecmult_digits dg;
        ecmult_split_into(sc_mul(sv, rinv), dg, 0);
        flags = u2_flags(dg);
        post_u2_digits(s_slot, IBFT_SPLIT_SIGS, i, dg);
      }
      s_slot[IBFT_SLOT_F1 * IBFT_SPLIT_SIGS + i] = flags;
      __threadfence_block();
      named_bar_arrive(1 + p, 64);
    }
    IBFT_ROLLED
    for (uint32_t p = 0; p < IBFT_SPLIT_CHAINS; p++) {
      const uint32_t i = 32 * p + lane;
      if ((okmask >> p) & 1u) {
        uint32_t flags = s_slot[IBFT_SLOT_F1 * IBFT_SPLIT_SIGS + i];
        ibft_sig_item it;
        load_item(it, s_items, i);
        resolved_item ri;
        bool have = false;
        resolve_item(it, arena, arena_len, ri, &have, true);  // this time with the digest
        sc rinv;
#pragma unroll
        for (int k = 0; k < 8; k++) rinv.v[k] = s_slot[(IBFT_SLOT_A + k) * IBFT_SPLIT_SIGS + i];
        ecmult_digits dg;
#pragma unroll
        for (int k = 0; k < 6; k++) dg.ks[0][k] = dg.ks[1][k] = 0;
        dg.kneg[0] = dg.kneg[1] = false;
        split_helper_u1(ri, rinv, dg);
        fe y, gx, gy;
        bool g_inf = false;
        if (split_helper_point(ri, dg, G, y, g_inf, gx, gy)) {
          flags |= IBFT_SF_ROOT | (g_inf ? IBFT_SF_GINF : 0u);
#pragma unroll
          for (int k = 0; k < 8; k++) {
            s_y[k * IBFT_SPLIT_SIGS + i] = y.v[k];
            if (!g_inf) {
              s_slot[(IBFT_SLOT_A + k) * IBFT_SPLIT_SIGS + i] = gx.v[k];
              s_slot[(IBFT_SLOT_B + k) * IBFT_SPLIT_SIGS + i] = gy.v[k];
            }
          }
        }
        s_slot[IBFT_SLOT_F2 * IBFT_SPLIT_SIGS + i] = flags;
      }
      __threadfence_block();
      named_bar_arrive(1 + IBFT_SPLIT_CHAINS + p, 64);
    }
    return;
  }
  // -------------------------------------------------------------------- chain warp
  const uint32_t i = tid, idx = base + i;  // tid = 32 * warp + lane
  const bool active = idx < shard_hi;
  ibft_sig_item it;
  resolved_item ri;
  bool have = false;
  int st = IBFT_ITEM_OK;
  rtab_view T{s_rtab + i, (uint32_t)IBFT_SPLIT_SIGS};
  fe gz = fe_from_u32(1);  // global Z of the table (ecmult_build_rtable_globalz)
  if (active) {
    load_item(it, s_items, i);
    st = resolve_item(it, arena, arena_len, ri, &have, false);  // fields only: the chain never needs the digest
    if (have) gz = ecmult_build_rtable_globalz(split_chain_point(ri.r), T);  // table on a second isomorphic curve: no inversion
  }
  named_bar_sync(1 + warp, 64);  // the helper has posted the digits of u2
  jac acc;
  acc.x = fe_zero(); acc.y = fe_zero(); acc.z = fe_zero();
  acc.inf = true;
  bool go = false;
  if (active && have) {
    uint32_t flags = s_slot[IBFT_SLOT_F1 * IBFT_SPLIT_SIGS + i];
    if (flags & IBFT_SF_VALID) {
      ecmult_digits dg;
      take_u2_digits(s_slot, IBFT_SPLIT_SIGS, i, flags, dg);
      acc = ecmult_streams(dg, G, T, false);
      go = true;
    }
  }
  named_bar_sync(1 + IBFT_SPLIT_CHAINS + warp, 64);  // the helper has posted y and u1*G
  aff K;
  K.x = fe_zero(); K.y = fe_zero();
  uint8_t addr[20];
#pragma unroll
  for (int k = 0; k < 20; k++) addr[k] = 0;
  bool ok = false;
  if (go) {
    uint32_t flags = s_slot[IBFT_SLOT_F2 * IBFT_SPLIT_SIGS + i];
    if (flags & IBFT_SF_ROOT) {
      fe y, gx, gy;
      take_root_u1g(s_slot, s_y, IBFT_SPLIT_SIGS, i, y, gx, gy);
      ok = split_chain_finish(acc, fe_mul(y, gz), (flags & IBFT_SF_GINF) != 0, gx, gy, addr, &K);  // Z' -> Z' * Z_8 * y
    }
  }
  if (active) {
#pragma unroll
    for (int k = 0; k < 20; k++) ok = ok && (addr[k] == ri.signer[k]);
    int vi = -1;
    uint32_t vslot = IBFT_NO_TABLE;
    if (ok) ok = member_and_vote(groups, n_groups, slots, n_slots, it.group, ri.signer, sink, true, &vi, &vslot);
    if (ok) learn_key(slots, vslot, vi, K);
    if (status != nullptr) status[idx] = (uint8_t)st;
    if (recovered != nullptr) {
#pragma unroll
      for (int k = 0; k < 20; k++) recovered[(size_t)idx * 20 + k] = addr[k];
    }
  } else {
    ok = false;
  }
  uint32_t word = __ballot_sync(0xFFFFFFFFu, ok);
  if (lane == 0 && active) bitmap[idx >> 5] = word;
}
#endif

#if IBFT_WC > 0
// ------------------------------------------------------------------------------------------------------------
// Known-key LATENCY variant (engine flag IBFT_FLAG_KEY_CACHE, mid-size rounds): k_recover_split's chain + helper layout, but
// the signature is VERIFIED against the validator's learned key instead of recovered (verify_core.cuh "Verification against a
// KNOWN public key").  The helper warp supplies w = s^-1 (one inversion for the lane's three signatures), the digits of
// u2 = r w, and later the affine u1*G = (z w) G from the comb tables; the chain warp walks u2*Q over the validator's table of
// multiples -- 17 rounds of 8 doublings + at most two additions, no per-signature table, no square root, no address hash --
// adds u1*G and accepts iff the point is exactly R = (r, y) with parity(y) = v.  An accept IS the recover path's verdict 1.
// Everything else that could still be valid -- key not learned yet, or the verification rejected -- goes to the worklist and is
// decided by the recover path (k_recover_qsplit in worklist mode, launched right behind this kernel); items that can never be
// valid (malformed, out of range, unknown group, signer not in the set) are settled here.  A round in which every signature
// verifies (the normal case of consensus) never runs a second chain.
// ------------------------------------------------------------------------------------------------------------
#define IBFT_VF_GREADY 8u     // phase 2: u1*G posted
#define IBFT_VF_RECOVER 32u   // phase 1: member, but the key is not known yet: worklist
__global__ void __launch_bounds__(32 * (IBFT_SPLIT_CHAINS + 1), 1)
k_verify_split(const ibft_sig_item* __restrict__ items, uint32_t n, const uint8_t* __restrict__ arena, size_t arena_len,
               uint32_t shard_lo, uint32_t shard_hi, const ibft_group_desc* __restrict__ groups, uint32_t n_groups,
               const slot_dev* __restrict__ slots, uint32_t n_slots, uint32_t* __restrict__ bitmap, uint8_t* __restrict__ status,
               const uint32_t* __restrict__ ctable, vote_sink sink, uint32_t* __restrict__ worklist) {
  extern __shared__ uint32_t s_dyn[];
  uint32_t* s_items = s_dyn;
  uint32_t* s_slot = s_items + IBFT_SPLIT_SIGS * IBFT_ITEM_ROW_WORDS;  // word w of signature i at [w * 96 + i]
  const uint32_t S = IBFT_SPLIT_SIGS;
  const uint32_t tid = threadIdx.x, warp = tid >> 5, lane = tid & 31u;
  const uint32_t base = shard_lo + blockIdx.x * IBFT_SPLIT_SIGS;
  stage_items<IBFT_SPLIT_SIGS, 32 * (IBFT_SPLIT_CHAINS + 1)>(s_items, items, base, shard_hi, tid);
  __syncthreads();
  gtab_view G{g_gtable};
  G.comb = ctable;
  if (warp == IBFT_SPLIT_CHAINS) {
    // ------------------------------------------------------------------ helper warp
    uint32_t okmask = 0;
    IBFT_ROLLED
    for (uint32_t p = 0; p < IBFT_SPLIT_CHAINS; p++) {
      const uint32_t i = 32 * p + lane, idx = base + i;
      uint32_t flags = 0;
      if (idx < shard_hi) {
        ibft_sig_item it;
        load_item(it, s_items, i);
        resolved_item ri;
        bool have = false;
        int st = resolve_item(it, arena, arena_len, ri, &have, false);
        if (status != nullptr) status[idx] = (uint8_t)st;
        have = have && split_sig_in_range(ri);
        int v = -1;
        uint32_t slot = IBFT_NO_TABLE;
        if (have && group_member(groups, n_groups, slots, n_slots, it.group, ri.signer, &v, &slot)) {
          bool ready = false;
          uint32_t t = 0;
          if (v >= 0 && slots[slot].key_ref != nullptr) t = key_lookup(slots[slot], slots[slot].key_ref[v], &ready);
          if (ready) {
            sc r = sc_from_be(ri.r), sv = sc_from_be(ri.s);
            slot_put8(s_slot, S, i, sv.v, r.v);  // s (inverted below), then r
            s_slot[IBFT_VSLOT_SIGNER * S + i] = (uint32_t)v | (slot << 16);
            s_slot[IBFT_VSLOT_TAB * S + i] = t;
            okmask |= 1u << p;
          } else {
            flags = IBFT_VF_RECOVER;               // member whose key is not known (or no table: v < 0): the recover path decides
          }
        }
      }
      s_slot[IBFT_SLOT_F1 * S + i] = flags;
    }
    {
      // w = s^-1 for the lane's signatures with ONE inversion (Montgomery's trick; an absent one contributes 1)
      sc one;
#pragma unroll
      for (int k = 0; k < 8; k++) one.v[k] = k == 0;
      sc ss[IBFT_SPLIT_CHAINS], pre[IBFT_SPLIT_CHAINS];
#pragma unroll
      for (uint32_t p = 0; p < IBFT_SPLIT_CHAINS; p++) {
        ss[p] = one;
        if ((okmask >> p) & 1u) {
#pragma unroll
          for (int k = 0; k < 8; k++) ss[p].v[k] = s_slot[(IBFT_SLOT_A + k) * S + 32 * p + lane];
        }
        pre[p] = p ? sc_mul(pre[p - 1], ss[p]) : ss[p];
      }
      sc inv = IBFT_SC_INV(pre[IBFT_SPLIT_CHAINS - 1]);
#pragma unroll
      for (int p = IBFT_SPLIT_CHAINS - 1; p >= 0; p--) {
        sc wi = p ? sc_mul(inv, pre[p - 1]) : inv;
        if (p) inv = sc_mul(inv, ss[p]);
#pragma unroll
        for (int k = 0; k < 8; k++) s_slot[(IBFT_SLOT_A + k) * S + 32 * p + lane] = wi.v[k];  // w replaces s
      }
    }
    IBFT_ROLLED
    for (uint32_t p = 0; p < IBFT_SPLIT_CHAINS; p++) {
      const uint32_t i = 32 * p + lane;
      if ((okmask >> p) & 1u) {
        sc w, r;
        slot_get8(s_slot, S, i, w.v, r.v);
        ecmult_digits dg;
        ecmult_split_into(sc_mul(r, w), dg, 0);
        post_u2_digits(s_slot, S, i, dg);
        s_slot[IBFT_SLOT_F1 * S + i] = u2_flags(dg);
      }
      __threadfence_block();
      named_bar_arrive(1 + p, 64);
    }
    IBFT_ROLLED
    for (uint32_t p = 0; p < IBFT_SPLIT_CHAINS; p++) {
      const uint32_t i = 32 * p + lane;
      if ((okmask >> p) & 1u) {
        ibft_sig_item it;
        load_item(it, s_items, i);
        resolved_item ri;
        bool have = false;
        resolve_item(it, arena, arena_len, ri, &have, true);  // this time with the digest
        sc w;
        slot_get8(s_slot, S, i, w.v);
        fe gx = fe_zero(), gy = fe_zero();
        bool g_inf = false;
        known_helper_u1g(ri, w, G, g_inf, gx, gy);
        slot_put8(s_slot, S, i, gx.v, gy.v);
        s_slot[IBFT_VSLOT_F2 * S + i] = IBFT_VF_GREADY | (g_inf ? IBFT_SF_GINF : 0u);
      }
      __threadfence_block();
      named_bar_arrive(1 + IBFT_SPLIT_CHAINS + p, 64);
    }
    return;
  }
  // -------------------------------------------------------------------- chain warp: u2 * Q from the validator's table
  const uint32_t i = tid, idx = base + i;
  const bool active = idx < shard_hi;
  named_bar_sync(1 + warp, 64);  // digits of u2 (and the verdict of the structural checks) are posted
  jac acc;
  acc.x = fe_zero(); acc.y = fe_zero(); acc.z = fe_zero();
  acc.inf = true;
  uint32_t flags = active ? s_slot[IBFT_SLOT_F1 * S + i] : 0u;
  uint32_t vslot = 0;
  if (flags & IBFT_SF_VALID) {
    ecmult_digits dg;
    take_u2_digits(s_slot, S, i, flags, dg);
    vslot = s_slot[IBFT_VSLOT_SIGNER * S + i];
    gtab_view Qt{key_table_of(slots[vslot >> 16].key_chunks, s_slot[IBFT_VSLOT_TAB * S + i])};
    acc = ecmult_streams_known(dg, G, Qt, false);
  }
  named_bar_sync(1 + IBFT_SPLIT_CHAINS + warp, 64);  // u1*G is posted
  bool ok = false;
  if (flags & IBFT_SF_VALID) {
    const uint32_t f2 = s_slot[IBFT_VSLOT_F2 * S + i];
    fe gx, gy;
    slot_get8(s_slot, S, i, gx.v, gy.v);
    ibft_sig_item it;
    load_item(it, s_items, i);
    resolved_item ri;
    bool have = false;
    resolve_item(it, arena, arena_len, ri, &have, false);
    ok = known_chain_finish(acc, (f2 & IBFT_SF_GINF) != 0, gx, gy, ri);
    if (ok) record_vote(sink, groups, it.group, (int)(vslot & 0xFFFFu));
  }
  // whatever was not accepted but could still be valid goes to the recover pass
  if (active && !ok && (flags & (IBFT_SF_VALID | IBFT_VF_RECOVER))) worklist[1 + atomicAdd(&worklist[0], 1u)] = idx;
  uint32_t word = __ballot_sync(0xFFFFFFFFu, ok);
  if (lane == 0 && active) bitmap[idx >> 5] = word;
}
#endif

#if IBFT_WC > 0
// ------------------------------------------------------------------------------------------------------------
// K1 + K2, small-round latency variant: the two ideas above combined.  CTA = 3 four-lane CHAIN warps (8 signatures each)
// + 1 HELPER warp (one lane per signature, a single pass over the CTA's 24), one CTA per SM, one warp per scheduler.
// The quads walk only u2*phi(R) (XYZZ levels, projective table, no square root, no inversion before the final one);
// the helper supplies the digits of u2 early and y, u1*G later.  Verdict bits are OR-ed into a pre-zeroed bitmap
// (24 signatures per CTA do not align with the 32-bit words).  Capacity of one wave: SMs x 24 signatures.
// ------------------------------------------------------------------------------------------------------------
#ifndef IBFT_QSPLIT_MIN_CTAS
#define IBFT_QSPLIT_MIN_CTAS 1
#endif
__global__ void __launch_bounds__(128, IBFT_QSPLIT_MIN_CTAS)
k_recover_qsplit(const ibft_sig_item* __restrict__ items, uint32_t n, const uint8_t* __restrict__ arena, size_t arena_len,
                 uint32_t shard_lo, uint32_t shard_hi, const ibft_group_desc* __restrict__ groups, uint32_t n_groups,
                 const slot_dev* __restrict__ slots, uint32_t n_slots, uint32_t* __restrict__ bitmap,
                 uint8_t* __restrict__ recovered, uint8_t* __restrict__ status, const uint32_t* __restrict__ ctable, vote_sink sink,
                 const uint32_t* __restrict__ list) {
  // list != nullptr: WORKLIST mode (second pass of the known-key latency path): list[0] = count, list[1..] = item indices; the
  // t-th signature of the grid is item list[1 + t]; CTAs beyond the count leave at once; verdict bits are OR-ed in.
  __shared__ uint32_t s_items[IBFT_QSPLIT_SIGS * IBFT_ITEM_ROW_WORDS];
  __shared__ uint32_t s_idx[IBFT_QSPLIT_SIGS];
  __shared__ uint32_t s_qtab[IBFT_QSPLIT_SIGS * IBFT_QTAB_WORDS];
  __shared__ uint32_t s_slot[IBFT_QSPLIT_SIGS * IBFT_SLOT_WORDS];
  __shared__ uint32_t s_y[IBFT_QSPLIT_SIGS * 8];
  __shared__ uint4 s_xb[4 * 128];
  const uint32_t tid = threadIdx.x, warp = tid >> 5, lane = tid & 31u;
  const uint32_t base = list ? blockIdx.x * IBFT_QSPLIT_SIGS : shard_lo + blockIdx.x * IBFT_QSPLIT_SIGS;
  const uint32_t limit = list ? list[0] : shard_hi;   // rows [base, limit) of this CTA exist
  if (base >= limit) return;                            // (uniform over the CTA)
  {
    uint32_t avail = min((uint32_t)IBFT_QSPLIT_SIGS, limit - base);
    if (tid < IBFT_QSPLIT_SIGS) s_idx[tid] = tid < avail ? (list ? list[1 + base + tid] : base + tid) : 0xFFFFFFFFu;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 2; k++) {
      uint32_t u = tid + k * 128;
      uint32_t row = u >> 3, col = u & 7;
      if (row < avail) {
        uint4 v = __ldg(reinterpret_cast<const uint4*>(items + s_idx[row]) + col);
        uint32_t* d = s_items + row * IBFT_ITEM_ROW_WORDS + col * 4;
        d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
      }
    }
  }
  __syncthreads();
  gtab_view G{g_gtable};
  G.comb = ctable;
  const uint32_t S = IBFT_QSPLIT_SIGS;
  if (warp == 3) {
    // ---------------------------------------------------------------- helper warp: lane l serves signature l (l < 24)
    const uint32_t i = lane, idx = lane < S ? s_idx[lane] : 0xFFFFFFFFu;
    const bool mine = lane < S && idx != 0xFFFFFFFFu;
    ibft_sig_item it;
    resolved_item ri;
    sc rinv;
    uint32_t flags = 0;
    if (mine) {
      load_item(it, s_items, i);
      bool have = false;
      resolve_item(it, arena, arena_len, ri, &have, false);
      if (have && split_sig_in_range(ri)) {
        rinv = IBFT_SC_INV(sc_from_be(ri.r));
        ecmult_digits dg;
        split_helper_u2(ri, rinv, dg);
        flags = u2_flags(dg);
        post_u2_digits(s_slot, S, i, dg);
      }
    }
    if (lane < S) s_slot[IBFT_SLOT_F1 * S + i] = flags;
    __threadfence_block();
    named_bar_arrive(1, 64); named_bar_arrive(2, 64); named_bar_arrive(3, 64);
    if (flags & IBFT_SF_VALID) {
      bool have = false;
      resolve_item(it, arena, arena_len, ri, &have, true);  // with the digest
      ecmult_digits dg;
#pragma unroll
      for (int k = 0; k < 6; k++) dg.ks[0][k] = dg.ks[1][k] = 0;
      dg.kneg[0] = dg.kneg[1] = false;
      split_helper_u1(ri, rinv, dg);
      fe y, gx, gy;
      bool g_inf = false;
      if (split_helper_point(ri, dg, G, y, g_inf, gx, gy)) {
        flags |= IBFT_SF_ROOT | (g_inf ? IBFT_SF_GINF : 0u);
#pragma unroll
        for (int k = 0; k < 8; k++) {
          s_y[k * S + i] = y.v[k];
          if (!g_inf) {
            s_slot[(IBFT_SLOT_A + k) * S + i] = gx.v[k];
            s_slot[(IBFT_SLOT_B + k) * S + i] = gy.v[k];
          }
        }
      }
      s_slot[IBFT_SLOT_F2 * S + i] = flags;
    }
    __threadfence_block();
    named_bar_arrive(4, 64); named_bar_arrive(5, 64); named_bar_arrive(6, 64);
    return;
  }
  // ------------------------------------------------------------------ chain warps: four lanes per signature
  const uint32_t q = tid >> 2, idx = s_idx[q];
  const bool active = idx != 0xFFFFFFFFu;
  exec_quad ex;
  ex.role = (int)(tid & 3u);
  ex.mask = 0xFu << (tid & 28u);
  ex.xb = s_xb;
  ex.par = 0;
  ibft_sig_item it;
  resolved_item ri;
  bool have = false;
  int st = IBFT_ITEM_OK;
  fe c = fe_zero();
  qtab_view T{s_qtab + q, S};
  if (active) {
    load_item(it, s_items, q);
    st = resolve_item(it, arena, arena_len, ri, &have, false);
    if (have) ecmult_build_qtable(ex, split_chain_point(ri.r, &c), T);
  }
  named_bar_sync(1 + warp, 64);
  xyzz acc;
  acc.x = fe_zero(); acc.y = fe_zero(); acc.zz = fe_zero(); acc.zzz = fe_zero();
  acc.inf = true;
  bool go = false;
  if (active && have) {
    uint32_t flags = s_slot[IBFT_SLOT_F1 * S + q];
    if (flags & IBFT_SF_VALID) {
      ecmult_digits dg;
      take_u2_digits(s_slot, S, q, flags, dg);
      acc = ecmult_streams_x(ex, dg, G, T, false);
      go = true;
    }
  }
  named_bar_sync(4 + warp, 64);
  aff K;
  K.x = fe_zero(); K.y = fe_zero();
  uint8_t addr[20];
#pragma unroll
  for (int k = 0; k < 20; k++) addr[k] = 0;
  bool ok = false;
  if (go) {
    uint32_t flags = s_slot[IBFT_SLOT_F2 * S + q];
    if (flags & IBFT_SF_ROOT) {
      fe y, gx, gy;
      take_root_u1g(s_slot, s_y, S, q, y, gx, gy);
      ok = split_chain_finish_x(ex, acc, c, y, (flags & IBFT_SF_GINF) != 0, gx, gy, addr, &K);
    }
  }
  if (active) {
#pragma unroll
    for (int k = 0; k < 20; k++) ok = ok && (addr[k] == ri.signer[k]);
    int vi = -1;
    uint32_t vslot = IBFT_NO_TABLE;
    if (ok) ok = member_and_vote(groups, n_groups, slots, n_slots, it.group, ri.signer, sink, ex.leader(), &vi, &vslot);
    if (ok && ex.leader()) learn_key(slots, vslot, vi, K);
    if (ex.leader()) {
      if (status != nullptr && list == nullptr) status[idx] = (uint8_t)st;
      if (recovered != nullptr) {
#pragma unroll
        for (int k = 0; k < 20; k++) recovered[(size_t)idx * 20 + k] = addr[k];
      }
      if (ok) atomicOr(&bitmap[idx >> 5], 1u << (idx & 31u));
    }
  }
}
#endif

// ------------------------------------------------------------------------------------------------------------
// K3: quorum
// ------------------------------------------------------------------------------------------------------------

// the vote of a counted item of group g: its signer's bit in the group's voted set (*bit = 0: the group has no table, the item
// no signer, or the signer is not in the table)
__device__ __forceinline__ void quorum_vote(const item_tail& t, uint32_t g, const uint8_t* __restrict__ arena, size_t arena_len,
                                            const ibft_group_desc* __restrict__ groups, const group_dev* __restrict__ gdev,
                                            const slot_dev* __restrict__ slots, uint32_t n_slots, uint32_t* word, uint32_t* bit) {
  const uint32_t slot = groups[g].table_slot;
  if (slot == IBFT_NO_TABLE || slot >= n_slots || !slots[slot].valid) return;
  uint32_t a[5];
  if (!item_signer_words(t, arena, arena_len, a)) return;
  const int v = lookup_validator_words(slots[slot], a);
  if (v < 0) return;
  *word = gdev[g].voted_off + ((uint32_t)v >> 5);
  *bit = 1u << (v & 31);
}

__global__ void k_quorum_mark(const ibft_sig_item* __restrict__ items, uint32_t n, const uint8_t* __restrict__ arena, size_t arena_len,
                              const uint32_t* __restrict__ bitmap,
                              const ibft_group_desc* __restrict__ groups, const group_dev* __restrict__ gdev,
                              uint32_t n_groups, const slot_dev* __restrict__ slots, uint32_t n_slots,
                              uint32_t* __restrict__ voted, uint32_t* __restrict__ n_valid, uint32_t lo, uint32_t hi) {
  const uint32_t i = lo + blockIdx.x * blockDim.x + threadIdx.x;
  const bool set = i < hi && i < n && ((bitmap[i >> 5] >> (i & 31)) & 1u);
  if (__ballot_sync(0xFFFFFFFFu, set) == 0) return;  // a warp of rejected items reads nothing else
  item_tail t{};
  if (set) t = load_item_tail(items + i);
  const uint32_t g = t.group();
  const bool valid = set && g < n_groups;
  count_valid_warp(n_valid, valid, g);
  uint32_t word = 0, bit = 0;
  if (valid) quorum_vote(t, g, arena, arena_len, groups, gdev, slots, n_slots, &word, &bit);
  or_votes_warp(voted, word, bit);
}

// k_quorum_mark for calls in which a group is bound to the accepted proposal's hash (ibft_group_hash): an item of a bound group
// counts -- enters the voted set and the valid count -- only when it names the bound hash (item_names_hash, group_hash.cuh); an
// item of an unbound group counts when its verdict bit is set, as in k_quorum_mark.  counted (nullptr: not wanted) receives one
// bit per item of [lo, hi), each by an atomic bit update, so that shards may share a bitmap whatever their bounds.  A separate
// kernel: k_quorum_mark and the recover kernels' fused marking stay as they are, and the recover kernels run without a vote sink
// when a call binds hashes (DESIGN.md §3.2).
__global__ void k_quorum_mark_hashed(const ibft_sig_item* __restrict__ items, uint32_t n, const uint8_t* __restrict__ arena,
                                     size_t arena_len, const uint32_t* __restrict__ bitmap, const ibft_group_desc* __restrict__ groups,
                                     const ibft_group_hash* __restrict__ ghash, const group_dev* __restrict__ gdev, uint32_t n_groups,
                                     const slot_dev* __restrict__ slots, uint32_t n_slots, uint32_t* __restrict__ voted,
                                     uint32_t* __restrict__ n_valid, uint32_t* __restrict__ counted, uint32_t lo, uint32_t hi) {
  const uint32_t i = lo + blockIdx.x * blockDim.x + threadIdx.x;
  const bool in = i < hi && i < n;
  const ibft_sig_item* it = items + i;
  item_tail t{};
  if (in) t = load_item_tail(it);
  const uint32_t g = t.group();
  bool c = in && ((bitmap[i >> 5] >> (i & 31)) & 1u) && g < n_groups;
  if (c) {
    const uint32_t mt = ghash != nullptr ? ghash[g].msg_type : IBFT_HASH_UNBOUND;
    if (mt != IBFT_HASH_UNBOUND) c = item_names_hash(*it, arena, arena_len, mt, ghash[g].hash);
  }
  if (counted != nullptr && in) {
    if (c) atomicOr(&counted[i >> 5], 1u << (i & 31));
    else atomicAnd(&counted[i >> 5], ~(1u << (i & 31)));
  }
  count_valid_warp(n_valid, c, g);
  uint32_t word = 0, bit = 0;
  if (c) quorum_vote(t, g, arena, arena_len, groups, gdev, slots, n_slots, &word, &bit);
  or_votes_warp(voted, word, bit);
}

// multi-GPU: OR the ranks' partial voted sets and add their valid counts (partial layout: voted words, then one count per group)
__global__ void k_quorum_merge(const uint32_t* __restrict__ parts, uint32_t n_parts, uint32_t part_stride, uint32_t voted_words,
                               uint32_t n_groups, uint32_t* __restrict__ voted, uint32_t* __restrict__ n_valid) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= voted_words + n_groups) return;
  uint32_t acc = 0;
  for (uint32_t r = 0; r < n_parts; r++) {
    uint32_t v = parts[(size_t)r * part_stride + i];
    acc = i < voted_words ? (acc | v) : (acc + v);
  }
  if (i < voted_words) voted[i] = acc;
  else n_valid[i - voted_words] = acc;
}

// Multi-GPU exchange WITHOUT a library collective: every rank's (bitmap words | partial voted sets | valid counts) sit in a
// buffer its peers have mapped over NVLink (CUDA IPC); this kernel publishes "my round `epoch` is complete", waits for the
// peers' flags, then reads their words straight out of peer memory -- OR-ing the voted sets, summing the counts, and assembling
// the complete bitmap -- so that the all-gather and the merge are ONE launch (the NCCL path costs a collective launch + the
// merge kernel).  Buffer of rank r: [2 parities][words_per_rank] words, then flags[2].  Rounds
// alternate parities: a rank can only start writing parity p for round e+2 after it has seen every peer's flag for round e+1,
// i.e. after every peer has finished reading round e.  The wait is bounded (spin_limit polls): on timeout the kernel reports
// through *timeout_flag and merges nothing -- it never hangs the device.
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_relaxed_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
struct peer_bufs {
  uint32_t* buf[8];  // one node: at most 8 ranks
};
__global__ void k_quorum_exchange(peer_bufs peers, uint32_t world, uint32_t rank, uint32_t words_per_rank, uint32_t bitmap_words,
                                  uint32_t voted_words, uint32_t n_groups, uint32_t epoch, uint32_t spin_limit,
                                  uint32_t* __restrict__ full_bitmap, uint32_t* __restrict__ voted, uint32_t* __restrict__ n_valid,
                                  uint32_t* __restrict__ timeout_flag) {
  __shared__ uint32_t s_ok;
  const uint32_t par = epoch & 1u;
  const size_t flags_off = 2 * (size_t)words_per_rank;
  if (threadIdx.x == 0) {
    if (blockIdx.x == 0) {
      __threadfence_system();  // the verify / mark kernels' writes to my buffer are visible to the peers before the flag is
      st_release_sys(peers.buf[rank] + flags_off + par, epoch);
    }
    uint32_t ok = 1;
    for (uint32_t r = 0; r < world && ok; r++) {
      const uint32_t* f = peers.buf[r] + flags_off + par;
      uint32_t spins = 0;
      while ((int32_t)(ld_acquire_sys(f) - epoch) < 0) {
        if (++spins > spin_limit) { ok = 0; break; }
        __nanosleep(64);
      }
    }
    if (!ok) atomicExch(timeout_flag, 1u);
    s_ok = ok;
  }
  __syncthreads();
  if (!s_ok) return;
  const uint32_t per_rank_bitmap = bitmap_words;  // words [0, bitmap_words) of a rank's buffer: its slice of the bitmap
  const uint32_t total = world * per_rank_bitmap + voted_words + n_groups;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    if (i < world * per_rank_bitmap) {
      const uint32_t r = i / per_rank_bitmap, w = i % per_rank_bitmap;
      full_bitmap[i] = ld_relaxed_sys(peers.buf[r] + (size_t)par * words_per_rank + w);
    } else {
      const uint32_t j = i - world * per_rank_bitmap;  // index into (voted sets | counts)
      uint32_t acc = 0;
      for (uint32_t r = 0; r < world; r++) {
        uint32_t v = ld_relaxed_sys(peers.buf[r] + (size_t)par * words_per_rank + per_rank_bitmap + j);
        acc = j < voted_words ? (acc | v) : (acc + v);
      }
      if (j < voted_words) voted[j] = acc;
      else n_valid[j - voted_words] = acc;
    }
  }
}

// The group's decision (hasQuorumByMsgType, reference core/ibft.go:1273-1284) from what the CTA that summed the group's power
// holds: the quorum rule and proposer of the descriptor, the voted set, the summed power (updated in place: under the PREPARE
// rule the proposer's power joins the sum), the valid count and the slot's threshold.  Rule 0 is HasQuorum.
__device__ __forceinline__ uint32_t group_decision(uint32_t rule, uint32_t proposer, const uint32_t* __restrict__ voted,
                                                   const slot_dev& s, uint32_t n_valid, uint64_t power[5]) {
  if (rule == IBFT_QUORUM_PREPREPARE) return n_valid >= 1 ? 1u : 0u;  // len(msgs) >= 1
  if (rule == IBFT_QUORUM_PREPARE) {                                    // HasPrepareQuorum (validator_manager.go:99-127)
    if (proposer == IBFT_PROPOSER_UNSET) return 0u;                     // no proposal message
    if (proposer != IBFT_PROPOSER_NONE) {
      if (proposer >= s.n) return 0u;                                   // table replaced since the groups were planned: no verdict
      if ((voted[proposer >> 5] >> (proposer & 31)) & 1u) return 0u;    // the proposer is among the senders
      const uint64_t* p = s.powers + 4 * (size_t)proposer;              // the proposer joins the sender set
      unsigned long long c = 0;
#pragma unroll
      for (int k = 0; k < 5; k++) {
        unsigned long long add = k < 4 ? p[k] : 0ull;
        unsigned long long t = power[k] + add;
        unsigned long long c1 = t < add;
        unsigned long long t2 = t + c;
        c1 += t2 < c;
        power[k] = t2;
        c = c1;
      }
    }
  }
  int cmp = 0;  // power >= quorum ?
  for (int k = 4; k >= 0; k--) {
    uint64_t q = s.quorum[k];
    if (cmp == 0 && power[k] != q) cmp = power[k] < q ? -1 : 1;
  }
  return cmp >= 0 ? 1u : 0u;
}

// one CTA per group: 320-bit sum of the voting power of the voted validators, then the group's decision (group_decision)
#define IBFT_REDUCE_THREADS 1024  // one CTA per group; a 10k-validator set is 10 strided passes instead of 40
__global__ void __launch_bounds__(IBFT_REDUCE_THREADS)
k_quorum_reduce(const ibft_group_desc* __restrict__ groups, const group_dev* __restrict__ gdev, uint32_t n_groups,
                const slot_dev* __restrict__ slots, uint32_t n_slots, const uint32_t* __restrict__ voted,
                const uint32_t* __restrict__ n_valid, ibft_group_result* __restrict__ results) {
  __shared__ uint64_t s_sum[IBFT_REDUCE_THREADS][5];
  __shared__ uint32_t s_cnt[IBFT_REDUCE_THREADS];
  uint32_t g = blockIdx.x;
  if (g >= n_groups) return;
  uint32_t slot = groups[g].table_slot;
  bool has_table = slot != IBFT_NO_TABLE && slot < n_slots && slots[slot].valid;
  uint64_t acc[5] = {0, 0, 0, 0, 0};
  uint32_t cnt = 0;
  if (has_table) {
    const slot_dev& s = slots[slot];
    const uint32_t* vw = voted + gdev[g].voted_off;
    for (uint32_t v = threadIdx.x; v < s.n; v += blockDim.x) {
      if ((vw[v >> 5] >> (v & 31)) & 1u) {
        cnt++;
        const uint64_t* p = s.powers + 4 * (size_t)v;
        unsigned long long c = 0;
#pragma unroll
        for (int k = 0; k < 5; k++) {
          unsigned long long add = k < 4 ? p[k] : 0ull;
          unsigned long long t = acc[k] + add;
          unsigned long long c1 = t < add;
          unsigned long long t2 = t + c;
          c1 += t2 < c;
          acc[k] = t2;
          c = c1;
        }
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 5; k++) s_sum[threadIdx.x][k] = acc[k];
  s_cnt[threadIdx.x] = cnt;
  __syncthreads();
  for (uint32_t stride = blockDim.x >> 1; stride > 0; stride >>= 1) {
    if (threadIdx.x < stride) {
      unsigned long long c = 0;
#pragma unroll
      for (int k = 0; k < 5; k++) {
        unsigned long long a = s_sum[threadIdx.x][k], b = s_sum[threadIdx.x + stride][k];
        unsigned long long t = a + b;
        unsigned long long c1 = t < b;
        unsigned long long t2 = t + c;
        c1 += t2 < c;
        s_sum[threadIdx.x][k] = t2;
        c = c1;
      }
      s_cnt[threadIdx.x] += s_cnt[threadIdx.x + stride];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    ibft_group_result r;
#pragma unroll
    for (int k = 0; k < 5; k++) r.power[k] = s_sum[0][k];
    r.n_valid = n_valid[g];
    r.n_distinct = s_cnt[0];
    r.has_quorum = 0;
    r.reserved = 0;
    if (has_table)
      r.has_quorum = group_decision(groups[g].flags & IBFT_QUORUM_RULE_MASK, groups[g].reserved, voted + gdev[g].voted_off, slots[slot],
                                    r.n_valid, r.power);
    results[g] = r;
  }
}

// ------------------------------------------------------------------------------------------------------------
// Reject reasons (ibft_explain_batch): the rejected items only, compacted on the host, one thread each in one-warp CTAs, each
// decided again step by step by explain_item (verify_core.cuh) with the one-thread recovery of k_recover and its membership test.
// A cold path kept apart from the verify kernels, whose register budget and hot loop it leaves alone.  WIDE: u1*G from the wide
// comb, as in k_recover.  Dynamic shared memory: the per-signature R tables, 32 x IBFT_RTAB_WORDS words.
// ------------------------------------------------------------------------------------------------------------
template <bool WIDE>
__global__ void __launch_bounds__(32)
k_explain(const ibft_sig_item* __restrict__ items, uint32_t n, const uint8_t* __restrict__ arena, size_t arena_len,
          const ibft_group_desc* __restrict__ groups, uint32_t n_groups, const slot_dev* __restrict__ slots, uint32_t n_slots,
          const uint32_t* __restrict__ ctable, const uint32_t* __restrict__ wtable, uint8_t* __restrict__ reasons,
          uint8_t* __restrict__ recovered) {
  extern __shared__ uint32_t s_rtab[];
  const uint32_t i = blockIdx.x * 32 + threadIdx.x;
  if (i >= n) return;
  ibft_sig_item it;
  const uint4* src = reinterpret_cast<const uint4*>(items + i);
  uint4* w = reinterpret_cast<uint4*>(&it);
#pragma unroll
  for (int k = 0; k < 8; k++) w[k] = __ldg(src + k);
  gtab_view G{g_gtable};
  G.comb = ctable;
  G.wide = WIDE ? wtable : nullptr;
  rtab_view T{s_rtab + threadIdx.x, 32u};
  auto member = [&](uint32_t group, const uint8_t* signer) {
    int v;
    uint32_t slot;
    return group_member(groups, n_groups, slots, n_slots, group, signer, &v, &slot);
  };
  uint8_t addr[20];
  uint8_t why;
#if IBFT_GEN_WIDE > 0
  if (WIDE) why = explain_item(exec_serial_wide{}, it, arena, arena_len, groups != nullptr, n_groups, G, T, member, addr);
  else
#endif
    why = explain_item(exec_serial{}, it, arena, arena_len, groups != nullptr, n_groups, G, T, member, addr);
  reasons[i] = why;
#pragma unroll
  for (int k = 0; k < 20; k++) recovered[(size_t)i * 20 + k] = addr[k];
}

// ------------------------------------------------------------------------------------------------------------
// Reject reasons of device-resident items (ibft_explain_batch_device), in two launches per chunk of a shard.
// k_explain_compact: one thread per item of [lo, hi) (lo a multiple of 32, so each warp reads one bitmap word).  A one bit gets
// IBFT_REASON_OK and a zero address; the zero bits are appended to worklist[1..] with one atomic per warp (order is free: every
// output is written by index), and their number is added to worklist[0] and to *count (when given).
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_explain_compact(const uint32_t* __restrict__ bitmap, uint32_t lo, uint32_t hi, uint8_t* __restrict__ reasons,
                  uint8_t* __restrict__ recovered, uint32_t* __restrict__ worklist, uint32_t* __restrict__ count) {
  const uint32_t i = lo + blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t lane = threadIdx.x & 31u;
  bool zero = false;
  if (i < hi) {
    const bool one = (__ldg(bitmap + (i >> 5)) >> lane) & 1u;
    zero = !one;
    if (one) {
      reasons[i] = IBFT_REASON_OK;
      if (recovered)
#pragma unroll
        for (int k = 0; k < 20; k++) recovered[(size_t)i * 20 + k] = 0;
    }
  }
  const uint32_t m = __ballot_sync(0xFFFFFFFFu, zero);
  if (m == 0) return;
  uint32_t base = 0;
  if (lane == 0) {
    base = atomicAdd(worklist, (uint32_t)__popc(m));
    if (count) atomicAdd(count, (uint32_t)__popc(m));
  }
  base = __shfl_sync(0xFFFFFFFFu, base, 0);
  if (zero) worklist[1 + base + __popc(m & ((1u << lane) - 1u))] = i;
}

// k_explain_list: k_explain over the worklist of k_explain_compact, launched for the most items the list can hold (the count is
// on the device); threads beyond it leave at once, as in k_recover's worklist mode.  Every listed item has verdict bit 0, so an
// item the pass accepts is IBFT_REASON_INCONSISTENT.  recovered may be null.
template <bool WIDE>
__global__ void __launch_bounds__(32)
k_explain_list(const ibft_sig_item* __restrict__ items, const uint8_t* __restrict__ arena, size_t arena_len,
               const ibft_group_desc* __restrict__ groups, uint32_t n_groups, const slot_dev* __restrict__ slots, uint32_t n_slots,
               const uint32_t* __restrict__ ctable, const uint32_t* __restrict__ wtable, const uint32_t* __restrict__ worklist,
               uint8_t* __restrict__ reasons, uint8_t* __restrict__ recovered) {
  extern __shared__ uint32_t s_rtab[];
  const uint32_t k = blockIdx.x * 32 + threadIdx.x;
  if (k >= worklist[0]) return;
  const uint32_t i = worklist[1 + k];
  ibft_sig_item it;
  const uint4* src = reinterpret_cast<const uint4*>(items + i);
  uint4* w = reinterpret_cast<uint4*>(&it);
#pragma unroll
  for (int j = 0; j < 8; j++) w[j] = __ldg(src + j);
  gtab_view G{g_gtable};
  G.comb = ctable;
  G.wide = WIDE ? wtable : nullptr;
  rtab_view T{s_rtab + threadIdx.x, 32u};
  auto member = [&](uint32_t group, const uint8_t* signer) {
    int v;
    uint32_t slot;
    return group_member(groups, n_groups, slots, n_slots, group, signer, &v, &slot);
  };
  uint8_t addr[20];
  uint8_t why;
#if IBFT_GEN_WIDE > 0
  if (WIDE) why = explain_item(exec_serial_wide{}, it, arena, arena_len, groups != nullptr, n_groups, G, T, member, addr);
  else
#endif
    why = explain_item(exec_serial{}, it, arena, arena_len, groups != nullptr, n_groups, G, T, member, addr);
  reasons[i] = why == IBFT_REASON_OK ? (uint8_t)IBFT_REASON_INCONSISTENT : why;
  if (recovered)
#pragma unroll
    for (int j = 0; j < 20; j++) recovered[(size_t)i * 20 + j] = addr[j];
}

// ------------------------------------------------------------------------------------------------------------
// hash-only batch (IsValidProposalHash)
// ------------------------------------------------------------------------------------------------------------
__global__ void k_keccak_batch(const uint8_t* __restrict__ arena, size_t arena_len, const uint32_t* __restrict__ offs,
                               const uint32_t* __restrict__ lens, const uint64_t* __restrict__ rounds, uint32_t n,
                               uint8_t* __restrict__ out) {
  // rounds == nullptr: out[i] = Keccak-256(message i).
  // rounds != nullptr: the proposal hash of this engine's synthetic convention (SURVEY.md §8c), both sponges in ONE launch:
  //                    out[i] = Keccak-256(Keccak-256(rawProposal_i) || u64_be(round_i))   (IsValidProposalHash)
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint8_t h[40];
  if ((size_t)offs[i] + lens[i] > arena_len) {
#pragma unroll
    for (int k = 0; k < 32; k++) h[k] = 0;
  } else {
    keccak256_bytes(arena + offs[i], lens[i], h);
    if (rounds != nullptr) {
      uint64_t r = rounds[i];
#pragma unroll
      for (int k = 0; k < 8; k++) h[32 + k] = (uint8_t)(r >> (8 * (7 - k)));
      uint8_t h2[32];
      keccak256_bytes(h, 40, h2);
#pragma unroll
      for (int k = 0; k < 32; k++) h[k] = h2[k];
    }
  }
#pragma unroll
  for (int k = 0; k < 32; k++) out[(size_t)i * 32 + k] = h[k];
}

// ------------------------------------------------------------------------------------------------------------
// combined generator table (IBFT_WC > 0): entry (d1, d2) = d1*G + d2*lambda*G, computed with the kernel's own scalar
// multiplication as (d1 + d2*lambda mod n) * G and checked against the oracle in tests/test_gpu_primitives.py
// ------------------------------------------------------------------------------------------------------------
#if IBFT_WC > 0
__global__ void __launch_bounds__(64)
k_build_ctable(uint32_t* __restrict__ out) {  // blockIdx.y = comb position: entries scaled by 2^(WC * position)
  __shared__ uint32_t s_gtab[IBFT_GTAB_ENTRY_WORDS * IBFT_GTAB_ENTRIES];
  __shared__ uint32_t s_rtab[64 * IBFT_RTAB_WORDS];
  for (uint32_t i = threadIdx.x; i < IBFT_GTAB_ENTRY_WORDS * IBFT_GTAB_ENTRIES; i += 64) s_gtab[i] = g_gtable[i];
  __syncthreads();
  size_t e = (size_t)blockIdx.x * 64 + threadIdx.x;
  if (e >= (size_t)IBFT_CTAB_ENTRIES) return;
  int d1 = (int)(e / IBFT_CTAB_D2), d2 = (int)(e % IBFT_CTAB_D2) - (1 << (IBFT_WC - 1));
  const uint32_t lam[8] = {0x1B23BD72u, 0xDF02967Cu, 0x20816678u, 0x122E22EAu, 0x8812645Au, 0xA5261C02u, 0xC05C30E0u, 0x5363AD4Cu};
  sc a, b, l;
#pragma unroll
  for (int i = 0; i < 8; i++) { a.v[i] = 0; b.v[i] = 0; l.v[i] = lam[i]; }
  a.v[0] = (uint32_t)d1;
  b.v[0] = (uint32_t)(d2 < 0 ? -d2 : d2);
  sc t = sc_mul(b, l);
  if (d2 < 0) t = sc_neg(t);
  sc k = sc_add(a, t);
  const uint32_t pos = blockIdx.y;
  if (pos) {
    sc m;
#pragma unroll
    for (int i = 0; i < 8; i++) m.v[i] = 0;
    m.v[(pos * IBFT_WC) / 32] = 1u << ((pos * IBFT_WC) % 32);
    k = sc_mul(k, m);
  }
  uint32_t* o = out + IBFT_GTAB_ENTRY_WORDS * ((size_t)pos * IBFT_CTAB_ENTRIES + e);
  gtab_view G{s_gtab};
  rtab_view T{s_rtab + threadIdx.x, 64u};
  aff g1;
  G.load(0, g1.x, g1.y);
  sc zero;
#pragma unroll
  for (int i = 0; i < 8; i++) zero.v[i] = 0;
  jac P = ecmult_double(k, zero, g1, G, T);
  if (P.inf || fe_is_zero(P.z)) {
#pragma unroll
    for (int i = 0; i < 16; i++) o[i] = 0;  // (0, 0): never looked up
    return;
  }
  fe zi = IBFT_FE_INV(P.z), zi2 = fe_sqr(zi);
  fe x = fe_normalize(fe_mul(P.x, zi2)), y = fe_normalize(fe_mul(P.y, fe_mul(zi2, zi)));
#pragma unroll
  for (int i = 0; i < 8; i++) { o[i] = x.v[i]; o[8 + i] = y.v[i]; }
}
#endif

#if IBFT_GEN_WIDE > 0
// ------------------------------------------------------------------------------------------------------------
// wide generator comb (secp_ec.cuh, IBFT_GEN_WIDE): built once per process and device.  A thread builds a run of IBFT_WIDE_RUN
// consecutive entries of one position: the first by a scalar multiplication, the others by chained mixed additions of the
// position's base 2^(w p) G, all normalised with one inversion (Montgomery's trick).  Every entry is checked on the curve; an
// entry off the curve sets *bad.
// ------------------------------------------------------------------------------------------------------------
#define IBFT_WIDE_RUN 8  // 2 x 7 field elements of the run fit the thread's IBFT_RTAB_WORDS slice of shared memory
// m * 2^(w pos) mod n
__device__ sc wide_scalar(uint32_t pos, uint32_t m) {
  sc a, t;
#pragma unroll
  for (int i = 0; i < 8; i++) { a.v[i] = 0; t.v[i] = 0; }
  a.v[0] = m;
  t.v[(pos * IBFT_GEN_WIDE) / 32] = 1u << ((pos * IBFT_GEN_WIDE) % 32);  // 2^(w pos) <= 2^242 < n
  return sc_mul(a, t);
}
// k * G (k in [1, n)) affine, by the kernel's own double-scalar multiplication with u2 = 0
__device__ void wide_mult_affine(const sc& k, const rtab_view& T, fe& x, fe& y) {
  gtab_view G{g_gtable};
  aff g1;
  G.load(0, g1.x, g1.y);
  sc zero;
#pragma unroll
  for (int i = 0; i < 8; i++) zero.v[i] = 0;
  const jac P = ecmult_double(k, zero, g1, G, T);
  const fe zi = IBFT_FE_INV(P.z), zi2 = fe_sqr(zi);
  x = fe_normalize(fe_mul(P.x, zi2));
  y = fe_normalize(fe_mul(P.y, fe_mul(zi2, zi)));
}
__device__ void wide_store_checked(uint32_t* o, const fe& x, const fe& y, uint32_t* bad) {
  if (!fe_equal(fe_sqr(y), fe_add(fe_mul(fe_sqr(x), x), fe_from_u32(7)))) atomicOr(bad, 1u);
#pragma unroll
  for (int i = 0; i < 8; i++) { o[i] = x.v[i]; o[8 + i] = y.v[i]; }
}
// bases[p] = 2^(w p) G, p = 0 .. IBFT_GW_POSITIONS - 1
__global__ void __launch_bounds__(32) k_wide_bases(uint32_t* __restrict__ bases, uint32_t* __restrict__ bad) {
  __shared__ uint32_t s_rtab[32 * IBFT_RTAB_WORDS];
  const uint32_t p = threadIdx.x;
  if (p >= IBFT_GW_POSITIONS) return;
  fe x, y;
  wide_mult_affine(wide_scalar(p, 1), rtab_view{s_rtab + p, 32u}, x, y);
  wide_store_checked(bases + IBFT_GTAB_ENTRY_WORDS * p, x, y, bad);
}
// blockIdx.y = position; entry index e (m = e + 1) of a position at out + 16 * (pos * IBFT_GW_ENTRIES + e)
__global__ void __launch_bounds__(64) k_build_wtable(uint32_t* __restrict__ out, const uint32_t* __restrict__ bases, uint32_t* __restrict__ bad) {
  __shared__ uint32_t s_rtab[64 * IBFT_RTAB_WORDS];
  const uint32_t pos = blockIdx.y;
  const uint32_t count = pos + 1 < IBFT_GW_POSITIONS ? IBFT_GW_ENTRIES : IBFT_GW_TOP_ENTRIES;
  const uint32_t first = (blockIdx.x * 64 + threadIdx.x) * IBFT_WIDE_RUN;
  if (first >= count) return;
  const int len = (int)min((uint32_t)IBFT_WIDE_RUN, count - first);
  const rtab_view T{s_rtab + threadIdx.x, 64u};  // entry i of the run: (Z_i, Z_1 ... Z_i)
  uint32_t* o = out + IBFT_GTAB_ENTRY_WORDS * ((size_t)pos * IBFT_GW_ENTRIES + first);
  fe bx, by;
#pragma unroll
  for (int i = 0; i < 8; i++) { bx.v[i] = bases[IBFT_GTAB_ENTRY_WORDS * pos + i]; by.v[i] = bases[IBFT_GTAB_ENTRY_WORDS * pos + 8 + i]; }
  jac P;
  wide_mult_affine(wide_scalar(pos, first + 1), T, P.x, P.y);
  P.z = fe_from_u32(1);
  P.inf = false;
  wide_store_checked(o, P.x, P.y, bad);
  // entries 1 .. len-1: P + base (m = 1 makes the first addition a doubling, which the adder handles); Jacobian X, Y parked
  // in the output
  fe pre = P.z;
  IBFT_ROLLED
  for (int i = 1; i < len; i++) {
    P = jac_add_affine(P, bx, by);
    pre = i == 1 ? P.z : fe_mul(pre, P.z);
    T.store(i, P.z, pre);
#pragma unroll
    for (int k = 0; k < 8; k++) { o[16 * i + k] = P.x.v[k]; o[16 * i + 8 + k] = P.y.v[k]; }
  }
  if (len < 2) return;
  fe acc = IBFT_FE_INV(pre);  // 1 / (Z_1 ... Z_{len-1})
  IBFT_ROLLED
  for (int i = len - 1; i >= 1; i--) {
    fe zi = acc, z, t;
    T.load(i, z, t);
    if (i > 1) {
      fe prev;
      T.load(i - 1, t, prev);
      zi = fe_mul(acc, prev);  // 1 / Z_i
      acc = fe_mul(acc, z);
    }
    fe x, y;
#pragma unroll
    for (int k = 0; k < 8; k++) { x.v[k] = o[16 * i + k]; y.v[k] = o[16 * i + 8 + k]; }
    const fe zi2 = fe_sqr(zi);
    wide_store_checked(o + 16 * i, fe_normalize(fe_mul(x, zi2)), fe_normalize(fe_mul(y, fe_mul(zi2, zi))), bad);
  }
}
#endif

#if IBFT_WC > 0
// key registry: comb tables for every registry entry whose key has been learned but whose table is missing.  One thread per
// (entry, comb position): 8*pos doublings, 128 additions and 128 inversions each -- a whole 10k-validator set (170,000
// threads, 21.8 M table entries, 1.39 GB) is built once per engine, whatever the number of resident heights that list it;
// k_keytabs_step then publishes the tables.  tab: the bounded registry's table slot of each entry (nullptr: slot r).
__global__ void __launch_bounds__(64)
k_build_keytabs(const uint32_t* __restrict__ state, const uint32_t* __restrict__ key_xy, const uint32_t* __restrict__ tab,
                uint32_t* const* __restrict__ chunks, uint32_t n_entries) {
  const uint32_t t = blockIdx.x * 64 + threadIdx.x;
  const uint32_t r = t / IBFT_KEYTAB_POSITIONS, pos = t % IBFT_KEYTAB_POSITIONS;
  if (r >= n_entries || state[r] != IBFT_KEY_BUILDING) return;
  aff Q;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    Q.x.v[i] = key_xy[16 * (size_t)r + i];
    Q.y.v[i] = key_xy[16 * (size_t)r + 8 + i];
  }
  const uint32_t slot = tab != nullptr ? tab[r] : r;
  build_keytab_pos(Q, (int)pos, key_table_of(chunks, slot) + (size_t)pos * IBFT_KEYTAB_ENTRIES * IBFT_GTAB_ENTRY_WORDS);
}
// state steps around the build, one launch each on the same stream: LEARNED -> BUILDING (claim: the set of entries this pass
// builds is fixed here -- recover kernels of another lane may keep learning keys meanwhile, those wait for the next pass),
// BUILDING -> READY (publish).  A bounded registry (tab != nullptr) claims only the entries that hold a table slot.
__global__ void __launch_bounds__(256)
k_keytabs_step(uint32_t* __restrict__ state, const uint32_t* __restrict__ tab, uint32_t n_entries, uint32_t from, uint32_t to) {
  const uint32_t r = blockIdx.x * 256 + threadIdx.x;
  if (r < n_entries && state[r] == from && (tab == nullptr || tab[r] != IBFT_KEY_NO_TAB)) state[r] = to;
}
// ibft_set_validators: the new table's key_ref arrives with bit 31 set on the entries just given to an address the registry
// did not hold -- a fresh or a retired entry, whose state (and key) may still be that of another address.  Reset those to
// unknown (and, in a bounded registry, without a table slot), then clear the mark.  Runs while every lane is held and the
// device is idle, before the table is published.
__global__ void __launch_bounds__(256)
k_adopt_entries(uint32_t* __restrict__ key_ref, uint32_t n, uint32_t* __restrict__ state, uint32_t* __restrict__ tab) {
  const uint32_t v = blockIdx.x * 256 + threadIdx.x;
  if (v >= n) return;
  const uint32_t r = key_ref[v];
  if (r & IBFT_KEY_REF_FRESH) {
    state[r & ~IBFT_KEY_REF_FRESH] = IBFT_KEY_UNKNOWN;
    if (tab != nullptr) tab[r & ~IBFT_KEY_REF_FRESH] = IBFT_KEY_NO_TAB;
    key_ref[v] = r & ~IBFT_KEY_REF_FRESH;
  }
}
// Multi-device engines: take the keys another device of the engine has learned.  src_state / src_xy: a copy of that device's
// state and keys of entries [0, n).  The sub-engines number their entries alike (they take every registry-changing call in the
// same order), so entry r names the same address on both -- except after a replication rolled back part way, when it may not:
// key_matches_address against this device's own address of entry r refuses such a key, and the entry learns by recovery.  An
// adopted key is written as learn_key writes a recovered one (first writer wins, every writer stores the same key), so the
// kernel may run beside the verify kernels of any lane; `adopted` counts the keys this launch took.
__global__ void __launch_bounds__(256)
k_adopt_peer_keys(const uint32_t* __restrict__ src_state, const uint32_t* __restrict__ src_xy, uint32_t n, uint32_t* state,
                  uint32_t* key_xy, const uint8_t* __restrict__ addr, uint32_t* learn_count, uint32_t* adopted) {
  const uint32_t r = blockIdx.x * 256 + threadIdx.x;
  if (r >= n) return;
  const uint32_t ss = src_state[r];
  if (!(ss == IBFT_KEY_LEARNED || ss == IBFT_KEY_READY || ss == IBFT_KEY_EVICTED) || state[r] != IBFT_KEY_UNKNOWN) return;
  fe x, y;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    x.v[i] = src_xy[16 * (size_t)r + i];
    y.v[i] = src_xy[16 * (size_t)r + 8 + i];
  }
  if (!key_matches_address(x, y, addr + 20 * (size_t)r)) return;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    key_xy[16 * (size_t)r + i] = x.v[i];
    key_xy[16 * (size_t)r + 8 + i] = y.v[i];
  }
  __threadfence();
  if (atomicCAS(&state[r], IBFT_KEY_UNKNOWN, IBFT_KEY_LEARNED) == IBFT_KEY_UNKNOWN) {
    atomicAdd(learn_count, 1u);
    atomicAdd(adopted, 1u);
  }
}

// Key sharing between engines of separate processes (ibft_key_share_*; block format and decisions in key_share.cuh).
// ibft_set_validators: an entry given to another address forgets that it was exported (runs before k_adopt_entries clears the
// marks of the new table's key_ref).
__global__ void __launch_bounds__(256) k_key_share_forget(const uint32_t* __restrict__ key_ref, uint32_t n, uint32_t* __restrict__ shared) {
  const uint32_t v = blockIdx.x * 256 + threadIdx.x;
  if (v < n && (key_ref[v] & IBFT_KEY_REF_FRESH)) shared[key_ref[v] & ~IBFT_KEY_REF_FRESH] = 0;
}
// Export: one CTA walks entries [0, n_entries) a thousand at a time and writes a record for each exportable one, in ascending
// entry order (a block-wide prefix count gives every record its place), until the block holds IBFT_KEY_SHARE_RECORDS.  The state
// is read before the key: learn_key stores the key, fences, then publishes the state.
__global__ void __launch_bounds__(1024) k_key_export(const uint32_t* state, uint32_t* __restrict__ shared, const uint32_t* key_xy,
                                                     const uint8_t* __restrict__ addr, uint32_t n_entries, uint32_t* __restrict__ block) {
  __shared__ uint32_t s_warp[32];
  __shared__ uint32_t s_total;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  uint32_t base_out = 0;
  for (uint32_t base = 0; base < n_entries && base_out < IBFT_KEY_SHARE_RECORDS; base += 1024) {
    const uint32_t r = base + tid;
    const bool pick = r < n_entries && key_share_exportable(*(volatile const uint32_t*)&state[r], shared[r]);
    const uint32_t ballot = __ballot_sync(0xFFFFFFFFu, pick);
    if (lane == 0) s_warp[warp] = __popc(ballot);
    __syncthreads();
    if (warp == 0) {
      const uint32_t c = s_warp[lane];
      uint32_t incl = c;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, d);
        if (lane >= (uint32_t)d) incl += t;
      }
      s_warp[lane] = incl - c;
      if (lane == 31) s_total = incl;
    }
    __syncthreads();
    const uint32_t pos = base_out + s_warp[warp] + __popc(ballot & ((1u << lane) - 1u));
    if (pick && pos < IBFT_KEY_SHARE_RECORDS) {
      __threadfence();
      uint32_t xy[16];
#pragma unroll
      for (int i = 0; i < 16; i++) xy[i] = key_xy[16 * (size_t)r + i];
      key_share_put(block + 1 + IBFT_KEY_SHARE_RECORD_WORDS * pos, addr + 20 * (size_t)r, xy);
      shared[r] = 1;
    }
    base_out = min(IBFT_KEY_SHARE_RECORDS, base_out + s_total);
    __syncthreads();  // s_warp / s_total are rewritten by the next step
  }
  if (tid == 0) block[0] = base_out;
}
struct key_share_parts {
  const uint32_t* part[IBFT_KEY_SHARE_MAX_PARTS];
};
// Adopt: one thread per record slot of every block but the engine's own (blockIdx.y = block).  The blocks may lie in peer memory
// a peer wrote before publishing a flag this device has seen, so they are read with system-scope loads.  The write of an adopted
// key is learn_key's (first writer wins, every writer stores the same key), so the kernel may run beside the verify kernels;
// the entry is marked exported, so the key is never sent back.  counts (may be nullptr): { adopted, refused }.
__global__ void __launch_bounds__(256)
k_key_adopt(key_share_parts parts, uint32_t self_part, const slot_dev* __restrict__ slots, uint32_t n_slots, uint32_t* state,
            uint32_t* key_xy, const uint8_t* __restrict__ addr, uint32_t* __restrict__ shared, uint32_t* learn_count,
            uint32_t* __restrict__ counts) {
  if (blockIdx.y == self_part) return;
  const uint32_t* blk = parts.part[blockIdx.y];
  const uint32_t i = blockIdx.x * 256 + threadIdx.x;
  const uint32_t count = ld_relaxed_sys(blk);
  if (count > IBFT_KEY_SHARE_RECORDS) {
    if (i == 0 && counts != nullptr) atomicAdd(&counts[1], 1u);
    return;
  }
  if (i >= count) return;
  uint32_t rec[IBFT_KEY_SHARE_RECORD_WORDS];
#pragma unroll
  for (int k = 0; k < (int)IBFT_KEY_SHARE_RECORD_WORDS; k++) rec[k] = ld_relaxed_sys(blk + 1 + IBFT_KEY_SHARE_RECORD_WORDS * i + k);
  auto lookup = [&](uint32_t s, const uint8_t* a) -> int {
    const slot_dev& sd = slots[s];
    if (!sd.valid || sd.key_ref == nullptr) return -1;
    const int v = lookup_validator(sd, a);
    return v < 0 ? -1 : (int)sd.key_ref[v];
  };
  uint32_t r = 0;
  fe x, y;
  const uint32_t d = key_share_decide(rec, n_slots, lookup, state, addr, &r, &x, &y);
  if (d == IBFT_KEY_SHARE_REFUSE && counts != nullptr) atomicAdd(&counts[1], 1u);
  if (d != IBFT_KEY_SHARE_ADOPT) return;
#pragma unroll
  for (int k = 0; k < 8; k++) {
    key_xy[16 * (size_t)r + k] = x.v[k];
    key_xy[16 * (size_t)r + 8 + k] = y.v[k];
  }
  __threadfence();
  if (atomicCAS(&state[r], IBFT_KEY_UNKNOWN, IBFT_KEY_LEARNED) == IBFT_KEY_UNKNOWN) {
    shared[r] = 1;
    atomicAdd(learn_count, 1u);
    if (counts != nullptr) atomicAdd(&counts[0], 1u);
  }
}
#endif

// ------------------------------------------------------------------------------------------------------------
// batched signing (MessageConstructor side)
// ------------------------------------------------------------------------------------------------------------
// Three nonce modes: given (nonces != nullptr), Keccak-derived (nonces == nullptr), and libsecp256k1's RFC 6979 nonce (rfc6979,
// ibft_sign_batch_rfc6979; nonces is then ignored).
__global__ void __launch_bounds__(64)
k_sign(const uint8_t* __restrict__ privkeys, const uint8_t* __restrict__ digests, const uint8_t* __restrict__ nonces, bool rfc6979,
       uint32_t n, uint8_t* __restrict__ sigs) {
  __shared__ uint32_t s_gtab[IBFT_GTAB_ENTRY_WORDS * IBFT_GTAB_ENTRIES];
  __shared__ uint32_t s_rtab[64 * IBFT_RTAB_WORDS];
  for (uint32_t i = threadIdx.x; i < IBFT_GTAB_ENTRY_WORDS * IBFT_GTAB_ENTRIES; i += 64) s_gtab[i] = g_gtable[i];
  __syncthreads();
  uint32_t i = blockIdx.x * 64 + threadIdx.x;
  if (i >= n) return;
  uint8_t d[32], z[32], k[32], sig[65];
#pragma unroll
  for (int j = 0; j < 32; j++) { d[j] = privkeys[32 * (size_t)i + j]; z[j] = digests[32 * (size_t)i + j]; }
  gtab_view G{s_gtab};
  rtab_view T{s_rtab + threadIdx.x, 64u};
  bool ok = false;
  if (rfc6979) {
    ok = ecdsa_sign_rfc6979(d, z, G, T, sig);
  } else if (nonces != nullptr) {
#pragma unroll
    for (int j = 0; j < 32; j++) k[j] = nonces[32 * (size_t)i + j];
    ok = ecdsa_sign(d, z, k, G, T, sig);
  } else {
    // derived nonce: k = Keccak-256(d || z || ctr), ctr = 0, 1, ... until usable (deterministic, unique per (key, digest))
    for (uint32_t ctr = 0; ctr < 4 && !ok; ctr++) {
      uint8_t buf[65];
#pragma unroll
      for (int j = 0; j < 32; j++) { buf[j] = d[j]; buf[32 + j] = z[j]; }
      buf[64] = (uint8_t)ctr;
      keccak256_bytes(buf, 65, k);
      ok = ecdsa_sign(d, z, k, G, T, sig);
    }
  }
#pragma unroll
  for (int j = 0; j < 65; j++) sigs[65 * (size_t)i + j] = ok ? sig[j] : (uint8_t)0;
}

// ------------------------------------------------------------------------------------------------------------
// primitive parity hooks + integer-pipe probes
// ------------------------------------------------------------------------------------------------------------
__global__ void k_debug_op(int op, const uint8_t* a, const uint8_t* b, const uint8_t* c, uint32_t n, uint8_t* out,
                           uint32_t stride) {
#if IBFT_GTAB_SMEM
  __shared__ uint32_t s_gtab[IBFT_GTAB_ENTRY_WORDS * IBFT_GTAB_ENTRIES];
  for (uint32_t i = threadIdx.x; i < IBFT_GTAB_ENTRY_WORDS * IBFT_GTAB_ENTRIES; i += blockDim.x) s_gtab[i] = g_gtable[i];
  __syncthreads();
#else
  const uint32_t* s_gtab = g_gtable;
#endif
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t* pa = a + 32 * (size_t)i;
  const uint8_t* pb = b ? b + 32 * (size_t)i : pa;
  uint8_t* o = out + (size_t)stride * i;
  switch (op) {
    case IBFT_DBG_FE_MUL: fe_to_be(fe_normalize(fe_mul(fe_from_be(pa), fe_from_be(pb))), o); break;
    case IBFT_DBG_FE_SQR: fe_to_be(fe_normalize(fe_sqr(fe_from_be(pa))), o); break;
    case IBFT_DBG_FE_INV: fe_to_be(fe_normalize(IBFT_FE_INV(fe_from_be(pa))), o); break;
    case IBFT_DBG_FE_SQRT: fe_to_be(fe_normalize(fe_sqrt_candidate(fe_from_be(pa))), o); break;
    case IBFT_DBG_FE_ADD: fe_to_be(fe_normalize(fe_add(fe_from_be(pa), fe_from_be(pb))), o); break;
    case IBFT_DBG_FE_SUB: fe_to_be(fe_normalize(fe_sub(fe_from_be(pa), fe_from_be(pb))), o); break;
    case IBFT_DBG_SC_MUL: sc_to_be(sc_mul(sc_from_be(pa), sc_from_be(pb)), o); break;
    case IBFT_DBG_SC_INV: sc_to_be(IBFT_SC_INV(sc_reduce_once(sc_from_be(pa))), o); break;
    case IBFT_DBG_GLV: {
      glv_half h1, h2;
      glv_split(sc_reduce_once(sc_from_be(pa)), h1, h2);
      for (int k = 0; k < 64; k++) o[k] = 0;
      for (int k = 0; k < 5; k++)
        for (int j = 0; j < 4; j++) {
          o[4 * k + j] = (uint8_t)(h1.k[k] >> (8 * j));
          o[24 + 4 * k + j] = (uint8_t)(h2.k[k] >> (8 * j));
        }
      o[20] = h1.neg;
      o[44] = h2.neg;
      break;
    }
    case IBFT_DBG_ECMULT: {
      gtab_view G{s_gtab};
      const uint8_t* pc = c + 64 * (size_t)i;
      aff P;
      P.x = fe_from_be(pc);
      P.y = fe_from_be(pc + 32);
      uint32_t rtab[IBFT_RTAB_WORDS];
      rtab_view T{rtab, 1};
      jac Q = ecmult_double(sc_reduce_once(sc_from_be(pa)), sc_reduce_once(sc_from_be(pb)), P, G, T);
      for (int k = 0; k < 64; k++) o[k] = 0;
      if (!(Q.inf || fe_is_zero(Q.z))) {
        fe zi = IBFT_FE_INV(Q.z), zi2 = fe_sqr(zi);
        fe_to_be(fe_normalize(fe_mul(Q.x, zi2)), o);
        fe_to_be(fe_normalize(fe_mul(Q.y, fe_mul(zi2, zi))), o + 32);
      }
      break;
    }
    case IBFT_DBG_KEY_ADDRESS: o[0] = key_matches_address(fe_from_be(pa), fe_from_be(pb), c + 64 * (size_t)i) ? 1 : 0; break;
    default: debug_arith_op(op, pa, pb, o, c ? c + 64 * (size_t)i : nullptr); break;
  }
}

#define PROBE_ITERS 2048
#define PROBE_UNROLL 16
__global__ void k_probe_imad(uint32_t* out, uint32_t a, uint32_t b) {
  uint32_t x[8];
#pragma unroll
  for (int k = 0; k < 8; k++) x[k] = threadIdx.x + k;
  for (int i = 0; i < PROBE_ITERS; i++) {
#pragma unroll
    for (int u = 0; u < PROBE_UNROLL; u++) {
#pragma unroll
      for (int k = 0; k < 8; k++) asm volatile("mad.lo.u32 %0,%0,%1,%2;" : "+r"(x[k]) : "r"(a), "r"(b));
    }
  }
  uint32_t s = 0;
#pragma unroll
  for (int k = 0; k < 8; k++) s ^= x[k];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
__global__ void k_probe_wide(uint32_t* out, uint32_t a, uint32_t b) {
  uint32_t x[4][8];
#pragma unroll
  for (int k = 0; k < 4; k++)
#pragma unroll
    for (int j = 0; j < 8; j++) x[k][j] = threadIdx.x + k + j;
  for (int i = 0; i < PROBE_ITERS; i++) {
#pragma unroll
    for (int u = 0; u < PROBE_UNROLL / 4; u++) {
#pragma unroll
      for (int k = 0; k < 4; k++) {
        asm volatile(
            "mad.lo.cc.u32 %0,%8,%9,%0; madc.hi.cc.u32 %1,%8,%9,%1;"
            "madc.lo.cc.u32 %2,%8,%9,%2; madc.hi.cc.u32 %3,%8,%9,%3;"
            "madc.lo.cc.u32 %4,%8,%9,%4; madc.hi.cc.u32 %5,%8,%9,%5;"
            "madc.lo.cc.u32 %6,%8,%9,%6; madc.hi.u32 %7,%8,%9,%7;"
            : "+r"(x[k][0]), "+r"(x[k][1]), "+r"(x[k][2]), "+r"(x[k][3]), "+r"(x[k][4]), "+r"(x[k][5]), "+r"(x[k][6]),
              "+r"(x[k][7])
            : "r"(a), "r"(b));
      }
    }
  }
  uint32_t s = 0;
#pragma unroll
  for (int k = 0; k < 4; k++)
#pragma unroll
    for (int j = 0; j < 8; j++) s ^= x[k][j];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// ------------------------------------------------------------------------------------------------------------
// host side: engine object + C ABI
// ------------------------------------------------------------------------------------------------------------
static thread_local char tl_err[512] = "";
static void set_err(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(tl_err, sizeof tl_err, fmt, ap);
  va_end(ap);
}
#define CU(call)                                                                                        \
  do {                                                                                                  \
    cudaError_t _e = (call);                                                                            \
    if (_e != cudaSuccess) {                                                                            \
      set_err("%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__);              \
      return IBFT_ERR_CUDA;                                                                             \
    }                                                                                                   \
  } while (0)

struct slot_host {
  bool valid = false;
  uint64_t height = 0;
  uint32_t n = 0;
  uint32_t* d_keys = nullptr;
  uint64_t* d_powers = nullptr;
  uint64_t quorum[5] = {0, 0, 0, 0, 0};
  // key registry (IBFT_FLAG_KEY_CACHE): registry entry of each validator, on the device and here
  uint32_t* d_key_ref = nullptr;
  std::vector<uint32_t> key_ref;
};

// 20-byte address as a hash-map key
struct addr20 {
  uint8_t b[20];
  bool operator==(const addr20& o) const { return memcmp(b, o.b, 20) == 0; }
};
struct addr20_hash {
  size_t operator()(const addr20& a) const {
    uint64_t x, y;
    uint32_t z;
    memcpy(&x, a.b, 8); memcpy(&y, a.b + 8, 8); memcpy(&z, a.b + 16, 4);
    return (size_t)((x * 0x9E3779B97F4A7C15ull) ^ (y + 0x632BE59BD9B4E019ull + (x << 6) + (x >> 2)) ^ ((uint64_t)z << 29));
  }
};

// The engine's key registry (IBFT_FLAG_KEY_CACHE): one entry per distinct address listed by at least one resident table.
// Device: state and key of every possible entry (allocated at engine creation), comb tables in chunks of IBFT_KEY_CHUNK
// entries allocated as the registry grows (only in ibft_set_validators, which holds every lane and drains the device).
// Host: address -> entry, per-entry reference counts (one per table row that lists the address) and a free list.  An entry
// whose count drops to 0 is retired: its address is forgotten, and the entry goes to the next new address with its state
// reset to unknown.
struct key_registry {
  uint32_t capacity = 0;                 // entries that state / key_xy / the chunk-pointer array can hold
  uint32_t* d_state = nullptr;           // capacity words
  uint32_t* d_key_xy = nullptr;          // capacity x 16 words
  uint8_t* d_addr = nullptr;             // capacity x 20 bytes: the address of each entry handed out (k_adopt_peer_keys checks
                                         // an adopted key against it)
  uint32_t** d_chunks = nullptr;         // capacity / IBFT_KEY_CHUNK (rounded up) chunk base pointers
  uint32_t* d_learn_count = nullptr;     // keys learned so far (learn_key)
  uint32_t* h_learn_count = nullptr;     // pinned
  uint32_t built_count = 0;              // value of *d_learn_count when the tables were last brought up to date
  std::vector<uint32_t*> chunks;         // host copy of the allocated chunk pointers
  uint32_t used = 0;                     // entries [0, used) have been handed out at least once (high-water mark)
  std::unordered_map<addr20, uint32_t, addr20_hash> by_addr;
  std::vector<addr20> addr_of;           // address of each entry in use (a retired entry keeps its last one, here and in d_addr)
  std::vector<uint32_t> refs;            // reference count of each entry
  std::vector<uint32_t> free_list;       // retired entries, reused before the high-water mark moves
  // Bounded registry (ibft_set_key_table_budget, for the rest of the engine's life): `chunks` is a pool of budget.max_tables
  // table slots, chunk i holding chunk_tables[i] of them (0: not allocated yet; the last one may be partial), and an entry
  // holds a slot or none (budget.table, mirrored in d_tab).  Slots are taken away only at reclaim points (every lane held,
  // device drained); the per-call refresh only hands out free ones.
  bool bounded = false;
  ibft::key_budget budget;
  std::vector<uint32_t> chunk_tables;
  uint32_t* d_tab = nullptr;             // capacity words
  uint8_t* d_used = nullptr;             // capacity bytes: used flags of the known-key pass
  bool build_due = false;                // entries admitted at the last reclaim point wait for the next refresh
  // Key sharing between engines (ibft_key_share_*; allocated by the first such call): per entry, 1 once its key was exported
  // or adopted (key_share_exportable)
  uint32_t* d_shared = nullptr;          // capacity words
};

struct pending_call {
  bool active = false;
  uint32_t n = 0, n_groups = 0;
  uint32_t* bitmap_out = nullptr;
  ibft_group_result* results_out = nullptr;
  uint8_t* recovered_out = nullptr;
  uint32_t* counted_out = nullptr;
  bool hashed = false;  // counted bits on the device (a group was bound); else they are the verdict bits
};

// One LANE = everything a host-buffer verify call needs while it is in flight: streams, events, device buffers, pinned
// staging.  The engine has two, so that two handlers do not serialise (the reference runs the COMMIT fan-in, a ROUND_CHANGE
// watcher and the gossip ingress concurrently: core/ibft.go:335-347, :1128):
//   lane 0  full capacity (max_items): bulk handler batches, the async submit/poll/wait API, the device-resident entry points;
//   lane 1  a small lane (IBFT_LANE1_ITEMS) for the ingress coalescer's batches and other small concurrent calls.
// A call holds its lane's mutex from staging to the copy-out; validator tables and the key registry are shared.
#define IBFT_LANES 2
#define IBFT_LANE1_ITEMS 16384u
#define IBFT_LANE1_ARENA (4u << 20)
struct lane {
  std::mutex mu;
  uint32_t cap_items = 0;
  size_t cap_arena = 0;
  cudaStream_t stream = nullptr;
  cudaStream_t copy_stream = nullptr;       // H2D of chunk k+1 overlaps the recover kernel of chunk k
  std::vector<cudaEvent_t> chunk_ev;
  cudaStream_t lat_stream[4] = {nullptr, nullptr, nullptr, nullptr};  // one round in four pieces: copy + kernel of piece k
  cudaEvent_t lat_ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};  // overlap the staging of piece k+1 (latency path)
  cudaEvent_t done_ev = nullptr;
  // device
  ibft_sig_item* d_items = nullptr;
  uint8_t* d_arena = nullptr;
  uint32_t* d_bitmap = nullptr;
  uint8_t* d_recovered = nullptr;
  uint8_t* d_status = nullptr;
  uint8_t* h_status = nullptr;
  uint32_t last_status_n = 0;
  ibft_group_desc* d_groups = nullptr;
  group_dev* d_gdev = nullptr;
  ibft_group_result* d_results = nullptr;
  uint32_t* d_voted = nullptr;
  uint32_t* d_nvalid = nullptr;
  size_t voted_words_cap = 0;
  ibft_group_hash* d_ghash = nullptr;  // hash bindings of the groups (ibft_group_hash), when last_hashes is not empty
  uint32_t* d_counted = nullptr;       // counted bits of a call that binds hashes
  // pinned host staging
  ibft_sig_item* h_items = nullptr;
  uint8_t* h_arena = nullptr;
  uint32_t* h_bitmap = nullptr;
  uint8_t* h_recovered = nullptr;
  ibft_group_desc* h_groups = nullptr;
  group_dev* h_gdev = nullptr;
  ibft_group_result* h_results = nullptr;
  ibft_group_hash* h_ghash = nullptr;
  uint32_t* h_counted = nullptr;
  std::vector<group_dev> last_gdev;  // layout of the voted sets of the most recent reduce
  std::vector<ibft_group_desc> last_groups;
  std::vector<ibft_group_hash> last_hashes;  // hash bindings of last_groups; empty when no group is bound
  pending_call pending;
  uint32_t* d_worklist = nullptr;  // key-registry path: [0] = count, [1..] = indices left to the recover pass
  cudaEvent_t wl_ev[4] = {nullptr, nullptr, nullptr, nullptr};  // last use of each worklist (orders launches that arrive on different streams)
  // worklists the known-key passes of the current host-buffer call filled (bit k = worklist k), and whether one of them was
  // filled twice (its head then holds only the later pass); copied to last_wl_* when the call completes
  uint32_t wl_used = 0, last_wl_used = 0;
  bool wl_reused = false, last_wl_reused = false;
  const uint8_t* dev_arena = nullptr;
  size_t dev_arena_len = 0;
};

struct ibft_engine {
  ibft_engine_params p;
  lane lanes[IBFT_LANES];
  std::atomic<int> last_lane{0};  // lane of the most recently COMPLETED host-buffer call (ibft_last_item_status, ibft_get_voted_bitmap)
  slot_dev* d_slots = nullptr;
  std::vector<slot_host> slots;
  std::vector<slot_dev> slots_shadow;
  std::atomic<uint64_t> launches{0};
  std::atomic<int> recover_path{IBFT_PATH_AUTO};
  std::mutex keys_mu;  // key registry upkeep (reg.built_count); ibft_set_validators changes the registry under every lane's lock
  key_registry reg;
  int sm_count = 132;  // replaced by the device's count at engine creation
  uint32_t* d_ctable = nullptr;  // combined generator table (IBFT_WC > 0)
  uint32_t* d_wtable = nullptr;  // wide generator comb of the device (IBFT_GEN_WIDE > 0), shared; nullptr when it did not fit
  cudaFuncAttributes recover_attr{};
  // ibft_explain_batch_device: [0] = count, [1..max_items] = the zero bits of one chunk of a shard; explain_ev = its last use
  // (calls may arrive on different streams)
  uint32_t* d_explain_wl = nullptr;
  cudaEvent_t explain_ev = nullptr;
  // hashing (ibft_keccak256_batch / ibft_proposal_hash_batch): own lock, own stream, own grow-only scratch -- a hash call
  // never waits for a verify call and never allocates on the per-call path
  std::mutex hash_mu;
  cudaStream_t hash_stream = nullptr;
  uint8_t *hs_arena = nullptr, *hs_h_arena = nullptr, *hs_meta = nullptr, *hs_h_meta = nullptr;
  size_t hs_arena_cap = 0;
  uint32_t hs_n_cap = 0;
  // multi-device engines (ibft_engine_create_multi): a coordinator holds one ordinary engine per device and allocates nothing
  // above; a view is the borrowed diagnostics handle of one of them (ibft_engine_sub)
  struct multi_engine* multi = nullptr;
  ibft_engine* view_of = nullptr;
  bool coordinated = false;  // a sub-engine of a multi-device engine: its coordinator shares and refreshes the learned keys
};
// Entry points of a coordinator or a view (defined with ibft_engine_create_multi at the end of this file)
static int multi_refused(ibft_engine* e, const char* fn);
static ibft_engine* diag_engine(ibft_engine* e);
static void multi_destroy(ibft_engine* e);
static int multi_set_validators(ibft_engine* e, uint32_t table_slot, uint64_t height, const uint8_t* addrs, const uint8_t* powers_be,
                                uint32_t n);
static int multi_verify(ibft_engine* e, const ibft_sig_item* items, uint32_t n, const uint8_t* arena, size_t arena_len,
                        const ibft_group_desc* groups, uint32_t n_groups, uint32_t* bitmap_out, ibft_group_result* results_out,
                        uint8_t* recovered_out, uint8_t* status_out, uint32_t* voted_out, uint32_t voted_stride_words,
                        const ibft_group_hash* ghash = nullptr, uint32_t* counted_out = nullptr);
static int multi_submit(ibft_engine* e, const ibft_sig_item* items, uint32_t n, const uint8_t* arena, size_t arena_len,
                        const ibft_group_desc* groups, uint32_t n_groups, uint32_t* bitmap_out, ibft_group_result* results_out,
                        uint8_t* recovered_out);
static int multi_poll(ibft_engine* e, int* done);
static int multi_wait(ibft_engine* e);
static int multi_last_item_status(ibft_engine* e, uint8_t* status_out, uint32_t n);
static int multi_explain(ibft_engine* e, const ibft_sig_item* items, uint32_t n, const uint8_t* arena, size_t arena_len,
                         const ibft_group_desc* groups, uint32_t n_groups, const uint32_t* bitmap, uint8_t* reasons_out,
                         uint8_t* recovered_out);
static int multi_known_handed_back(ibft_engine* e, uint32_t* n_out);
static int multi_hash(ibft_engine* e, const uint8_t* arena, size_t arena_len, const uint32_t* offsets, const uint32_t* lens,
                      const uint64_t* rounds, uint32_t n, uint8_t* out32);
static int multi_sign(ibft_engine* e, const uint8_t* privkeys, const uint8_t* digests, const uint8_t* nonces, bool rfc6979, uint32_t n,
                      uint8_t* sigs65_out);
static int multi_refresh_key_tables(ibft_engine* e, uint32_t* n_keys_out);
static int multi_set_key_table_budget(ibft_engine* e, uint32_t max_tables);
static int multi_set_recover_path(ibft_engine* e, int path);
static uint64_t multi_launch_count(ibft_engine* e);
// a coordinator or a view: device-pointer calls name memory of one device, and a view only answers diagnostics
#define IBFT_REFUSE_MULTI(e) \
  if ((e) && ((e)->multi || (e)->view_of)) return multi_refused((e), __func__)
#define IBFT_REFUSE_VIEW(e) \
  if ((e) && (e)->view_of) return multi_refused((e), __func__)
// the one-thread recover kernel of an engine: u1*G from the wide comb when the engine holds it
template <int BLOCK>
static decltype(&k_recover<BLOCK, false>) recover_kernel(const ibft_engine* e) {
  return e->d_wtable != nullptr ? k_recover<BLOCK, true> : k_recover<BLOCK, false>;
}
// launches kernel k on st, counts it (ibft_launch_count) and returns its launch error
template <typename... P, typename... A>
static cudaError_t launch(ibft_engine* e, void (*k)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, A... args) {
  k<<<grid, block, smem, st>>>(args...);
  e->launches++;
  return cudaGetLastError();
}
// every lane, in index order (validator-table replacement and other engine-wide operations)
struct all_lanes_lock {
  ibft_engine* e;
  explicit all_lanes_lock(ibft_engine* e_) : e(e_) { for (auto& L : e->lanes) L.mu.lock(); }
  ~all_lanes_lock() { for (int i = IBFT_LANES - 1; i >= 0; i--) e->lanes[i].mu.unlock(); }
};

extern "C" int ibft_abi_version(void) { return IBFT_ABI_VERSION; }
extern "C" const char* ibft_last_error(void) { return tl_err; }

static void lane_free(lane* L) {
  cudaFree(L->d_status); cudaFreeHost(L->h_status);
  cudaFree(L->d_worklist);
  cudaFree(L->d_items); cudaFree(L->d_arena); cudaFree(L->d_bitmap); cudaFree(L->d_recovered); cudaFree(L->d_groups);
  cudaFree(L->d_gdev); cudaFree(L->d_results); cudaFree(L->d_voted); cudaFree(L->d_nvalid);
  cudaFreeHost(L->h_items); cudaFreeHost(L->h_arena); cudaFreeHost(L->h_bitmap); cudaFreeHost(L->h_recovered);
  cudaFreeHost(L->h_groups); cudaFreeHost(L->h_gdev); cudaFreeHost(L->h_results);
  cudaFree(L->d_ghash); cudaFree(L->d_counted); cudaFreeHost(L->h_ghash); cudaFreeHost(L->h_counted);
  if (L->done_ev) cudaEventDestroy(L->done_ev);
  for (auto ev : L->chunk_ev) cudaEventDestroy(ev);
  if (L->copy_stream) cudaStreamDestroy(L->copy_stream);
  for (auto ls : L->lat_stream) if (ls) cudaStreamDestroy(ls);
  for (auto ev : L->lat_ev) if (ev) cudaEventDestroy(ev);
  for (auto ev : L->wl_ev) if (ev) cudaEventDestroy(ev);
  if (L->stream) cudaStreamDestroy(L->stream);
}

// The wide generator comb: 1.38 GiB at w = 22, so ONE per device, shared by every engine of the process and freed by the last
// engine on the device to close.  Built on the first engine's lane-0 stream while the registry lock is held.
struct wide_table_ref {
  uint32_t* d = nullptr;
  int refs = 0;
};
static std::mutex g_wide_mu;
static std::unordered_map<int, wide_table_ref> g_wide;

static int wide_acquire(ibft_engine* e, cudaStream_t st) {
#if IBFT_GEN_WIDE > 0
  std::lock_guard<std::mutex> lk(g_wide_mu);
  wide_table_ref& w = g_wide[e->p.device];
  if (w.refs == 0) {
    // the table, then the positions' bases 2^(w p) G, then the on-curve flag (one entry's worth of words)
    const size_t entries = IBFT_GW_TOTAL + IBFT_GW_POSITIONS + 1;
    uint32_t* d = nullptr;
    if (cudaMalloc(&d, entries * IBFT_GTAB_ENTRY_WORDS * 4) != cudaSuccess) {
      (void)cudaGetLastError();  // does not fit: this engine adds u1*G by the per-position comb, with the same verdicts
      g_wide.erase(e->p.device);
      return IBFT_OK;
    }
    uint32_t* bases = d + IBFT_GW_TOTAL * IBFT_GTAB_ENTRY_WORDS;
    uint32_t* bad = bases + IBFT_GW_POSITIONS * IBFT_GTAB_ENTRY_WORDS;
    uint32_t h_bad = 0;
    cudaError_t ce = cudaMemsetAsync(bad, 0, 4, st);
    if (ce == cudaSuccess) {
      k_wide_bases<<<1, 32, 0, st>>>(bases, bad);
      k_build_wtable<<<dim3((IBFT_GW_ENTRIES + 64 * IBFT_WIDE_RUN - 1) / (64 * IBFT_WIDE_RUN), IBFT_GW_POSITIONS), 64, 0, st>>>(d, bases, bad);
      e->launches += 2;
      ce = cudaGetLastError();
    }
    if (ce == cudaSuccess) ce = cudaMemcpyAsync(&h_bad, bad, 4, cudaMemcpyDeviceToHost, st);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
    if (ce != cudaSuccess || h_bad) {
      cudaFree(d);
      g_wide.erase(e->p.device);
      if (ce != cudaSuccess) set_err("wide generator comb: %s", cudaGetErrorString(ce));
      else set_err("wide generator comb: an entry built on the device is not on the curve");
      return IBFT_ERR_CUDA;
    }
    w.d = d;
  }
  w.refs++;
  e->d_wtable = w.d;
#else
  (void)e;
  (void)st;
#endif
  return IBFT_OK;
}

static void wide_release(ibft_engine* e) {
  if (!e->d_wtable) return;
  std::lock_guard<std::mutex> lk(g_wide_mu);
  auto it = g_wide.find(e->p.device);
  if (--it->second.refs == 0) {
    cudaFree(it->second.d);
    g_wide.erase(it);
  }
  e->d_wtable = nullptr;
}

static void engine_free(ibft_engine* e) {
  if (!e) return;
  cudaSetDevice(e->p.device);
  cudaDeviceSynchronize();
  wide_release(e);
  for (auto& s : e->slots) {
    if (s.d_keys) cudaFree(s.d_keys);
    if (s.d_powers) cudaFree(s.d_powers);
    cudaFree(s.d_key_ref);
  }
  for (auto& L : e->lanes) lane_free(&L);
  cudaFree(e->d_ctable);
  for (auto c : e->reg.chunks) cudaFree(c);
  cudaFree(e->reg.d_tab); cudaFree(e->reg.d_used); cudaFree(e->reg.d_shared);
  cudaFree(e->reg.d_state); cudaFree(e->reg.d_key_xy); cudaFree(e->reg.d_addr); cudaFree(e->reg.d_chunks); cudaFree(e->reg.d_learn_count);
  cudaFreeHost(e->reg.h_learn_count);
  cudaFree(e->d_slots);
  cudaFree(e->d_explain_wl);
  if (e->explain_ev) cudaEventDestroy(e->explain_ev);
  if (e->hash_stream) cudaStreamDestroy(e->hash_stream);
  cudaFree(e->hs_arena); cudaFreeHost(e->hs_h_arena); cudaFree(e->hs_meta); cudaFreeHost(e->hs_h_meta);
  delete e;
}

static int lane_alloc(ibft_engine* e, lane* L, uint32_t cap_items, size_t cap_arena) {
  const ibft_engine_params& p = e->p;
  L->cap_items = cap_items;
  L->cap_arena = cap_arena;
  CU(cudaStreamCreateWithFlags(&L->stream, cudaStreamNonBlocking));
  CU(cudaStreamCreateWithFlags(&L->copy_stream, cudaStreamNonBlocking));
  for (auto& ls : L->lat_stream) CU(cudaStreamCreateWithFlags(&ls, cudaStreamNonBlocking));
  for (auto& ev : L->lat_ev) CU(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
  for (auto& ev : L->wl_ev) CU(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
  CU(cudaEventCreateWithFlags(&L->done_ev, cudaEventDisableTiming));
  size_t n = cap_items, words = (n + 31) / 32;
  CU(cudaMalloc(&L->d_items, n * sizeof(ibft_sig_item)));
  if (p.flags & IBFT_FLAG_KEY_CACHE)
    CU(cudaMalloc(&L->d_worklist, 4 * (n + 1) * 4));  // four lists: chunks of a large host batch alternate between two streams, the
                                                      // four pieces of a mid-size round (latency path) run side by side
  CU(cudaMalloc(&L->d_arena, std::max<size_t>(cap_arena, 16)));
  CU(cudaMalloc(&L->d_bitmap, std::max<size_t>(words, 1) * 4));
  CU(cudaMalloc(&L->d_recovered, n * 20));
  CU(cudaMalloc(&L->d_status, n));
  CU(cudaHostAlloc(&L->h_status, n, cudaHostAllocDefault));
  CU(cudaMalloc(&L->d_groups, (size_t)p.max_groups * sizeof(ibft_group_desc)));
  CU(cudaMalloc(&L->d_gdev, (size_t)p.max_groups * sizeof(group_dev)));
  CU(cudaMalloc(&L->d_results, (size_t)p.max_groups * sizeof(ibft_group_result)));
  L->voted_words_cap = (size_t)p.max_groups * ((p.max_validators + 31) / 32);
  CU(cudaMalloc(&L->d_voted, std::max<size_t>(L->voted_words_cap, 1) * 4));
  CU(cudaMalloc(&L->d_nvalid, (size_t)p.max_groups * 4));
  CU(cudaHostAlloc(&L->h_items, n * sizeof(ibft_sig_item), cudaHostAllocDefault));
  CU(cudaHostAlloc(&L->h_arena, std::max<size_t>(cap_arena, 16), cudaHostAllocDefault));
  CU(cudaHostAlloc(&L->h_bitmap, std::max<size_t>(words, 1) * 4, cudaHostAllocDefault));
  CU(cudaHostAlloc(&L->h_recovered, n * 20, cudaHostAllocDefault));
  CU(cudaHostAlloc(&L->h_groups, (size_t)p.max_groups * sizeof(ibft_group_desc), cudaHostAllocDefault));
  CU(cudaHostAlloc(&L->h_gdev, (size_t)p.max_groups * sizeof(group_dev), cudaHostAllocDefault));
  CU(cudaHostAlloc(&L->h_results, (size_t)p.max_groups * sizeof(ibft_group_result), cudaHostAllocDefault));
  CU(cudaMalloc(&L->d_ghash, std::max<size_t>(p.max_groups, 1) * sizeof(ibft_group_hash)));
  CU(cudaMalloc(&L->d_counted, std::max<size_t>(words, 1) * 4));
  CU(cudaHostAlloc(&L->h_ghash, std::max<size_t>(p.max_groups, 1) * sizeof(ibft_group_hash), cudaHostAllocDefault));
  CU(cudaHostAlloc(&L->h_counted, std::max<size_t>(words, 1) * 4, cudaHostAllocDefault));
  return IBFT_OK;
}

static int engine_alloc(ibft_engine* e) {
  const ibft_engine_params& p = e->p;
  CU(cudaSetDevice(p.device));
  CU(cudaStreamCreateWithFlags(&e->hash_stream, cudaStreamNonBlocking));
  int rc = lane_alloc(e, &e->lanes[0], p.max_items, p.max_payload_bytes);
  if (rc != IBFT_OK) return rc;
  rc = lane_alloc(e, &e->lanes[1], std::min<uint32_t>(p.max_items, IBFT_LANE1_ITEMS), std::min<size_t>(p.max_payload_bytes, IBFT_LANE1_ARENA));
  if (rc != IBFT_OK) return rc;
  lane* L = &e->lanes[0];
  if (p.flags & IBFT_FLAG_KEY_CACHE) {
    // the most entries there can ever be: every slot full of distinct addresses, plus the table ibft_set_validators is
    // installing (its references are taken before the slot's previous content lets go of its own)
    key_registry& R = e->reg;
    const size_t cap = ((size_t)p.max_table_slots + 1) * p.max_validators;
    if (cap >= IBFT_KEY_REF_FRESH) { set_err("key registry of %zu entries: at most 2^31 - 1", cap); return IBFT_ERR_INVALID_ARG; }
    R.capacity = (uint32_t)cap;
    const size_t n_chunks = (cap + IBFT_KEY_CHUNK - 1) / IBFT_KEY_CHUNK;
    CU(cudaMalloc(&R.d_state, std::max<size_t>(cap, 1) * 4));
    CU(cudaMalloc(&R.d_key_xy, std::max<size_t>(cap, 1) * 64));
    CU(cudaMalloc(&R.d_addr, std::max<size_t>(cap, 1) * 20));
    CU(cudaMalloc(&R.d_chunks, std::max<size_t>(n_chunks, 1) * sizeof(uint32_t*)));
    CU(cudaMemset(R.d_chunks, 0, std::max<size_t>(n_chunks, 1) * sizeof(uint32_t*)));
    CU(cudaMalloc(&R.d_learn_count, 4));
    CU(cudaMemset(R.d_learn_count, 0, 4));
    CU(cudaHostAlloc(&R.h_learn_count, 4, cudaHostAllocDefault));
  }
  CU(cudaMalloc(&e->d_slots, (size_t)p.max_table_slots * sizeof(slot_dev)));
  CU(cudaMemset(e->d_slots, 0, (size_t)p.max_table_slots * sizeof(slot_dev)));
  CU(cudaMalloc(&e->d_explain_wl, ((size_t)p.max_items + 1) * 4));
  CU(cudaEventCreateWithFlags(&e->explain_ev, cudaEventDisableTiming));
  e->slots.resize(p.max_table_slots);
  e->slots_shadow.assign(p.max_table_slots, slot_dev{});
  CU(cudaMemcpyToSymbol(g_gtable, IBFT_GTABLE, sizeof(uint32_t) * IBFT_GTAB_ENTRY_WORDS * IBFT_GTAB_ENTRIES));
  for (bool wide : {false, true}) {
    CU(cudaFuncSetAttribute(wide ? k_recover<IBFT_BLOCK, true> : k_recover<IBFT_BLOCK, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            IBFT_BLOCK * IBFT_RTAB_WORDS * 4));
    CU(cudaFuncSetAttribute(wide ? k_recover<32, true> : k_recover<32, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            32 * IBFT_RTAB_WORDS * 4));
  }
#if IBFT_WC > 0
  CU(cudaFuncSetAttribute(k_recover_split, cudaFuncAttributeMaxDynamicSharedMemorySize, IBFT_SPLIT_SMEM));
  CU(cudaFuncSetAttribute(k_verify_split, cudaFuncAttributeMaxDynamicSharedMemorySize, IBFT_VSPLIT_SMEM));
#endif
  {
    cudaDeviceProp prop;
    CU(cudaGetDeviceProperties(&prop, p.device));
    e->sm_count = prop.multiProcessorCount;
  }
#if IBFT_WC > 0
  {
    // position 0 is the combined table of the interleaved window loop; positions 1.. are the comb tables of the split
    // latency kernel's helper warps (36 MB in all: they fit in the H100's 50 MB L2 while a round is being verified)
    size_t entries = (size_t)IBFT_CTAB_ENTRIES;
    CU(cudaMalloc(&e->d_ctable, (size_t)IBFT_CTAB_POSITIONS * entries * IBFT_GTAB_ENTRY_WORDS * 4));
    CU(launch(e, k_build_ctable, dim3((unsigned)((entries + 63) / 64), IBFT_CTAB_POSITIONS), 64, 0, L->stream, e->d_ctable));
  }
#endif
  rc = wide_acquire(e, L->stream);
  if (rc != IBFT_OK) return rc;
  CU(cudaFuncGetAttributes(&e->recover_attr, recover_kernel<IBFT_BLOCK>(e)));
  CU(cudaDeviceSynchronize());
  return IBFT_OK;
}

// test hook: copy `count` entries of the generator comb tables starting at entry `first` (64 bytes each, x then y as 8
// little-endian words); entry p * entries + i is entry i of comb position p (position 0 = the combined table).  Returns
// IBFT_ERR_INVALID_ARG when the library was built without a combined table
extern "C" int ibft_debug_ctable(ibft_engine* e, uint32_t first, uint32_t count, uint8_t* out, int* wc, uint32_t* entries) {
  e = diag_engine(e);
  if (!e) { set_err("null engine"); return IBFT_ERR_INVALID_ARG; }
  if (wc) *wc = IBFT_WC;
#if IBFT_WC > 0
  if (entries) *entries = (uint32_t)IBFT_CTAB_ENTRIES;
  if (count == 0) return IBFT_OK;
  if (!out || (size_t)first + count > (size_t)IBFT_CTAB_POSITIONS * IBFT_CTAB_ENTRIES) { set_err("range"); return IBFT_ERR_INVALID_ARG; }
  CU(cudaSetDevice(e->p.device));
  CU(cudaMemcpy(out, e->d_ctable + (size_t)first * IBFT_GTAB_ENTRY_WORDS, (size_t)count * 64, cudaMemcpyDeviceToHost));
  return IBFT_OK;
#else
  if (entries) *entries = 0;
  (void)first; (void)out;
  return count == 0 ? IBFT_OK : IBFT_ERR_INVALID_ARG;
#endif
}

// test hook: copy `count` entries of the wide generator comb starting at entry `first` (entry p * entries + m - 1 = m * 2^(w p) G)
extern "C" int ibft_debug_wtable(ibft_engine* e, uint32_t first, uint32_t count, uint8_t* out, int* w, uint32_t* entries, uint32_t* total) {
  e = diag_engine(e);
  if (!e) { set_err("null engine"); return IBFT_ERR_INVALID_ARG; }
  if (w) *w = e->d_wtable ? IBFT_GEN_WIDE : 0;
#if IBFT_GEN_WIDE > 0
  if (entries) *entries = IBFT_GW_ENTRIES;
  if (total) *total = (uint32_t)IBFT_GW_TOTAL;
  if (count == 0) return IBFT_OK;
  if (!e->d_wtable || !out || (size_t)first + count > IBFT_GW_TOTAL) { set_err("range"); return IBFT_ERR_INVALID_ARG; }
  CU(cudaSetDevice(e->p.device));
  CU(cudaMemcpy(out, e->d_wtable + (size_t)first * IBFT_GTAB_ENTRY_WORDS, (size_t)count * 64, cudaMemcpyDeviceToHost));
  return IBFT_OK;
#else
  if (entries) *entries = 0;
  if (total) *total = 0;
  (void)first; (void)out;
  return count == 0 ? IBFT_OK : IBFT_ERR_INVALID_ARG;
#endif
}

// test hook: the key registry entry of validator `validator` (validator-index order) of a table slot -- its state
// (IBFT_KEY_*), the learned affine key (x, y as 8 little-endian words each) and `count` comb entries starting at `first`
// (entry j * 128 + m - 1 = m * 2^(8j) * Q, same format as ibft_debug_ctable).  Read through the slot's key_ref into the
// engine's registry.  Waits for the device.
extern "C" int ibft_debug_keytab(ibft_engine* e, uint32_t table_slot, uint32_t validator, uint32_t first, uint32_t count, uint8_t* out,
                                 uint32_t* state_out, uint8_t* key_out) {
  e = diag_engine(e);
  if (!e) { set_err("null engine"); return IBFT_ERR_INVALID_ARG; }
#if IBFT_WC > 0
  all_lanes_lock lk(e);
  if (table_slot >= e->p.max_table_slots || !e->slots[table_slot].valid) { set_err("slot %u not set", table_slot); return IBFT_ERR_NO_TABLE; }
  const slot_host& s = e->slots[table_slot];
  if (!e->reg.d_state) { set_err("engine has no key registry"); return IBFT_ERR_INVALID_ARG; }
  if (validator >= s.n || (count && !out) || (size_t)first + count > (size_t)IBFT_KEYTAB_POSITIONS * IBFT_KEYTAB_ENTRIES) {
    set_err("range");
    return IBFT_ERR_INVALID_ARG;
  }
  const uint32_t r = s.key_ref[validator];
  const uint32_t t = e->reg.bounded ? e->reg.budget.table[r] : r;
  CU(cudaSetDevice(e->p.device));
  CU(cudaDeviceSynchronize());
  if (state_out) {
    CU(cudaMemcpy(state_out, e->reg.d_state + r, 4, cudaMemcpyDeviceToHost));
    if (*state_out == IBFT_KEY_EVICTED) *state_out = IBFT_KEY_LEARNED;
  }
  if (key_out) CU(cudaMemcpy(key_out, e->reg.d_key_xy + 16 * (size_t)r, 64, cudaMemcpyDeviceToHost));
  if (count) {
    if (t == IBFT_KEY_NO_TAB) { set_err("validator %u has no comb table", validator); return IBFT_ERR_INVALID_ARG; }
    const uint32_t* tab = e->reg.chunks[t / IBFT_KEY_CHUNK] + (size_t)(t % IBFT_KEY_CHUNK) * IBFT_KEYTAB_WORDS;
    CU(cudaMemcpy(out, tab + (size_t)first * IBFT_GTAB_ENTRY_WORDS, (size_t)count * 64, cudaMemcpyDeviceToHost));
  }
  return IBFT_OK;
#else
  (void)table_slot; (void)validator; (void)first; (void)count; (void)out; (void)state_out; (void)key_out;
  set_err("library built without a key registry");
  return IBFT_ERR_INVALID_ARG;
#endif
}

// test hook: the key registry as a whole -- entries in use (distinct addresses of the resident tables), how many of those have a
// finished comb table, and the bytes of comb-table chunks allocated so far.  Any output may be NULL.  Waits for the device.
extern "C" int ibft_debug_key_registry(ibft_engine* e, uint32_t* entries_in_use, uint32_t* entries_ready, uint64_t* bytes_reserved) {
  e = diag_engine(e);
  if (!e) { set_err("null engine"); return IBFT_ERR_INVALID_ARG; }
  all_lanes_lock lk(e);
  const key_registry& R = e->reg;
  if (!R.d_state) { set_err("engine has no key registry"); return IBFT_ERR_INVALID_ARG; }
  CU(cudaSetDevice(e->p.device));
  CU(cudaDeviceSynchronize());
  std::vector<uint32_t> state(R.used);
  if (R.used) CU(cudaMemcpy(state.data(), R.d_state, (size_t)R.used * 4, cudaMemcpyDeviceToHost));
  uint32_t ready = 0;
  for (const auto& kv : R.by_addr) ready += state[kv.second] == IBFT_KEY_READY;
  if (entries_in_use) *entries_in_use = (uint32_t)R.by_addr.size();
  if (entries_ready) *entries_ready = ready;
  uint64_t tables = (uint64_t)R.chunks.size() * IBFT_KEY_CHUNK;
  if (R.bounded) { tables = 0; for (uint32_t c : R.chunk_tables) tables += c; }
  if (bytes_reserved) *bytes_reserved = tables * IBFT_KEYTAB_WORDS * 4;
  return IBFT_OK;
}

// test hook: number of items the known-key pass of the most recent completed host-buffer call handed to the recover pass
// (the sum of the heads of the worklists that call filled; 0 when it took no known-key pass)
extern "C" int ibft_debug_known_handed_back(ibft_engine* e, uint32_t* n_out) {
  if (!e || !n_out) { set_err("null argument"); return IBFT_ERR_INVALID_ARG; }
  if (e->multi) return multi_known_handed_back(e, n_out);
  e = diag_engine(e);
  lane* L = &e->lanes[e->last_lane.load()];
  std::lock_guard<std::mutex> lk(L->mu);
  if (L->pending.active) { set_err("a submitted call is still pending"); return IBFT_ERR_INVALID_ARG; }
  if (L->last_wl_reused) { set_err("the last call filled one worklist twice: its count is not kept"); return IBFT_ERR_INVALID_ARG; }
  uint32_t total = 0;
  CU(cudaSetDevice(e->p.device));
  for (uint32_t k = 0; k < 4; k++) {
    if (!((L->last_wl_used >> k) & 1u)) continue;
    uint32_t head = 0;
    CU(cudaMemcpy(&head, L->d_worklist + (size_t)k * ((size_t)L->cap_items + 1), 4, cudaMemcpyDeviceToHost));
    total += head;
  }
  *n_out = total;
  return IBFT_OK;
}

extern "C" int ibft_engine_create(const ibft_engine_params* params, ibft_engine** out) {
  if (!params || !out) { set_err("null argument"); return IBFT_ERR_INVALID_ARG; }
  *out = nullptr;
  int count = 0;
  cudaError_t ce = cudaGetDeviceCount(&count);
  if (ce != cudaSuccess || count <= 0) {
    set_err("no CUDA device available (%s): this engine has no CPU fallback", ce != cudaSuccess ? cudaGetErrorString(ce) : "device count 0");
    return IBFT_ERR_NO_DEVICE;
  }
  if (params->device < 0 || params->device >= count || params->max_items == 0 || params->max_groups == 0 ||
      params->max_groups > 65535 || params->max_table_slots == 0 || params->max_table_slots > 65535) {
    set_err("invalid engine parameters");
    return IBFT_ERR_INVALID_ARG;
  }
  ibft_engine* e = new ibft_engine();
  e->p = *params;
  e->p.max_items = (e->p.max_items + 31u) & ~31u;
  int rc = engine_alloc(e);
  if (rc != IBFT_OK) { engine_free(e); return rc; }
  *out = e;
  return IBFT_OK;
}

extern "C" void ibft_engine_destroy(ibft_engine* e) {
  if (e && e->view_of) return;  // borrowed: it goes with its coordinator
  if (e && e->multi) return multi_destroy(e);
  engine_free(e);
}

extern "C" int ibft_engine_device_info(ibft_engine* e, ibft_device_info* out) {
  e = diag_engine(e);
  if (!e || !out) { set_err("null argument"); return IBFT_ERR_INVALID_ARG; }
  cudaDeviceProp prop;
  CU(cudaGetDeviceProperties(&prop, e->p.device));
  memset(out, 0, sizeof *out);
  snprintf(out->name, sizeof out->name, "%.63s", prop.name);
  out->sm_count = prop.multiProcessorCount;
  out->cc_major = prop.major;
  out->cc_minor = prop.minor;
  int khz = 0;
  cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, e->p.device);
  out->clock_khz = khz;
  out->total_mem = prop.totalGlobalMem;
  out->abi_version = IBFT_ABI_VERSION;
  out->kernel_regs = e->recover_attr.numRegs;
  out->kernel_smem_bytes = (int32_t)e->recover_attr.sharedSizeBytes + IBFT_BLOCK * IBFT_RTAB_WORDS * 4;
  out->block_threads = IBFT_BLOCK;
  return IBFT_OK;
}

// 256-bit big-endian -> 4 little-endian u64 limbs
static void be32_to_limbs(const uint8_t* b, uint64_t l[4]) {
  for (int i = 0; i < 4; i++) {
    uint64_t w = 0;
    for (int j = 0; j < 8; j++) w = (w << 8) | b[(3 - i) * 8 + j];
    l[i] = w;
  }
}

// Key registry (caller holds every lane, device idle): one reference per row of a table being installed.  An address the
// registry does not hold takes a retired entry, or the next one above the high-water mark; its row of `refs` carries
// IBFT_KEY_REF_FRESH.  The comb-table pool grows by whole chunks when the high-water mark passes its last one.  On failure
// (IBFT_ERR_CAPACITY: the pool could not grow) the registry is exactly as it was.
static int registry_acquire(ibft_engine* e, const uint8_t* addrs, uint32_t n, std::vector<uint32_t>& refs) {
  key_registry& R = e->reg;
  const uint32_t used0 = R.used;
  const size_t chunks0 = R.chunks.size();
  std::vector<uint32_t> fresh;  // entries given to new addresses, in the order they were taken
  refs.assign(n, 0);
  for (uint32_t v = 0; v < n; v++) {
    addr20 a;
    memcpy(a.b, addrs + 20 * (size_t)v, 20);
    auto ins = R.by_addr.emplace(a, 0u);
    if (ins.second) {
      uint32_t r;
      if (!R.free_list.empty()) { r = R.free_list.back(); R.free_list.pop_back(); }
      else r = R.used++;
      ins.first->second = r;
      if (R.addr_of.size() <= r) { R.addr_of.resize((size_t)r + 1); R.refs.resize((size_t)r + 1, 0u); }
      R.addr_of[r] = a;
      fresh.push_back(r);
      refs[v] = r | IBFT_KEY_REF_FRESH;
    } else {
      refs[v] = ins.first->second;
    }
  }
  cudaError_t ce = cudaSuccess;
  const size_t need = R.bounded ? 0 : ((size_t)R.used + IBFT_KEY_CHUNK - 1) / IBFT_KEY_CHUNK;  // a bounded pool grows lazily
  while (R.used <= R.capacity && R.chunks.size() < need) {
    uint32_t* c = nullptr;
    ce = cudaMalloc(&c, (size_t)IBFT_KEY_CHUNK * IBFT_KEYTAB_WORDS * 4);
    if (ce != cudaSuccess) break;
    R.chunks.push_back(c);
  }
  if (ce == cudaSuccess && R.chunks.size() > chunks0)
    ce = cudaMemcpy(R.d_chunks + chunks0, R.chunks.data() + chunks0, (R.chunks.size() - chunks0) * sizeof(uint32_t*), cudaMemcpyHostToDevice);
  if (ce != cudaSuccess || R.used > R.capacity) {
    set_err("key registry: %zu new addresses do not fit (%u entries in use, %zu chunks of %u): %s", fresh.size(),
            (uint32_t)(R.by_addr.size() - fresh.size()), chunks0, IBFT_KEY_CHUNK,
            ce != cudaSuccess ? cudaGetErrorString(ce) : "registry capacity");
    (void)cudaGetLastError();
    for (size_t i = fresh.size(); i-- > 0;) {  // forget the new addresses; retired entries go back in the order they left
      R.by_addr.erase(R.addr_of[fresh[i]]);
      if (fresh[i] < used0) R.free_list.push_back(fresh[i]);
    }
    R.used = used0;
    while (R.chunks.size() > chunks0) { cudaFree(R.chunks.back()); R.chunks.pop_back(); }
    refs.clear();
    return ce == cudaSuccess || ce == cudaErrorMemoryAllocation ? IBFT_ERR_CAPACITY : IBFT_ERR_CUDA;
  }
  for (uint32_t v = 0; v < n; v++) R.refs[refs[v] & ~IBFT_KEY_REF_FRESH]++;
  if (R.bounded) R.budget.ensure(R.used);
  return IBFT_OK;
}
// ... and one reference less per row of a table being dropped; an entry no resident table lists any more is retired
static void registry_release(ibft_engine* e, const std::vector<uint32_t>& refs) {
  key_registry& R = e->reg;
  for (uint32_t r : refs) {
    if (--R.refs[r] == 0) {
      R.by_addr.erase(R.addr_of[r]);
      R.free_list.push_back(r);
    }
  }
}

#if IBFT_WC > 0
// Bounded registry: tables chunk i holds under a budget of m table slots (the last chunk may be partial)
static uint32_t pool_chunk_tables(uint32_t m, size_t i) {
  const size_t lo = i * IBFT_KEY_CHUNK;
  return lo >= m ? 0u : (uint32_t)std::min<size_t>(IBFT_KEY_CHUNK, m - lo);
}
// make sure the chunk of table slot t is allocated (lazily, at its size under the current budget); false when it cannot be
static bool pool_reserve(key_registry& R, uint32_t t, bool* grew) {
  const size_t i = t / IBFT_KEY_CHUNK;
  if (R.chunk_tables[i]) return true;
  const uint32_t k = pool_chunk_tables(R.budget.max_tables, i);
  uint32_t* c = nullptr;
  if (cudaMalloc(&c, (size_t)k * IBFT_KEYTAB_WORDS * 4) != cudaSuccess) { (void)cudaGetLastError(); return false; }
  R.chunks[i] = c;
  R.chunk_tables[i] = k;
  *grew = true;
  return true;
}
static uint32_t* pool_table(key_registry& R, uint32_t t) {
  return R.chunks[t / IBFT_KEY_CHUNK] + (size_t)(t % IBFT_KEY_CHUNK) * IBFT_KEYTAB_WORDS;
}

// A reclaim point of the bounded registry (caller holds every lane, device drained): read and clear the used flags, rank the
// entries with a known key (key_budget.hpp), evict, move the kept tables that sit at or above the (new) budget down, resize or
// free the chunks the new budget does not cover, and give slots to the admitted entries (built by the next refresh).  A chunk
// that cannot be allocated costs tables, never an error: the entries concerned keep their key and take the recover path.
// Invariant: an entry is READY only while its slot holds the comb table of its own current key.
static int budget_reclaim(ibft_engine* e, uint32_t new_max) {
  key_registry& R = e->reg;
  ibft::key_budget& B = R.budget;
  const uint32_t n = R.used;
  std::vector<uint32_t> state(n);
  std::vector<uint8_t> used(n), listed(n), known(n), addr((size_t)n * 20);
  if (n) {
    CU(cudaMemcpy(state.data(), R.d_state, (size_t)n * 4, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(used.data(), R.d_used, n, cudaMemcpyDeviceToHost));
    CU(cudaMemset(R.d_used, 0, n));
  }
  for (uint32_t r = 0; r < n; r++) {
    listed[r] = R.refs[r] > 0;
    known[r] = state[r] == IBFT_KEY_LEARNED || state[r] == IBFT_KEY_READY || state[r] == IBFT_KEY_EVICTED;
    memcpy(&addr[20 * (size_t)r], R.addr_of[r].b, 20);
  }
  const ibft::key_budget::plan p = B.reclaim(n, listed.data(), known.data(), used.data(), addr.data(), new_max);
  std::vector<uint32_t> lost;  // entries whose table could not be placed
  bool grew = false;
  for (const auto& mv : p.moves) {
    if (!pool_reserve(R, mv.to, &grew)) { lost.push_back(mv.entry); continue; }
    CU(cudaMemcpy(pool_table(R, mv.to), pool_table(R, mv.from), (size_t)IBFT_KEYTAB_WORDS * 4, cudaMemcpyDeviceToDevice));
  }
  for (uint32_t r : lost) B.drop(r);
  lost.clear();
  // chunks whose size changes with the budget: freed when it no longer covers them, otherwise reallocated at the new size with
  // the tables they keep (only tables below the new budget are live by now)
  const size_t n_chunks = R.chunks.size();
  for (size_t i = 0; i < n_chunks; i++) {
    const uint32_t have = R.chunk_tables[i], want = pool_chunk_tables(new_max, i);
    if (!have || have == want) continue;
    uint32_t* c = nullptr;
    if (want && cudaMalloc(&c, (size_t)want * IBFT_KEYTAB_WORDS * 4) == cudaSuccess) {
      CU(cudaMemcpy(c, R.chunks[i], (size_t)std::min(have, want) * IBFT_KEYTAB_WORDS * 4, cudaMemcpyDeviceToDevice));
    } else {
      (void)cudaGetLastError();
      c = nullptr;
      for (uint32_t t = (uint32_t)(i * IBFT_KEY_CHUNK); t < i * IBFT_KEY_CHUNK + have && t < B.owner.size(); t++)
        if (B.owner[t] != ibft::kNoTable) lost.push_back(B.owner[t]);
    }
    CU(cudaFree(R.chunks[i]));
    R.chunks[i] = c;
    R.chunk_tables[i] = c ? want : 0u;
  }
  for (uint32_t r : lost) B.drop(r);
  for (uint32_t r : p.admitted) {
    const uint32_t t = B.table[r];
    if (t != ibft::kNoTable && !pool_reserve(R, t, &grew)) B.drop(r);
  }
  // states: a slot that holds the entry's table stays READY, an admitted one is LEARNED (built by the next refresh), and every
  // other known key of a listed entry is EVICTED -- so LEARNED without a slot means "learned since this reclaim point"
  R.build_due = false;
  for (uint32_t r = 0; r < n; r++) {
    if (!listed[r] || !known[r]) continue;
    if (B.table[r] == ibft::kNoTable) state[r] = IBFT_KEY_EVICTED;
    else if (state[r] != IBFT_KEY_READY) { state[r] = IBFT_KEY_LEARNED; R.build_due = true; }
  }
  if (n) {
    CU(cudaMemcpy(R.d_tab, B.table.data(), (size_t)n * 4, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(R.d_state, state.data(), (size_t)n * 4, cudaMemcpyHostToDevice));
  }
  CU(cudaMemcpy(R.d_chunks, R.chunks.data(), R.chunks.size() * sizeof(uint32_t*), cudaMemcpyHostToDevice));
  return IBFT_OK;
}

// Switch the engine to a bounded registry (every lane held, device drained).  The tables built so far stay where they are:
// entry r's table is slot r of the pool, then the first reclaim point brings the pool to its budget.
static int budget_enable(ibft_engine* e) {
  key_registry& R = e->reg;
  const size_t n_chunks = ((size_t)R.capacity + IBFT_KEY_CHUNK - 1) / IBFT_KEY_CHUNK;
  uint32_t* d_tab = nullptr;
  uint8_t* d_used = nullptr;
  cudaError_t ce = cudaMalloc(&d_tab, std::max<size_t>(R.capacity, 1) * 4);
  if (ce == cudaSuccess) ce = cudaMalloc(&d_used, std::max<size_t>(R.capacity, 1));
  if (ce == cudaSuccess) ce = cudaMemset(d_used, 0, std::max<size_t>(R.capacity, 1));
  if (ce != cudaSuccess) {
    cudaFree(d_tab); cudaFree(d_used);
    (void)cudaGetLastError();
    set_err("key table budget: %s", cudaGetErrorString(ce));
    return ce == cudaErrorMemoryAllocation ? IBFT_ERR_CAPACITY : IBFT_ERR_CUDA;
  }
  R.d_tab = d_tab;
  R.d_used = d_used;
  std::vector<uint32_t> state(R.used);
  if (R.used) CU(cudaMemcpy(state.data(), R.d_state, (size_t)R.used * 4, cudaMemcpyDeviceToHost));
  std::vector<uint8_t> holds(R.chunks.size() * IBFT_KEY_CHUNK, 0);
  for (uint32_t r = 0; r < R.used; r++) holds[r] = state[r] == IBFT_KEY_READY && R.refs[r] > 0;
  R.budget.adopt_identity(R.used, holds);
  R.chunk_tables.assign(n_chunks, 0);
  for (size_t i = 0; i < R.chunks.size(); i++) R.chunk_tables[i] = IBFT_KEY_CHUNK;
  R.chunks.resize(n_chunks, nullptr);
  R.bounded = true;
  for (size_t k = 0; k < e->slots.size(); k++) {
    if (!e->slots[k].d_key_ref) continue;
    e->slots_shadow[k].key_tab = R.d_tab;
    e->slots_shadow[k].key_used = R.d_used;
    CU(cudaMemcpy(e->d_slots + k, &e->slots_shadow[k], sizeof(slot_dev), cudaMemcpyHostToDevice));
  }
  return IBFT_OK;
}
#endif

extern "C" int ibft_set_validators(ibft_engine* e, uint32_t table_slot, uint64_t height, const uint8_t* addrs,
                                   const uint8_t* powers_be, uint32_t n) {
  IBFT_REFUSE_VIEW(e);
  if (e && e->multi) return multi_set_validators(e, table_slot, height, addrs, powers_be, n);
  if (!e || (!addrs && n)) { set_err("null argument"); return IBFT_ERR_INVALID_ARG; }
  if (table_slot >= e->p.max_table_slots) { set_err("table slot %u out of range", table_slot); return IBFT_ERR_INVALID_ARG; }
  if (n > e->p.max_validators) { set_err("validator table of %u exceeds capacity %u", n, e->p.max_validators); return IBFT_ERR_CAPACITY; }
  // total voting power and quorum = floor(2*total/3) + 1 in 320-bit arithmetic (validator_manager.go:130-135)
  std::vector<uint64_t> powers((size_t)n * 4);
  uint64_t total[5] = {0, 0, 0, 0, 0};
  for (uint32_t i = 0; i < n; i++) {
    uint64_t l[4] = {1, 0, 0, 0};
    if (powers_be) be32_to_limbs(powers_be + 32 * (size_t)i, l);
    memcpy(&powers[4 * (size_t)i], l, sizeof l);
    unsigned __int128 c = 0;
    for (int k = 0; k < 5; k++) {
      c += (unsigned __int128)total[k] + (k < 4 ? l[k] : 0);
      total[k] = (uint64_t)c;
      c >>= 64;
    }
  }
  if ((total[0] | total[1] | total[2] | total[3] | total[4]) == 0) {
    set_err("total voting power is zero or less");
    return IBFT_ERR_VOTING_POWER;
  }
  uint64_t twice[6] = {0, 0, 0, 0, 0, 0};
  {
    uint64_t c = 0;
    for (int k = 0; k < 5; k++) { twice[k] = (total[k] << 1) | c; c = total[k] >> 63; }
    twice[5] = c;
  }
  uint64_t q[6];
  {
    unsigned __int128 rem = 0;
    for (int k = 5; k >= 0; k--) {
      unsigned __int128 cur = (rem << 64) | twice[k];
      q[k] = (uint64_t)(cur / 3);
      rem = cur % 3;
    }
    unsigned __int128 c = 1;
    for (int k = 0; k < 6; k++) { c += q[k]; q[k] = (uint64_t)c; c >>= 64; }
  }
  // sorted key table: 5 big-endian words + validator index
  std::vector<uint32_t> order(n);
  for (uint32_t i = 0; i < n; i++) order[i] = i;
  std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) {
    int c = memcmp(addrs + 20 * (size_t)a, addrs + 20 * (size_t)b, 20);
    return c != 0 ? c < 0 : a < b;
  });
  // go-ibft keys voting power by address (a map: core/validator_manager.go), so a table cannot list an address twice.  A
  // duplicate would count its power twice in the quorum and credit its votes to whichever copy the search meets first: refuse it
  // before anything changes, so the slot keeps its previous table and the key registry its entries
  for (uint32_t r = 1; r < n; r++)
    if (memcmp(addrs + 20 * (size_t)order[r - 1], addrs + 20 * (size_t)order[r], 20) == 0) {
      set_err("validator table lists one address twice: validators %u and %u", order[r - 1], order[r]);
      return IBFT_ERR_INVALID_ARG;
    }
  std::vector<uint32_t> keys((size_t)n * 6);
  for (uint32_t r = 0; r < n; r++) {
    const uint8_t* a = addrs + 20 * (size_t)order[r];
    for (int w = 0; w < 5; w++)
      keys[6 * (size_t)r + w] = ((uint32_t)a[4 * w] << 24) | ((uint32_t)a[4 * w + 1] << 16) | ((uint32_t)a[4 * w + 2] << 8) | a[4 * w + 3];
    keys[6 * (size_t)r + 5] = order[r];
  }
  // replacing a table frees device memory the kernels of ANY lane may be reading: take every lane and drain the device
  all_lanes_lock lk(e);
  for (auto& L : e->lanes)
    if (L.pending.active) { set_err("a submitted call is still pending; wait for it first"); return IBFT_ERR_INVALID_ARG; }
  CU(cudaSetDevice(e->p.device));
  slot_host& s = e->slots[table_slot];
  CU(cudaDeviceSynchronize());
  // the slot's previous content keeps its registry references until the new table holds its own
  slot_host old = std::move(s);
  s = slot_host{};
  const bool registry = (e->p.flags & IBFT_FLAG_KEY_CACHE) && e->reg.d_state && IBFT_WC > 0;
  int rc_alloc = IBFT_OK;
  do {
    cudaError_t ce = cudaMalloc(&s.d_keys, std::max<size_t>(keys.size(), 6) * 4);
    if (ce == cudaSuccess) ce = cudaMalloc(&s.d_powers, std::max<size_t>(powers.size(), 4) * 8);
    if (ce == cudaSuccess && n) ce = cudaMemcpy(s.d_keys, keys.data(), keys.size() * 4, cudaMemcpyHostToDevice);
    if (ce == cudaSuccess && n) ce = cudaMemcpy(s.d_powers, powers.data(), powers.size() * 8, cudaMemcpyHostToDevice);
    if (ce == cudaSuccess && registry && n) ce = cudaMalloc(&s.d_key_ref, (size_t)n * 4);
    if (ce != cudaSuccess) {
      set_err("validator table of %u validators: %s", n, cudaGetErrorString(ce));
      rc_alloc = ce == cudaErrorMemoryAllocation ? IBFT_ERR_CAPACITY : IBFT_ERR_CUDA;
      (void)cudaGetLastError();
    }
  } while (0);
  // one registry entry per address: the addresses the registry already holds keep their entry (and key); new ones get an entry
  if (rc_alloc == IBFT_OK && registry && n) rc_alloc = registry_acquire(e, addrs, n, s.key_ref);
  if (rc_alloc != IBFT_OK) {  // the slot keeps its previous table, the registry its previous references
    cudaFree(s.d_keys); cudaFree(s.d_powers); cudaFree(s.d_key_ref);
    s = std::move(old);
    return rc_alloc;
  }
#if IBFT_WC > 0
  if (s.d_key_ref) {
    // upload key_ref; entries new to their address are reset to unknown before any kernel can read them through this table
    cudaError_t ce = cudaMemcpy(s.d_key_ref, s.key_ref.data(), (size_t)n * 4, cudaMemcpyHostToDevice);
    uint32_t lo = UINT32_MAX, hi = 0;  // the entries new to their address lie in [lo, hi)
    for (uint32_t v = 0; v < n; v++)
      if (s.key_ref[v] & IBFT_KEY_REF_FRESH) {
        lo = std::min(lo, s.key_ref[v] & ~IBFT_KEY_REF_FRESH);
        hi = std::max(hi, (s.key_ref[v] & ~IBFT_KEY_REF_FRESH) + 1);
      }
    const bool adopt = lo < hi;
    static_assert(sizeof(addr20) == 20, "addr_of is uploaded as packed 20-byte addresses");
    if (ce == cudaSuccess && adopt)  // the others of [lo, hi) hold their address already
      ce = cudaMemcpy(e->reg.d_addr + 20 * (size_t)lo, e->reg.addr_of[lo].b, 20 * (size_t)(hi - lo), cudaMemcpyHostToDevice);
    if (ce == cudaSuccess && adopt && e->reg.d_shared) {
      ce = launch(e, k_key_share_forget, (n + 255) / 256, 256, 0, nullptr, s.d_key_ref, n, e->reg.d_shared);
    }
    if (ce == cudaSuccess && adopt) {
      ce = launch(e, k_adopt_entries, (n + 255) / 256, 256, 0, nullptr, s.d_key_ref, n, e->reg.d_state,
                  e->reg.bounded ? e->reg.d_tab : nullptr);
      if (ce == cudaSuccess) ce = cudaDeviceSynchronize();
    }
    for (auto& r : s.key_ref) r &= ~IBFT_KEY_REF_FRESH;
    if (ce != cudaSuccess) {
      set_err("validator table of %u validators: key registry entries: %s", n, cudaGetErrorString(ce));
      registry_release(e, s.key_ref);
      cudaFree(s.d_keys); cudaFree(s.d_powers); cudaFree(s.d_key_ref);
      s = std::move(old);
      return IBFT_ERR_CUDA;
    }
  }
#endif
  s.n = n;
  s.height = height;
  memcpy(s.quorum, q, sizeof s.quorum);
  s.valid = true;
  slot_dev sd{};
  sd.keys = s.d_keys;
  sd.powers = s.d_powers;
  if (s.d_key_ref) {
    sd.key_ref = s.d_key_ref;
    sd.key_state = e->reg.d_state;
    sd.key_xy = e->reg.d_key_xy;
    sd.key_chunks = e->reg.d_chunks;
    sd.learn_count = e->reg.d_learn_count;
    if (e->reg.bounded) { sd.key_tab = e->reg.d_tab; sd.key_used = e->reg.d_used; }
  }
  memcpy(sd.quorum, q, sizeof sd.quorum);
  sd.n = n;
  sd.valid = 1;
  // the previous content lets go of its entries: an address no resident table lists any more is forgotten
  registry_release(e, old.key_ref);
  if (old.d_keys) cudaFree(old.d_keys);
  if (old.d_powers) cudaFree(old.d_powers);
  cudaFree(old.d_key_ref);
  e->slots_shadow[table_slot] = sd;
  CU(cudaMemcpy(e->d_slots + table_slot, &sd, sizeof sd, cudaMemcpyHostToDevice));
#if IBFT_WC > 0
  if (e->reg.bounded) return budget_reclaim(e, e->reg.budget.max_tables);  // entries retired here give their slots back
#endif
  return IBFT_OK;
}

// Key registry upkeep: build the comb tables of the keys learned since the last call -- one claim / build / publish pass over
// the engine's registry, whichever tables the keys were learned through.  Cheap when nothing is new (one 4-byte read).
// ibft_verify_batch / ibft_verify_wait call it on their way out; callers of the device-resident entry points call it between
// rounds.  n_ready_out: the members of the resident tables whose key is known, summed over the tables.  The caller holds
// keys_mu; the work goes on stream st.
static int refresh_key_tables_held(ibft_engine* e, cudaStream_t st, uint32_t* n_ready_out) {
  uint32_t total = 0;
#if IBFT_WC > 0
  if ((e->p.flags & IBFT_FLAG_KEY_CACHE) && e->reg.d_state) {
    key_registry& R = e->reg;
    CU(cudaSetDevice(e->p.device));
    CU(cudaMemcpyAsync(R.h_learn_count, R.d_learn_count, 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    const uint32_t learned = *R.h_learn_count;
    bool build = learned != R.built_count && R.used;
    if (R.bounded && build) {
      // the other lane's kernels may be running: only FREE slots are handed out here, to the keys learned since the last
      // reclaim point (LEARNED without a slot), in ascending address order
      std::vector<uint32_t> state(R.used), fresh;
      CU(cudaMemcpyAsync(state.data(), R.d_state, (size_t)R.used * 4, cudaMemcpyDeviceToHost, st));
      CU(cudaStreamSynchronize(st));
      for (uint32_t r = 0; r < R.used; r++)
        if (state[r] == IBFT_KEY_LEARNED && R.refs[r] > 0 && R.budget.table[r] == ibft::kNoTable) fresh.push_back(r);
      std::sort(fresh.begin(), fresh.end(), [&](uint32_t a, uint32_t b) { return memcmp(R.addr_of[a].b, R.addr_of[b].b, 20) < 0; });
      bool grew = false, assigned = false;
      for (uint32_t r : fresh) {
        const uint32_t t = R.budget.take_free(r);
        if (t == ibft::kNoTable) break;
        if (!pool_reserve(R, t, &grew)) { R.budget.drop(r); break; }  // the pool cannot grow: builds stop at what it holds
        CU(cudaMemcpyAsync(R.d_tab + r, &R.budget.table[r], 4, cudaMemcpyHostToDevice, st));
        assigned = true;
      }
      if (grew) CU(cudaMemcpyAsync(R.d_chunks, R.chunks.data(), R.chunks.size() * sizeof(uint32_t*), cudaMemcpyHostToDevice, st));
      CU(cudaStreamSynchronize(st));  // the host copies above read pageable memory that changes on the next call
      R.built_count = learned;
      build = assigned;
    }
    if (R.bounded && R.build_due) build = true;
    if (build) {
      // the pass covers [0, used), retired entries included: one that was retired while still LEARNED (a table replaced
      // before any refresh ran) gets its table built once for nothing -- 17 threads -- and is reset when it is reused.  A
      // bounded registry builds only the entries that hold a slot.
      const uint32_t* tab = R.bounded ? R.d_tab : nullptr;
      k_keytabs_step<<<(R.used + 255) / 256, 256, 0, st>>>(R.d_state, tab, R.used, IBFT_KEY_LEARNED, IBFT_KEY_BUILDING);
      k_build_keytabs<<<(uint32_t)(((size_t)R.used * IBFT_KEYTAB_POSITIONS + 63) / 64), 64, 0, st>>>(R.d_state, R.d_key_xy,
                                                                                                          tab, R.d_chunks, R.used);
      k_keytabs_step<<<(R.used + 255) / 256, 256, 0, st>>>(R.d_state, tab, R.used, IBFT_KEY_BUILDING, IBFT_KEY_READY);
      R.build_due = false;
      e->launches += 3;
      CU(cudaGetLastError());
      R.built_count = learned;
      // the tables are complete before anybody can launch the next round on another stream
      CU(cudaStreamSynchronize(st));
    }
    if (n_ready_out && R.used) {
      std::vector<uint32_t> state(R.used);
      CU(cudaMemcpyAsync(state.data(), R.d_state, (size_t)R.used * 4, cudaMemcpyDeviceToHost, st));
      CU(cudaStreamSynchronize(st));
      for (const slot_host& s : e->slots)
        if (s.valid)
          for (uint32_t r : s.key_ref) total += state[r] != IBFT_KEY_UNKNOWN;
    }
  }
#endif
  if (n_ready_out) *n_ready_out = total;
  return IBFT_OK;
}
static int refresh_key_tables_locked(ibft_engine* e, lane* L, uint32_t* n_ready_out) {
  std::lock_guard<std::mutex> kl(e->keys_mu);
  return refresh_key_tables_held(e, L->stream, n_ready_out);
}
extern "C" int ibft_refresh_key_tables(ibft_engine* e, uint32_t* n_keys_out) {
  if (!e) { set_err("null engine"); return IBFT_ERR_INVALID_ARG; }
  IBFT_REFUSE_VIEW(e);
  if (e->multi) return multi_refresh_key_tables(e, n_keys_out);
  lane* L = &e->lanes[0];
  std::unique_lock<std::mutex> lk(L->mu), lk1;
  if (L->pending.active) { set_err("a submitted call is still pending"); return IBFT_ERR_INVALID_ARG; }
#if IBFT_WC > 0
  if (e->reg.bounded) {  // a reclaim point: every lane (in index order), device drained
    lk1 = std::unique_lock<std::mutex>(e->lanes[1].mu);
    CU(cudaSetDevice(e->p.device));
    CU(cudaDeviceSynchronize());
    int rc = budget_reclaim(e, e->reg.budget.max_tables);
    if (rc != IBFT_OK) return rc;
  }
#endif
  return refresh_key_tables_locked(e, L, n_keys_out);
}

extern "C" int ibft_set_key_table_budget(ibft_engine* e, uint32_t max_tables) {
  if (!e) { set_err("null engine"); return IBFT_ERR_INVALID_ARG; }
  IBFT_REFUSE_VIEW(e);
  if (e->multi) return multi_set_key_table_budget(e, max_tables);
#if IBFT_WC > 0
  if (!(e->p.flags & IBFT_FLAG_KEY_CACHE) || !e->reg.d_state) { set_err("engine has no key registry"); return IBFT_ERR_INVALID_ARG; }
  all_lanes_lock lk(e);
  for (auto& L : e->lanes)
    if (L.pending.active) { set_err("a submitted call is still pending; wait for it first"); return IBFT_ERR_INVALID_ARG; }
  CU(cudaSetDevice(e->p.device));
  CU(cudaDeviceSynchronize());
  if (!e->reg.bounded) {
    int rc = budget_enable(e);
    if (rc != IBFT_OK) return rc;
  }
  // more slots than the registry can ever have entries would never be used
  return budget_reclaim(e, std::min(max_tables, e->reg.capacity));
#else
  (void)max_tables;
  set_err("library built without a key registry");
  return IBFT_ERR_INVALID_ARG;
#endif
}

// Key sharing between engines of separate processes (include/ibft_verify.h).  Both device calls hold lane 0 while they launch:
// ibft_set_validators, which changes the tables and the entries' addresses, takes every lane and drains the device first.
extern "C" int ibft_key_share_words(ibft_engine* e, uint32_t* words_out) {
  if (!e || !words_out) { set_err("null argument"); return IBFT_ERR_INVALID_ARG; }
  *words_out = IBFT_KEY_SHARE_WORDS;
  return IBFT_OK;
}
// the checks both calls share, and the export marks (zero: nothing exported yet), allocated by the first call; caller holds lane 0
static int key_share_begin(ibft_engine* e) {
  if (!(e->p.flags & IBFT_FLAG_KEY_CACHE) || !e->reg.d_state || IBFT_WC == 0) { set_err("engine has no key registry"); return IBFT_ERR_INVALID_ARG; }
  if (e->lanes[0].pending.active) { set_err("a submitted call is still pending"); return IBFT_ERR_INVALID_ARG; }
  CU(cudaSetDevice(e->p.device));
  if (!e->reg.d_shared) {
    uint32_t* d = nullptr;
    CU(cudaMalloc(&d, (size_t)e->reg.capacity * 4));
    if (cudaMemset(d, 0, (size_t)e->reg.capacity * 4) != cudaSuccess) { cudaFree(d); CU(cudaGetLastError()); }
    e->reg.d_shared = d;
  }
  return IBFT_OK;
}
extern "C" int ibft_key_share_export_device(ibft_engine* e, void* d_block, void* stream) {
  IBFT_REFUSE_MULTI(e);
  if (!e || !d_block) { set_err("null argument"); return IBFT_ERR_INVALID_ARG; }
#if IBFT_WC > 0
  lane* L = &e->lanes[0];
  std::lock_guard<std::mutex> lk(L->mu);
  int rc = key_share_begin(e);
  if (rc != IBFT_OK) return rc;
  const key_registry& R = e->reg;
  CU(launch(e, k_key_export, 1, 1024, 0, stream ? (cudaStream_t)stream : L->stream, R.d_state, R.d_shared, R.d_key_xy, R.d_addr, R.used,
            (uint32_t*)d_block));
  return IBFT_OK;
#else
  (void)stream;
  set_err("library built without a key registry");
  return IBFT_ERR_INVALID_ARG;
#endif
}
extern "C" int ibft_key_share_adopt_device(ibft_engine* e, const uint64_t* part_ptrs, uint32_t n_parts, uint32_t self_part,
                                           void* d_counts_out, void* stream) {
  IBFT_REFUSE_MULTI(e);
  if (!e || !part_ptrs || n_parts == 0 || n_parts > IBFT_KEY_SHARE_MAX_PARTS || self_part >= n_parts) {
    set_err("bad argument: %u parts (1 to %u), own part %u", n_parts, IBFT_KEY_SHARE_MAX_PARTS, self_part);
    return IBFT_ERR_INVALID_ARG;
  }
  key_share_parts parts{};
  for (uint32_t k = 0; k < n_parts; k++) {
    if (k != self_part && part_ptrs[k] == 0) { set_err("key block %u is null", k); return IBFT_ERR_INVALID_ARG; }
    parts.part[k] = (const uint32_t*)(uintptr_t)part_ptrs[k];
  }
#if IBFT_WC > 0
  lane* L = &e->lanes[0];
  std::lock_guard<std::mutex> lk(L->mu);
  int rc = key_share_begin(e);
  if (rc != IBFT_OK) return rc;
  cudaStream_t st = stream ? (cudaStream_t)stream : L->stream;
  if (d_counts_out) CU(cudaMemsetAsync(d_counts_out, 0, 8, st));
  key_registry& R = e->reg;
  CU(launch(e, k_key_adopt, dim3(IBFT_KEY_SHARE_RECORDS / 256, n_parts), 256, 0, st, parts, self_part, e->d_slots, e->p.max_table_slots,
            R.d_state, R.d_key_xy, R.d_addr, R.d_shared, R.d_learn_count, (uint32_t*)d_counts_out));
  return IBFT_OK;
#else
  (void)d_counts_out; (void)stream;
  set_err("library built without a key registry");
  return IBFT_ERR_INVALID_ARG;
#endif
}

extern "C" int ibft_get_quorum(ibft_engine* e, uint32_t table_slot, uint64_t quorum_out[5], uint64_t* height_out,
                               uint32_t* n_out) {
  e = diag_engine(e);
  if (!e || table_slot >= e->p.max_table_slots) { set_err("bad slot"); return IBFT_ERR_INVALID_ARG; }
  std::lock_guard<std::mutex> lk(e->lanes[0].mu);
  const slot_host& s = e->slots[table_slot];
  if (!s.valid) { set_err("slot %u not set", table_slot); return IBFT_ERR_NO_TABLE; }
  if (quorum_out) memcpy(quorum_out, s.quorum, sizeof s.quorum);
  if (height_out) *height_out = s.height;
  if (n_out) *n_out = s.n;
  return IBFT_OK;
}

// lay out the voted sets of the call's groups; validates table slots and quorum rules (IBFT_QUORUM_*)
static int plan_groups(ibft_engine* e, lane* L, const ibft_group_desc* groups, uint32_t n_groups, group_dev* gdev, size_t* total_words) {
  size_t off = 0;
  for (uint32_t g = 0; g < n_groups; g++) {
    uint32_t slot = groups[g].table_slot;
    const uint32_t rule = groups[g].flags & IBFT_QUORUM_RULE_MASK, proposer = groups[g].reserved;
    if (rule == 3u) { set_err("group %u: quorum rule 3 is reserved", g); return IBFT_ERR_INVALID_ARG; }
    if (rule != IBFT_QUORUM_DEFAULT && slot == IBFT_NO_TABLE) {
      set_err("group %u: quorum rule %u needs a validator table", g, rule);
      return IBFT_ERR_INVALID_ARG;
    }
    uint32_t nw = 0;
    if (slot != IBFT_NO_TABLE) {
      if (slot >= e->p.max_table_slots || !e->slots[slot].valid) {
        set_err("group %u references validator-table slot %u which is not set", g, slot);
        return IBFT_ERR_NO_TABLE;
      }
      // IsValidValidator answers for the validator set AT THE MESSAGE'S HEIGHT (core/backend.go:41-45): a slot that has been
      // recycled for another height must never answer for this one
      if (e->slots[slot].height != groups[g].height) {
        set_err("group %u is for height %llu but validator-table slot %u holds height %llu", g, (unsigned long long)groups[g].height,
                slot, (unsigned long long)e->slots[slot].height);
        return IBFT_ERR_NO_TABLE;
      }
      if (rule == IBFT_QUORUM_PREPARE && proposer != IBFT_PROPOSER_NONE && proposer != IBFT_PROPOSER_UNSET && proposer >= e->slots[slot].n) {
        set_err("group %u: proposer index %u is outside the %u-validator table of slot %u", g, proposer, e->slots[slot].n, slot);
        return IBFT_ERR_INVALID_ARG;
      }
      nw = (e->slots[slot].n + 31) / 32;
    }
    gdev[g].voted_off = (uint32_t)off;
    gdev[g].n_words = nw;
    off += nw;
  }
  if (off > L->voted_words_cap) { set_err("voted sets of the call exceed capacity"); return IBFT_ERR_CAPACITY; }
  *total_words = off;
  return IBFT_OK;
}

// Validates the hash bindings of a call's groups (ibft_group_hash); *any_bound = at least one group is bound
static int check_group_hashes(const ibft_group_desc* groups, uint32_t n_groups, const ibft_group_hash* hashes, bool* any_bound) {
  *any_bound = false;
  for (uint32_t g = 0; g < n_groups; g++) {
    const ibft_group_hash& h = hashes[g];
    if (h.reserved[0] | h.reserved[1] | h.reserved[2]) { set_err("group hash %u: reserved words must be zero", g); return IBFT_ERR_INVALID_ARG; }
    if (h.msg_type == IBFT_HASH_UNBOUND) continue;
    const uint32_t rule = groups[g].flags & IBFT_QUORUM_RULE_MASK;
    if (h.msg_type != IBFT_HASH_PREPARE && h.msg_type != IBFT_HASH_COMMIT) {
      set_err("group hash %u: msg_type %u is not PREPARE (1), COMMIT (2) or IBFT_HASH_UNBOUND", g, h.msg_type);
      return IBFT_ERR_INVALID_ARG;
    }
    const bool fits = rule == IBFT_QUORUM_DEFAULT || (rule == IBFT_QUORUM_PREPARE && h.msg_type == IBFT_HASH_PREPARE);
    if (!fits) {
      set_err("group %u: quorum rule %u cannot be bound to %s hashes", g, rule, h.msg_type == IBFT_HASH_PREPARE ? "PREPARE" : "COMMIT");
      return IBFT_ERR_INVALID_ARG;
    }
    *any_bound = true;
  }
  return IBFT_OK;
}

// The arguments every signature kernel takes, for one recover step over items [lo, hi)
struct sig_args {
  const ibft_sig_item* items; uint32_t n;
  const uint8_t* arena; size_t arena_len;
  uint32_t lo, hi;
  const ibft_group_desc* groups; uint32_t n_groups;
  const slot_dev* slots; uint32_t n_slots;
  uint32_t* bitmap; uint8_t* recovered; uint8_t* status;
  const uint32_t* ctable; vote_sink sink;
};

// Launches signature kernel k over a's items.  list: the worklist a known-key pass fills, or the one a recover kernel takes its
// items from; such a worklist pass leaves the recovered addresses and the statuses to the known-key pass.
static cudaError_t launch_sig(ibft_engine* e, sig_kernel k, const sig_args& a, uint32_t* list, cudaStream_t st) {
  auto grid = [&](uint32_t cta_sigs) { return (a.hi - a.lo + cta_sigs - 1) / cta_sigs; };
  uint8_t* const recovered = list ? nullptr : a.recovered;
  uint8_t* const status = list ? nullptr : a.status;
  const uint32_t chain_cta = 32 * (IBFT_SPLIT_CHAINS + 1), rtab_smem = IBFT_RTAB_WORDS * 4;
#define IBFT_SIG_ARGS a.items, a.n, a.arena, a.arena_len, a.lo, a.hi, a.groups, a.n_groups, a.slots, a.n_slots, a.bitmap
  switch (k) {
    case SK_RECOVER_32:
      return launch(e, recover_kernel<32>(e), grid(32), 32, 32 * rtab_smem, st, IBFT_SIG_ARGS, recovered, status, a.ctable, a.sink, list,
                    e->d_wtable);
    case SK_RECOVER_128:
      return launch(e, recover_kernel<IBFT_BLOCK>(e), grid(IBFT_BLOCK), IBFT_BLOCK, IBFT_BLOCK * rtab_smem, st, IBFT_SIG_ARGS, recovered,
                    status, a.ctable, a.sink, list, e->d_wtable);
    case SK_QUAD:
      return launch(e, k_recover_quad, grid(IBFT_QUAD_SIGS), 4 * IBFT_QUAD_SIGS, 0, st, IBFT_SIG_ARGS, recovered, status, a.ctable, a.sink);
#if IBFT_WC > 0
    case SK_SPLIT:
      return launch(e, k_recover_split, grid(IBFT_SPLIT_SIGS), chain_cta, IBFT_SPLIT_SMEM, st, IBFT_SIG_ARGS, recovered, status, a.ctable,
                    a.sink);
    case SK_QSPLIT:
      return launch(e, k_recover_qsplit, grid(IBFT_QSPLIT_SIGS), 128, 0, st, IBFT_SIG_ARGS, recovered, status, a.ctable, a.sink, list);
    case SK_VERIFY_KNOWN_32:
      return launch(e, k_verify_known<32>, grid(32), 32, 0, st, IBFT_SIG_ARGS, a.status, a.ctable, a.sink, list);
    case SK_VERIFY_KNOWN_128:
      return launch(e, k_verify_known<IBFT_BLOCK>, grid(IBFT_BLOCK), IBFT_BLOCK, 0, st, IBFT_SIG_ARGS, a.status, a.ctable, a.sink, list);
    case SK_VERIFY_SPLIT:
      return launch(e, k_verify_split, grid(IBFT_SPLIT_SIGS), chain_cta, IBFT_VSPLIT_SMEM, st, IBFT_SIG_ARGS, a.status, a.ctable, a.sink,
                    list);
#endif
    default:
      return cudaErrorInvalidDeviceFunction;  // a kernel this build does not have
  }
#undef IBFT_SIG_ARGS
}

// One recover step over items [lo, hi) on `path` (ibft_set_recover_path): the kernels plan_recover picks (recover_plan.hpp)
static int launch_recover(ibft_engine* e, lane* L, const ibft_sig_item* d_items, uint32_t n, const uint8_t* d_arena, size_t arena_len,
                          uint32_t lo, uint32_t hi, const ibft_group_desc* d_groups, uint32_t n_groups, uint32_t* d_bitmap,
                          uint8_t* d_recovered, cudaStream_t st, int path, uint8_t* d_status = nullptr,
                          vote_sink sink = vote_sink{nullptr, nullptr, nullptr}, uint32_t worklist_index = 0) {
  if (hi <= lo) return IBFT_OK;
  const uint32_t cnt = hi - lo;
  uint32_t* const worklist = L->d_worklist ? L->d_worklist + (size_t)worklist_index * ((size_t)L->cap_items + 1) : nullptr;
  const bool known = known_key_ok((e->p.flags & IBFT_FLAG_KEY_CACHE) != 0, d_recovered != nullptr, d_groups != nullptr,
                                  worklist != nullptr, cnt, L->cap_items);
  const recover_plan plan = plan_recover(path, cnt, arena_len, (uint32_t)e->sm_count, known, IBFT_WC > 0);
  const sig_args a{d_items, n, d_arena, arena_len, lo, hi, d_groups, n_groups, e->d_slots, e->p.max_table_slots, d_bitmap,
                   d_recovered, d_status, e->d_ctable, sink};
  if (plan.worklist == SK_NONE) {
    if (plan.first == SK_QSPLIT)  // its verdict bits are OR-ed in
      CU(cudaMemsetAsync(d_bitmap + (lo >> 5), 0, (size_t)((hi + 31) / 32 - (lo >> 5)) * 4, st));
    CU(launch_sig(e, plan.first, a, nullptr, st));
    return IBFT_OK;
  }
  // the known-key pass, then the recover pass over the worklist of what it did not accept (which finds it empty, and returns at
  // once, when every signature verified).  Device-resident callers may use different streams: launches sharing a worklist are
  // ordered on the device.
  const uint32_t bit = 1u << (worklist_index & 3u);  // host-side record for ibft_debug_known_handed_back
  if (L->wl_used & bit) L->wl_reused = true;
  L->wl_used |= bit;
  CU(cudaStreamWaitEvent(st, L->wl_ev[worklist_index & 3u], 0));
  CU(cudaMemsetAsync(worklist, 0, 4, st));
  CU(launch_sig(e, plan.first, a, worklist, st));
  CU(launch_sig(e, plan.worklist, a, worklist, st));
  CU(cudaEventRecord(L->wl_ev[worklist_index & 3u], st));
  return IBFT_OK;
}

// Marks the votes of the passing items of [lo, hi) into voted / nvalid: k_quorum_mark_hashed when a group is bound to a hash
// (d_ghash) or the counted bits are wanted, else k_quorum_mark
static cudaError_t mark_votes(ibft_engine* e, lane* L, const ibft_sig_item* d_items, uint32_t n, const uint8_t* d_arena, size_t arena_len,
                              const uint32_t* d_bitmap, uint32_t n_groups, const ibft_group_hash* d_ghash, uint32_t* d_counted,
                              uint32_t* voted, uint32_t* nvalid, uint32_t lo, uint32_t hi, cudaStream_t st) {
  const uint32_t grid = (hi - lo + 255) / 256;
  if (d_ghash || d_counted)
    return launch(e, k_quorum_mark_hashed, grid, 256, 0, st, d_items, n, d_arena, arena_len, d_bitmap, L->d_groups, d_ghash, L->d_gdev,
                  n_groups, e->d_slots, e->p.max_table_slots, voted, nvalid, d_counted, lo, hi);
  return launch(e, k_quorum_mark, grid, 256, 0, st, d_items, n, d_arena, arena_len, d_bitmap, L->d_groups, L->d_gdev, n_groups,
                e->d_slots, e->p.max_table_slots, voted, nvalid, lo, hi);
}

// the quorum decision of each of the lane's groups from its voted sets
static cudaError_t reduce_votes(ibft_engine* e, lane* L, uint32_t n_groups, ibft_group_result* d_results, cudaStream_t st) {
  return launch(e, k_quorum_reduce, n_groups, IBFT_REDUCE_THREADS, 0, st, L->d_groups, L->d_gdev, n_groups, e->d_slots,
                e->p.max_table_slots, L->d_voted, L->d_nvalid, d_results);
}

// words of the voted sets of the lane's groups
static size_t lane_voted_words(const lane* L) {
  size_t words = 0;
  for (const group_dev& g : L->last_gdev) words += g.n_words;
  return words;
}

// Staging copy of a chunk of pageable caller memory (a cgo caller's Go heap) into the lane's pinned buffer.  One thread moves
// ~4 GB/s on the GPU boxes' hosts -- 134 MB of tuples would take longer than the kernels that consume them -- so large chunks are
// split over a few short-lived helper threads (the copy of chunk k+1 already overlaps the device work on chunk k).
static void stage_copy(void* dst, const void* src, size_t bytes) {
  const size_t kMin = 2u << 20;
  if (bytes < 2 * kMin) { memcpy(dst, src, bytes); return; }
  const unsigned parts = (unsigned)std::min<size_t>(4, bytes / kMin);
  const size_t per = (bytes / parts + 63) & ~(size_t)63;
  std::thread th[3];
  unsigned started = 0;
  for (unsigned k = 1; k < parts; k++) {
    size_t off = k * per, len = k + 1 == parts ? bytes - off : per;
    th[started++] = std::thread([=]() { memcpy((char*)dst + off, (const char*)src + off, len); });
  }
  memcpy(dst, src, std::min(per, bytes));
  for (unsigned k = 0; k < started; k++) th[k].join();
}

static int submit_locked(ibft_engine* e, lane* L, const ibft_sig_item* items, uint32_t n, const uint8_t* arena, size_t arena_len,
                         const ibft_group_desc* groups, uint32_t n_groups, uint32_t* bitmap_out,
                         ibft_group_result* results_out, uint8_t* recovered_out, bool votes_only = false,
                         const ibft_group_hash* ghash = nullptr, uint32_t* counted_out = nullptr, bool async_call = false) {
  // votes_only: a shard of a multi-device call -- record the votes, leave the reduce to the coordinator's merge
  // ghash: the groups' hash bindings, given only when at least one group is bound (checked by check_group_hashes)
  // async_call: the call returns before its copies have run (ibft_verify_submit), so no caller buffer may be read after it
  if (L->pending.active) { set_err("a submitted call is still pending; wait for it first"); return IBFT_ERR_INVALID_ARG; }
  if ((n && !items) || (n && !bitmap_out) || (arena_len && !arena) || (n_groups && !groups)) { set_err("null argument"); return IBFT_ERR_INVALID_ARG; }
  if (n > L->cap_items || arena_len > L->cap_arena || n_groups > e->p.max_groups) {
    set_err("batch (%u items, %zu payload bytes, %u groups) exceeds engine capacity (%u, %zu, %u)", n, arena_len, n_groups,
            L->cap_items, L->cap_arena, e->p.max_groups);
    return IBFT_ERR_CAPACITY;
  }
  CU(cudaSetDevice(e->p.device));
  L->wl_used = 0;
  L->wl_reused = false;
  size_t voted_words = 0;
  if (n_groups) {
    int rc = plan_groups(e, L, groups, n_groups, L->h_gdev, &voted_words);
    if (rc != IBFT_OK) return rc;
    memcpy(L->h_groups, groups, (size_t)n_groups * sizeof(ibft_group_desc));
    L->last_gdev.assign(L->h_gdev, L->h_gdev + n_groups);
    L->last_groups.assign(groups, groups + n_groups);
  } else {
    L->last_gdev.clear();
    L->last_groups.clear();
  }
  if (ghash && n_groups) L->last_hashes.assign(ghash, ghash + n_groups);
  else L->last_hashes.clear();
  const bool hashed = !L->last_hashes.empty();
  cudaStream_t st = L->stream;
  if (arena_len) {
    if (arena != L->h_arena) memcpy(L->h_arena, arena, arena_len);  // a shard is planned straight into the staging
    CU(cudaMemcpyAsync(L->d_arena, L->h_arena, arena_len, cudaMemcpyHostToDevice, st));
  }
  if (n_groups) {
    CU(cudaMemcpyAsync(L->d_groups, L->h_groups, (size_t)n_groups * sizeof(ibft_group_desc), cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(L->d_gdev, L->h_gdev, (size_t)n_groups * sizeof(group_dev), cudaMemcpyHostToDevice, st));
  }
  if (hashed) {
    memcpy(L->h_ghash, ghash, (size_t)n_groups * sizeof(ibft_group_hash));
    CU(cudaMemcpyAsync(L->d_ghash, L->h_ghash, (size_t)n_groups * sizeof(ibft_group_hash), cudaMemcpyHostToDevice, st));
  }
  // quorum requested: the recover kernels record the votes themselves (no k_quorum_mark pass over the tuples afterwards) -- unless
  // a group is bound to a hash, which their fused marking cannot test: k_quorum_mark_hashed marks the counted items afterwards
  vote_sink sink{nullptr, nullptr, nullptr};
  if (n_groups && (results_out || votes_only || hashed)) {
    CU(cudaMemsetAsync(L->d_voted, 0, std::max<size_t>(voted_words, 1) * 4, st));
    CU(cudaMemsetAsync(L->d_nvalid, 0, (size_t)n_groups * 4, st));
    if (!hashed) sink = vote_sink{L->d_voted, L->d_nvalid, L->d_gdev};
  }
  // Tuples go up in chunks: while the recover kernel works on chunk k, the host stages chunk k+1 into pinned memory and the
  // copy engine moves it (two streams + events).  Small batches are a single chunk.
  const uint32_t CHUNK = 1u << 17;
  uint32_t n_chunks = n ? (n + CHUNK - 1) / CHUNK : 0;  // (not const: the latency path below takes the round over)
  while (L->chunk_ev.size() < n_chunks + 1) {
    cudaEvent_t ev;
    CU(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    L->chunk_ev.push_back(ev);
  }
  if (n_chunks > 1) {  // the copy stream must see the arena / groups uploads of this call
    CU(cudaEventRecord(L->chunk_ev[n_chunks], st));
    CU(cudaStreamWaitEvent(L->copy_stream, L->chunk_ev[n_chunks], 0));
  }
  // A caller that already holds the tuples in page-locked memory (cudaHostAlloc / cudaHostRegister, e.g. torch pin_memory)
  // is copied from directly by a synchronous call, which waits for its copies before it returns.  Pageable memory (Go heap
  // through cgo) goes through the engine's pinned staging first -- and so does every tuple of an asynchronous call, whose DMA
  // would otherwise read the caller's buffer after the call has returned it.
  bool direct = false;
  if (n && !async_call) {
    cudaPointerAttributes pa;
    if (cudaPointerGetAttributes(&pa, items) == cudaSuccess) direct = pa.type == cudaMemoryTypeHost;
    else (void)cudaGetLastError();
  }
  int rc = IBFT_OK;
  const int path = e->recover_path.load();  // read once: a concurrent ibft_set_recover_path cannot mix kernels within the call
  // a mid-size round in latency pieces (recover_plan.hpp); the main stream joins them before the quorum kernels
  const bool known = known_key_ok((e->p.flags & IBFT_FLAG_KEY_CACHE) != 0, recovered_out != nullptr, n_groups != 0,
                                  L->d_worklist != nullptr, n, L->cap_items);
  const piece_plan pieces = plan_pieces(path, n, arena_len, (uint32_t)e->sm_count, known, IBFT_WC > 0);
  if (pieces.per) {
    CU(cudaEventRecord(L->lat_ev[4], st));  // arena / groups uploads of this call
    for (uint32_t c = 0; c < IBFT_LAT_PIECES; c++) {
      uint32_t lo = std::min(n, c * pieces.per), hi = std::min(n, lo + pieces.per);
      if (hi <= lo) break;
      cudaStream_t ls = L->lat_stream[c];
      const ibft_sig_item* src = items + lo;
      if (!direct) {
        memcpy(L->h_items + lo, items + lo, (size_t)(hi - lo) * sizeof(ibft_sig_item));
        src = L->h_items + lo;
      }
      CU(cudaStreamWaitEvent(ls, L->lat_ev[4], 0));
      CU(cudaMemcpyAsync(L->d_items + lo, src, (size_t)(hi - lo) * sizeof(ibft_sig_item), cudaMemcpyHostToDevice, ls));
      rc = launch_recover(e, L, L->d_items, n, L->d_arena, arena_len, lo, hi, n_groups ? L->d_groups : nullptr, n_groups, L->d_bitmap,
                          recovered_out ? L->d_recovered : nullptr, ls, pieces.path, L->d_status, sink, c);
      if (rc != IBFT_OK) return rc;
      CU(cudaEventRecord(L->lat_ev[c], ls));
      CU(cudaStreamWaitEvent(st, L->lat_ev[c], 0));
    }
    n_chunks = 0;  // the generic chunk loop below has nothing left to do
  }
  // Several chunks: chunk c's kernels run on one of two alternating streams, so that the tail of one chunk (the last CTAs of a
  // 1,024-CTA launch on 444 resident slots) overlaps the head of the next instead of idling the SMs eight times per batch.
  if (n_chunks > 1) {
    CU(cudaEventRecord(L->lat_ev[4], st));  // arena / groups uploads and the vote-sink memsets of this call
    CU(cudaStreamWaitEvent(L->lat_stream[0], L->lat_ev[4], 0));
    CU(cudaStreamWaitEvent(L->lat_stream[1], L->lat_ev[4], 0));
  }
  for (uint32_t c = 0; c < n_chunks; c++) {
    uint32_t lo = c * CHUNK, hi = std::min(n, lo + CHUNK);
    const ibft_sig_item* src = items + lo;
    if (!direct) {
      stage_copy(L->h_items + lo, items + lo, (size_t)(hi - lo) * sizeof(ibft_sig_item));
      src = L->h_items + lo;
    }
    cudaStream_t cs = n_chunks > 1 ? L->copy_stream : st;
    cudaStream_t ks = n_chunks > 1 ? L->lat_stream[c & 1u] : st;
    CU(cudaMemcpyAsync(L->d_items + lo, src, (size_t)(hi - lo) * sizeof(ibft_sig_item), cudaMemcpyHostToDevice, cs));
    if (n_chunks > 1) {
      CU(cudaEventRecord(L->chunk_ev[c], cs));
      CU(cudaStreamWaitEvent(ks, L->chunk_ev[c], 0));
    }
    rc = launch_recover(e, L, L->d_items, n, L->d_arena, arena_len, lo, hi, n_groups ? L->d_groups : nullptr, n_groups, L->d_bitmap,
                        recovered_out ? L->d_recovered : nullptr, ks, path, L->d_status, sink, c & 1u);
    if (rc != IBFT_OK) return rc;
  }
  if (n_chunks > 1) {
    for (int k = 0; k < 2; k++) {
      CU(cudaEventRecord(L->lat_ev[k], L->lat_stream[k]));
      CU(cudaStreamWaitEvent(st, L->lat_ev[k], 0));
    }
  }
  if (hashed && n) {
    CU(mark_votes(e, L, L->d_items, n, L->d_arena, arena_len, L->d_bitmap, n_groups, L->d_ghash, L->d_counted, L->d_voted, L->d_nvalid, 0u, n,
                  st));
    if (counted_out) CU(cudaMemcpyAsync(L->h_counted, L->d_counted, (size_t)((n + 31) / 32) * 4, cudaMemcpyDeviceToHost, st));
  }
  if (n_groups && results_out) {
    CU(reduce_votes(e, L, n_groups, L->d_results, st));
    CU(cudaMemcpyAsync(L->h_results, L->d_results, (size_t)n_groups * sizeof(ibft_group_result), cudaMemcpyDeviceToHost, st));
  }
  if (n) {
    CU(cudaMemcpyAsync(L->h_status, L->d_status, (size_t)n, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(L->h_bitmap, L->d_bitmap, (size_t)((n + 31) / 32) * 4, cudaMemcpyDeviceToHost, st));
    if (recovered_out) CU(cudaMemcpyAsync(L->h_recovered, L->d_recovered, (size_t)n * 20, cudaMemcpyDeviceToHost, st));
  }
  CU(cudaEventRecord(L->done_ev, st));
  L->pending.active = true;
  L->pending.n = n;
  L->pending.n_groups = (n_groups && results_out) ? n_groups : 0;
  L->pending.bitmap_out = bitmap_out;
  L->pending.results_out = results_out;
  L->pending.recovered_out = recovered_out;
  L->pending.counted_out = counted_out;
  L->pending.hashed = hashed;
  return IBFT_OK;
}

static int wait_locked(ibft_engine* e, lane* L) {
  if (!L->pending.active) { set_err("no submitted call to wait for"); return IBFT_ERR_INVALID_ARG; }
  CU(cudaSetDevice(e->p.device));
  cudaError_t ce = cudaEventSynchronize(L->done_ev);
  pending_call pc = L->pending;
  L->pending.active = false;
  if (ce != cudaSuccess) {
    // launch/execution failure: NO verdict is produced (outputs untouched) -- never `true` (SURVEY.md §5)
    set_err("device execution failed: %s", cudaGetErrorString(ce));
    return IBFT_ERR_CUDA;
  }
  L->last_status_n = pc.n;
  L->last_wl_used = L->wl_used;
  L->last_wl_reused = L->wl_reused;
  if (pc.n) {
    size_t words = (pc.n + 31) / 32;
    memcpy(pc.bitmap_out, L->h_bitmap, words * 4);
    if (pc.n & 31) pc.bitmap_out[words - 1] &= (1u << (pc.n & 31)) - 1u;
    if (pc.recovered_out) memcpy(pc.recovered_out, L->h_recovered, (size_t)pc.n * 20);
    if (pc.counted_out) {
      memcpy(pc.counted_out, pc.hashed ? L->h_counted : L->h_bitmap, words * 4);
      if (pc.n & 31) pc.counted_out[words - 1] &= (1u << (pc.n & 31)) - 1u;
    }
  }
  if (pc.n_groups) memcpy(pc.results_out, L->h_results, (size_t)pc.n_groups * sizeof(ibft_group_result));
  e->last_lane.store((int)(L - e->lanes));
  // new keys -> tables, for the next call (a multi-device engine's coordinator does it once it has shared the keys)
  if ((e->p.flags & IBFT_FLAG_KEY_CACHE) && !e->coordinated) return refresh_key_tables_locked(e, L, nullptr);
  return IBFT_OK;
}

// Lane selection for a synchronous host-buffer call: a call that fits the small lane takes whichever lane is free (small lane
// first, so that bulk callers find lane 0 free); a large call always takes lane 0.  Returns with the lane's mutex HELD.
static lane* acquire_lane(ibft_engine* e, uint32_t n, size_t arena_len) {
  lane* big = &e->lanes[0];
  lane* small = &e->lanes[1];
  const bool fits_small = n <= small->cap_items && arena_len <= small->cap_arena;
  if (fits_small) {
    if (small->mu.try_lock()) return small;
    if (big->mu.try_lock()) {
      if (!big->pending.active) return big;
      big->mu.unlock();
    }
    small->mu.lock();
    return small;
  }
  big->mu.lock();
  return big;
}

// the voted sets of the lane's last call into voted_out (n_groups rows of voted_stride_words words)
static int copy_voted(ibft_engine* e, lane* L, uint32_t n_groups, bool recorded, uint32_t* voted_out, uint32_t voted_stride_words) {
  if (voted_out && n_groups) {
    CU(cudaSetDevice(e->p.device));
    for (uint32_t g = 0; g < n_groups; g++) {
      const group_dev& gd = L->last_gdev[g];
      uint32_t* dst = voted_out + (size_t)g * voted_stride_words;
      uint32_t w = std::min<uint32_t>(gd.n_words, voted_stride_words);
      // without results_out the recover kernels recorded no votes: the sets are all-zero by definition
      if (w && recorded) CU(cudaMemcpyAsync(dst, L->d_voted + gd.voted_off, (size_t)w * 4, cudaMemcpyDeviceToHost, L->stream));
      else w = 0;
      for (uint32_t i = w; i < voted_stride_words; i++) dst[i] = 0;
    }
    CU(cudaStreamSynchronize(L->stream));
  }
  return IBFT_OK;
}

static int verify_batch_on_lane(ibft_engine* e, lane* L, const ibft_sig_item* items, uint32_t n, const uint8_t* arena, size_t arena_len,
                                const ibft_group_desc* groups, uint32_t n_groups, uint32_t* bitmap_out, ibft_group_result* results_out,
                                uint8_t* recovered_out, uint8_t* status_out, uint32_t* voted_out, uint32_t voted_stride_words,
                                const ibft_group_hash* ghash = nullptr, uint32_t* counted_out = nullptr) {
  int rc = submit_locked(e, L, items, n, arena, arena_len, groups, n_groups, bitmap_out, results_out, recovered_out, false, ghash, counted_out);
  if (rc != IBFT_OK) return rc;
  rc = wait_locked(e, L);
  if (rc != IBFT_OK) return rc;
  if (status_out && n) memcpy(status_out, L->h_status, n);
  return copy_voted(e, L, n_groups, results_out != nullptr, voted_out, voted_stride_words);
}

extern "C" int ibft_verify_batch(ibft_engine* e, const ibft_sig_item* items, uint32_t n, const uint8_t* arena, size_t arena_len,
                                 const ibft_group_desc* groups, uint32_t n_groups, uint32_t* bitmap_out,
                                 ibft_group_result* results_out, uint8_t* recovered_out) {
  if (!e) { set_err("null engine"); return IBFT_ERR_INVALID_ARG; }
  IBFT_REFUSE_VIEW(e);
  if (e->multi)
    return multi_verify(e, items, n, arena, arena_len, groups, n_groups, bitmap_out, results_out, recovered_out, nullptr, nullptr, 0);
  lane* L = acquire_lane(e, n, arena_len);
  std::lock_guard<std::mutex> lk(L->mu, std::adopt_lock);
  return verify_batch_on_lane(e, L, items, n, arena, arena_len, groups, n_groups, bitmap_out, results_out, recovered_out, nullptr, nullptr, 0);
}

extern "C" int ibft_verify_batch_ex(ibft_engine* e, const ibft_sig_item* items, uint32_t n, const uint8_t* arena, size_t arena_len,
                                    const ibft_group_desc* groups, uint32_t n_groups, uint32_t* bitmap_out,
                                    ibft_group_result* results_out, uint8_t* recovered_out, uint8_t* status_out, uint32_t* voted_out,
                                    uint32_t voted_stride_words) {
  if (!e) { set_err("null engine"); return IBFT_ERR_INVALID_ARG; }
  if (voted_out && !results_out) { set_err("voted_out needs results_out (votes are recorded only when quorum results are requested)"); return IBFT_ERR_INVALID_ARG; }
  IBFT_REFUSE_VIEW(e);
  if (e->multi)
    return multi_verify(e, items, n, arena, arena_len, groups, n_groups, bitmap_out, results_out, recovered_out, status_out, voted_out,
                        voted_stride_words);
  lane* L = acquire_lane(e, n, arena_len);
  std::lock_guard<std::mutex> lk(L->mu, std::adopt_lock);
  return verify_batch_on_lane(e, L, items, n, arena, arena_len, groups, n_groups, bitmap_out, results_out, recovered_out, status_out, voted_out,
                              voted_stride_words);
}

extern "C" int ibft_verify_batch_hashed(ibft_engine* e, const ibft_sig_item* items, uint32_t n, const uint8_t* arena, size_t arena_len,
                                        const ibft_group_desc* groups, uint32_t n_groups, uint32_t* bitmap_out,
                                        ibft_group_result* results_out, uint8_t* recovered_out, uint8_t* status_out, uint32_t* voted_out,
                                        uint32_t voted_stride_words, const ibft_group_hash* group_hashes, uint32_t* counted_out) {
  if (!e) { set_err("null engine"); return IBFT_ERR_INVALID_ARG; }
  if (voted_out && !results_out) { set_err("voted_out needs results_out (votes are recorded only when quorum results are requested)"); return IBFT_ERR_INVALID_ARG; }
  IBFT_REFUSE_VIEW(e);
  if (n_groups && !groups) { set_err("null argument"); return IBFT_ERR_INVALID_ARG; }
  bool bound = false;
  if (group_hashes) {
    if (n_groups > e->p.max_groups) {
      set_err("batch (%u groups) exceeds engine capacity (%u)", n_groups, e->p.max_groups);
      return IBFT_ERR_CAPACITY;
    }
    int rc = check_group_hashes(groups, n_groups, group_hashes, &bound);
    if (rc != IBFT_OK) return rc;
  }
  const ibft_group_hash* ghash = bound ? group_hashes : nullptr;  // no group bound: the call is ibft_verify_batch_ex
  if (e->multi)
    return multi_verify(e, items, n, arena, arena_len, groups, n_groups, bitmap_out, results_out, recovered_out, status_out, voted_out,
                        voted_stride_words, ghash, counted_out);
  lane* L = acquire_lane(e, n, arena_len);
  std::lock_guard<std::mutex> lk(L->mu, std::adopt_lock);
  return verify_batch_on_lane(e, L, items, n, arena, arena_len, groups, n_groups, bitmap_out, results_out, recovered_out, status_out, voted_out,
                              voted_stride_words, ghash, counted_out);
}

extern "C" int ibft_last_item_status(ibft_engine* e, uint8_t* status_out, uint32_t n) {
  if (!e || (n && !status_out)) { set_err("null argument"); return IBFT_ERR_INVALID_ARG; }
  if (e->multi) return multi_last_item_status(e, status_out, n);
  e = diag_engine(e);
  lane* L = &e->lanes[e->last_lane.load()];
  std::lock_guard<std::mutex> lk(L->mu);
  if (L->pending.active) { set_err("a submitted call is still pending"); return IBFT_ERR_INVALID_ARG; }
  if (n > L->last_status_n) { set_err("last call had %u items", L->last_status_n); return IBFT_ERR_INVALID_ARG; }
  memcpy(status_out, L->h_status, n);
  return IBFT_OK;
}

// ibft_explain_batch on one device's engine
static int explain_batch(ibft_engine* e, const ibft_sig_item* items, uint32_t n, const uint8_t* arena, size_t arena_len,
                         const ibft_group_desc* groups, uint32_t n_groups, const uint32_t* bitmap, uint8_t* reasons_out,
                         uint8_t* recovered_out) {
  if (n > e->p.max_items || arena_len > e->p.max_payload_bytes || n_groups > e->p.max_groups) {
    set_err("batch (%u items, %zu payload bytes, %u groups) exceeds engine capacity (%u, %u, %u)", n, arena_len, n_groups, e->p.max_items,
            e->p.max_payload_bytes, e->p.max_groups);
    return IBFT_ERR_CAPACITY;
  }
  std::vector<uint32_t> idx;  // the items to explain: those whose verdict bit is 0
  for (uint32_t i = 0; i < n; i++)
    if (bitmap == nullptr || !((bitmap[i >> 5] >> (i & 31u)) & 1u)) idx.push_back(i);
  const uint32_t m = (uint32_t)idx.size();
  lane* L = acquire_lane(e, m, arena_len);
  std::lock_guard<std::mutex> lk(L->mu, std::adopt_lock);
  if (L->pending.active) { set_err("a submitted call is still pending; wait for it first"); return IBFT_ERR_INVALID_ARG; }
  if (n_groups) {  // the verify calls' checks of slots, heights and quorum rules
    std::vector<group_dev> gdev(n_groups);
    size_t voted_words = 0;
    int rc = plan_groups(e, L, groups, n_groups, gdev.data(), &voted_words);
    if (rc != IBFT_OK) return rc;
  }
  std::vector<uint8_t> why(m);
  std::vector<uint8_t> rec(recovered_out ? (size_t)m * 20 : 0);
  if (m) {
    CU(cudaSetDevice(e->p.device));
    cudaStream_t st = L->stream;
    for (uint32_t k = 0; k < m; k++) L->h_items[k] = items[idx[k]];
    if (arena_len) {
      memcpy(L->h_arena, arena, arena_len);
      CU(cudaMemcpyAsync(L->d_arena, L->h_arena, arena_len, cudaMemcpyHostToDevice, st));
    }
    // The groups go through the lane's quorum-result buffer (56 bytes per group, no longer needed once a call has returned):
    // d_groups of lane 0 holds the groups bound for the device-resident calls, which this call must not replace.
    ibft_group_desc* d_groups = reinterpret_cast<ibft_group_desc*>(L->d_results);
    if (n_groups) {
      memcpy(L->h_groups, groups, (size_t)n_groups * sizeof(ibft_group_desc));
      CU(cudaMemcpyAsync(d_groups, L->h_groups, (size_t)n_groups * sizeof(ibft_group_desc), cudaMemcpyHostToDevice, st));
    }
    CU(cudaMemcpyAsync(L->d_items, L->h_items, (size_t)m * sizeof(ibft_sig_item), cudaMemcpyHostToDevice, st));
    auto kernel = e->d_wtable != nullptr ? k_explain<true> : k_explain<false>;
    CU(launch(e, kernel, (m + 31) / 32, 32, 32 * IBFT_RTAB_WORDS * 4, st, L->d_items, m, L->d_arena, arena_len,
              n_groups ? d_groups : nullptr, n_groups, e->d_slots, e->p.max_table_slots, e->d_ctable, e->d_wtable, L->d_status,
              L->d_recovered));
    // the answers land in the pinned tuple staging, which the upload above (same stream) has finished with
    uint8_t* h_out = reinterpret_cast<uint8_t*>(L->h_items);
    CU(cudaMemcpyAsync(h_out, L->d_status, m, cudaMemcpyDeviceToHost, st));
    if (recovered_out) CU(cudaMemcpyAsync(h_out + m, L->d_recovered, (size_t)m * 20, cudaMemcpyDeviceToHost, st));
    cudaError_t ce = cudaStreamSynchronize(st);
    if (ce != cudaSuccess) {
      set_err("device execution failed: %s", cudaGetErrorString(ce));
      return IBFT_ERR_CUDA;
    }
    memcpy(why.data(), h_out, m);
    if (recovered_out) memcpy(rec.data(), h_out + m, (size_t)m * 20);
  }
  if (n) memset(reasons_out, IBFT_REASON_OK, n);
  if (recovered_out && n) memset(recovered_out, 0, (size_t)n * 20);
  for (uint32_t k = 0; k < m; k++) {
    reasons_out[idx[k]] = bitmap != nullptr && why[k] == IBFT_REASON_OK ? (uint8_t)IBFT_REASON_INCONSISTENT : why[k];
    if (recovered_out) memcpy(recovered_out + (size_t)idx[k] * 20, rec.data() + (size_t)k * 20, 20);
  }
  return IBFT_OK;
}

extern "C" int ibft_explain_batch(ibft_engine* e, const ibft_sig_item* items, uint32_t n, const uint8_t* arena, size_t arena_len,
                                  const ibft_group_desc* groups, uint32_t n_groups, const uint32_t* bitmap, uint8_t* reasons_out,
                                  uint8_t* recovered_out) {
  if (!e || (n && (!items || !reasons_out)) || (arena_len && !arena) || (n_groups && !groups)) { set_err("null argument"); return IBFT_ERR_INVALID_ARG; }
  IBFT_REFUSE_VIEW(e);
  if (e->multi) return multi_explain(e, items, n, arena, arena_len, groups, n_groups, bitmap, reasons_out, recovered_out);
  return explain_batch(e, items, n, arena, arena_len, groups, n_groups, bitmap, reasons_out, recovered_out);
}

// The asynchronous API lives on lane 0 (one call pending at a time, as before); synchronous calls that fit the small lane keep
// working while it is pending.
extern "C" int ibft_verify_submit(ibft_engine* e, const ibft_sig_item* items, uint32_t n, const uint8_t* arena, size_t arena_len,
                                  const ibft_group_desc* groups, uint32_t n_groups, uint32_t* bitmap_out,
                                  ibft_group_result* results_out, uint8_t* recovered_out) {
  if (!e) { set_err("null engine"); return IBFT_ERR_INVALID_ARG; }
  IBFT_REFUSE_VIEW(e);
  if (e->multi) return multi_submit(e, items, n, arena, arena_len, groups, n_groups, bitmap_out, results_out, recovered_out);
  lane* L = &e->lanes[0];
  std::lock_guard<std::mutex> lk(L->mu);
  return submit_locked(e, L, items, n, arena, arena_len, groups, n_groups, bitmap_out, results_out, recovered_out, false, nullptr, nullptr,
                       /*async_call=*/true);
}

extern "C" int ibft_verify_poll(ibft_engine* e, int* done) {
  if (!e || !done) { set_err("null argument"); return IBFT_ERR_INVALID_ARG; }
  IBFT_REFUSE_VIEW(e);
  if (e->multi) return multi_poll(e, done);
  lane* L = &e->lanes[0];
  std::lock_guard<std::mutex> lk(L->mu);
  if (!L->pending.active) { *done = 1; return IBFT_OK; }
  CU(cudaSetDevice(e->p.device));
  cudaError_t ce = cudaEventQuery(L->done_ev);
  if (ce == cudaSuccess) { *done = 1; return IBFT_OK; }
  if (ce == cudaErrorNotReady) { *done = 0; return IBFT_OK; }
  set_err("device execution failed: %s", cudaGetErrorString(ce));
  return IBFT_ERR_CUDA;
}

extern "C" int ibft_verify_wait(ibft_engine* e) {
  if (!e) { set_err("null engine"); return IBFT_ERR_INVALID_ARG; }
  IBFT_REFUSE_VIEW(e);
  if (e->multi) return multi_wait(e);
  lane* L = &e->lanes[0];
  std::lock_guard<std::mutex> lk(L->mu);
  return wait_locked(e, L);
}

extern "C" int ibft_verify_batch_device(ibft_engine* e, const void* d_items, uint32_t n, const void* d_arena, size_t arena_len,
                                        uint32_t shard_lo, uint32_t shard_hi, void* d_bitmap, void* d_recovered, void* stream) {
  IBFT_REFUSE_MULTI(e);
  if (!e || (n && (!d_items || !d_bitmap))) { set_err("null argument"); return IBFT_ERR_INVALID_ARG; }
  if (shard_hi > n || shard_lo > shard_hi || (shard_lo & 31) || ((shard_hi & 31) && shard_hi != n)) {
    set_err("shard [%u,%u) of %u must be 32-aligned", shard_lo, shard_hi, n);
    return IBFT_ERR_INVALID_ARG;
  }
  lane* L = &e->lanes[0];
  std::lock_guard<std::mutex> lk(L->mu);
  CU(cudaSetDevice(e->p.device));
  cudaStream_t st = stream ? (cudaStream_t)stream : L->stream;
  L->dev_arena = (const uint8_t*)d_arena;  // remembered for ibft_quorum_reduce_device (raw-frame items carry their signer in the arena)
  L->dev_arena_len = arena_len;
  // membership is applied by ibft_quorum_reduce_device / the host mirror in this mode when no groups are bound
  return launch_recover(e, L, (const ibft_sig_item*)d_items, n, (const uint8_t*)d_arena, arena_len, shard_lo, shard_hi,
                        L->last_groups.empty() ? nullptr : L->d_groups, (uint32_t)L->last_groups.size(), (uint32_t*)d_bitmap,
                        (uint8_t*)d_recovered, st, e->recover_path.load());
}

extern "C" int ibft_explain_batch_device(ibft_engine* e, const void* d_items, uint32_t n, const void* d_arena, size_t arena_len,
                                         uint32_t shard_lo, uint32_t shard_hi, const void* d_bitmap, void* d_reasons, void* d_recovered,
                                         void* d_count_out, void* stream) {
  IBFT_REFUSE_MULTI(e);
  if (!e || (n && (!d_items || !d_bitmap || !d_reasons)) || (arena_len && !d_arena)) { set_err("null argument"); return IBFT_ERR_INVALID_ARG; }
  if (shard_hi > n || shard_lo > shard_hi || (shard_lo & 31) || ((shard_hi & 31) && shard_hi != n)) {
    set_err("shard [%u,%u) of %u must be 32-aligned", shard_lo, shard_hi, n);
    return IBFT_ERR_INVALID_ARG;
  }
  lane* L = &e->lanes[0];
  std::lock_guard<std::mutex> lk(L->mu);
  CU(cudaSetDevice(e->p.device));
  cudaStream_t st = stream ? (cudaStream_t)stream : L->stream;
  uint32_t* count = (uint32_t*)d_count_out;
  if (count) CU(cudaMemsetAsync(count, 0, 4, st));
  if (shard_hi == shard_lo) return IBFT_OK;
  // membership as ibft_verify_batch_device decides it: the bound groups, or none
  const uint32_t n_groups = (uint32_t)L->last_groups.size();
  const ibft_group_desc* groups = n_groups ? L->d_groups : nullptr;
  auto kernel = e->d_wtable != nullptr ? k_explain_list<true> : k_explain_list<false>;
  uint32_t* wl = e->d_explain_wl;
  CU(cudaStreamWaitEvent(st, e->explain_ev, 0));
  // chunks of max_items, a multiple of 32 (ibft_engine_create rounds it up), so that every chunk starts on a bitmap word
  const uint32_t chunk = e->p.max_items;
  for (uint32_t lo = shard_lo; lo < shard_hi; lo += std::min(chunk, shard_hi - lo)) {
    const uint32_t cnt = std::min(chunk, shard_hi - lo);
    CU(cudaMemsetAsync(wl, 0, 4, st));
    CU(launch(e, k_explain_compact, (cnt + 255) / 256, 256, 0, st, (const uint32_t*)d_bitmap, lo, lo + cnt, (uint8_t*)d_reasons,
              (uint8_t*)d_recovered, wl, count));
    CU(launch(e, kernel, (cnt + 31) / 32, 32, 32 * IBFT_RTAB_WORDS * 4, st, (const ibft_sig_item*)d_items, (const uint8_t*)d_arena,
              arena_len, groups, n_groups, e->d_slots, e->p.max_table_slots, e->d_ctable, e->d_wtable, wl, (uint8_t*)d_reasons,
              (uint8_t*)d_recovered));
  }
  CU(cudaEventRecord(e->explain_ev, st));
  return IBFT_OK;
}

// binds the groups used by the device-resident entry points (copied to the engine's device buffers)
extern "C" int ibft_bind_groups(ibft_engine* e, const ibft_group_desc* groups, uint32_t n_groups) {
  IBFT_REFUSE_MULTI(e);
  if (!e || (n_groups && !groups)) { set_err("null argument"); return IBFT_ERR_INVALID_ARG; }
  if (n_groups > e->p.max_groups) { set_err("too many groups"); return IBFT_ERR_CAPACITY; }
  lane* L = &e->lanes[0];
  std::lock_guard<std::mutex> lk(L->mu);
  CU(cudaSetDevice(e->p.device));
  size_t voted_words = 0;
  if (n_groups) {
    int rc = plan_groups(e, L, groups, n_groups, L->h_gdev, &voted_words);
    if (rc != IBFT_OK) return rc;
    memcpy(L->h_groups, groups, (size_t)n_groups * sizeof(ibft_group_desc));
    CU(cudaMemcpy(L->d_groups, L->h_groups, (size_t)n_groups * sizeof(ibft_group_desc), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(L->d_gdev, L->h_gdev, (size_t)n_groups * sizeof(group_dev), cudaMemcpyHostToDevice));
    L->last_gdev.assign(L->h_gdev, L->h_gdev + n_groups);
    L->last_groups.assign(groups, groups + n_groups);
  } else {
    L->last_gdev.clear();
    L->last_groups.clear();
  }
  L->last_hashes.clear();  // new groups: any hash binding was for the previous ones
  return IBFT_OK;
}

// binds the groups of the device-resident calls to the accepted proposal's hash (ibft_group_hash); NULL unbinds
extern "C" int ibft_bind_group_hashes(ibft_engine* e, const ibft_group_hash* hashes, uint32_t n_groups) {
  IBFT_REFUSE_MULTI(e);
  if (!e) { set_err("null argument"); return IBFT_ERR_INVALID_ARG; }
  lane* L = &e->lanes[0];
  std::lock_guard<std::mutex> lk(L->mu);
  if (hashes == nullptr) {
    L->last_hashes.clear();
    return IBFT_OK;
  }
  if (n_groups != L->last_groups.size()) {
    set_err("%u hash bindings for %zu bound groups: call ibft_bind_groups with the same groups first", n_groups, L->last_groups.size());
    return IBFT_ERR_INVALID_ARG;
  }
  bool bound = false;
  int rc = check_group_hashes(L->last_groups.data(), n_groups, hashes, &bound);
  if (rc != IBFT_OK) return rc;
  if (!bound) {
    L->last_hashes.clear();
    return IBFT_OK;
  }
  CU(cudaSetDevice(e->p.device));
  memcpy(L->h_ghash, hashes, (size_t)n_groups * sizeof(ibft_group_hash));
  CU(cudaMemcpy(L->d_ghash, L->h_ghash, (size_t)n_groups * sizeof(ibft_group_hash), cudaMemcpyHostToDevice));
  L->last_hashes.assign(hashes, hashes + n_groups);
  return IBFT_OK;
}

extern "C" int ibft_quorum_reduce_device(ibft_engine* e, const void* d_items, uint32_t n, const void* d_bitmap,
                                         const void* d_groups, uint32_t n_groups, void* d_results, void* stream) {
  return ibft_quorum_reduce_device_ex(e, d_items, n, d_bitmap, d_groups, n_groups, d_results, nullptr, stream);
}

extern "C" int ibft_quorum_reduce_device_ex(ibft_engine* e, const void* d_items, uint32_t n, const void* d_bitmap, const void* d_groups,
                                            uint32_t n_groups, void* d_results, void* d_counted, void* stream) {
  IBFT_REFUSE_MULTI(e);
  if (!e || !d_results || (n && (!d_items || !d_bitmap))) { set_err("null argument"); return IBFT_ERR_INVALID_ARG; }
  lane* L = &e->lanes[0];
  std::lock_guard<std::mutex> lk(L->mu);
  if (n_groups != L->last_groups.size()) { set_err("call ibft_bind_groups with the same groups first"); return IBFT_ERR_INVALID_ARG; }
  (void)d_groups;  // the bound copy is authoritative (its voted-set layout was planned on the host)
  CU(cudaSetDevice(e->p.device));
  cudaStream_t st = stream ? (cudaStream_t)stream : L->stream;
  if (n_groups == 0) return IBFT_OK;
  CU(cudaMemsetAsync(L->d_voted, 0, std::max<size_t>(lane_voted_words(L), 1) * 4, st));
  CU(cudaMemsetAsync(L->d_nvalid, 0, (size_t)n_groups * 4, st));
  if (n)
    CU(mark_votes(e, L, (const ibft_sig_item*)d_items, n, L->dev_arena, L->dev_arena_len, (const uint32_t*)d_bitmap, n_groups,
                  L->last_hashes.empty() ? nullptr : L->d_ghash, (uint32_t*)d_counted, L->d_voted, L->d_nvalid, 0u, n, st));
  CU(reduce_votes(e, L, n_groups, (ibft_group_result*)d_results, st));
  return IBFT_OK;
}

extern "C" int ibft_quorum_partial_words(ibft_engine* e, uint32_t* words_out) {
  IBFT_REFUSE_MULTI(e);
  if (!e || !words_out) { set_err("null argument"); return IBFT_ERR_INVALID_ARG; }
  lane* L = &e->lanes[0];
  std::lock_guard<std::mutex> lk(L->mu);
  *words_out = (uint32_t)(lane_voted_words(L) + L->last_groups.size());
  return IBFT_OK;
}

extern "C" int ibft_quorum_mark_device(ibft_engine* e, const void* d_items, uint32_t n, uint32_t shard_lo, uint32_t shard_hi,
                                       const void* d_bitmap, void* d_partial, void* stream) {
  return ibft_quorum_mark_device_ex(e, d_items, n, shard_lo, shard_hi, d_bitmap, d_partial, nullptr, stream);
}

extern "C" int ibft_quorum_mark_device_ex(ibft_engine* e, const void* d_items, uint32_t n, uint32_t shard_lo, uint32_t shard_hi,
                                          const void* d_bitmap, void* d_partial, void* d_counted, void* stream) {
  IBFT_REFUSE_MULTI(e);
  if (!e || !d_partial || (n && (!d_items || !d_bitmap))) { set_err("null argument"); return IBFT_ERR_INVALID_ARG; }
  if (shard_hi > n || shard_lo > shard_hi) { set_err("bad shard"); return IBFT_ERR_INVALID_ARG; }
  lane* L = &e->lanes[0];
  std::lock_guard<std::mutex> lk(L->mu);
  uint32_t n_groups = (uint32_t)L->last_groups.size();
  if (n_groups == 0) { set_err("call ibft_bind_groups first"); return IBFT_ERR_INVALID_ARG; }
  CU(cudaSetDevice(e->p.device));
  cudaStream_t st = stream ? (cudaStream_t)stream : L->stream;
  const size_t voted_words = lane_voted_words(L);
  uint32_t* part = (uint32_t*)d_partial;
  CU(cudaMemsetAsync(part, 0, (voted_words + n_groups) * 4, st));
  if (shard_hi > shard_lo)
    CU(mark_votes(e, L, (const ibft_sig_item*)d_items, n, L->dev_arena, L->dev_arena_len, (const uint32_t*)d_bitmap, n_groups,
                  L->last_hashes.empty() ? nullptr : L->d_ghash, (uint32_t*)d_counted, part, part + voted_words, shard_lo, shard_hi, st));
  return IBFT_OK;
}

extern "C" int ibft_quorum_merge_device(ibft_engine* e, const void* d_partials, uint32_t n_parts, uint32_t part_stride_words,
                                        void* d_results, void* stream) {
  IBFT_REFUSE_MULTI(e);
  if (!e || !d_partials || !d_results || n_parts == 0) { set_err("null argument"); return IBFT_ERR_INVALID_ARG; }
  lane* L = &e->lanes[0];
  std::lock_guard<std::mutex> lk(L->mu);
  uint32_t n_groups = (uint32_t)L->last_groups.size();
  if (n_groups == 0) { set_err("call ibft_bind_groups first"); return IBFT_ERR_INVALID_ARG; }
  CU(cudaSetDevice(e->p.device));
  cudaStream_t st = stream ? (cudaStream_t)stream : L->stream;
  const size_t voted_words = lane_voted_words(L);
  if (part_stride_words < voted_words + n_groups) { set_err("partial stride too small"); return IBFT_ERR_INVALID_ARG; }
  uint32_t total = (uint32_t)(voted_words + n_groups);
  CU(launch(e, k_quorum_merge, (total + 255) / 256, 256, 0, st, (const uint32_t*)d_partials, n_parts, part_stride_words,
            (uint32_t)voted_words, n_groups, L->d_voted, L->d_nvalid));
  CU(reduce_votes(e, L, n_groups, (ibft_group_result*)d_results, st));
  return IBFT_OK;
}

// Exchange buffers of the peer-memory path: allocated by the engine (a plain cudaMalloc block, so that its IPC handle names
// exactly this buffer), exported as a 64-byte CUDA IPC handle, and opened by the peers ON THEIR OWN DEVICE with lazy peer access --
// which is what makes the mapping dereferenceable from the peer's kernels over NVLink.
static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle is 64 bytes");
extern "C" int ibft_exchange_alloc(ibft_engine* e, uint32_t words, void** d_buf_out, uint8_t handle_out[64]) {
  IBFT_REFUSE_MULTI(e);
  if (!e || !d_buf_out || !handle_out || words == 0) { set_err("bad argument"); return IBFT_ERR_INVALID_ARG; }
  CU(cudaSetDevice(e->p.device));
  void* p = nullptr;
  CU(cudaMalloc(&p, (size_t)words * 4));
  CU(cudaMemset(p, 0, (size_t)words * 4));
  cudaIpcMemHandle_t h;
  cudaError_t ce = cudaIpcGetMemHandle(&h, p);
  if (ce != cudaSuccess) { cudaFree(p); set_err("cudaIpcGetMemHandle: %s", cudaGetErrorString(ce)); return IBFT_ERR_CUDA; }
  memcpy(handle_out, &h, 64);
  *d_buf_out = p;
  return IBFT_OK;
}
extern "C" int ibft_exchange_open(ibft_engine* e, const uint8_t handle[64], void** d_peer_out) {
  IBFT_REFUSE_MULTI(e);
  if (!e || !handle || !d_peer_out) { set_err("bad argument"); return IBFT_ERR_INVALID_ARG; }
  CU(cudaSetDevice(e->p.device));
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, 64);
  void* p = nullptr;
  CU(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
  *d_peer_out = p;
  return IBFT_OK;
}
extern "C" int ibft_exchange_close(ibft_engine* e, void* d_peer) {
  IBFT_REFUSE_MULTI(e);
  if (!e || !d_peer) { set_err("bad argument"); return IBFT_ERR_INVALID_ARG; }
  CU(cudaSetDevice(e->p.device));
  CU(cudaIpcCloseMemHandle(d_peer));
  return IBFT_OK;
}
extern "C" int ibft_exchange_free(ibft_engine* e, void* d_buf) {
  IBFT_REFUSE_MULTI(e);
  if (!e || !d_buf) { set_err("bad argument"); return IBFT_ERR_INVALID_ARG; }
  CU(cudaSetDevice(e->p.device));
  CU(cudaDeviceSynchronize());
  CU(cudaFree(d_buf));
  return IBFT_OK;
}
extern "C" int ibft_exchange_clear(ibft_engine* e, void* d_buf, uint32_t word_off, uint32_t words, void* stream) {
  IBFT_REFUSE_MULTI(e);
  if (!e || !d_buf) { set_err("bad argument"); return IBFT_ERR_INVALID_ARG; }
  CU(cudaSetDevice(e->p.device));
  CU(cudaMemsetAsync((uint32_t*)d_buf + word_off, 0, (size_t)words * 4, stream ? (cudaStream_t)stream : e->lanes[0].stream));
  return IBFT_OK;
}

extern "C" int ibft_quorum_exchange_device(ibft_engine* e, const uint64_t* peer_bufs_in, uint32_t world, uint32_t rank,
                                           uint32_t words_per_rank, uint32_t bitmap_words_per_rank, uint32_t epoch, void* d_bitmap_full,
                                           void* d_results, void* d_timeout_flag, void* stream) {
  IBFT_REFUSE_MULTI(e);
  if (!e || !peer_bufs_in || !d_bitmap_full || !d_results || !d_timeout_flag || world == 0 || world > 8 || rank >= world || epoch == 0) {
    set_err("bad argument");
    return IBFT_ERR_INVALID_ARG;
  }
  lane* L = &e->lanes[0];
  std::lock_guard<std::mutex> lk(L->mu);
  uint32_t n_groups = (uint32_t)L->last_groups.size();
  if (n_groups == 0) { set_err("call ibft_bind_groups first"); return IBFT_ERR_INVALID_ARG; }
  const size_t voted_words = lane_voted_words(L);
  if (words_per_rank < bitmap_words_per_rank + voted_words + n_groups) { set_err("exchange buffer too small"); return IBFT_ERR_INVALID_ARG; }
  CU(cudaSetDevice(e->p.device));
  cudaStream_t st = stream ? (cudaStream_t)stream : L->stream;
  peer_bufs pb{};
  for (uint32_t r = 0; r < world; r++) {
    pb.buf[r] = (uint32_t*)(uintptr_t)peer_bufs_in[r];
  }
  const uint32_t total = world * bitmap_words_per_rank + (uint32_t)voted_words + n_groups;
  const uint32_t blocks = std::max(1u, std::min(64u, (total + 255u) / 256u));
  CU(launch(e, k_quorum_exchange, blocks, 256, 0, st, pb, world, rank, words_per_rank, bitmap_words_per_rank, (uint32_t)voted_words,
            n_groups, epoch, /*spin_limit=*/400000u, (uint32_t*)d_bitmap_full, L->d_voted, L->d_nvalid, (uint32_t*)d_timeout_flag));
  CU(reduce_votes(e, L, n_groups, (ibft_group_result*)d_results, st));
  return IBFT_OK;
}

extern "C" int ibft_get_voted_bitmap(ibft_engine* e, uint32_t group, uint32_t* words_out, uint32_t n_words) {
  e = diag_engine(e);  // a coordinator's merged voted sets are on its lead device
  if (!e || !words_out) { set_err("null argument"); return IBFT_ERR_INVALID_ARG; }
  lane* L = &e->lanes[e->last_lane.load()];
  std::lock_guard<std::mutex> lk(L->mu);
  if (group >= L->last_gdev.size()) { set_err("group %u not part of the last call", group); return IBFT_ERR_INVALID_ARG; }
  const group_dev& g = L->last_gdev[group];
  if (n_words < g.n_words) { set_err("need %u words", g.n_words); return IBFT_ERR_CAPACITY; }
  CU(cudaSetDevice(e->p.device));
  CU(cudaStreamSynchronize(L->stream));
  if (g.n_words) CU(cudaMemcpy(words_out, L->d_voted + g.voted_off, (size_t)g.n_words * 4, cudaMemcpyDeviceToHost));
  for (uint32_t i = g.n_words; i < n_words; i++) words_out[i] = 0;
  return IBFT_OK;
}

// Hash scratch is engine-owned and only ever grows (no cudaMalloc / cudaFree on the per-call path).
static int hash_scratch_reserve(ibft_engine* e, size_t arena_len, uint32_t n) {
  if (arena_len > e->hs_arena_cap) {
    size_t cap = std::max<size_t>(arena_len, std::max<size_t>(e->hs_arena_cap * 2, 1 << 16));
    cudaFree(e->hs_arena); e->hs_arena = nullptr; e->hs_arena_cap = 0;
    cudaFreeHost(e->hs_h_arena); e->hs_h_arena = nullptr;
    CU(cudaMalloc(&e->hs_arena, cap));
    CU(cudaHostAlloc(&e->hs_h_arena, cap, cudaHostAllocDefault));
    e->hs_arena_cap = cap;
  }
  if (n > e->hs_n_cap) {
    uint32_t cap = std::max<uint32_t>(n, std::max<uint32_t>(e->hs_n_cap * 2, 256));
    cudaFree(e->hs_meta); e->hs_meta = nullptr; e->hs_n_cap = 0;
    cudaFreeHost(e->hs_h_meta); e->hs_h_meta = nullptr;
    // per message: offset (4) + length (4) + round (8) in, 32 bytes out
    CU(cudaMalloc(&e->hs_meta, (size_t)cap * 48));
    CU(cudaHostAlloc(&e->hs_h_meta, (size_t)cap * 48, cudaHostAllocDefault));
    e->hs_n_cap = cap;
  }
  return IBFT_OK;
}

static int hash_batch_locked(ibft_engine* e, const uint8_t* arena, size_t arena_len, const uint32_t* offsets, const uint32_t* lens,
                             const uint64_t* rounds, uint32_t n, uint8_t* out32) {
  CU(cudaSetDevice(e->p.device));
  int rc = hash_scratch_reserve(e, arena_len, n);
  if (rc != IBFT_OK) return rc;
  // layout of the meta block (host mirror and device): rounds[n] | offsets[n] | lens[n] | out[n][32]
  uint8_t* hm = e->hs_h_meta;
  uint8_t* dm = e->hs_meta;
  const size_t o_off = (size_t)n * 8, o_len = o_off + (size_t)n * 4, o_out = o_len + (size_t)n * 4;
  if (rounds) memcpy(hm, rounds, (size_t)n * 8);
  memcpy(hm + o_off, offsets, (size_t)n * 4);
  memcpy(hm + o_len, lens, (size_t)n * 4);
  cudaStream_t st = e->hash_stream;
  if (arena_len) {
    memcpy(e->hs_h_arena, arena, arena_len);
    CU(cudaMemcpyAsync(e->hs_arena, e->hs_h_arena, arena_len, cudaMemcpyHostToDevice, st));
  }
  CU(cudaMemcpyAsync(dm, hm, o_out, cudaMemcpyHostToDevice, st));
  CU(launch(e, k_keccak_batch, (n + 63) / 64, 64, 0, st, e->hs_arena, arena_len, (const uint32_t*)(dm + o_off),
            (const uint32_t*)(dm + o_len), rounds ? (const uint64_t*)dm : nullptr, n, dm + o_out));
  CU(cudaMemcpyAsync(hm + o_out, dm + o_out, (size_t)n * 32, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  memcpy(out32, hm + o_out, (size_t)n * 32);
  return IBFT_OK;
}

extern "C" int ibft_keccak256_batch(ibft_engine* e, const uint8_t* arena, size_t arena_len, const uint32_t* offsets,
                                    const uint32_t* lens, uint32_t n, uint8_t* out32) {
  if (!e || (n && (!offsets || !lens || !out32)) || (arena_len && !arena)) { set_err("null argument"); return IBFT_ERR_INVALID_ARG; }
  IBFT_REFUSE_VIEW(e);
  if (n == 0) return IBFT_OK;
  if (e->multi) return multi_hash(e, arena, arena_len, offsets, lens, nullptr, n, out32);
  std::lock_guard<std::mutex> lk(e->hash_mu);
  return hash_batch_locked(e, arena, arena_len, offsets, lens, nullptr, n, out32);
}

extern "C" int ibft_proposal_hash_batch(ibft_engine* e, const uint8_t* arena, size_t arena_len, const uint32_t* offsets,
                                        const uint32_t* lens, const uint64_t* rounds, uint32_t n, uint8_t* out32) {
  if (!e || (n && (!offsets || !lens || !rounds || !out32)) || (arena_len && !arena)) { set_err("null argument"); return IBFT_ERR_INVALID_ARG; }
  IBFT_REFUSE_VIEW(e);
  if (n == 0) return IBFT_OK;
  if (e->multi) return multi_hash(e, arena, arena_len, offsets, lens, rounds, n, out32);
  std::lock_guard<std::mutex> lk(e->hash_mu);
  return hash_batch_locked(e, arena, arena_len, offsets, lens, rounds, n, out32);
}

static int sign_batch(ibft_engine* e, const uint8_t* privkeys, const uint8_t* digests, const uint8_t* nonces, bool rfc6979,
                      uint32_t n, uint8_t* sigs65_out) {
  if (!e || (n && (!privkeys || !digests || !sigs65_out))) { set_err("null argument"); return IBFT_ERR_INVALID_ARG; }
  IBFT_REFUSE_VIEW(e);
  if (n == 0) return IBFT_OK;
  if (e->multi) return multi_sign(e, privkeys, digests, nonces, rfc6979, n, sigs65_out);
  lane* L = &e->lanes[0];
  std::lock_guard<std::mutex> lk(L->mu);
  CU(cudaSetDevice(e->p.device));
  uint8_t *d_d = nullptr, *d_z = nullptr, *d_k = nullptr, *d_s = nullptr;
  int rc = IBFT_OK;
  cudaError_t ce;
#define CUK(call) if ((ce = (call)) != cudaSuccess) { set_err("%s failed: %s", #call, cudaGetErrorString(ce)); rc = IBFT_ERR_CUDA; goto done; }
  CUK(cudaMalloc(&d_d, (size_t)n * 32));
  CUK(cudaMalloc(&d_z, (size_t)n * 32));
  CUK(cudaMalloc(&d_s, (size_t)n * 65));
  CUK(cudaMemcpyAsync(d_d, privkeys, (size_t)n * 32, cudaMemcpyHostToDevice, L->stream));
  CUK(cudaMemcpyAsync(d_z, digests, (size_t)n * 32, cudaMemcpyHostToDevice, L->stream));
  if (nonces) {
    CUK(cudaMalloc(&d_k, (size_t)n * 32));
    CUK(cudaMemcpyAsync(d_k, nonces, (size_t)n * 32, cudaMemcpyHostToDevice, L->stream));
  }
  CUK(launch(e, k_sign, (n + 63) / 64, 64, 0, L->stream, d_d, d_z, d_k, rfc6979, n, d_s));
  CUK(cudaMemcpyAsync(sigs65_out, d_s, (size_t)n * 65, cudaMemcpyDeviceToHost, L->stream));
  CUK(cudaStreamSynchronize(L->stream));
  // private keys do not stay on the device
  cudaMemsetAsync(d_d, 0, (size_t)n * 32, L->stream);
  if (d_k) cudaMemsetAsync(d_k, 0, (size_t)n * 32, L->stream);
  cudaStreamSynchronize(L->stream);
done:
#undef CUK
  cudaFree(d_d); cudaFree(d_z); cudaFree(d_k); cudaFree(d_s);
  return rc;
}

extern "C" int ibft_sign_batch(ibft_engine* e, const uint8_t* privkeys, const uint8_t* digests, const uint8_t* nonces, uint32_t n,
                               uint8_t* sigs65_out) {
  return sign_batch(e, privkeys, digests, nonces, false, n, sigs65_out);
}

extern "C" int ibft_sign_batch_rfc6979(ibft_engine* e, const uint8_t* privkeys, const uint8_t* digests, uint32_t n,
                                       uint8_t* sigs65_out) {
  return sign_batch(e, privkeys, digests, nullptr, true, n, sigs65_out);
}

extern "C" int ibft_set_recover_path(ibft_engine* e, int path) {
  if (e == nullptr || path < IBFT_PATH_AUTO || path > IBFT_PATH_QSPLIT) { set_err("bad recover path"); return IBFT_ERR_INVALID_ARG; }
  IBFT_REFUSE_VIEW(e);
  if (e->multi) return multi_set_recover_path(e, path);
  e->recover_path.store(path);
  return IBFT_OK;
}

extern "C" uint64_t ibft_engine_launch_count(ibft_engine* e) {
  if (e && e->multi) return multi_launch_count(e);
  e = diag_engine(e);
  return e ? e->launches.load() : 0;
}

extern "C" int ibft_probe_int_peak(ibft_engine* e, double* imad_per_s, double* wide_mac_per_s) {
  e = diag_engine(e);
  if (!e || !imad_per_s || !wide_mac_per_s) { set_err("null argument"); return IBFT_ERR_INVALID_ARG; }
  lane* L = &e->lanes[0];
  std::lock_guard<std::mutex> lk(L->mu);
  CU(cudaSetDevice(e->p.device));
  cudaDeviceProp prop;
  CU(cudaGetDeviceProperties(&prop, e->p.device));
  int blocks = prop.multiProcessorCount * 8, threads = 256;
  uint32_t* d_out = nullptr;
  CU(cudaMalloc(&d_out, (size_t)blocks * threads * 4));
  cudaEvent_t e0, e1;
  CU(cudaEventCreate(&e0));
  CU(cudaEventCreate(&e1));
  double best[2] = {0, 0};
  for (int which = 0; which < 2; which++) {
    for (int rep = 0; rep < 4; rep++) {
      CU(cudaEventRecord(e0, L->stream));
      if (which == 0) k_probe_imad<<<blocks, threads, 0, L->stream>>>(d_out, 3, 5);
      else k_probe_wide<<<blocks, threads, 0, L->stream>>>(d_out, 3, 5);
      CU(cudaEventRecord(e1, L->stream));
      CU(cudaEventSynchronize(e1));
      float ms = 0;
      CU(cudaEventElapsedTime(&ms, e0, e1));
      double instr = (double)PROBE_ITERS * PROBE_UNROLL * (which == 0 ? 8 : 4) * (double)blocks * threads;
      double rate = instr / (ms * 1e-3);
      if (rep > 0 && rate > best[which]) best[which] = rate;
    }
  }
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  cudaFree(d_out);
  *imad_per_s = best[0];
  *wide_mac_per_s = best[1];
  return IBFT_OK;
}

extern "C" int ibft_debug_op(ibft_engine* e, int op, const uint8_t* a, const uint8_t* b, const uint8_t* c, uint32_t n,
                             uint8_t* out, uint32_t out_stride) {
  e = diag_engine(e);
  if (!e || !a || !out || n == 0 || ((op == IBFT_DBG_RFC6979 || op == IBFT_DBG_KEY_ADDRESS || op == IBFT_DBG_FE_FUSED) && (!b || !c))) {
    set_err("null argument");
    return IBFT_ERR_INVALID_ARG;
  }
  lane* L = &e->lanes[0];
  std::lock_guard<std::mutex> lk(L->mu);
  CU(cudaSetDevice(e->p.device));
  uint8_t *d_a = nullptr, *d_b = nullptr, *d_c = nullptr, *d_o = nullptr;
  int rc = IBFT_OK;
  cudaError_t ce;
#define CUK(call) if ((ce = (call)) != cudaSuccess) { set_err("%s failed: %s", #call, cudaGetErrorString(ce)); rc = IBFT_ERR_CUDA; goto done; }
  // Operands, the cleared output and the kernel all go on the lane's stream.  That stream is non-blocking, so a copy or memset
  // on the legacy default stream is not ordered before the kernel: a pageable cudaMemcpy may return before its DMA lands and
  // cudaMemset returns before it runs, and the kernel could read the previous call's operands (cudaMalloc hands the same
  // blocks back) or have a lane's result cleared after it was written.
  CUK(cudaMalloc(&d_a, (size_t)n * 32));
  CUK(cudaMemcpyAsync(d_a, a, (size_t)n * 32, cudaMemcpyHostToDevice, L->stream));
  if (b) { CUK(cudaMalloc(&d_b, (size_t)n * 32)); CUK(cudaMemcpyAsync(d_b, b, (size_t)n * 32, cudaMemcpyHostToDevice, L->stream)); }
  if (c) { CUK(cudaMalloc(&d_c, (size_t)n * 64)); CUK(cudaMemcpyAsync(d_c, c, (size_t)n * 64, cudaMemcpyHostToDevice, L->stream)); }
  CUK(cudaMalloc(&d_o, (size_t)n * out_stride));
  CUK(cudaMemsetAsync(d_o, 0, (size_t)n * out_stride, L->stream));
  CUK(launch(e, k_debug_op, (n + 63) / 64, 64, 0, L->stream, op, d_a, d_b, d_c, n, d_o, out_stride));
  CUK(cudaMemcpyAsync(out, d_o, (size_t)n * out_stride, cudaMemcpyDeviceToHost, L->stream));
  CUK(cudaStreamSynchronize(L->stream));
done:
#undef CUK
  cudaFree(d_a); cudaFree(d_b); cudaFree(d_c); cudaFree(d_o);
  return rc;
}

// ------------------------------------------------------------------------------------------------------------
// multi-device engines (ibft_engine_create_multi)
// ------------------------------------------------------------------------------------------------------------
// A coordinator holds one ordinary engine per listed device (its sub-engines; the first is the lead).  A host-buffer verify call
// is cut into contiguous 32-aligned shards (shard_plan.hpp); each shard is planned straight into its device's pinned staging with
// an arena of its own, and each device verifies it through the usual staging, chunking and key-registry paths, recording its votes
// without a reduce.  The lead then gathers every device's voted sets and valid counts with peer copies (ordered by the devices'
// completion events; they work with or without peer access and on a repeated ordinal) and runs the merge and the weighted reduce
// of the device-resident multi-GPU path.  Caller buffers are written only once every device has succeeded.

// one host-buffer call in flight on a lane kind
struct multi_call {
  bool active = false;
  uint32_t n = 0, n_groups = 0, used = 0;  // used: devices [0, used) hold its shards
  bool merge = false;                      // quorum results of a call on more than one device: merged on the lead
  uint32_t* bitmap_out = nullptr;
  ibft_group_result* results_out = nullptr;
  uint8_t* recovered_out = nullptr;
  uint32_t* counted_out = nullptr;
  std::vector<std::vector<uint32_t>> bitmap;   // each shard's verdict words, recovered addresses and counted words, until every
  std::vector<std::vector<uint8_t>> recovered; // device is done
  std::vector<std::vector<uint32_t>> counted;
};

// a slot's table as the devices hold it, for the roll-back of a replication that failed part way
struct multi_table {
  bool valid = false;
  uint64_t height = 0;
  uint32_t n = 0;
  std::vector<uint8_t> addrs, powers;  // powers empty: unit power
};

struct multi_engine {
  std::vector<ibft_engine*> subs;   // one per listed device, in list order
  std::vector<ibft_engine*> views;  // their ibft_engine_sub handles
  // verify, hash and sign calls share it; the calls that replace tables or change the key registries hold it alone, so that no
  // call ever sees the devices disagree
  std::shared_mutex state_mu;
  uint32_t* d_parts[IBFT_LANES] = {nullptr, nullptr};  // on the lead, per lane kind: one partial (voted words | valid counts) per device
  cudaEvent_t merged[IBFT_LANES] = {nullptr, nullptr};
  multi_call pending;  // the asynchronous API (lane 0); guarded by the lead's lane-0 mutex
  std::mutex last_mu;  // the most recent completed host-buffer call
  std::vector<uint8_t> last_status;
  uint32_t last_used = 0;
  std::vector<multi_table> tables;
  // key sharing (IBFT_FLAG_KEY_CACHE; all empty otherwise), guarded by every device's keys_mu.  Per device: a stream for key
  // upkeep (a call that ran on the lead alone holds no lane of the others), a scratch of 17 words per registry entry plus one
  // (another device's state words, then its keys, then the adoption counter), and the value of its learn counter the last
  // share step accounted for
  std::vector<cudaStream_t> key_stream;
  std::vector<uint32_t*> key_scratch;
  std::vector<uint32_t> key_seen;
  uint32_t* h_key_counts = nullptr;  // pinned, 2 words per device: learn counter, keys adopted
};

static int multi_refused(ibft_engine* e, const char* fn) {
  if (e->view_of) set_err("%s: a sub-engine handle (ibft_engine_sub) answers diagnostics only", fn);
  else set_err("%s takes device pointers of one device: a multi-device engine has no such call; use one engine per device "
               "(go-ibft_b200/sharding.py)", fn);
  return IBFT_ERR_INVALID_ARG;
}

static ibft_engine* diag_engine(ibft_engine* e) {
  if (e && e->multi) return e->multi->subs[0];
  if (e && e->view_of) return e->view_of;
  return e;
}

// lane `kind` of devices [0, used), in device-list order: two calls never wait for each other in a cycle
struct multi_lanes_lock {
  multi_engine* M;
  int kind;
  uint32_t used;
  multi_lanes_lock(multi_engine* M_, int kind_, uint32_t used_) : M(M_), kind(kind_), used(used_) {
    for (uint32_t k = 0; k < used; k++) M->subs[k]->lanes[kind].mu.lock();
  }
  ~multi_lanes_lock() {
    for (uint32_t k = used; k-- > 0;) M->subs[k]->lanes[kind].mu.unlock();
  }
};

// fn(k) for every device k < used, each on a thread of its own (k = 0 on the caller's) when `parallel`; returns the first failure,
// with its error text on the calling thread
static int for_devices(uint32_t used, bool parallel, const std::function<int(uint32_t)>& fn) {
  std::vector<int> rc(used, IBFT_OK);
  std::vector<std::string> err(used);
  auto one = [&](uint32_t k) {
    rc[k] = fn(k);
    if (rc[k] != IBFT_OK) err[k] = tl_err;
  };
  std::vector<std::thread> th;
  for (uint32_t k = parallel ? 1 : used; k < used; k++) th.emplace_back(one, k);
  if (parallel) one(0);
  else
    for (uint32_t k = 0; k < used; k++) one(k);
  for (auto& t : th) t.join();
  for (uint32_t k = 0; k < used; k++)
    if (rc[k] != IBFT_OK) {
      set_err("device %u: %s", k, err[k].c_str());
      return rc[k];
    }
  return IBFT_OK;
}

// the lead gathers every shard's voted sets and valid counts and reduces them; enqueued on the lead's lane stream
static int multi_merge_enqueue(multi_engine* M, int kind, uint32_t used, uint32_t n_groups) {
  ibft_engine* lead = M->subs[0];
  lane* L0 = &lead->lanes[kind];
  const size_t vw = lane_voted_words(L0);
  const size_t stride = vw + n_groups;
  CU(cudaSetDevice(lead->p.device));
  cudaStream_t st = L0->stream;
  uint32_t parts = 0;
  for (uint32_t k = 0; k < used; k++) {
    ibft_engine* s = M->subs[k];
    lane* L = &s->lanes[kind];
    if (!L->pending.active) continue;  // an empty trailing shard
    if (k) CU(cudaStreamWaitEvent(st, L->done_ev, 0));
    uint32_t* dst = M->d_parts[kind] + parts * stride;
    if (vw) CU(cudaMemcpyPeerAsync(dst, lead->p.device, L->d_voted, s->p.device, vw * 4, st));
    CU(cudaMemcpyPeerAsync(dst + vw, lead->p.device, L->d_nvalid, s->p.device, (size_t)n_groups * 4, st));
    parts++;
  }
  CU(launch(lead, k_quorum_merge, (uint32_t)((stride + 255) / 256), 256, 0, st, M->d_parts[kind], parts, (uint32_t)stride, (uint32_t)vw,
            n_groups, L0->d_voted, L0->d_nvalid));
  CU(reduce_votes(lead, L0, n_groups, L0->d_results, st));
  CU(cudaMemcpyAsync(L0->h_results, L0->d_results, (size_t)n_groups * sizeof(ibft_group_result), cudaMemcpyDeviceToHost, st));
  CU(cudaEventRecord(M->merged[kind], st));
  return IBFT_OK;
}

// Stages and enqueues a call on lane `kind` of devices [0, used), whose mutexes the caller holds.  Nothing is written to the
// caller's buffers here.
static int multi_submit_locked(ibft_engine* E, int kind, uint32_t used, const ibft_sig_item* items, uint32_t n, const uint8_t* arena,
                               size_t arena_len, const ibft_group_desc* groups, uint32_t n_groups, uint32_t* bitmap_out,
                               ibft_group_result* results_out, uint8_t* recovered_out, multi_call& mc,
                               const ibft_group_hash* ghash = nullptr, uint32_t* counted_out = nullptr, bool async_call = false) {
  multi_engine* M = E->multi;
  ibft_engine* lead = M->subs[0];
  lane* L0 = &lead->lanes[kind];
  for (uint32_t k = 0; k < used; k++)
    if (M->subs[k]->lanes[kind].pending.active) { set_err("a submitted call is still pending; wait for it first"); return IBFT_ERR_INVALID_ARG; }
  mc = multi_call{};
  mc.n = n;
  mc.n_groups = n_groups;
  mc.used = used;
  mc.bitmap_out = bitmap_out;
  mc.results_out = results_out;
  mc.recovered_out = recovered_out;
  mc.counted_out = counted_out;
  if (used == 1) {  // the lead's own call, as on a single-device engine
    int rc = submit_locked(lead, L0, items, n, arena, arena_len, groups, n_groups, bitmap_out, results_out, recovered_out, false, ghash,
                           counted_out, async_call);
    mc.active = rc == IBFT_OK;
    return rc;
  }
  // the checks of a single-device call, on the host before any device is touched
  if ((n && !items) || (n && !bitmap_out) || (arena_len && !arena) || (n_groups && !groups)) { set_err("null argument"); return IBFT_ERR_INVALID_ARG; }
  if (n > L0->cap_items || arena_len > L0->cap_arena || n_groups > E->p.max_groups) {
    set_err("batch (%u items, %zu payload bytes, %u groups) exceeds engine capacity (%u, %zu, %u)", n, arena_len, n_groups,
            L0->cap_items, L0->cap_arena, E->p.max_groups);
    return IBFT_ERR_CAPACITY;
  }
  if (n_groups) {
    std::vector<group_dev> gdev(n_groups);
    size_t voted_words = 0;
    int rc = plan_groups(lead, L0, groups, n_groups, gdev.data(), &voted_words);
    if (rc != IBFT_OK) return rc;
  }
  mc.merge = n_groups && results_out;
  mc.bitmap.resize(used);
  mc.recovered.resize(used);
  mc.counted.resize(used);
  // each device plans its shard into its own pinned staging: large pageable batches are staged on all devices at once
  const bool parallel = (uint64_t)n * sizeof(ibft_sig_item) + arena_len >= (4u << 20);
  int rc = for_devices(used, parallel, [&](uint32_t k) {
    ibft_engine* s = M->subs[k];
    lane* L = &s->lanes[kind];
    uint32_t lo, hi;
    shard_bounds(n, used, k, &lo, &hi);
    if (hi == lo) return IBFT_OK;
    std::vector<arena_run> runs;
    const size_t len = plan_shard(items, lo, hi, arena_len, L->h_items, runs);
    copy_runs(arena, runs, L->h_arena);
    mc.bitmap[k].assign((hi - lo + 31) / 32, 0);
    if (recovered_out) mc.recovered[k].assign((size_t)(hi - lo) * 20, 0);
    if (counted_out) mc.counted[k].assign((hi - lo + 31) / 32, 0);
    // a bound group's filter runs per shard (k_quorum_mark_hashed), so the partials the lead merges hold counted items only
    return submit_locked(s, L, L->h_items, hi - lo, L->h_arena, len, groups, n_groups, mc.bitmap[k].data(), nullptr,
                         recovered_out ? mc.recovered[k].data() : nullptr, /*votes_only=*/mc.merge, ghash,
                         counted_out ? mc.counted[k].data() : nullptr);
  });
  if (rc == IBFT_OK && mc.merge) rc = multi_merge_enqueue(M, kind, used, n_groups);
  if (rc != IBFT_OK) {  // drain what was enqueued; its outputs go to this call's own buffers
    const std::string err = tl_err;
    for (uint32_t k = 0; k < used; k++)
      if (M->subs[k]->lanes[kind].pending.active) (void)wait_locked(M->subs[k], &M->subs[k]->lanes[kind]);
    if (mc.merge) {
      cudaSetDevice(lead->p.device);
      (void)cudaStreamSynchronize(L0->stream);
    }
    set_err("%s", err.c_str());
    return rc;
  }
  mc.active = true;
  return IBFT_OK;
}

// Key sharing.  Every device learns the keys of its own shards; after each host-buffer call the devices whose learn counter
// moved since the last share step are the sources, and every other device adopts their keys: a peer copy of the source's state
// and keys of the entries in use into the destination's scratch (with or without peer access, and on a repeated ordinal), then
// k_adopt_peer_keys, which checks each key against the destination's own address of the entry.  Then every device builds the
// tables of its new keys -- after the adoption, so that a bounded registry hands its free slots to the keys learned on any
// device, in address order, as a single-device engine does.

// every device's keys_mu, in device-list order (taken after any lane: nobody waits for a lane while holding one)
struct multi_keys_lock {
  std::vector<std::unique_lock<std::mutex>> lk;
  explicit multi_keys_lock(multi_engine* M) { for (ibft_engine* s : M->subs) lk.emplace_back(s->keys_mu); }
};
// every lane of every device, device by device in list order, lanes in index order (the reclaim points)
struct multi_all_lanes_lock {
  std::vector<std::unique_lock<std::mutex>> lk;
  explicit multi_all_lanes_lock(multi_engine* M) {
    for (ibft_engine* s : M->subs)
      for (lane& L : s->lanes) lk.emplace_back(L.mu);
  }
};

// The adoption (caller holds every keys_mu).  Afterwards a device's baseline is its counter as read here plus the keys it
// adopted: adopted keys are not sent back as new, and keys a concurrent call learns meanwhile go out with the next step.
static int multi_adopt_keys(multi_engine* M) {
#if IBFT_WC > 0
  const uint32_t n_dev = (uint32_t)M->subs.size();
  uint32_t* h = M->h_key_counts;
  for (uint32_t k = 0; k < n_dev; k++) {
    CU(cudaSetDevice(M->subs[k]->p.device));
    CU(cudaMemcpyAsync(h + 2 * k, M->subs[k]->reg.d_learn_count, 4, cudaMemcpyDeviceToHost, M->key_stream[k]));
  }
  std::vector<uint32_t> src;
  for (uint32_t k = 0; k < n_dev; k++) {
    CU(cudaSetDevice(M->subs[k]->p.device));
    CU(cudaStreamSynchronize(M->key_stream[k]));
    if (h[2 * k] != M->key_seen[k]) src.push_back(k);
  }
  if (src.empty()) return IBFT_OK;
  for (uint32_t d = 0; d < n_dev; d++) {
    ibft_engine* D = M->subs[d];
    key_registry& R = D->reg;
    cudaStream_t ks = M->key_stream[d];
    uint32_t* sc = M->key_scratch[d];
    uint32_t* adopted = sc + 17 * (size_t)R.capacity;
    h[2 * d + 1] = 0;
    CU(cudaSetDevice(D->p.device));
    CU(cudaMemsetAsync(adopted, 0, 4, ks));
    for (uint32_t k : src) {
      const ibft_engine* S = M->subs[k];
      const uint32_t n = std::min(S->reg.used, R.used);
      if (k == d || n == 0) continue;
      // state first: a key the state copy shows as learned was written before that state (learn_key's fence)
      CU(cudaMemcpyPeerAsync(sc, D->p.device, S->reg.d_state, S->p.device, (size_t)n * 4, ks));
      CU(cudaMemcpyPeerAsync(sc + R.capacity, D->p.device, S->reg.d_key_xy, S->p.device, (size_t)n * 64, ks));
      CU(launch(D, k_adopt_peer_keys, (n + 255) / 256, 256, 0, ks, sc, sc + R.capacity, n, R.d_state, R.d_key_xy, R.d_addr,
                R.d_learn_count, adopted));
    }
    CU(cudaMemcpyAsync(h + 2 * d + 1, adopted, 4, cudaMemcpyDeviceToHost, ks));
  }
  for (uint32_t d = 0; d < n_dev; d++) {
    CU(cudaSetDevice(M->subs[d]->p.device));
    CU(cudaStreamSynchronize(M->key_stream[d]));
    M->key_seen[d] = h[2 * d] + h[2 * d + 1];
  }
#else
  (void)M;
#endif
  return IBFT_OK;
}

// every device builds the tables of the keys it learned or adopted (caller holds every keys_mu); a device with nothing new
// since its last refresh costs nothing
static int multi_refresh_keys(multi_engine* M) {
  for (uint32_t k = 0; k < M->subs.size(); k++) {
    ibft_engine* s = M->subs[k];
    if (M->key_seen[k] == s->reg.built_count && !(s->reg.bounded && s->reg.build_due)) continue;
    int rc = refresh_key_tables_held(s, M->key_stream[k], nullptr);
    if (rc != IBFT_OK) return rc;
  }
  return IBFT_OK;
}

// the share step that closes every host-buffer call
static int multi_share_keys(multi_engine* M) {
  if (M->key_stream.empty()) return IBFT_OK;
  multi_keys_lock kl(M);
  int rc = multi_adopt_keys(M);
  return rc != IBFT_OK ? rc : multi_refresh_keys(M);
}

// A reclaim point of a bounded registry (caller holds every lane of every device, devices drained): every device takes the used
// flags of all, matched by address, so that every budget ranks the keys by their use on any device.  The flags only rank keys:
// no device check is needed.
static int multi_merge_used_flags(multi_engine* M) {
#if IBFT_WC > 0
  if (M->key_stream.empty() || !M->subs[0]->reg.bounded) return IBFT_OK;
  std::unordered_set<addr20, addr20_hash> hot;
  std::vector<std::vector<uint8_t>> used(M->subs.size());
  for (size_t k = 0; k < M->subs.size(); k++) {
    const key_registry& R = M->subs[k]->reg;
    used[k].assign(R.used, 0);
    CU(cudaSetDevice(M->subs[k]->p.device));
    if (R.used) CU(cudaMemcpy(used[k].data(), R.d_used, R.used, cudaMemcpyDeviceToHost));
    for (const auto& kv : R.by_addr)
      if (used[k][kv.second]) hot.insert(kv.first);
  }
  for (size_t k = 0; k < M->subs.size(); k++) {
    const key_registry& R = M->subs[k]->reg;
    for (const auto& kv : R.by_addr) used[k][kv.second] |= hot.count(kv.first) ? 1 : 0;
    CU(cudaSetDevice(M->subs[k]->p.device));
    if (R.used) CU(cudaMemcpy(R.d_used, used[k].data(), R.used, cudaMemcpyHostToDevice));
  }
#else
  (void)M;
#endif
  return IBFT_OK;
}

// before the sub-engines' own reclaim points (ibft_set_validators, ibft_set_key_table_budget): merge the used flags.  With a
// call pending nothing is merged: the sub-engines refuse the call themselves.
static int multi_before_reclaim(multi_engine* M) {
  if (M->key_stream.empty() || !M->subs[0]->reg.bounded) return IBFT_OK;
  multi_all_lanes_lock lk(M);
  for (ibft_engine* s : M->subs)
    for (lane& L : s->lanes)
      if (L.pending.active) return IBFT_OK;
  for (ibft_engine* s : M->subs) {
    CU(cudaSetDevice(s->p.device));
    CU(cudaDeviceSynchronize());
  }
  return multi_merge_used_flags(M);
}

// Waits for a call of multi_submit_locked (same lanes held) and, once every device has succeeded, writes the caller's buffers.
static int multi_wait_locked(ibft_engine* E, int kind, multi_call& mc, uint8_t* status_out, uint32_t* voted_out,
                             uint32_t voted_stride_words) {
  multi_engine* M = E->multi;
  if (!mc.active) { set_err("no submitted call to wait for"); return IBFT_ERR_INVALID_ARG; }
  mc.active = false;
  ibft_engine* lead = M->subs[0];
  lane* L0 = &lead->lanes[kind];
  if (mc.used == 1) {
    int rc = wait_locked(lead, L0);
    if (rc != IBFT_OK) return rc;
  } else {
    int rc = IBFT_OK;
    std::string err;
    for (uint32_t k = 0; k < mc.used; k++) {
      lane* L = &M->subs[k]->lanes[kind];
      if (!L->pending.active) continue;
      int r = wait_locked(M->subs[k], L);
      if (r != IBFT_OK && rc == IBFT_OK) { rc = r; err = tl_err; }
    }
    if (mc.merge) {
      cudaError_t ce = cudaSetDevice(lead->p.device);
      if (ce == cudaSuccess) ce = cudaEventSynchronize(M->merged[kind]);
      if (ce != cudaSuccess && rc == IBFT_OK) {
        rc = IBFT_ERR_CUDA;
        err = std::string("quorum merge on the lead device failed: ") + cudaGetErrorString(ce);
      }
    }
    if (rc != IBFT_OK) { set_err("%s", err.c_str()); return rc; }
    for (uint32_t k = 0; k < mc.used; k++) {
      uint32_t lo, hi;
      shard_bounds(mc.n, mc.used, k, &lo, &hi);
      if (hi == lo) continue;
      memcpy(mc.bitmap_out + lo / 32, mc.bitmap[k].data(), mc.bitmap[k].size() * 4);
      if (mc.recovered_out) memcpy(mc.recovered_out + (size_t)lo * 20, mc.recovered[k].data(), mc.recovered[k].size());
      if (mc.counted_out) memcpy(mc.counted_out + lo / 32, mc.counted[k].data(), mc.counted[k].size() * 4);
    }
    if (mc.merge) memcpy(mc.results_out, L0->h_results, (size_t)mc.n_groups * sizeof(ibft_group_result));
  }
  {
    std::lock_guard<std::mutex> lk(M->last_mu);
    M->last_status.resize(mc.n);
    for (uint32_t k = 0; k < mc.used; k++) {
      uint32_t lo, hi;
      shard_bounds(mc.n, mc.used, k, &lo, &hi);
      if (hi > lo) memcpy(M->last_status.data() + lo, M->subs[k]->lanes[kind].h_status, hi - lo);
    }
    M->last_used = mc.used;
    if (status_out && mc.n) memcpy(status_out, M->last_status.data(), mc.n);
  }
  // new keys -> every device, then tables, for the next call; a failure here is reported as a single engine reports its refresh
  int rc = multi_share_keys(M);
  if (rc != IBFT_OK) return rc;
  return copy_voted(lead, L0, mc.n_groups, mc.results_out != nullptr, voted_out, voted_stride_words);
}

static int multi_verify(ibft_engine* E, const ibft_sig_item* items, uint32_t n, const uint8_t* arena, size_t arena_len,
                        const ibft_group_desc* groups, uint32_t n_groups, uint32_t* bitmap_out, ibft_group_result* results_out,
                        uint8_t* recovered_out, uint8_t* status_out, uint32_t* voted_out, uint32_t voted_stride_words,
                        const ibft_group_hash* ghash, uint32_t* counted_out) {
  multi_engine* M = E->multi;
  std::shared_lock<std::shared_mutex> st(M->state_mu);
  const lane& small = M->subs[0]->lanes[1];
  const int kind = n <= small.cap_items && arena_len <= small.cap_arena ? 1 : 0;  // chosen once, for every device
  const uint32_t used = shard_devices(n, (uint32_t)M->subs.size());
  multi_lanes_lock lk(M, kind, used);
  multi_call mc;
  int rc = multi_submit_locked(E, kind, used, items, n, arena, arena_len, groups, n_groups, bitmap_out, results_out, recovered_out, mc, ghash,
                               counted_out);
  if (rc != IBFT_OK) return rc;
  return multi_wait_locked(E, kind, mc, status_out, voted_out, voted_stride_words);
}

// the lead explains: every device holds the same tables, and the items to explain are few
static int multi_explain(ibft_engine* E, const ibft_sig_item* items, uint32_t n, const uint8_t* arena, size_t arena_len,
                         const ibft_group_desc* groups, uint32_t n_groups, const uint32_t* bitmap, uint8_t* reasons_out,
                         uint8_t* recovered_out) {
  multi_engine* M = E->multi;
  std::shared_lock<std::shared_mutex> st(M->state_mu);
  return explain_batch(M->subs[0], items, n, arena, arena_len, groups, n_groups, bitmap, reasons_out, recovered_out);
}

static int multi_submit(ibft_engine* E, const ibft_sig_item* items, uint32_t n, const uint8_t* arena, size_t arena_len,
                        const ibft_group_desc* groups, uint32_t n_groups, uint32_t* bitmap_out, ibft_group_result* results_out,
                        uint8_t* recovered_out) {
  multi_engine* M = E->multi;
  std::shared_lock<std::shared_mutex> st(M->state_mu);
  multi_lanes_lock lk(M, 0, (uint32_t)M->subs.size());
  return multi_submit_locked(E, 0, shard_devices(n, (uint32_t)M->subs.size()), items, n, arena, arena_len, groups, n_groups, bitmap_out,
                             results_out, recovered_out, M->pending, nullptr, nullptr, /*async_call=*/true);
}

static int multi_poll(ibft_engine* E, int* done) {
  multi_engine* M = E->multi;
  multi_lanes_lock lk(M, 0, (uint32_t)M->subs.size());
  *done = 1;
  if (!M->pending.active) return IBFT_OK;
  auto query = [&](ibft_engine* s, cudaEvent_t ev) {
    CU(cudaSetDevice(s->p.device));
    cudaError_t ce = cudaEventQuery(ev);
    if (ce == cudaErrorNotReady) *done = 0;
    else if (ce != cudaSuccess) { set_err("device execution failed: %s", cudaGetErrorString(ce)); return IBFT_ERR_CUDA; }
    return IBFT_OK;
  };
  for (uint32_t k = 0; k < M->pending.used && *done; k++) {
    ibft_engine* s = M->subs[k];
    if (!s->lanes[0].pending.active) continue;
    int rc = query(s, s->lanes[0].done_ev);
    if (rc != IBFT_OK) return rc;
  }
  if (M->pending.merge && *done) return query(M->subs[0], M->merged[0]);
  return IBFT_OK;
}

static int multi_wait(ibft_engine* E) {
  multi_engine* M = E->multi;
  multi_lanes_lock lk(M, 0, (uint32_t)M->subs.size());
  return multi_wait_locked(E, 0, M->pending, nullptr, nullptr, 0);
}

static int multi_last_item_status(ibft_engine* E, uint8_t* status_out, uint32_t n) {
  multi_engine* M = E->multi;
  {
    std::lock_guard<std::mutex> lk(M->subs[0]->lanes[0].mu);
    if (M->pending.active) { set_err("a submitted call is still pending"); return IBFT_ERR_INVALID_ARG; }
  }
  std::lock_guard<std::mutex> lk(M->last_mu);
  if (n > M->last_status.size()) { set_err("last call had %zu items", M->last_status.size()); return IBFT_ERR_INVALID_ARG; }
  memcpy(status_out, M->last_status.data(), n);
  return IBFT_OK;
}

static int multi_known_handed_back(ibft_engine* E, uint32_t* n_out) {
  multi_engine* M = E->multi;
  uint32_t used;
  {
    std::lock_guard<std::mutex> lk(M->last_mu);
    used = M->last_used;
  }
  uint32_t total = 0;
  for (uint32_t k = 0; k < used; k++) {
    uint32_t c = 0;
    int rc = ibft_debug_known_handed_back(M->subs[k], &c);
    if (rc != IBFT_OK) return rc;
    total += c;
  }
  *n_out = total;
  return IBFT_OK;
}

static int multi_hash(ibft_engine* E, const uint8_t* arena, size_t arena_len, const uint32_t* offsets, const uint32_t* lens,
                      const uint64_t* rounds, uint32_t n, uint8_t* out32) {
  multi_engine* M = E->multi;
  std::shared_lock<std::shared_mutex> st(M->state_mu);
  const uint32_t used = shard_devices(n, (uint32_t)M->subs.size());
  std::vector<uint8_t> out((size_t)n * 32);
  int rc = for_devices(used, true, [&](uint32_t k) {
    uint32_t lo, hi;
    shard_bounds(n, used, k, &lo, &hi);
    if (hi == lo) return IBFT_OK;
    ibft_engine* s = M->subs[k];
    std::lock_guard<std::mutex> lk(s->hash_mu);
    return hash_batch_locked(s, arena, arena_len, offsets + lo, lens + lo, rounds ? rounds + lo : nullptr, hi - lo, out.data() + (size_t)lo * 32);
  });
  if (rc == IBFT_OK) memcpy(out32, out.data(), out.size());
  return rc;
}

static int multi_sign(ibft_engine* E, const uint8_t* privkeys, const uint8_t* digests, const uint8_t* nonces, bool rfc6979, uint32_t n,
                      uint8_t* sigs65_out) {
  multi_engine* M = E->multi;
  std::shared_lock<std::shared_mutex> st(M->state_mu);
  const uint32_t used = shard_devices(n, (uint32_t)M->subs.size());
  std::vector<uint8_t> out((size_t)n * 65);
  int rc = for_devices(used, true, [&](uint32_t k) {
    uint32_t lo, hi;
    shard_bounds(n, used, k, &lo, &hi);
    if (hi == lo) return IBFT_OK;
    return sign_batch(M->subs[k], privkeys + (size_t)lo * 32, digests + (size_t)lo * 32, nonces ? nonces + (size_t)lo * 32 : nullptr, rfc6979,
                      hi - lo, out.data() + (size_t)lo * 65);
  });
  if (rc == IBFT_OK) memcpy(sigs65_out, out.data(), out.size());
  return rc;
}

// Unsets a slot: the roll-back, on the devices that already took it, of a table another device refused
static void slot_clear(ibft_engine* e, uint32_t slot) {
  all_lanes_lock lk(e);
  cudaSetDevice(e->p.device);
  cudaDeviceSynchronize();
  slot_host old = std::move(e->slots[slot]);
  e->slots[slot] = slot_host{};
  registry_release(e, old.key_ref);
  cudaFree(old.d_keys); cudaFree(old.d_powers); cudaFree(old.d_key_ref);
  e->slots_shadow[slot] = slot_dev{};
  cudaMemcpy(e->d_slots + slot, &e->slots_shadow[slot], sizeof(slot_dev), cudaMemcpyHostToDevice);
#if IBFT_WC > 0
  if (e->reg.bounded) (void)budget_reclaim(e, e->reg.budget.max_tables);
#endif
}

static int multi_set_validators(ibft_engine* E, uint32_t table_slot, uint64_t height, const uint8_t* addrs, const uint8_t* powers_be,
                                uint32_t n) {
  multi_engine* M = E->multi;
  std::unique_lock<std::shared_mutex> st(M->state_mu);
  int rc = multi_before_reclaim(M);
  if (rc != IBFT_OK) return rc;
  // the lead checks every argument on the host before it touches its device: a refused table leaves every device as it was
  rc = ibft_set_validators(M->subs[0], table_slot, height, addrs, powers_be, n);
  if (rc != IBFT_OK) return rc;
  for (size_t k = 1; k < M->subs.size(); k++) {
    rc = ibft_set_validators(M->subs[k], table_slot, height, addrs, powers_be, n);
    if (rc == IBFT_OK) continue;
    const std::string err = tl_err;
    const multi_table& old = M->tables[table_slot];
    for (size_t j = 0; j < k; j++) {  // the devices that took the new table get the slot's previous content back
      if (old.valid) (void)ibft_set_validators(M->subs[j], table_slot, old.height, old.addrs.data(), old.powers.empty() ? nullptr : old.powers.data(), old.n);
      else slot_clear(M->subs[j], table_slot);
    }
    set_err("device %zu: %s", k, err.c_str());
    return rc;
  }
  multi_table& t = M->tables[table_slot];
  t.valid = true;
  t.height = height;
  t.n = n;
  t.addrs.assign(addrs, addrs + (size_t)n * 20);
  if (powers_be) t.powers.assign(powers_be, powers_be + (size_t)n * 32);
  else t.powers.clear();
  return IBFT_OK;
}

// per (slot, validator): whether device e knows the validator's key
static int known_members(ibft_engine* e, std::vector<std::vector<uint8_t>>& known) {
  known.resize(e->slots.size());
#if IBFT_WC > 0
  if (!(e->p.flags & IBFT_FLAG_KEY_CACHE) || !e->reg.d_state) return IBFT_OK;
  all_lanes_lock lk(e);
  const key_registry& R = e->reg;
  CU(cudaSetDevice(e->p.device));
  CU(cudaDeviceSynchronize());
  std::vector<uint32_t> state(R.used);
  if (R.used) CU(cudaMemcpy(state.data(), R.d_state, (size_t)R.used * 4, cudaMemcpyDeviceToHost));
  for (size_t s = 0; s < e->slots.size(); s++) {
    const slot_host& sh = e->slots[s];
    if (!sh.valid) continue;
    known[s].resize(sh.key_ref.size());
    for (size_t v = 0; v < sh.key_ref.size(); v++) known[s][v] |= state[sh.key_ref[v]] != IBFT_KEY_UNKNOWN;
  }
#endif
  return IBFT_OK;
}

static int multi_refresh_key_tables(ibft_engine* E, uint32_t* n_keys_out) {
  multi_engine* M = E->multi;
  std::unique_lock<std::shared_mutex> st(M->state_mu);
  if (M->key_stream.empty()) {
    for (ibft_engine* s : M->subs) {
      int rc = ibft_refresh_key_tables(s, nullptr);
      if (rc != IBFT_OK) return rc;
    }
  } else {
    // adopt first, then (bounded) the reclaim point on every device with the merged flags, then the tables
    multi_all_lanes_lock lk(M);
    for (ibft_engine* s : M->subs)
      if (s->lanes[0].pending.active) { set_err("a submitted call is still pending"); return IBFT_ERR_INVALID_ARG; }
    multi_keys_lock kl(M);
    int rc = multi_adopt_keys(M);
#if IBFT_WC > 0
    if (rc == IBFT_OK && M->subs[0]->reg.bounded) {
      for (ibft_engine* s : M->subs) {
        CU(cudaSetDevice(s->p.device));
        CU(cudaDeviceSynchronize());
      }
      rc = multi_merge_used_flags(M);
      for (size_t k = 0; k < M->subs.size() && rc == IBFT_OK; k++) rc = budget_reclaim(M->subs[k], M->subs[k]->reg.budget.max_tables);
    }
#endif
    if (rc == IBFT_OK) rc = multi_refresh_keys(M);
    if (rc != IBFT_OK) return rc;
  }
  if (!n_keys_out) return IBFT_OK;
  // the tables are the same on every device: a member counts once when any device knows its key
  std::vector<std::vector<uint8_t>> known;
  for (ibft_engine* s : M->subs) {
    int rc = known_members(s, known);
    if (rc != IBFT_OK) return rc;
  }
  uint32_t total = 0;
  for (const auto& row : known)
    for (uint8_t b : row) total += b;
  *n_keys_out = total;
  return IBFT_OK;
}

static int multi_set_key_table_budget(ibft_engine* E, uint32_t max_tables) {
  multi_engine* M = E->multi;
  std::unique_lock<std::shared_mutex> st(M->state_mu);
  int rc = multi_before_reclaim(M);
  if (rc != IBFT_OK) return rc;
  for (ibft_engine* s : M->subs) {
    rc = ibft_set_key_table_budget(s, max_tables);
    if (rc != IBFT_OK) return rc;
  }
  return IBFT_OK;
}

static int multi_set_recover_path(ibft_engine* E, int path) {
  for (ibft_engine* s : E->multi->subs) s->recover_path.store(path);
  return IBFT_OK;
}

static uint64_t multi_launch_count(ibft_engine* E) {
  uint64_t total = 0;
  for (ibft_engine* s : E->multi->subs) total += s->launches.load();
  return total;
}

static void multi_destroy(ibft_engine* E) {
  multi_engine* M = E->multi;
  if (!M->subs.empty()) {
    cudaSetDevice(M->subs[0]->p.device);
    cudaDeviceSynchronize();
    for (int k = 0; k < IBFT_LANES; k++) {
      cudaFree(M->d_parts[k]);
      if (M->merged[k]) cudaEventDestroy(M->merged[k]);
    }
  }
  for (size_t k = 0; k < M->key_stream.size(); k++) {
    cudaSetDevice(M->subs[k]->p.device);
    cudaDeviceSynchronize();
    if (M->key_stream[k]) cudaStreamDestroy(M->key_stream[k]);
    cudaFree(M->key_scratch[k]);
  }
  cudaFreeHost(M->h_key_counts);
  for (ibft_engine* s : M->subs) engine_free(s);
  for (ibft_engine* v : M->views) delete v;
  delete M;
  delete E;
}

extern "C" int ibft_engine_create_multi(const ibft_engine_params* params, const int32_t* devices, uint32_t n_devices, ibft_engine** out) {
  if (!params || !out || (n_devices && !devices)) { set_err("null argument"); return IBFT_ERR_INVALID_ARG; }
  *out = nullptr;
  if (n_devices == 0 || n_devices > 8) { set_err("a multi-device engine takes 1 to 8 devices, not %u", n_devices); return IBFT_ERR_INVALID_ARG; }
  ibft_engine_params p = *params;
  p.device = devices[0];
  if (n_devices == 1) return ibft_engine_create(&p, out);
  ibft_engine* E = new ibft_engine();
  E->multi = new multi_engine();
  multi_engine* M = E->multi;
  for (uint32_t k = 0; k < n_devices; k++) {
    p.device = devices[k];
    ibft_engine* s = nullptr;
    int rc = ibft_engine_create(&p, &s);
    if (rc != IBFT_OK) {
      const std::string err = tl_err;
      multi_destroy(E);
      set_err("device %u (ordinal %d): %s", k, (int)devices[k], err.c_str());
      return rc;
    }
    M->subs.push_back(s);
    ibft_engine* v = new ibft_engine();
    v->view_of = s;
    v->p = s->p;
    M->views.push_back(v);
  }
  ibft_engine* lead = M->subs[0];
  E->p = lead->p;
  M->tables.resize(E->p.max_table_slots);
  cudaError_t ce = cudaSetDevice(lead->p.device);
  const size_t part_words = lead->lanes[0].voted_words_cap + E->p.max_groups;
  for (int k = 0; k < IBFT_LANES && ce == cudaSuccess; k++) {
    ce = cudaMalloc(&M->d_parts[k], (size_t)n_devices * part_words * 4);
    if (ce == cudaSuccess) ce = cudaEventCreateWithFlags(&M->merged[k], cudaEventDisableTiming);
  }
  if (ce != cudaSuccess) {
    set_err("merge buffers on the lead device: %s", cudaGetErrorString(ce));
    multi_destroy(E);
    return IBFT_ERR_CUDA;
  }
  for (ibft_engine* s : M->subs) s->coordinated = true;
#if IBFT_WC > 0
  if ((E->p.flags & IBFT_FLAG_KEY_CACHE) && lead->reg.d_state) {
    const size_t scratch = (17 * (size_t)lead->reg.capacity + 1) * 4;
    M->key_stream.assign(n_devices, nullptr);
    M->key_scratch.assign(n_devices, nullptr);
    M->key_seen.assign(n_devices, 0);
    ce = cudaHostAlloc(&M->h_key_counts, 8 * (size_t)n_devices, cudaHostAllocPortable);
    for (uint32_t k = 0; k < n_devices && ce == cudaSuccess; k++) {
      ce = cudaSetDevice(M->subs[k]->p.device);
      if (ce == cudaSuccess) ce = cudaStreamCreateWithFlags(&M->key_stream[k], cudaStreamNonBlocking);
      if (ce == cudaSuccess) ce = cudaMalloc(&M->key_scratch[k], scratch);
    }
    if (ce != cudaSuccess) {
      set_err("key sharing buffers: %s", cudaGetErrorString(ce));
      multi_destroy(E);
      return ce == cudaErrorMemoryAllocation ? IBFT_ERR_CAPACITY : IBFT_ERR_CUDA;
    }
  }
#endif
  *out = E;
  return IBFT_OK;
}

extern "C" int ibft_engine_device_count(ibft_engine* e, uint32_t* n_out) {
  if (!e || !n_out) { set_err("null argument"); return IBFT_ERR_INVALID_ARG; }
  *n_out = e->multi ? (uint32_t)e->multi->subs.size() : 1u;
  return IBFT_OK;
}

extern "C" int ibft_engine_sub(ibft_engine* e, uint32_t k, ibft_engine** sub_out) {
  if (!e || !sub_out) { set_err("null argument"); return IBFT_ERR_INVALID_ARG; }
  const uint32_t n = e->multi ? (uint32_t)e->multi->subs.size() : 1u;
  if (k >= n) { set_err("device %u of an engine over %u", k, n); return IBFT_ERR_INVALID_ARG; }
  *sub_out = e->multi ? e->multi->views[k] : e;  // a single-device engine is its own only device engine
  return IBFT_OK;
}
