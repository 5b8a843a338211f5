// shard_plan.hpp -- host-only planner of a multi-device host-buffer call (ibft_engine_create_multi): which devices a call of n
// items uses, the contiguous 32-aligned shard of each, and each shard's own tuples and payload arena.
//
// A shard's arena is the union of the byte ranges its items reference, each byte copied once, rounded out to the call arena's
// 16-byte blocks: a coverage bitmap marks every block a span touches, the marked blocks are packed in order, and every payload
// offset (payload_off of the kinds that carry a payload, the second-span offset in digest[0..8) of IBFT_KIND_PAYLOAD2) is
// rewritten into them.  A certificate's nested IBFT_KIND_WIRE frames lie inside their outer frame, and the ROUND_CHANGE messages
// of a round share one certificate tail, so copying per item would duplicate those bytes and could push a shard past
// max_payload_bytes where the whole call fits.  A shard's arena holds a subset of the call's blocks, so it is never longer than
// the call's, and every span keeps its offset mod 16 (the sponge sees the same alignment).  The plan costs one pass over the
// items plus one over the bitmap (arena_len / 128 bytes), with no sort.  Spans outside the call's arena are left as they are:
// they stay outside the (shorter) shard arena, verdict 0 either way.  Zero-length spans inside the arena become offset 0.
#ifndef IBFT_SHARD_PLAN_HPP
#define IBFT_SHARD_PLAN_HPP

#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../include/ibft_verify.h"

// A multi-device call of n items runs on min(devices, ceil(n / IBFT_MULTI_MIN_SHARD)) devices (at least one).  The value is a
// guess, not a measurement: below it the cost of another device's launches and merge copies is assumed to outweigh its share.
#define IBFT_MULTI_MIN_SHARD 1024u

namespace ibft {

inline uint32_t shard_devices(uint32_t n, uint32_t n_devices) {
  const uint64_t want = ((uint64_t)n + IBFT_MULTI_MIN_SHARD - 1) / IBFT_MULTI_MIN_SHARD;
  return (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(n_devices, want));
}

// [lo, hi) of shard `rank` of `world`: contiguous, disjoint, covering [0, n), every boundary except n a multiple of 32 (the rule of
// sharding.shard_bounds).  Trailing shards may be empty (lo == hi == n).
inline void shard_bounds(uint32_t n, uint32_t world, uint32_t rank, uint32_t* lo, uint32_t* hi) {
  const uint64_t words = ((uint64_t)n + 31) / 32, per = (words + world - 1) / world;
  *lo = (uint32_t)std::min<uint64_t>((uint64_t)rank * per * 32, n);
  *hi = (uint32_t)std::min<uint64_t>(((uint64_t)rank + 1) * per * 32, n);
}

// one copy into the shard arena: arena[src, src + len) -> shard_arena[dst, dst + len)
struct arena_run {
  uint64_t src, dst, len;
};

inline bool kind_has_payload(uint8_t kind) {
  return kind == IBFT_KIND_PAYLOAD || kind == IBFT_KIND_WIRE || kind == IBFT_KIND_WIRE_SEAL || kind == IBFT_KIND_PAYLOAD2;
}

inline uint64_t payload2_off(const ibft_sig_item& it) {
  uint64_t v = 0;
  for (int i = 0; i < 8; i++) v |= (uint64_t)it.digest[i] << (8 * i);
  return v;
}
inline uint32_t payload2_len(const ibft_sig_item& it) {
  return (uint32_t)it.digest[8] | ((uint32_t)it.digest[9] << 8) | ((uint32_t)it.digest[10] << 16) | ((uint32_t)it.digest[11] << 24);
}

// Plans items[lo, hi) of a call whose arena is arena_len bytes: local[0, hi - lo) receives the tuples with their offsets rewritten,
// runs the copies that build the shard arena (ascending, disjoint).  Returns the shard arena's length (<= arena_len).
inline size_t plan_shard(const ibft_sig_item* items, uint32_t lo, uint32_t hi, size_t arena_len, ibft_sig_item* local,
                         std::vector<arena_run>& runs) {
  runs.clear();
  const uint32_t cnt = hi - lo;
  const uint64_t blocks = ((uint64_t)arena_len + 15) / 16, words = (blocks + 63) / 64;
  std::vector<uint64_t> cover(words, 0);
  auto in_range2 = [&](const ibft_sig_item& it) {
    const uint64_t off2 = payload2_off(it), len2 = payload2_len(it);
    return off2 <= arena_len && len2 <= arena_len - off2;
  };
  auto mark = [&](uint64_t off, uint64_t len) {  // blocks [b0, b1) of a non-empty in-range span
    const uint64_t b0 = off / 16, b1 = (off + len - 1) / 16 + 1, w0 = b0 / 64, w1 = (b1 - 1) / 64;
    const uint64_t head = ~0ull << (b0 % 64), tail = ~0ull >> (63 - (b1 - 1) % 64);
    if (w0 == w1) { cover[w0] |= head & tail; return; }
    cover[w0] |= head;
    for (uint64_t w = w0 + 1; w < w1; w++) cover[w] = ~0ull;
    cover[w1] |= tail;
  };
  for (uint32_t i = 0; i < cnt; i++) {  // one pass copies the tuples and marks their spans
    memcpy(&local[i], &items[lo + i], sizeof(ibft_sig_item));
    const ibft_sig_item& it = local[i];
    if (!kind_has_payload(it.kind)) continue;
    if (it.payload_len && (uint64_t)it.payload_off + it.payload_len <= arena_len) mark(it.payload_off, it.payload_len);
    if (it.kind == IBFT_KIND_PAYLOAD2 && payload2_len(it) && in_range2(it)) mark(payload2_off(it), payload2_len(it));
  }
  // rank[w] = marked blocks before word w; the shard offset of global byte o is 16 * (marked blocks before o's block) + o % 16
  std::vector<uint64_t> rank(words + 1, 0);
  for (uint64_t w = 0; w < words; w++) rank[w + 1] = rank[w] + (uint64_t)__builtin_popcountll(cover[w]);
  auto rebase = [&](uint64_t off, uint64_t len) -> uint64_t {
    if (len == 0) return 0;
    const uint64_t b = off / 16, w = b / 64;
    return 16 * (rank[w] + (uint64_t)__builtin_popcountll(cover[w] & ((1ull << (b % 64)) - 1))) + off % 16;
  };
  // the runs of marked blocks (the last block of the arena may be short)
  auto next = [&](uint64_t from, bool set) -> uint64_t {  // first block >= from whose bit is `set`, or blocks
    uint64_t w = from / 64;
    if (w >= words) return blocks;
    uint64_t x = (set ? cover[w] : ~cover[w]) & (~0ull << (from % 64));
    while (!x && ++w < words) x = set ? cover[w] : ~cover[w];
    return w < words ? std::min(blocks, w * 64 + (uint64_t)__builtin_ctzll(x)) : blocks;
  };
  uint64_t dst = 0;
  for (uint64_t b = next(0, true); b < blocks; b = next(b, true)) {
    const uint64_t end = next(b, false), len = std::min<uint64_t>(end * 16, arena_len) - b * 16;
    runs.push_back(arena_run{b * 16, dst, len});
    dst += len;
    b = end;
  }
  for (uint32_t i = 0; i < cnt; i++) {
    ibft_sig_item& it = local[i];
    if (!kind_has_payload(it.kind)) continue;
    if ((uint64_t)it.payload_off + it.payload_len <= arena_len) it.payload_off = (uint32_t)rebase(it.payload_off, it.payload_len);
    if (it.kind == IBFT_KIND_PAYLOAD2 && in_range2(it)) {
      const uint64_t o = rebase(payload2_off(it), payload2_len(it));
      for (int b = 0; b < 8; b++) it.digest[b] = (uint8_t)(o >> (8 * b));
    }
  }
  return (size_t)dst;
}

// builds the shard arena planned by plan_shard
inline void copy_runs(const uint8_t* arena, const std::vector<arena_run>& runs, uint8_t* shard_arena) {
  for (const arena_run& r : runs) memcpy(shard_arena + r.dst, arena + r.src, (size_t)r.len);
}

}  // namespace ibft

#endif  // IBFT_SHARD_PLAN_HPP
