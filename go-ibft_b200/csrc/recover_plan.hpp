// recover_plan.hpp -- host-only planner of the recover step: which signature kernels (sig_kernel) one step launches, and
// whether a host-buffer call is cut into latency pieces.  The verdicts are the same on every path; only latency and throughput
// differ.  engine.cu launches what these functions return, and its kernels size their CTAs by the values below.  The split
// kernels, k_verify_known and the key registry exist only with a combined generator table (IBFT_WC > 0: `wc` below).
//
// For a step of cnt items on S SMs:
//   small  cnt <= S * 256: one-warp CTAs (eight per SM) still cover the step in one wave
//   long   arena_len / cnt > 256 (integer division): ROUND_CHANGE messages with their certificates, up to 909 KB of signed bytes
//          each, whose sponges a helper warp would hash one after the other; one thread per signature hashes them in parallel
//   K      the known-key pass may run (known_key_ok): engine flag IBFT_FLAG_KEY_CACHE, no recovered addresses wanted, groups
//          bound, and a worklist that holds the step (a larger device-resident shard takes the plain recover path)
// AUTO (ibft_set_recover_path) resolves, with a combined table: K or long -> THREAD (verifying against the learned key's comb
// table, 51 additions and no doubling, beats every recover kernel at every size); else cnt <= S * 48 -> QSPLIT (two CTAs of 24
// per SM); else cnt <= S * 192 -> SPLIT (two CTAs of 96 per SM: a 10k-validator COMMIT round); else THREAD.  Without one:
// QUAD up to S * 32 (one wave of its CTAs), else THREAD.  The resolved path runs, with a combined table:
//   QSPLIT      bitmap range zeroed (its verdict bits are OR-ed in), then k_recover_qsplit -- even with K
//   SPLIT       with K k_verify_split, then k_recover_qsplit over its worklist; else k_recover_split
//   QUAD        k_recover_quad -- even with K; also without a combined table
//   THREAD      with K k_verify_known<32 if small, else 128>, then over its worklist k_recover_qsplit if small and not long,
//               else k_recover<128>; else (and on every path but QUAD without a combined table) k_recover<32 if small, else 128>
//
// Latency pieces: a host-buffer call of n items with a combined table, path AUTO, S * 48 < n <= S * 96 and not long (e.g.
// 10,000 seals, 1.28 MB of tuples) would have its staging copy and upload sit in front of a kernel that cannot start before its
// last tuple has arrived.  It goes in IBFT_LAT_PIECES pieces of ceil(ceil(n / 4) / 96) * 96 items, each on its own stream:
// piece k+1 is staged while piece k is copied and verified, and the pieces' kernels run side by side on different SMs.  Piece k
// uses worklist k and is forced to THREAD with K (the known-key pass in one-warp CTAs), else to SPLIT.  Every other call goes
// in upload chunks of 2^17 items on the engine's path, chunk c using worklist c & 1.
#ifndef IBFT_RECOVER_PLAN_HPP
#define IBFT_RECOVER_PLAN_HPP

#include <cstddef>
#include <cstdint>

#include "../../include/ibft_verify.h"

#define IBFT_BLOCK 128                // threads (= signatures) per CTA of the throughput kernels
#define IBFT_QUAD_SIGS 32             // signatures per k_recover_quad CTA (four lanes each: 128 threads, one bitmap word)
#define IBFT_SPLIT_CHAINS 3           // chain warps per k_recover_split / k_verify_split CTA, besides the helper warp
#define IBFT_SPLIT_SIGS (32 * IBFT_SPLIT_CHAINS)
#define IBFT_QSPLIT_SIGS 24           // signatures per k_recover_qsplit CTA: three four-lane chain warps of 8
#define IBFT_SMALL_SIGS_PER_SM 256u   // small step: at most this many signatures per SM
#define IBFT_LONG_PAYLOAD 256u        // long step: more payload bytes than this per item
#define IBFT_LAT_PIECES 4u

namespace ibft {

enum sig_kernel : int {
  SK_NONE = 0,
  SK_RECOVER_32,        // k_recover<32>: one thread per signature, one-warp CTAs
  SK_RECOVER_128,       // k_recover<IBFT_BLOCK>: the throughput kernel
  SK_QUAD,              // k_recover_quad: four lanes per signature
  SK_SPLIT,             // k_recover_split: chain warps (one lane per signature) + a helper warp (digest, r^-1, root, u1*G)
  SK_QSPLIT,            // k_recover_qsplit: four-lane chain warps + a helper warp; also the worklist pass
  SK_VERIFY_KNOWN_32,   // k_verify_known<32>: the known-key pass, one thread per signature
  SK_VERIFY_KNOWN_128,  // k_verify_known<IBFT_BLOCK>
  SK_VERIFY_SPLIT,      // k_verify_split: the known-key pass on chain + helper warps
};

struct recover_plan {
  sig_kernel first;     // SK_QSPLIT: its range of the bitmap is zeroed first
  sig_kernel worklist;  // the pass over what the known-key first pass left, or SK_NONE
};

inline bool known_key_ok(bool key_cache, bool want_recovered, bool groups, bool worklist, uint32_t cnt, uint32_t worklist_cap) {
  return key_cache && !want_recovered && groups && worklist && cnt <= worklist_cap;
}

inline bool long_payloads(uint32_t cnt, size_t arena_len) { return arena_len / cnt > IBFT_LONG_PAYLOAD; }

// the kernels of one recover step of cnt > 0 items on `path` (ibft_set_recover_path's values)
inline recover_plan plan_recover(int path, uint32_t cnt, size_t arena_len, uint32_t sms, bool known, bool wc) {
  if (path == IBFT_PATH_AUTO) {
    if (!wc) path = cnt <= sms * IBFT_QUAD_SIGS ? IBFT_PATH_QUAD : IBFT_PATH_THREAD;
    else if (known || long_payloads(cnt, arena_len)) path = IBFT_PATH_THREAD;
    else if (cnt <= sms * 2u * IBFT_QSPLIT_SIGS) path = IBFT_PATH_QSPLIT;
    else if (cnt <= sms * 2u * IBFT_SPLIT_SIGS) path = IBFT_PATH_SPLIT;
    else path = IBFT_PATH_THREAD;
  }
  const bool small = cnt <= sms * IBFT_SMALL_SIGS_PER_SM;
  if (path == IBFT_PATH_QUAD) return {SK_QUAD, SK_NONE};
  if (wc && path == IBFT_PATH_QSPLIT) return {SK_QSPLIT, SK_NONE};
  if (wc && path == IBFT_PATH_SPLIT) return known ? recover_plan{SK_VERIFY_SPLIT, SK_QSPLIT} : recover_plan{SK_SPLIT, SK_NONE};
  if (wc && known)
    return {small ? SK_VERIFY_KNOWN_32 : SK_VERIFY_KNOWN_128, small && !long_payloads(cnt, arena_len) ? SK_QSPLIT : SK_RECOVER_128};
  return {small ? SK_RECOVER_32 : SK_RECOVER_128, SK_NONE};
}

struct piece_plan {
  uint32_t per;  // items per piece (IBFT_LAT_PIECES pieces at most); 0: the call goes in upload chunks on its own path
  int path;      // the path every piece is forced to
};

// how a host-buffer call of n items on the engine's `path` is cut (known: K for the whole call)
inline piece_plan plan_pieces(int path, uint32_t n, size_t arena_len, uint32_t sms, bool known, bool wc) {
  if (!wc || path != IBFT_PATH_AUTO || n <= sms * 2u * IBFT_QSPLIT_SIGS || n > sms * IBFT_SPLIT_SIGS || long_payloads(n, arena_len))
    return {0, path};
  const uint32_t quarter = (n + IBFT_LAT_PIECES - 1) / IBFT_LAT_PIECES;
  return {(quarter + IBFT_SPLIT_SIGS - 1) / IBFT_SPLIT_SIGS * IBFT_SPLIT_SIGS, known ? IBFT_PATH_THREAD : IBFT_PATH_SPLIT};
}

}  // namespace ibft

#endif  // IBFT_RECOVER_PLAN_HPP
