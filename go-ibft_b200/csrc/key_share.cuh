// Key sharing between engines of separate processes (ibft_key_share_*, include/ibft_verify.h): the key block's records, which
// registry entries an export takes, and what an adoption does with a record.  Shared by k_key_export / k_key_adopt (engine.cu)
// and the host emulation (tests/emul/key_share_sync_driver.cpp).
#pragma once
#include "verify_core.cuh"

// key registry entry states (engine.cu)
#define IBFT_KEY_UNKNOWN 0u
#define IBFT_KEY_LEARNED 1u
#define IBFT_KEY_READY 2u
#define IBFT_KEY_BUILDING 3u  // claimed by a table-build pass (refresh_key_tables_locked)
#define IBFT_KEY_EVICTED 4u   // bounded registry: key known, no table slot (every kernel treats it as LEARNED)

static_assert(IBFT_KEY_SHARE_WORDS % 64 == 0 && IBFT_KEY_SHARE_WORDS >= 1 + IBFT_KEY_SHARE_RECORDS * IBFT_KEY_SHARE_RECORD_WORDS,
              "a key block holds its count word and IBFT_KEY_SHARE_RECORDS records, padded to 64 words");

namespace ibft {

// An export takes an entry whose key this engine learned by recovery and has not exported yet.  `shared` is the entry's export
// mark: set by the export that sent the key and by the adoption that took it (an adopted key is never sent back), cleared when
// ibft_set_validators gives the entry to another address.
IBFT_HD bool key_share_exportable(uint32_t state, uint32_t shared) {
  return shared == 0 && (state == IBFT_KEY_LEARNED || state == IBFT_KEY_READY || state == IBFT_KEY_EVICTED);
}

// One record: the entry's 20 address bytes in five words (byte 4k + j in byte j of word k), then x and y as 8 little-endian
// words each (the registry's key_xy format).
IBFT_HD void key_share_put(uint32_t* rec, const uint8_t* addr20, const uint32_t* xy16) {
#pragma unroll
  for (int k = 0; k < 5; k++)
    rec[k] = (uint32_t)addr20[4 * k] | ((uint32_t)addr20[4 * k + 1] << 8) | ((uint32_t)addr20[4 * k + 2] << 16) |
             ((uint32_t)addr20[4 * k + 3] << 24);
#pragma unroll
  for (int i = 0; i < 16; i++) rec[5 + i] = xy16[i];
}

#define IBFT_KEY_SHARE_DROP 0u    // no resident table lists the address
#define IBFT_KEY_SHARE_REFUSE 1u  // the key fails key_matches_address against the entry's address
#define IBFT_KEY_SHARE_KNOWN 2u   // a valid key of an entry that already has one
#define IBFT_KEY_SHARE_ADOPT 3u   // a valid key of an unknown entry: the caller writes it as learn_key does

// What an adoption does with a record.  The address is looked up in every resident table (lookup(slot, addr20) = the registry
// entry of the address in table slot `slot`, or -1 when that table does not list it); records name addresses, not entries,
// because two engines need not number their entries alike.  The key is checked before the entry's state is looked at, so a
// forged record counts as refused whether or not the entry is known.  *r_out = the entry (DROP: unset); *xy_out = the key.
template <class LOOKUP>
IBFT_HD uint32_t key_share_decide(const uint32_t* rec, uint32_t n_slots, const LOOKUP& lookup, const uint32_t* state,
                                  const uint8_t* entry_addr, uint32_t* r_out, fe* x_out, fe* y_out) {
  uint8_t a[20];
#pragma unroll
  for (int i = 0; i < 20; i++) a[i] = (uint8_t)(rec[i / 4] >> (8 * (i % 4)));
  int r = -1;
  for (uint32_t s = 0; s < n_slots && r < 0; s++) r = lookup(s, a);
  if (r < 0) return IBFT_KEY_SHARE_DROP;
  *r_out = (uint32_t)r;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    x_out->v[i] = rec[5 + i];
    y_out->v[i] = rec[13 + i];
  }
  if (!key_matches_address(*x_out, *y_out, entry_addr + 20 * (size_t)r)) return IBFT_KEY_SHARE_REFUSE;
  return state[r] == IBFT_KEY_UNKNOWN ? IBFT_KEY_SHARE_ADOPT : IBFT_KEY_SHARE_KNOWN;
}

}  // namespace ibft
