// C entry points over go-ibft_b200/csrc/group_hash.cuh (the proposal-hash extraction of groups bound to an accepted proposal) on
// the host, for tests/test_emul_group_hash.py.  Built on demand by that test:
//   g++ -O2 -fPIC -std=c++17 -shared -o libibft_group_hash.so group_hash_driver.cpp
#include "../../go-ibft_b200/csrc/group_hash.cuh"

extern "C" {

// extract_vote_hash over w[0, len): 1 with the hash copied to out (up to out_cap bytes) and its length in *out_len, 0 for nil
int gh_extract(const uint8_t* w, uint32_t len, uint32_t msg_type, uint8_t* out, uint32_t out_cap, uint32_t* out_len) {
  uint32_t off = 0, n = 0;
  if (!ibft::extract_vote_hash(w, len, msg_type, &off, &n)) return 0;
  for (uint32_t i = 0; i < n && i < out_cap; i++) out[i] = w[off + i];
  *out_len = n;
  return 1;
}

// item_names_hash for one packed tuple against a 32-byte bound hash
int gh_item_names_hash(const ibft_sig_item* it, const uint8_t* arena, size_t arena_len, uint32_t msg_type, const uint8_t* bound) {
  return ibft::item_names_hash(*it, arena, arena_len, msg_type, bound) ? 1 : 0;
}
}
