// The key-share decisions of k_key_export / k_key_adopt (key_share.cuh) on the host emulation (TEST ONLY): which entries an
// export takes and in what order, and what an adoption does with each record of the peers' key blocks.  The kernels' thread
// layout is not emulated: the export walks the entries in ascending order as the kernel's prefix count orders them, the
// adoption takes the records one at a time.  Built on demand by tests/test_emul_key_share_sync.py:
//   g++ -O2 -fPIC -std=c++17 -DEMUL_DIR=\"<tests/emul>\" -shared -o libibft_key_share_sync.so key_share_sync_driver.cpp -lpthread
#include "emul.cpp"
#include "../../go-ibft_b200/csrc/key_share.cuh"

extern "C" {

// Export of a registry of n entries (state, shared: n words; key_xy: 16 words per entry; addr: 20 bytes per entry) into
// `block` (IBFT_KEY_SHARE_WORDS words).  Marks the exported entries.  Returns the record count.
uint32_t emul_key_share_export(const uint32_t* state, uint32_t* shared, const uint32_t* key_xy, const uint8_t* addr, uint32_t n,
                               uint32_t* block) {
  uint32_t c = 0;
  for (uint32_t r = 0; r < n && c < IBFT_KEY_SHARE_RECORDS; r++)
    if (key_share_exportable(state[r], shared[r])) {
      key_share_put(block + 1 + IBFT_KEY_SHARE_RECORD_WORDS * c, addr + 20 * (size_t)r, key_xy + 16 * (size_t)r);
      shared[r] = 1;
      c++;
    }
  block[0] = c;
  return c;
}

// Adoption of the blocks [n_parts][IBFT_KEY_SHARE_WORDS] but block self_part.  Resident tables: slot s lists tab_n[s] addresses
// (ascending, 20 bytes each, at tab_addr + 20 * s * stride) whose registry entries are tab_ref[s * stride + row].  An adopted key is
// written and its entry marked LEARNED and exported, as k_key_adopt does.  decisions[p * IBFT_KEY_SHARE_RECORDS + i] =
// IBFT_KEY_SHARE_* of record i of block p (0xFF: not a record of the block).  counts = { adopted, refused }.
void emul_key_share_adopt(const uint32_t* blocks, uint32_t n_parts, uint32_t self_part, uint32_t n_slots, const uint8_t* tab_addr,
                          const uint32_t* tab_ref, const uint32_t* tab_n, uint32_t stride, uint32_t* state, uint32_t* key_xy,
                          const uint8_t* addr, uint32_t* shared, uint32_t* counts, uint8_t* decisions) {
  auto lookup = [&](uint32_t s, const uint8_t* a) -> int {
    uint32_t lo = 0, hi = tab_n[s];
    while (lo < hi) {
      const uint32_t mid = (lo + hi) / 2;
      const int c = memcmp(tab_addr + 20 * ((size_t)s * stride + mid), a, 20);
      if (c == 0) return (int)tab_ref[(size_t)s * stride + mid];
      if (c < 0) lo = mid + 1; else hi = mid;
    }
    return -1;
  };
  counts[0] = counts[1] = 0;
  memset(decisions, 0xFF, (size_t)n_parts * IBFT_KEY_SHARE_RECORDS);
  for (uint32_t p = 0; p < n_parts; p++) {
    if (p == self_part) continue;
    const uint32_t* blk = blocks + (size_t)p * IBFT_KEY_SHARE_WORDS;
    if (blk[0] > IBFT_KEY_SHARE_RECORDS) { counts[1]++; continue; }
    for (uint32_t i = 0; i < blk[0]; i++) {
      uint32_t r = 0;
      fe x, y;
      const uint32_t d = key_share_decide(blk + 1 + IBFT_KEY_SHARE_RECORD_WORDS * i, n_slots, lookup, state, addr, &r, &x, &y);
      decisions[(size_t)p * IBFT_KEY_SHARE_RECORDS + i] = (uint8_t)d;
      if (d == IBFT_KEY_SHARE_REFUSE) counts[1]++;
      if (d != IBFT_KEY_SHARE_ADOPT) continue;
      for (int k = 0; k < 8; k++) { key_xy[16 * (size_t)r + k] = x.v[k]; key_xy[16 * (size_t)r + 8 + k] = y.v[k]; }
      state[r] = IBFT_KEY_LEARNED;
      shared[r] = 1;
      counts[0]++;
    }
  }
}
}
