// explain_item (verify_core.cuh), the reason pass of ibft_explain_batch, on the host emulation (TEST ONLY): the same headers the
// kernel k_explain compiles, with the product's one-thread recovery (u1*G by the per-position comb, its entries computed on demand).
// Built on demand by tests/test_explain_oracle.py:
//   g++ -O2 -fPIC -std=c++17 -DEMUL_DIR=\"<tests/emul>\" -shared -o libibft_explain.so explain_driver.cpp -lpthread
#include "emul.cpp"

#include <mutex>

extern "C" {

// IBFT_REASON_* of one item; recovered20 = the recovered address (zero when recovery was not reached or failed).
//   grouped / n_groups: the call's groups (grouped = 0: a call without groups, which never yields IBFT_REASON_NO_GROUP)
//   table / table_n: the addresses (table_n x 20 bytes) of the validator table of the item's group; NULL for a group without one
int emul_explain_item(const ibft_sig_item* it, const uint8_t* arena, size_t arena_len, int grouped, uint32_t n_groups,
                      const uint8_t* table, uint32_t table_n, uint8_t* recovered20) {
  gtab_view G = emul_gview();
#if IBFT_WC > 0
  G.host_pos = emul_pos_entry;
#endif
  uint32_t rtab[IBFT_RTAB_WORDS];
  rtab_view T{rtab, 1};
  auto member = [&](uint32_t, const uint8_t* signer) {
    if (table == nullptr) return true;
    for (uint32_t i = 0; i < table_n; i++)
      if (memcmp(table + 20 * (size_t)i, signer, 20) == 0) return true;
    return false;
  };
  return explain_item(exec_serial{}, *it, arena, arena_len, grouped != 0, n_groups, G, T, member, recovered20);
}
}
