// The host emulation with the u1*G comb entries supplied (TEST / TOOL ONLY).
//
// The one-thread recovery of the product (verify_core.cuh, recover_key for exec_serial) adds u1*G by a comb over per-position
// tables; the plain emulation (emul.cpp) supplies no per-position entries, so its emul_verify_item runs the table-inversion
// composition.  This library runs the product's composition on the host, with the operation counters of opcount.cpp and the
// branch counters of its final addition (IBFT_BR_REC_*).  Built on demand by tests/test_emul_recover_comb.py and
// tools/fma_budget.py:
//   g++ -O2 -fPIC -std=c++17 -DEMUL_DIR=\"<tests/emul>\" -shared -o libibft_recover_comb.so recover_comb.cpp -lpthread
#include "opcount.cpp"

// comb entries computed on demand (emul_pos_entry) without touching the counters: the device reads them from its tables
static void pos_entry_uncounted(int pos, int d1, int d2, uint32_t* xy16) {
  unsigned long long ops[32], br[16];
  for (int i = 0; i < 32; i++) ops[i] = g_ops[i].load();
  for (int i = 0; i < 16; i++) br[i] = g_branch[i].load();
  emul_pos_entry(pos, d1, d2, xy16);
  for (int i = 0; i < 32; i++) g_ops[i].store(ops[i]);
  for (int i = 0; i < 16; i++) g_branch[i].store(br[i]);
}

extern "C" {

// emul_verify_item through the product's one-thread composition (single-threaded callers only: the counters are restored
// around every comb entry)
int emul_verify_item_comb(const ibft_sig_item* it, const uint8_t* arena, size_t arena_len, uint8_t* recovered20) {
  uint8_t addr[20];
  memset(recovered20, 0, 20);
  resolved_item ri;
  bool valid = false;
  int st = resolve_item(*it, arena, arena_len, ri, &valid);
  if (st != IBFT_ITEM_OK) return -1;
  if (!valid) return 0;
  gtab_view G = emul_gview();
  G.host_pos = pos_entry_uncounted;
  uint32_t rtab[IBFT_RTAB_WORDS];
  rtab_view T{rtab, 1};
  if (!ecrecover_address(ri.r, ri.s, ri.v, ri.z, G, T, addr)) return 0;
  memcpy(recovered20, addr, 20);
  return memcmp(addr, ri.signer, 20) == 0;
}

// out[i] = times IBFT_BR_REC_DBL + i was taken since emul_branch_reset (A = B, A = -B, u1 = 0, non-residue); returns 4
int emul_rec_branch_counts(unsigned long long* out /* 4 */) {
  for (int i = 0; i < 4; i++) out[i] = g_branch[IBFT_BR_REC_DBL + i].load();
  return 4;
}

// out[k] = IBFT_OP_k since emul_op_reset, the comb and final-step counters included; returns IBFT_OP_COUNT_ALL
int emul_op_counts_all(unsigned long long* out /* IBFT_OP_COUNT_ALL */) {
  for (int i = 0; i < IBFT_OP_COUNT_ALL; i++) out[i] = g_ops[i].load();
  return IBFT_OP_COUNT_ALL;
}

}  // extern "C"
