// The host emulation of the one-thread recovery with u1*G from the WIDE generator comb (TEST / TOOL ONLY).
//
// recover_key for exec_serial (verify_core.cuh) adds u1*G by the wide comb (ecmult_gen_wide) whenever the engine holds the
// table; this library runs that composition on the host, its entries m * 2^(w pos) * G computed on demand (the device holds
// a 1.38 GiB table), with the operation and branch counters of recover_comb.cpp.  Built on demand by
// tests/test_emul_wide_comb.py and tools/fma_budget.py:
//   g++ -O2 -fPIC -std=c++17 -DEMUL_DIR=\"<tests/emul>\" -shared -o libibft_recover_wide.so recover_wide.cpp -lpthread
#include "recover_comb.cpp"

static_assert(IBFT_GEN_WIDE > 0, "the emulation needs the wide comb");

// m * 2^(w pos) * G, affine, computed without touching the counters: the device reads it from its table
static void wide_entry_uncounted(int pos, int m, uint32_t* xy16) {
  unsigned long long ops[32], br[16];
  for (int i = 0; i < 32; i++) ops[i] = g_ops[i].load();
  for (int i = 0; i < 16; i++) br[i] = g_branch[i].load();
  sc a, t, zero;
  for (int i = 0; i < 8; i++) { a.v[i] = 0; t.v[i] = 0; zero.v[i] = 0; }
  a.v[0] = (uint32_t)m;
  t.v[(pos * IBFT_GEN_WIDE) / 32] = 1u << ((pos * IBFT_GEN_WIDE) % 32);
  gtab_view G = emul_gview();
  uint32_t rtab[IBFT_RTAB_WORDS];
  rtab_view T{rtab, 1};
  aff g1;
  G.load(0, g1.x, g1.y);
  jac P = ecmult_double(sc_mul(a, t), zero, g1, G, T);
  for (int i = 0; i < 16; i++) xy16[i] = 0;
  if (!(P.inf || fe_is_zero(P.z))) {
    fe zi = IBFT_FE_INV(P.z), zi2 = fe_sqr(zi);
    fe x = fe_normalize(fe_mul(P.x, zi2)), y = fe_normalize(fe_mul(P.y, fe_mul(zi2, zi)));
    for (int i = 0; i < 8; i++) { xy16[i] = x.v[i]; xy16[8 + i] = y.v[i]; }
  }
  for (int i = 0; i < 32; i++) g_ops[i].store(ops[i]);
  for (int i = 0; i < 16; i++) g_branch[i].store(br[i]);
}

// the same, counting the reads: one per non-zero digit of u1 per recovery
static std::atomic<unsigned long long> g_wide_reads{0};
static void wide_entry_counted(int pos, int m, uint32_t* xy16) {
  g_wide_reads.fetch_add(1, std::memory_order_relaxed);
  wide_entry_uncounted(pos, m, xy16);
}

extern "C" {

// emul_verify_item through the product's one-thread composition with the wide comb (single-threaded callers only)
int emul_verify_item_wide(const ibft_sig_item* it, const uint8_t* arena, size_t arena_len, uint8_t* recovered20) {
  uint8_t addr[20];
  memset(recovered20, 0, 20);
  resolved_item ri;
  bool valid = false;
  int st = resolve_item(*it, arena, arena_len, ri, &valid);
  if (st != IBFT_ITEM_OK) return -1;
  if (!valid) return 0;
  gtab_view G = emul_gview();
  G.host_wide = wide_entry_counted;
  uint32_t rtab[IBFT_RTAB_WORDS];
  rtab_view T{rtab, 1};
  if (!ecrecover_address(ri.r, ri.s, ri.v, ri.z, G, T, addr)) return 0;
  memcpy(recovered20, addr, 20);
  return memcmp(addr, ri.signer, 20) == 0;
}

// entry m of position pos as 64 bytes (x, y as 8 little-endian words each; the device table's format)
void emul_wide_entry(int pos, int m, uint32_t* xy16) { wide_entry_uncounted(pos, m, xy16); }

// the window and the layout: out = {w, positions, entries per position, entries of the top position}
void emul_wide_shape(uint32_t* out4) {
  out4[0] = IBFT_GEN_WIDE;
  out4[1] = IBFT_GW_POSITIONS;
  out4[2] = IBFT_GW_ENTRIES;
  out4[3] = IBFT_GW_TOP_ENTRIES;
}

// the Booth digits ecmult_gen_wide reads from u1 (8 little-endian words): out[j], j = 0 .. positions - 1
void emul_wide_digits(const uint32_t* u1, int32_t* out) {
  sc k;
  for (int i = 0; i < 8; i++) k.v[i] = u1[i];
  ecmult_digits dg;
  ecmult_wide_into(k, dg);
  for (int j = 0; j < IBFT_GW_POSITIONS; j++) out[j] = booth_digit<IBFT_GEN_WIDE, 12>(dg.flat + 12, j);
}

// wide-comb entries read since the last call (one per non-zero digit of u1 per recovery)
unsigned long long emul_wide_reads(void) { return g_wide_reads.exchange(0); }

}  // extern "C"
