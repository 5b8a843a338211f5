// Host emulation of the device arithmetic (TEST ONLY).
//
// Compiles the very same csrc/*.cuh headers with g++ (their portable C++ path) so that the complete
// per-signature pipeline -- GLV split, Booth digits, group law with exceptional cases, Keccak, address derivation --
// can be checked against the oracle on a CPU-only box.  This library is never loaded by the product; the product
// path (csrc/engine.cu) fails loudly without a CUDA device.  The PTX carry-chain multipliers are exercised on the
// GPU by tests/test_gpu_primitives.py through ibft_debug_op.
#include <atomic>
#include <cstring>

// exceptional branches of the group law taken since the last emul_branch_reset (IBFT_BR_* of secp_fe.cuh); entries
// [IBFT_BR_COUNT, 2 IBFT_BR_COUNT) count the same branches taken inside the split pipelines' final "+ u1 G" only
static std::atomic<unsigned long long> g_branch[16];
#define IBFT_BRANCH(i) g_branch[i].fetch_add(1, std::memory_order_relaxed)

#include "../../go-ibft_b200/csrc/verify_core.cuh"
#include "../../go-ibft_b200/csrc/debug_arith.cuh"
#include "../../go-ibft_b200/csrc/secp_gtable.inc"

#include <cstdio>
#include <array>
#include <map>
#include <mutex>
#include <thread>
#include <vector>

using namespace ibft;

// Combined generator table for the emulation: built once with the portable code (all host threads) and cached next to this
// file (tests/emul/ctable_wc<W>.bin, git-ignored).  The GPU builds its own copy in k_build_ctable.
#if IBFT_WC > 0
static const uint32_t* emul_ctable() {
  static std::vector<uint32_t> tab;
  if (!tab.empty()) return tab.data();
  const size_t entries = (size_t)IBFT_CTAB_ENTRIES;
  tab.assign(entries * 16, 0);
  char path[512];
  snprintf(path, sizeof path, "%s/ctable_wc%d.bin", EMUL_DIR, IBFT_WC);
  if (FILE* f = fopen(path, "rb")) {
    size_t got = fread(tab.data(), 4, tab.size(), f);
    fclose(f);
    if (got == tab.size()) return tab.data();
  }
  const uint32_t lam[8] = {0x1B23BD72u, 0xDF02967Cu, 0x20816678u, 0x122E22EAu, 0x8812645Au, 0xA5261C02u, 0xC05C30E0u, 0x5363AD4Cu};
  unsigned nt = std::max(1u, std::thread::hardware_concurrency());
  std::vector<std::thread> th;
  for (unsigned t = 0; t < nt; t++)
    th.emplace_back([&, t]() {
      gtab_view G{IBFT_GTABLE};
      uint32_t rtab[IBFT_RTAB_WORDS];
      rtab_view T{rtab, 1};
      for (size_t e = t; e < entries; e += nt) {
        int d1 = (int)(e / IBFT_CTAB_D2), d2 = (int)(e % IBFT_CTAB_D2) - (1 << (IBFT_WC - 1));
        sc a, b, l, zero;
        for (int i = 0; i < 8; i++) { a.v[i] = 0; b.v[i] = 0; zero.v[i] = 0; l.v[i] = lam[i]; }
        a.v[0] = (uint32_t)d1;
        b.v[0] = (uint32_t)(d2 < 0 ? -d2 : d2);
        sc tt = sc_mul(b, l);
        if (d2 < 0) tt = sc_neg(tt);
        sc k = sc_add(a, tt);
        aff g1;
        G.load(0, g1.x, g1.y);
        jac P = ecmult_double(k, zero, g1, G, T);
        if (P.inf || fe_is_zero(P.z)) continue;
        fe zi = IBFT_FE_INV(P.z), zi2 = fe_sqr(zi);
        fe x = fe_normalize(fe_mul(P.x, zi2)), y = fe_normalize(fe_mul(P.y, fe_mul(zi2, zi)));
        for (int i = 0; i < 8; i++) { tab[16 * e + i] = x.v[i]; tab[16 * e + 8 + i] = y.v[i]; }
      }
    });
  for (auto& x : th) x.join();
  if (FILE* f = fopen(path, "wb")) { fwrite(tab.data(), 4, tab.size(), f); fclose(f); }
  return tab.data();
}
static gtab_view emul_gview() {
  gtab_view G{IBFT_GTABLE};
  G.comb = emul_ctable();
  return G;
}
#else
static gtab_view emul_gview() { return gtab_view{IBFT_GTABLE}; }
#endif

// runs f and adds the branches it took to the final-add counters (single-threaded callers only: the tests)
template <class F>
static bool count_final_add(F f) {
  unsigned long long before[IBFT_BR_COUNT];
  for (int i = 0; i < IBFT_BR_COUNT; i++) before[i] = g_branch[i].load();
  bool r = f();
  for (int i = 0; i < IBFT_BR_COUNT; i++) g_branch[IBFT_BR_COUNT + i] += g_branch[i].load() - before[i];
  return r;
}

extern "C" {

int emul_verify_item(const ibft_sig_item* it, const uint8_t* arena, size_t arena_len, uint8_t* recovered20) {
  uint8_t addr[20];
  memset(recovered20, 0, 20);
  resolved_item ri;
  bool valid = false;
  int st = resolve_item(*it, arena, arena_len, ri, &valid);
  if (st != IBFT_ITEM_OK) return -1;  // NEEDS_HOST
  if (!valid) return 0;
  gtab_view G = emul_gview();
  uint32_t rtab[IBFT_RTAB_WORDS];
  rtab_view T{rtab, 1};
  if (!ecrecover_address(ri.r, ri.s, ri.v, ri.z, G, T, addr)) return 0;
  memcpy(recovered20, addr, 20);
  return memcmp(addr, ri.signer, 20) == 0;
}

// the same item through the LEVEL-structured group law of the four-lane kernel (products of a level computed one by one)
int emul_verify_item_levels(const ibft_sig_item* it, const uint8_t* arena, size_t arena_len, uint8_t* recovered20) {
  uint8_t addr[20];
  memset(recovered20, 0, 20);
  resolved_item ri;
  bool valid = false;
  int st = resolve_item(*it, arena, arena_len, ri, &valid);
  if (st != IBFT_ITEM_OK) return -1;
  if (!valid) return 0;
  gtab_view G = emul_gview();
  uint32_t rtab[IBFT_QTAB_WORDS];
  rtab_view T{rtab, 1};
  if (!ecrecover_address_x(exec_levels{}, ri.r, ri.s, ri.v, ri.z, G, T, addr)) return 0;
  memcpy(recovered20, addr, 20);
  return memcmp(addr, ri.signer, 20) == 0;
}

// out(64) = a*G + b*P through the level-structured XYZZ routine of the latency path; returns 1 for infinity
int emul_ecmult_levels(const uint8_t* a, const uint8_t* b, const uint8_t* c, uint8_t* out) {
  gtab_view G = emul_gview();
  aff P;
  P.x = fe_from_be(c);
  P.y = fe_from_be(c + 32);
  uint32_t rtab[IBFT_QTAB_WORDS];
  rtab_view T{rtab, 1};
  fe qx, qy;
  memset(out, 0, 64);
  if (!ecmult_affine(exec_levels{}, sc_reduce_once(sc_from_be(a)), sc_reduce_once(sc_from_be(b)), P, G, T, qx, qy)) return 1;
  fe_to_be(qx, out);
  fe_to_be(qy, out + 32);
  return 0;
}

#if IBFT_WC > 0
// per-position comb entries computed on demand (the device holds a 36 MB table): (d1 + d2 lambda) 2^(WC pos) G
static void emul_pos_entry(int pos, int d1, int d2, uint32_t* xy16) {
  static std::mutex mu;
  static std::map<uint64_t, std::array<uint32_t, 16>> cache;
  uint64_t key = ((uint64_t)pos << 40) | ((uint64_t)d1 << 20) | (uint64_t)(d2 + 4096);
  {
    std::lock_guard<std::mutex> g(mu);
    auto it = cache.find(key);
    if (it != cache.end()) { memcpy(xy16, it->second.data(), 64); return; }
  }
  const uint32_t lam[8] = {0x1B23BD72u, 0xDF02967Cu, 0x20816678u, 0x122E22EAu, 0x8812645Au, 0xA5261C02u, 0xC05C30E0u, 0x5363AD4Cu};
  sc a, b, l, m, zero;
  for (int i = 0; i < 8; i++) { a.v[i] = 0; b.v[i] = 0; l.v[i] = lam[i]; m.v[i] = 0; zero.v[i] = 0; }
  a.v[0] = (uint32_t)d1;
  b.v[0] = (uint32_t)(d2 < 0 ? -d2 : d2);
  m.v[(pos * IBFT_WC) / 32] = 1u << ((pos * IBFT_WC) % 32);
  sc t = sc_mul(b, l);
  if (d2 < 0) t = sc_neg(t);
  sc k = sc_mul(sc_add(a, t), m);
  gtab_view G = emul_gview();
  uint32_t rtab[IBFT_RTAB_WORDS];
  rtab_view T{rtab, 1};
  aff g1;
  G.load(0, g1.x, g1.y);
  jac P = ecmult_double(k, zero, g1, G, T);
  std::array<uint32_t, 16> e{};
  if (!(P.inf || fe_is_zero(P.z))) {
    fe zi = IBFT_FE_INV(P.z), zi2 = fe_sqr(zi);
    fe x = fe_normalize(fe_mul(P.x, zi2)), y = fe_normalize(fe_mul(P.y, fe_mul(zi2, zi)));
    for (int i = 0; i < 8; i++) { e[i] = x.v[i]; e[8 + i] = y.v[i]; }
  }
  memcpy(xy16, e.data(), 64);
  std::lock_guard<std::mutex> g(mu);
  cache[key] = e;
}

// the same item through the SPLIT pipeline of k_recover_split (helper / chain phases run one after the other)
int emul_verify_item_split(const ibft_sig_item* it, const uint8_t* arena, size_t arena_len, uint8_t* recovered20) {
  uint8_t addr[20];
  memset(recovered20, 0, 20);
  resolved_item ri;
  bool valid = false;
  int st = resolve_item(*it, arena, arena_len, ri, &valid);
  if (st != IBFT_ITEM_OK) return -1;
  if (!valid) return 0;
  gtab_view G = emul_gview();
  G.host_pos = emul_pos_entry;
  uint32_t rtab[IBFT_RTAB_WORDS];
  rtab_view T{rtab, 1};
  ecmult_digits dg;
  if (!split_helper_scalars(ri, dg)) return 0;             // helper phase 1
  aff Rp = split_chain_point(ri.r);                        // chain: inversion-free table + R streams on E' / E''
  fe gz = ecmult_build_rtable_globalz(Rp, T);
  jac acc = ecmult_streams(dg, G, T, false);
  fe y, gx, gy;
  bool g_inf = false;
  if (!split_helper_point(ri, dg, G, y, g_inf, gx, gy)) return 0;  // helper phase 2
  if (!count_final_add([&] { return split_chain_finish(acc, fe_mul(y, gz), g_inf, gx, gy, addr); })) return 0;  // chain: map back, + u1 G, address
  memcpy(recovered20, addr, 20);
  return memcmp(addr, ri.signer, 20) == 0;
}

// split pipeline with the level-structured (four-lane) chain
int emul_verify_item_qsplit(const ibft_sig_item* it, const uint8_t* arena, size_t arena_len, uint8_t* recovered20) {
  uint8_t addr[20];
  memset(recovered20, 0, 20);
  resolved_item ri;
  bool valid = false;
  int st = resolve_item(*it, arena, arena_len, ri, &valid);
  if (st != IBFT_ITEM_OK) return -1;
  if (!valid) return 0;
  gtab_view G = emul_gview();
  G.host_pos = emul_pos_entry;
  uint32_t qtab[IBFT_QTAB_WORDS];
  qtab_view T{qtab, 1};
  exec_levels ex;
  ecmult_digits dg;
  if (!split_helper_scalars(ri, dg)) return 0;
  fe c;
  aff Rp = split_chain_point(ri.r, &c);
  ecmult_build_qtable(ex, Rp, T);
  xyzz acc = ecmult_streams_x(ex, dg, G, T, false);
  fe y, gx, gy;
  bool g_inf = false;
  if (!split_helper_point(ri, dg, G, y, g_inf, gx, gy)) return 0;
  if (!count_final_add([&] { return split_chain_finish_x(ex, acc, c, y, g_inf, gx, gy, addr); })) return 0;
  memcpy(recovered20, addr, 20);
  return memcmp(addr, ri.signer, 20) == 0;
}

// verification against a known public key: key64 = X || Y big-endian; the table is built here for every call (test only).
// Returns the verdict of ecdsa_verify_known; *recovers_key = 1 when the recover path yields exactly that key.
int emul_verify_item_known(const ibft_sig_item* it, const uint8_t* arena, size_t arena_len, const uint8_t* key64, int* recovers_key) {
  resolved_item ri;
  bool valid = false;
  *recovers_key = 0;
  int st = resolve_item(*it, arena, arena_len, ri, &valid);
  if (st != IBFT_ITEM_OK) return -1;
  if (!valid) return 0;
  gtab_view G = emul_gview();
  aff Q;
  Q.x = fe_from_be(key64);
  Q.y = fe_from_be(key64 + 32);
  std::vector<uint32_t> kt(IBFT_KEYTAB_WORDS);  // the validator's comb: 17 positions x 128 entries
  build_keytab(Q, kt.data());
  G.host_pos = emul_pos_entry;  // the generator's per-position comb entries are computed on demand here
  gtab_view Qt{kt.data()};
  uint32_t rtab[IBFT_RTAB_WORDS];
  rtab_view T{rtab, 1};
  uint8_t addr[20];
  aff K;
  if (ecrecover_address(ri.r, ri.s, ri.v, ri.z, G, T, addr, &K)) {
    fe qx = fe_normalize(Q.x), qy = fe_normalize(Q.y);
    bool same = true;
    for (int i = 0; i < 8; i++) same = same && K.x.v[i] == qx.v[i] && K.y.v[i] == qy.v[i];
    *recovers_key = same ? 1 : 0;
  }
  int whole = ecdsa_verify_known(ri, G, Qt) ? 1 : 0;
  // the chain / helper cut of k_verify_split must give the same answer
  int cut = 0;
  if (split_sig_in_range(ri)) {
    G.host_pos = emul_pos_entry;
    sc w = IBFT_SC_INV(sc_from_be(ri.s));
    ecmult_digits dg;
    for (int k = 0; k < 6; k++) dg.ks[2][k] = dg.ks[3][k] = 0;
    dg.kneg[2] = dg.kneg[3] = false;
    known_helper_u2(ri, w, dg);
    jac acc = ecmult_streams_known(dg, G, Qt, false);
    bool g_inf = false;
    fe gx, gy;
    known_helper_u1g(ri, w, G, g_inf, gx, gy);
    cut = count_final_add([&] { return known_chain_finish(acc, g_inf, gx, gy, ri); }) ? 1 : 0;
  }
  if (cut != whole) return -2;
  return whole;
}
#endif

#if IBFT_WC > 0
// one comb position of a validator's key table (build_keytab_pos, the routine k_build_keytabs runs per (validator, position)):
// out = 128 entries x (X || Y big-endian), entry m-1 = m * 2^(8 pos) * Q
void emul_keytab_pos(const uint8_t* key64, int pos, uint8_t* out /* 128 * 64 bytes */) {
  aff Q;
  Q.x = fe_from_be(key64);
  Q.y = fe_from_be(key64 + 32);
  std::vector<uint32_t> kt((size_t)IBFT_KEYTAB_ENTRIES * 16);
  build_keytab_pos(Q, pos, kt.data());
  for (int m = 0; m < IBFT_KEYTAB_ENTRIES; m++) {
    fe x, y;
    for (int i = 0; i < 8; i++) { x.v[i] = kt[16 * m + i]; y.v[i] = kt[16 * m + 8 + i]; }
    fe_to_be(x, out + 64 * m);
    fe_to_be(y, out + 64 * m + 32);
  }
}
int emul_keytab_positions() { return IBFT_KEYTAB_POSITIONS; }

#endif
void emul_keccak256(const uint8_t* d, uint32_t n, uint8_t* out) { keccak256_bytes(d, n, out); }

// branch counters: out[i] = times branch IBFT_BR_i was taken since the last reset; returns IBFT_BR_COUNT
// out[IBFT_BR_COUNT + i] = those of them taken in a split pipeline's final add (emul_verify_item_split / _qsplit)
int emul_branch_counts(unsigned long long* out /* 2 * IBFT_BR_COUNT */) {
  for (int i = 0; i < 2 * IBFT_BR_COUNT; i++) out[i] = g_branch[i].load();
  return IBFT_BR_COUNT;
}
void emul_branch_reset() {
  for (auto& c : g_branch) c.store(0);
}

// op codes = IBFT_DBG_* of include/ibft_verify.h
int emul_debug_op(int op, const uint8_t* a, const uint8_t* b, const uint8_t* c, uint8_t* out) {
  switch (op) {
    case IBFT_DBG_FE_MUL: fe_to_be(fe_normalize(fe_mul(fe_from_be(a), fe_from_be(b))), out); return 0;
    case IBFT_DBG_FE_SQR: fe_to_be(fe_normalize(fe_sqr(fe_from_be(a))), out); return 0;
    case IBFT_DBG_FE_INV: fe_to_be(fe_normalize(IBFT_FE_INV(fe_from_be(a))), out); return 0;
    case IBFT_DBG_FE_SQRT: fe_to_be(fe_normalize(fe_sqrt_candidate(fe_from_be(a))), out); return 0;
    case IBFT_DBG_FE_ADD: fe_to_be(fe_normalize(fe_add(fe_from_be(a), fe_from_be(b))), out); return 0;
    case IBFT_DBG_FE_SUB: fe_to_be(fe_normalize(fe_sub(fe_from_be(a), fe_from_be(b))), out); return 0;
    case IBFT_DBG_SC_MUL: sc_to_be(sc_mul(sc_from_be(a), sc_from_be(b)), out); return 0;
    case IBFT_DBG_SC_INV: sc_to_be(IBFT_SC_INV(sc_reduce_once(sc_from_be(a))), out); return 0;
    case IBFT_DBG_GLV: {
      glv_half h1, h2;
      glv_split(sc_reduce_once(sc_from_be(a)), h1, h2);
      memset(out, 0, 64);
      for (int i = 0; i < 5; i++)
        for (int j = 0; j < 4; j++) {
          out[4 * i + j] = (uint8_t)(h1.k[i] >> (8 * j));       // little-endian magnitude, 20 bytes
          out[24 + 4 * i + j] = (uint8_t)(h2.k[i] >> (8 * j));
        }
      out[20] = h1.neg;
      out[44] = h2.neg;
      return 0;
    }
    case IBFT_DBG_ECMULT: {  // out = a*G + b*P, P = (c[0..31], c[32..63]) affine on the curve; all-zero out = infinity
      gtab_view G = emul_gview();
      aff P;
      P.x = fe_from_be(c);
      P.y = fe_from_be(c + 32);
      uint32_t rtab[IBFT_RTAB_WORDS];
      rtab_view T{rtab, 1};
      jac Q = ecmult_double(sc_reduce_once(sc_from_be(a)), sc_reduce_once(sc_from_be(b)), P, G, T);
      memset(out, 0, 64);
      if (Q.inf || fe_is_zero(Q.z)) return 1;
      fe zi = IBFT_FE_INV(Q.z), zi2 = fe_sqr(zi);
      fe_to_be(fe_normalize(fe_mul(Q.x, zi2)), out);
      fe_to_be(fe_normalize(fe_mul(Q.y, fe_mul(zi2, zi))), out + 32);
      return 0;
    }
    default: return debug_arith_op(op, a, b, out) ? 0 : -1;
  }
}
}

extern "C" int emul_sign(const uint8_t* d, const uint8_t* z, const uint8_t* k, uint8_t* sig65) {
  gtab_view G = emul_gview();
  uint32_t rtab[IBFT_RTAB_WORDS];
  rtab_view T{rtab, 1};
  return ecdsa_sign(d, z, k, G, T, sig65) ? 1 : 0;
}
