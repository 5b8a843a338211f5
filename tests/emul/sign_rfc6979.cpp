// The host emulation with the RFC 6979 signer's entry points (TEST ONLY).
//
// SHA-256, the DRBG's nonce candidates and ecdsa_sign_rfc6979 of the very csrc headers (sha256.cuh, verify_core.cuh), and the
// IBFT_DBG_RFC6979 body of debug_arith.cuh.  Built on demand by tests/test_emul_sign_rfc6979.py:
//   g++ -O2 -fPIC -std=c++17 -DEMUL_DIR=\"<tests/emul>\" -shared -o libibft_sign_rfc6979.so sign_rfc6979.cpp -lpthread
#include "emul.cpp"

// SHA-256 of n bytes through the device's compression function; the general padding lives here, the device only ever hashes
// the fixed lengths of sha256.cuh
extern "C" void emul_sha256(const uint8_t* m, uint32_t n, uint8_t* out32) {
  std::vector<uint8_t> buf(m, m + n);
  buf.push_back(0x80);
  while (buf.size() % 64 != 56) buf.push_back(0);
  const uint64_t bits = (uint64_t)n * 8;
  for (int i = 7; i >= 0; i--) buf.push_back((uint8_t)(bits >> (8 * i)));
  sha256_st st = sha256_iv();
  for (size_t off = 0; off < buf.size(); off += 64) {
    sha256_blk b;
    sha256_words_from_be(buf.data() + off, b.w, 16);
    st = sha256_compress(st, b);
  }
  sha256_words_to_be(st.h, out32, 8);
}

// raw nonce candidate c of ibft_sign_batch_rfc6979 for a key and a digest
extern "C" void emul_rfc6979_candidate(const uint8_t* key32, const uint8_t* digest32, uint32_t c, uint8_t* out32) {
  uint8_t zm[32];
  sc_to_be(sc_reduce_once(sc_from_be(digest32)), zm);
  rfc6979_candidate(key32, zm, c, out32);
}

// IBFT_DBG_RFC6979 through the body k_debug_op runs: a = key, b = digest, c = 64 bytes with the candidate in the last byte
extern "C" int emul_debug_rfc6979(const uint8_t* a, const uint8_t* b, const uint8_t* c, uint8_t* out32) {
  return debug_arith_op(IBFT_DBG_RFC6979, a, b, out32, c) ? 0 : -1;
}

// one row of ibft_sign_batch_rfc6979; returns 1 when signed, 0 when refused (sig65 all zero)
extern "C" int emul_sign_rfc6979(const uint8_t* d, const uint8_t* z, uint8_t* sig65) {
  gtab_view G = emul_gview();
  uint32_t rtab[IBFT_RTAB_WORDS];
  rtab_view T{rtab, 1};
  return ecdsa_sign_rfc6979(d, z, G, T, sig65) ? 1 : 0;
}
