// sha256.cuh -- SHA-256 (FIPS 180-4), HMAC-SHA256 keyed by 32 bytes (RFC 2104) and the HMAC-SHA256 DRBG of RFC 6979 §3.2
// that derives libsecp256k1's default ECDSA nonce (nonce_function_rfc6979, the nonce go-ethereum's crypto.Sign signs with).
//
// Every HMAC the DRBG computes has one of three fixed message lengths after the 64-byte pad block -- V (32 bytes),
// V || 0x00 (33) and V || sep || key || msg (97) -- so each length has its own block layout with the padding written in,
// and there is no general streaming hasher.  Values are kept as big-endian 32-bit words, the order SHA-256 reads them in.
// The compression is a real device function taking and returning its operands by value (registers, no stack): one body
// serves the ~20 compressions of a nonce instead of ~20 inlined copies of 64 rounds.
#pragma once
#include <stdint.h>

#include "secp_fe.cuh"

namespace ibft {

struct sha256_st { uint32_t h[8]; };
struct sha256_blk { uint32_t w[16]; };

IBFT_HD uint32_t sha256_rotr(uint32_t x, int n) { return (x >> n) | (x << (32 - n)); }

IBFT_HD uint32_t sha256_k(int i) {
  const uint32_t k[64] = {
      0x428a2f98u, 0x71374491u, 0xb5c0fbcfu, 0xe9b5dba5u, 0x3956c25bu, 0x59f111f1u, 0x923f82a4u, 0xab1c5ed5u,
      0xd807aa98u, 0x12835b01u, 0x243185beu, 0x550c7dc3u, 0x72be5d74u, 0x80deb1feu, 0x9bdc06a7u, 0xc19bf174u,
      0xe49b69c1u, 0xefbe4786u, 0x0fc19dc6u, 0x240ca1ccu, 0x2de92c6fu, 0x4a7484aau, 0x5cb0a9dcu, 0x76f988dau,
      0x983e5152u, 0xa831c66du, 0xb00327c8u, 0xbf597fc7u, 0xc6e00bf3u, 0xd5a79147u, 0x06ca6351u, 0x14292967u,
      0x27b70a85u, 0x2e1b2138u, 0x4d2c6dfcu, 0x53380d13u, 0x650a7354u, 0x766a0abbu, 0x81c2c92eu, 0x92722c85u,
      0xa2bfe8a1u, 0xa81a664bu, 0xc24b8b70u, 0xc76c51a3u, 0xd192e819u, 0xd6990624u, 0xf40e3585u, 0x106aa070u,
      0x19a4c116u, 0x1e376c08u, 0x2748774cu, 0x34b0bcb5u, 0x391c0cb3u, 0x4ed8aa4au, 0x5b9cca4fu, 0x682e6ff3u,
      0x748f82eeu, 0x78a5636fu, 0x84c87814u, 0x8cc70208u, 0x90befffau, 0xa4506cebu, 0xbef9a3f7u, 0xc67178f2u};
  return k[i];
}

IBFT_HD sha256_st sha256_iv() {
  return sha256_st{{0x6a09e667u, 0xbb67ae85u, 0x3c6ef372u, 0xa54ff53au, 0x510e527fu, 0x9b05688cu, 0x1f83d9abu, 0x5be0cd19u}};
}

// one compression: the state after hashing block b from state s
IBFT_FN sha256_st sha256_compress(sha256_st s, sha256_blk b) {
  uint32_t a = s.h[0], bb = s.h[1], c = s.h[2], d = s.h[3], e = s.h[4], f = s.h[5], g = s.h[6], h = s.h[7];
#pragma unroll
  for (int i = 0; i < 64; i++) {
    if (i >= 16) {  // message schedule in place: w[i mod 16] becomes W_i
      const uint32_t w15 = b.w[(i + 1) & 15], w2 = b.w[(i + 14) & 15];
      b.w[i & 15] += (sha256_rotr(w15, 7) ^ sha256_rotr(w15, 18) ^ (w15 >> 3)) + b.w[(i + 9) & 15] +
                     (sha256_rotr(w2, 17) ^ sha256_rotr(w2, 19) ^ (w2 >> 10));
    }
    const uint32_t t1 = h + (sha256_rotr(e, 6) ^ sha256_rotr(e, 11) ^ sha256_rotr(e, 25)) + ((e & f) ^ (~e & g)) + sha256_k(i) +
                        b.w[i & 15];
    const uint32_t t2 = (sha256_rotr(a, 2) ^ sha256_rotr(a, 13) ^ sha256_rotr(a, 22)) + ((a & bb) ^ (a & c) ^ (bb & c));
    h = g; g = f; f = e; e = d + t1;
    d = c; c = bb; bb = a; a = t1 + t2;
  }
  s.h[0] += a; s.h[1] += bb; s.h[2] += c; s.h[3] += d;
  s.h[4] += e; s.h[5] += f; s.h[6] += g; s.h[7] += h;
  return s;
}

IBFT_HD void sha256_words_from_be(const uint8_t* p, uint32_t* w, int n) {
#pragma unroll
  for (int i = 0; i < n; i++)
    w[i] = ((uint32_t)p[4 * i] << 24) | ((uint32_t)p[4 * i + 1] << 16) | ((uint32_t)p[4 * i + 2] << 8) | (uint32_t)p[4 * i + 3];
}

IBFT_HD void sha256_words_to_be(const uint32_t* w, uint8_t* p, int n) {
#pragma unroll
  for (int i = 0; i < n; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) p[4 * i + j] = (uint8_t)(w[i] >> (24 - 8 * j));
}

// The last block of a message whose final piece is the 32 bytes v, followed by word w8 (the 0x80 pad byte, with at most one
// message byte before it) and the length of the whole message in bits.
IBFT_HD sha256_blk sha256_blk_tail32(const uint32_t* v, uint32_t w8, uint32_t bits) {
  sha256_blk b;
#pragma unroll
  for (int i = 0; i < 8; i++) b.w[i] = v[i];
  b.w[8] = w8;
#pragma unroll
  for (int i = 9; i < 15; i++) b.w[i] = 0;
  b.w[15] = bits;
  return b;
}

// HMAC-SHA256 under one 32-byte key: the states after its inner (key ^ 0x36..) and outer (key ^ 0x5c..) pad blocks are
// computed once when the key is set; a tag then costs the message's blocks plus one outer block.
struct hmac_sha256 {
  sha256_st in, out;

  IBFT_HD void set_key(const uint32_t* key) {
    sha256_blk bi, bo;
#pragma unroll
    for (int i = 0; i < 16; i++) {
      const uint32_t k = i < 8 ? key[i] : 0u;
      bi.w[i] = k ^ 0x36363636u;
      bo.w[i] = k ^ 0x5c5c5c5cu;
    }
    in = sha256_compress(sha256_iv(), bi);
    out = sha256_compress(sha256_iv(), bo);
  }
  // outer hash over the inner digest (32 bytes after the 64-byte pad block: 768 bits)
  IBFT_HD void finish(const sha256_st& inner, uint32_t* tag) const {
    const sha256_st o = sha256_compress(out, sha256_blk_tail32(inner.h, 0x80000000u, 768u));
#pragma unroll
    for (int i = 0; i < 8; i++) tag[i] = o.h[i];
  }
  // tag = HMAC(key, v), 32-byte message
  IBFT_HD void mac32(const uint32_t* v, uint32_t* tag) const {
    finish(sha256_compress(in, sha256_blk_tail32(v, 0x80000000u, (64u + 32u) * 8u)), tag);
  }
  // tag = HMAC(key, v || sep), 33-byte message
  IBFT_HD void mac33(const uint32_t* v, uint32_t sep, uint32_t* tag) const {
    finish(sha256_compress(in, sha256_blk_tail32(v, (sep << 24) | 0x00800000u, (64u + 33u) * 8u)), tag);
  }
  // tag = HMAC(key, v || sep || x || m), 97-byte message: x || m (16 words) lands one byte late in the blocks
  IBFT_HD void mac97(const uint32_t* v, uint32_t sep, const uint32_t* x, const uint32_t* m, uint32_t* tag) const {
    uint32_t s[16];
#pragma unroll
    for (int i = 0; i < 8; i++) { s[i] = x[i]; s[8 + i] = m[i]; }
    sha256_blk b1, b2;
#pragma unroll
    for (int i = 0; i < 8; i++) b1.w[i] = v[i];
    b1.w[8] = (sep << 24) | (s[0] >> 8);
#pragma unroll
    for (int i = 1; i < 8; i++) b1.w[8 + i] = (s[i - 1] << 24) | (s[i] >> 8);
#pragma unroll
    for (int i = 0; i < 8; i++) b2.w[i] = (s[7 + i] << 24) | (s[8 + i] >> 8);
    b2.w[8] = (s[15] << 24) | 0x00800000u;
#pragma unroll
    for (int i = 9; i < 15; i++) b2.w[i] = 0;
    b2.w[15] = (64u + 97u) * 8u;
    finish(sha256_compress(sha256_compress(in, b1), b2), tag);
  }
};

// The HMAC-SHA256 DRBG of RFC 6979 §3.2 as libsecp256k1's nonce_function_rfc6979 runs it: seeded with key32 || msgmod32
// (the raw secret key and the digest reduced mod n; no extra data, no algorithm tag).  Output c of next() (c = 0, 1, ...) is
// the nonce candidate for libsecp256k1's attempt counter c.
struct rfc6979_state {
  hmac_sha256 k;
  uint32_t v[8];
  bool retry;

  IBFT_HD void init(const uint8_t* key32, const uint8_t* msgmod32) {
    uint32_t x[8], m[8], t[8];
    sha256_words_from_be(key32, x, 8);
    sha256_words_from_be(msgmod32, m, 8);
#pragma unroll
    for (int i = 0; i < 8; i++) { v[i] = 0x01010101u; t[i] = 0; }
    k.set_key(t);             // K = 0x00 * 32
    k.mac97(v, 0x00, x, m, t);  // K = HMAC_K(V || 0x00 || key || msg)
    k.set_key(t);
    k.mac32(v, v);            // V = HMAC_K(V)
    k.mac97(v, 0x01, x, m, t);  // K = HMAC_K(V || 0x01 || key || msg)
    k.set_key(t);
    k.mac32(v, v);            // V = HMAC_K(V)
    retry = false;
  }
  IBFT_HD void next(uint8_t* out32) {
    if (retry) {
      uint32_t t[8];
      k.mac33(v, 0x00, t);  // K = HMAC_K(V || 0x00)
      k.set_key(t);
      k.mac32(v, v);        // V = HMAC_K(V)
    }
    k.mac32(v, v);          // V = HMAC_K(V): the output
    sha256_words_to_be(v, out32, 8);
    retry = true;
  }
};

// nonce candidate c of libsecp256k1's nonce_function_rfc6979(key32, msgmod32, counter = c): the DRBG's (c+1)-th output.  Like
// libsecp256k1, every candidate runs the DRBG from its seed, so no DRBG state outlives the call.
IBFT_HD void rfc6979_candidate(const uint8_t* key32, const uint8_t* msgmod32, uint32_t c, uint8_t* out32) {
  rfc6979_state st;
  st.init(key32, msgmod32);
  for (uint32_t i = 0; i <= c; i++) st.next(out32);
}

}  // namespace ibft
