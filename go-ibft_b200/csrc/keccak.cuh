// keccak.cuh -- Keccak-256 (original padding 0x01) for the message-verification hot path.
//
// K1 of SURVEY.md §2.2: digest of IbftMessage.PayloadNoSig() (reference messages/proto/helper.go:13-27 produces the
// bytes; the hash itself is the embedder's, named only in comments core/ibft.go:648, messages.proto:51,61,67),
// of proposalHash||0x02 for committed seals, and of X||Y for the address.  One thread owns one sponge: the 25
// 64-bit lanes live in registers (50 x 32-bit), theta/rho/pi/chi are LOP3/SHF work on the ALU pipe, which the
// IMAD-bound EC arithmetic of neighbouring warps leaves idle.
#pragma once
#include <stdint.h>

#include "secp_fe.cuh"

namespace ibft {

IBFT_HD uint64_t rotl64(uint64_t v, int n) { return (v << n) | (v >> (64 - n)); }

IBFT_HD uint64_t keccak_rc(int i) {
  const uint64_t rc[24] = {
      0x0000000000000001ULL, 0x0000000000008082ULL, 0x800000000000808AULL, 0x8000000080008000ULL,
      0x000000000000808BULL, 0x0000000080000001ULL, 0x8000000080008081ULL, 0x8000000000008009ULL,
      0x000000000000008AULL, 0x0000000000000088ULL, 0x0000000080008009ULL, 0x000000008000000AULL,
      0x000000008000808BULL, 0x800000000000008BULL, 0x8000000000008089ULL, 0x8000000000008003ULL,
      0x8000000000008002ULL, 0x8000000000000080ULL, 0x000000000000800AULL, 0x800000008000000AULL,
      0x8000000080008081ULL, 0x8000000000008080ULL, 0x0000000080000001ULL, 0x8000000080008008ULL};
  return rc[i];
}

IBFT_HD void keccak_f1600(uint64_t* a) {
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int rnd = 0; rnd < 24; rnd++) {
    uint64_t c0 = a[0] ^ a[5] ^ a[10] ^ a[15] ^ a[20];
    uint64_t c1 = a[1] ^ a[6] ^ a[11] ^ a[16] ^ a[21];
    uint64_t c2 = a[2] ^ a[7] ^ a[12] ^ a[17] ^ a[22];
    uint64_t c3 = a[3] ^ a[8] ^ a[13] ^ a[18] ^ a[23];
    uint64_t c4 = a[4] ^ a[9] ^ a[14] ^ a[19] ^ a[24];
    uint64_t d0 = c4 ^ rotl64(c1, 1), d1 = c0 ^ rotl64(c2, 1), d2 = c1 ^ rotl64(c3, 1), d3 = c2 ^ rotl64(c4, 1),
             d4 = c3 ^ rotl64(c0, 1);
    // theta + rho + pi
    uint64_t b0 = a[0] ^ d0;
    uint64_t b1 = rotl64(a[6] ^ d1, 44);
    uint64_t b2 = rotl64(a[12] ^ d2, 43);
    uint64_t b3 = rotl64(a[18] ^ d3, 21);
    uint64_t b4 = rotl64(a[24] ^ d4, 14);
    uint64_t b5 = rotl64(a[3] ^ d3, 28);
    uint64_t b6 = rotl64(a[9] ^ d4, 20);
    uint64_t b7 = rotl64(a[10] ^ d0, 3);
    uint64_t b8 = rotl64(a[16] ^ d1, 45);
    uint64_t b9 = rotl64(a[22] ^ d2, 61);
    uint64_t b10 = rotl64(a[1] ^ d1, 1);
    uint64_t b11 = rotl64(a[7] ^ d2, 6);
    uint64_t b12 = rotl64(a[13] ^ d3, 25);
    uint64_t b13 = rotl64(a[19] ^ d4, 8);
    uint64_t b14 = rotl64(a[20] ^ d0, 18);
    uint64_t b15 = rotl64(a[4] ^ d4, 27);
    uint64_t b16 = rotl64(a[5] ^ d0, 36);
    uint64_t b17 = rotl64(a[11] ^ d1, 10);
    uint64_t b18 = rotl64(a[17] ^ d2, 15);
    uint64_t b19 = rotl64(a[23] ^ d3, 56);
    uint64_t b20 = rotl64(a[2] ^ d2, 62);
    uint64_t b21 = rotl64(a[8] ^ d3, 55);
    uint64_t b22 = rotl64(a[14] ^ d4, 39);
    uint64_t b23 = rotl64(a[15] ^ d0, 41);
    uint64_t b24 = rotl64(a[21] ^ d1, 2);
    // chi + iota
    a[0] = b0 ^ (~b1 & b2) ^ keccak_rc(rnd);
    a[1] = b1 ^ (~b2 & b3);
    a[2] = b2 ^ (~b3 & b4);
    a[3] = b3 ^ (~b4 & b0);
    a[4] = b4 ^ (~b0 & b1);
    a[5] = b5 ^ (~b6 & b7);
    a[6] = b6 ^ (~b7 & b8);
    a[7] = b7 ^ (~b8 & b9);
    a[8] = b8 ^ (~b9 & b5);
    a[9] = b9 ^ (~b5 & b6);
    a[10] = b10 ^ (~b11 & b12);
    a[11] = b11 ^ (~b12 & b13);
    a[12] = b12 ^ (~b13 & b14);
    a[13] = b13 ^ (~b14 & b10);
    a[14] = b14 ^ (~b10 & b11);
    a[15] = b15 ^ (~b16 & b17);
    a[16] = b16 ^ (~b17 & b18);
    a[17] = b17 ^ (~b18 & b19);
    a[18] = b18 ^ (~b19 & b15);
    a[19] = b19 ^ (~b15 & b16);
    a[20] = b20 ^ (~b21 & b22);
    a[21] = b21 ^ (~b22 & b23);
    a[22] = b22 ^ (~b23 & b24);
    a[23] = b23 ^ (~b24 & b20);
    a[24] = b24 ^ (~b20 & b21);
  }
}

IBFT_HD uint64_t load_le64_partial(const uint8_t* p, int n) {  // n in [0,8]
  uint64_t w = 0;
  for (int i = 0; i < n; i++) w |= (uint64_t)p[i] << (8 * i);
  return w;
}

// 8 message bytes from an ARBITRARILY aligned address as one little-endian lane.  Device: three aligned 32-bit loads + two
// funnel shifts instead of eight byte loads (a byte-wise absorb made the loads, not the permutation, the cost of a long sponge).  The aligned word that holds the last wanted byte is always inside the allocation.
IBFT_HD uint64_t load_le64_any(const uint8_t* p) {
#if defined(__CUDA_ARCH__)
  const uint32_t sh = ((uint32_t)(uintptr_t)p & 3u) * 8u;
  const uint32_t* a = reinterpret_cast<const uint32_t*>((uintptr_t)p & ~(uintptr_t)3);
  const uint32_t w0 = a[0], w1 = a[1];
  if (sh == 0) return (uint64_t)w0 | ((uint64_t)w1 << 32);
  const uint32_t w2 = a[2];
  return (uint64_t)__funnelshift_r(w0, w1, sh) | ((uint64_t)__funnelshift_r(w1, w2, sh) << 32);
#else
  return load_le64_partial(p, 8);
#endif
}

// Keccak-256 of an arbitrary byte string (multi-block), out = 32 bytes.
IBFT_HD void keccak256_bytes(const uint8_t* data, uint32_t len, uint8_t* out) {
  uint64_t st[25];
#pragma unroll
  for (int i = 0; i < 25; i++) st[i] = 0;
  while (len >= 136) {
#pragma unroll
    for (int i = 0; i < 17; i++) st[i] ^= load_le64_any(data + 8 * i);
    keccak_f1600(st);
    data += 136;
    len -= 136;
  }
  // final (partial) block with padding 0x01 ... 0x80
  int full = (int)(len >> 3), rem = (int)(len & 7);
  for (int i = 0; i < full; i++) st[i] ^= load_le64_any(data + 8 * i);
  st[full] ^= load_le64_partial(data + 8 * full, rem) | ((uint64_t)0x01 << (8 * rem));
  st[16] ^= 0x8000000000000000ULL;
  keccak_f1600(st);
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 8; j++) out[8 * i + j] = (uint8_t)(st[i] >> (8 * j));
}

// Keccak-256 of the concatenation of two byte spans (a wire frame with its signature field cut out; a ROUND_CHANGE head + its
// shared prepared certificate).  The first span is staged byte by byte up to a block boundary of the STREAM; from there on every
// rate block lies entirely inside the second span and is absorbed as 17 lanes read straight from memory (load_le64_any).
IBFT_HD void keccak256_two_spans(const uint8_t* p1, uint32_t n1, const uint8_t* p2, uint32_t n2, uint8_t* out) {
  uint64_t st[25];
#pragma unroll
  for (int i = 0; i < 25; i++) st[i] = 0;
  uint8_t blk[136];
  uint32_t pos = 0;
  // span 1, and the bytes of span 2 that complete its last block
  uint32_t i2 = 0;
  for (int span = 0; span < 2; span++) {
    const uint8_t* p = span ? p2 : p1;
    const uint32_t n = span ? n2 : n1;
    uint32_t i = 0;
    for (; i < n && !(span == 1 && pos == 0); i++) {
      blk[pos] = p[i];
      if (++pos == 136) {
#pragma unroll
        for (int k = 0; k < 17; k++) st[k] ^= load_le64_partial(blk + 8 * k, 8);
        keccak_f1600(st);
        pos = 0;
      }
    }
    if (span == 1) i2 = i;
  }
  // whole blocks of span 2
  while (n2 - i2 >= 136) {
#pragma unroll
    for (int k = 0; k < 17; k++) st[k] ^= load_le64_any(p2 + i2 + 8 * k);
    keccak_f1600(st);
    i2 += 136;
  }
  // tail (pos == 0 here unless span 2 ended inside the first loop)
  for (; i2 < n2; i2++) blk[pos++] = p2[i2];
  for (uint32_t i = pos; i < 136; i++) blk[i] = 0;
  blk[pos] = 0x01;
  blk[135] |= 0x80;
#pragma unroll
  for (int k = 0; k < 17; k++) st[k] ^= load_le64_partial(blk + 8 * k, 8);
  keccak_f1600(st);
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 8; j++) out[8 * i + j] = (uint8_t)(st[i] >> (8 * j));
}

// Keccak-256 of exactly 64 bytes given as two field elements (X||Y big-endian) -> last 20 bytes (the address)
// as five big-endian-loaded words: addr[0] = bytes 12..15 of the digest, ...
IBFT_HD void keccak256_xy_address(const fe& x, const fe& y, uint8_t* addr20) {
  uint64_t st[25];
#pragma unroll
  for (int i = 0; i < 25; i++) st[i] = 0;
  // message byte m[4k..4k+3] = big-endian limb (7-k) of x; lane i = bytes 8i..8i+7 little-endian
#pragma unroll
  for (int i = 0; i < 4; i++) {
    uint32_t w0 = x.v[7 - 2 * i], w1 = x.v[6 - 2 * i];  // bytes 8i..8i+3 and 8i+4..8i+7 (big-endian words)
    uint32_t l0 = (w0 >> 24) | ((w0 >> 8) & 0xFF00u) | ((w0 << 8) & 0xFF0000u) | (w0 << 24);
    uint32_t l1 = (w1 >> 24) | ((w1 >> 8) & 0xFF00u) | ((w1 << 8) & 0xFF0000u) | (w1 << 24);
    st[i] = (uint64_t)l0 | ((uint64_t)l1 << 32);
    uint32_t v0 = y.v[7 - 2 * i], v1 = y.v[6 - 2 * i];
    uint32_t m0 = (v0 >> 24) | ((v0 >> 8) & 0xFF00u) | ((v0 << 8) & 0xFF0000u) | (v0 << 24);
    uint32_t m1 = (v1 >> 24) | ((v1 >> 8) & 0xFF00u) | ((v1 << 8) & 0xFF0000u) | (v1 << 24);
    st[4 + i] = (uint64_t)m0 | ((uint64_t)m1 << 32);
  }
  st[8] ^= 0x01ULL;
  st[16] ^= 0x8000000000000000ULL;
  keccak_f1600(st);
  // digest bytes 12..31 = st[1] bytes 4..7, st[2], st[3]
#pragma unroll
  for (int j = 0; j < 4; j++) addr20[j] = (uint8_t)(st[1] >> (8 * (4 + j)));
#pragma unroll
  for (int j = 0; j < 8; j++) addr20[4 + j] = (uint8_t)(st[2] >> (8 * j));
#pragma unroll
  for (int j = 0; j < 8; j++) addr20[12 + j] = (uint8_t)(st[3] >> (8 * j));
}

}  // namespace ibft
