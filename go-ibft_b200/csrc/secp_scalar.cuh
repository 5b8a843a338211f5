// secp_scalar.cuh -- arithmetic modulo the group order n of secp256k1, GLV decomposition and signed
// fixed-window (Booth) digit extraction.
//
// Only a handful of mod-n operations happen per signature (z mod n, r^-1, u1 = -z r^-1, u2 = s r^-1),
// so this code is written in portable C++ on top of the field multiplier's 256x256 product; the GLV split
// itself is pure integer arithmetic (no reduction): with the lattice basis (a1,b1),(a2,b2) of
// {(x,y): x + y*lambda = 0 mod n},  k1 = k - c1*a1 - c2*a2,  k2 = -c1*b1 - c2*b2,  c_i = round(k*g_i/2^384).
// Constants were derived and bound-checked in Python (tools/gen_tables.py; |k1|,|k2| < 2^129).
#pragma once
#include "secp_fe.cuh"

namespace ibft {

struct sc {
  uint32_t v[8];
};

// n and 2^256 - n
#define IBFT_N_LIMBS {0xD0364141u, 0xBFD25E8Cu, 0xAF48A03Bu, 0xBAAEDCE6u, 0xFFFFFFFEu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu}
#define IBFT_NC_LIMBS {0x2FC9BEBFu, 0x402DA173u, 0x50B75FC4u, 0x45512319u, 0x00000001u}

IBFT_HD uint32_t sc_n_limb(int i) {
  const uint32_t n[8] = IBFT_N_LIMBS;
  return n[i];
}
IBFT_HD uint32_t sc_nc_limb(int i) {
  const uint32_t c[5] = IBFT_NC_LIMBS;
  return c[i];
}

IBFT_HD sc sc_from_be(const uint8_t* b) {
  fe t = fe_from_be(b);
  sc r;
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = t.v[i];
  return r;
}
IBFT_HD void sc_to_be(const sc& a, uint8_t* b) {
  fe t;
#pragma unroll
  for (int i = 0; i < 8; i++) t.v[i] = a.v[i];
  fe_to_be(t, b);
}
IBFT_HD bool sc_is_zero(const sc& a) {
  return (a.v[0] | a.v[1] | a.v[2] | a.v[3] | a.v[4] | a.v[5] | a.v[6] | a.v[7]) == 0;
}
// a >= n ?
IBFT_HD bool sc_ge_n(const sc& a) {
  // a + (2^256 - n) overflows 2^256  <=>  a >= n
  uint64_t c = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    c += (uint64_t)a.v[i] + (i < 5 ? sc_nc_limb(i) : 0u);
    c >>= 32;
  }
  return c != 0;
}
// a in [0, 2^256) -> a mod n (one conditional subtraction; 2^256 < 2n)
IBFT_HD sc sc_reduce_once(const sc& a) {
  sc t;
  uint64_t c = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    c += (uint64_t)a.v[i] + (i < 5 ? sc_nc_limb(i) : 0u);
    t.v[i] = (uint32_t)c;
    c >>= 32;
  }
  sc r;
  bool ge = c != 0;
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = ge ? t.v[i] : a.v[i];
  return r;
}
// -a mod n, a in [0, n)
IBFT_HD sc sc_neg(const sc& a) {
  sc r;
  int64_t c = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    c += (int64_t)sc_n_limb(i) - (int64_t)a.v[i];
    r.v[i] = (uint32_t)c;
    c >>= 32;
  }
  bool z = sc_is_zero(a);
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = z ? 0u : r.v[i];
  return r;
}

// a + b mod n, a, b in [0, n)
IBFT_HD sc sc_add(const sc& a, const sc& b) {
  sc t;
  uint64_t c = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    c += (uint64_t)a.v[i] + b.v[i];
    t.v[i] = (uint32_t)c;
    c >>= 32;
  }
  // a + b < 2n < 2^257: subtract n when the sum overflowed 2^256 or is >= n
  sc u;
  uint64_t d = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    d += (uint64_t)t.v[i] + (i < 5 ? sc_nc_limb(i) : 0u);
    u.v[i] = (uint32_t)d;
    d >>= 32;
  }
  bool ge = (c != 0) || (d != 0);  // (sum + 2^256 - n) carried  <=>  sum >= n
  sc r;
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = ge ? u.v[i] : t.v[i];
  return r;
}
// a > (n-1)/2 ?  (the "high-s" half)
IBFT_HD bool sc_is_high(const sc& a) {
  const uint32_t h[8] = {0x681B20A0u, 0xDFE92F46u, 0x57A4501Du, 0x5D576E73u, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0x7FFFFFFFu};  // (n-1)/2
  for (int i = 7; i >= 0; i--)
    if (a.v[i] != h[i]) return a.v[i] > h[i];
  return false;
}

// 512-bit R -> R mod n.  2^256 = NC (mod n), NC = 2^256 - n is 129 bits: three folds.
IBFT_HD sc sc_reduce512(const uint32_t* R) {
  // fold 1: acc1 = L + H * NC                      (< 2^386: 13 limbs + carry)
  uint32_t a1[14];
#pragma unroll
  for (int i = 0; i < 14; i++) a1[i] = i < 8 ? R[i] : 0u;
#pragma unroll
  for (int j = 0; j < 5; j++) {
    uint64_t c = 0;
    uint32_t m = sc_nc_limb(j);
#pragma unroll
    for (int i = 0; i < 8; i++) {
      c += (uint64_t)R[8 + i] * m + a1[i + j];
      a1[i + j] = (uint32_t)c;
      c >>= 32;
    }
#pragma unroll
    for (int i = 8 + j; i < 14; i++) {
      c += a1[i];
      a1[i] = (uint32_t)c;
      c >>= 32;
    }
  }
  // fold 2: acc2 = a1[0..7] + a1[8..13] * NC        (a1[8..13] < 2^130)
  uint32_t a2[12];
#pragma unroll
  for (int i = 0; i < 12; i++) a2[i] = i < 8 ? a1[i] : 0u;
#pragma unroll
  for (int j = 0; j < 5; j++) {
    uint64_t c = 0;
    uint32_t m = sc_nc_limb(j);
#pragma unroll
    for (int i = 0; i < 6; i++) {
      c += (uint64_t)a1[8 + i] * m + a2[i + j];
      a2[i + j] = (uint32_t)c;
      c >>= 32;
    }
#pragma unroll
    for (int i = 6 + j; i < 12; i++) {
      c += a2[i];
      a2[i] = (uint32_t)c;
      c >>= 32;
    }
  }
  // fold 3: acc3 = a2[0..7] + a2[8] * NC            (a2[8..] < 2^4, higher limbs are zero)
  uint32_t a3[9];
  {
    uint64_t c = 0;
    uint32_t h = a2[8];
#pragma unroll
    for (int i = 0; i < 8; i++) {
      c += (uint64_t)a2[i] + (i < 5 ? (uint64_t)h * sc_nc_limb(i) : 0ull);
      a3[i] = (uint32_t)c;
      c >>= 32;
    }
    a3[8] = (uint32_t)c;  // 0 or 1
  }
  // fold 4: a wrap leaves a small value; add NC once more
  sc r;
  {
    uint64_t c = 0;
    uint32_t h = a3[8];
#pragma unroll
    for (int i = 0; i < 8; i++) {
      c += (uint64_t)a3[i] + (i < 5 ? (uint64_t)h * sc_nc_limb(i) : 0ull);
      r.v[i] = (uint32_t)c;
      c >>= 32;
    }
  }
  return sc_reduce_once(r);
}

IBFT_HD sc sc_mul(const sc& a, const sc& b) {
  uint32_t R[16];
  mul_wide_8x8(R, a.v, b.v);
  return sc_reduce512(R);
}
IBFT_HD sc sc_sqr(const sc& a) { return sc_mul(a, a); }

// a^(n-2) mod n with a fixed 4-bit window (0 -> 0).  Replaced by safegcd in the tuned path.
IBFT_HD sc sc_inv_fermat(const sc& a) {
  // n - 2 as nibbles, most significant first
  const uint32_t e[8] = {0xD036413Fu, 0xBFD25E8Cu, 0xAF48A03Bu, 0xBAAEDCE6u, 0xFFFFFFFEu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu};
  sc tab[16];
  tab[0].v[0] = 1;
#pragma unroll
  for (int i = 1; i < 8; i++) tab[0].v[i] = 0;
  tab[1] = a;
  for (int i = 2; i < 16; i++) tab[i] = sc_mul(tab[i - 1], a);
  sc r = tab[(e[7] >> 28) & 15];
  for (int nib = 62; nib >= 0; nib--) {
    r = sc_sqr(r);
    r = sc_sqr(r);
    r = sc_sqr(r);
    r = sc_sqr(r);
    uint32_t d = (e[nib >> 3] >> (4 * (nib & 7))) & 15;
    if (d) r = sc_mul(r, tab[d]);
  }
  return r;
}

// ------------------------------------------------------------------------------------------------
// GLV decomposition
// ------------------------------------------------------------------------------------------------
struct glv_half {
  uint32_t k[5];  // magnitude, < 2^129
  bool neg;
};

// r[0..na+nb-1] = a[0..na-1] * b[0..nb-1]
template <int NA, int NB>
IBFT_HD void mul_small(uint32_t* r, const uint32_t* a, const uint32_t* b) {
#pragma unroll
  for (int i = 0; i < NA + NB; i++) r[i] = 0;
#pragma unroll
  for (int i = 0; i < NB; i++) {
    uint64_t c = 0;
#pragma unroll
    for (int j = 0; j < NA; j++) {
      c += (uint64_t)a[j] * b[i] + r[i + j];
      r[i + j] = (uint32_t)c;
      c >>= 32;
    }
    r[i + NA] = (uint32_t)c;
  }
}

// k in [0, n)  ->  k = k1 + k2*lambda (mod n), |k1|,|k2| < 2^129
IBFT_HD void glv_split(const sc& k, glv_half& h1, glv_half& h2) {
  const uint32_t g1[8] = {0x45DBB031u, 0xE893209Au, 0x71E8CA7Fu, 0x3DAA8A14u, 0x9284EB15u, 0xE86C90E4u, 0xA7D46BCDu, 0x3086D221u};
  const uint32_t g2[8] = {0x8AC47F71u, 0x1571B4AEu, 0x9DF506C6u, 0x221208ACu, 0x0ABFE4C4u, 0x6F547FA9u, 0x010E8828u, 0xE4437ED6u};
  const uint32_t a1[4] = {0x9284EB15u, 0xE86C90E4u, 0xA7D46BCDu, 0x3086D221u};                 // a1 = b2
  const uint32_t mb1[4] = {0x0ABFE4C3u, 0x6F547FA9u, 0x010E8828u, 0xE4437ED6u};                // -b1
  const uint32_t a2[5] = {0x9D44CFD8u, 0x57C1108Du, 0xA8E2F3F6u, 0x14CA50F7u, 0x00000001u};    // a2
  uint32_t W[16], c1[4], c2[4];
  mul_wide_8x8(W, k.v, g1);
  {
    uint64_t c = (uint64_t)W[12] + (W[11] >> 31);
    c1[0] = (uint32_t)c; c >>= 32;
    c += W[13]; c1[1] = (uint32_t)c; c >>= 32;
    c += W[14]; c1[2] = (uint32_t)c; c >>= 32;
    c += W[15]; c1[3] = (uint32_t)c;
  }
  mul_wide_8x8(W, k.v, g2);
  {
    uint64_t c = (uint64_t)W[12] + (W[11] >> 31);
    c2[0] = (uint32_t)c; c >>= 32;
    c += W[13]; c2[1] = (uint32_t)c; c >>= 32;
    c += W[14]; c2[2] = (uint32_t)c; c >>= 32;
    c += W[15]; c2[3] = (uint32_t)c;
  }
  // k2 = c1*(-b1) - c2*b2   (b2 = a1), exact signed integer, |k2| < 2^129: work modulo 2^192
  uint32_t p1[8], p2[8], q1[8], q2[9];
  mul_small<4, 4>(p1, c1, mb1);
  mul_small<4, 4>(p2, c2, a1);
  uint32_t k2[6];
  {
    int64_t c = 0;
#pragma unroll
    for (int i = 0; i < 6; i++) {
      c += (int64_t)p1[i] - (int64_t)p2[i];
      k2[i] = (uint32_t)c;
      c >>= 32;
    }
  }
  // k1 = k - c1*a1 - c2*a2
  mul_small<4, 4>(q1, c1, a1);
  mul_small<4, 5>(q2, c2, a2);
  uint32_t k1[6];
  {
    int64_t c = 0;
#pragma unroll
    for (int i = 0; i < 6; i++) {
      c += (int64_t)k.v[i] - (int64_t)q1[i] - (int64_t)q2[i];
      k1[i] = (uint32_t)c;
      c >>= 32;
    }
  }
  // sign / magnitude (two's complement in 192 bits)
  h1.neg = (k1[5] >> 31) != 0;
  h2.neg = (k2[5] >> 31) != 0;
  {
    uint64_t c = h1.neg ? 1 : 0;
#pragma unroll
    for (int i = 0; i < 5; i++) {
      c += h1.neg ? (uint32_t)~k1[i] : k1[i];
      h1.k[i] = (uint32_t)c;
      c >>= 32;
    }
  }
  {
    uint64_t c = h2.neg ? 1 : 0;
#pragma unroll
    for (int i = 0; i < 5; i++) {
      c += h2.neg ? (uint32_t)~k2[i] : k2[i];
      h2.k[i] = (uint32_t)c;
      c >>= 32;
    }
  }
}

// Signed fixed-window (Booth) digit j of a non-negative scalar stored as NL limbs (top limb zero-padded):
//   d_j = k[wj .. wj+w-1] + k[wj-1] - 2^w * k[wj+w-1]   in [-2^(w-1), 2^(w-1)],   k = sum d_j 2^(wj)
// Every window is independent of the others, so all lanes of a warp add at the same loop positions.
template <int W, int NL = 6>
IBFT_HD int booth_digit(const uint32_t* k6, int j) {
  int pos = W * j - 1;  // lowest bit of the (W+1)-bit field; -1 for j = 0
  uint32_t field;
  if (pos < 0) {
    field = (k6[0] << 1) & ((2u << W) - 1u);
  } else {
    int limb = pos >> 5, sh = pos & 31;
    uint64_t two = (uint64_t)k6[limb] | ((uint64_t)(limb + 1 < NL ? k6[limb + 1] : 0u) << 32);
    field = (uint32_t)(two >> sh) & ((2u << W) - 1u);
  }
  int d = (int)((field + 1u) >> 1);       // window value (bits 1..W) + carry-in bit 0
  d -= (int)((field >> W) & 1u) << W;     // minus 2^W if the window's top bit is set
  return d;
}

}  // namespace ibft
