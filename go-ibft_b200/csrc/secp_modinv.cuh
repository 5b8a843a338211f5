// secp_modinv.cuh -- modular inversion by Bernstein-Yang "safegcd" divsteps (variable time; nothing here is secret:
// signature verification only handles public data).
//
// Replaces the two Fermat ladders of the first kernel version (a^(p-2): 255 squarings; a^(n-2): ~320 generic mod-n
// multiplications, a large share of all instructions).  The algorithm works on 9 signed 30-bit limbs so that
// a 2x2 transition matrix of 30 divsteps can be applied with 32x32->64 multiply-adds without overflow:
//   repeat:  t = matrix of 30 divsteps on the low 30 bits of (f, g)            [ALU-pipe work: ctz, shifts, adds]
//            (d, e) <- t * (d, e) / 2^30  (mod m)                               [72 wide MACs]
//            (f, g) <- t * (f, g) / 2^30                                        [36 wide MACs]
//   until g == 0;   result = sign(f) * d  (mod m)
// ~19 iterations for 256-bit inputs, i.e. ~2k wide MACs per inversion.  Lanes of a warp iterate in lock step; only the
// trip counts of the inner (zero-skipping) and outer loops differ between lanes, and the warp runs the maximum.
// Parity: checked against Python pow(a, -1, m) and the Fermat ladders (tests/test_emul.py, tests/test_gpu_primitives.py).
#pragma once
#include "secp_fe.cuh"
#include "secp_scalar.cuh"

namespace ibft {

struct s30 {
  int32_t v[9];
};

struct modinfo30 {
  int32_t m[9];     // modulus, 30-bit limbs
  uint32_t minv30;  // modulus^-1 mod 2^30
};

IBFT_HD modinfo30 modinfo_p() {
  modinfo30 r = {{0x3FFFFC2F, 0x3FFFFFFB, 0x3FFFFFFF, 0x3FFFFFFF, 0x3FFFFFFF, 0x3FFFFFFF, 0x3FFFFFFF, 0x3FFFFFFF, 0x0000FFFF}, 0x2DDACACFu};
  return r;
}
IBFT_HD modinfo30 modinfo_n() {
  modinfo30 r = {{0x10364141, 0x3F497A33, 0x348A03BB, 0x2BB739AB, 0x3FFFFEBA, 0x3FFFFFFF, 0x3FFFFFFF, 0x3FFFFFFF, 0x0000FFFF}, 0x2A774EC1u};
  return r;
}

// 8 x 32-bit limbs (value < 2^256) -> 9 x 30-bit limbs
IBFT_HD s30 s30_from_u32x8(const uint32_t* a) {
  s30 r;
  const uint32_t M30 = 0x3FFFFFFFu;
  r.v[0] = (int32_t)(a[0] & M30);
  r.v[1] = (int32_t)(((a[0] >> 30) | (a[1] << 2)) & M30);
  r.v[2] = (int32_t)(((a[1] >> 28) | (a[2] << 4)) & M30);
  r.v[3] = (int32_t)(((a[2] >> 26) | (a[3] << 6)) & M30);
  r.v[4] = (int32_t)(((a[3] >> 24) | (a[4] << 8)) & M30);
  r.v[5] = (int32_t)(((a[4] >> 22) | (a[5] << 10)) & M30);
  r.v[6] = (int32_t)(((a[5] >> 20) | (a[6] << 12)) & M30);
  r.v[7] = (int32_t)(((a[6] >> 18) | (a[7] << 14)) & M30);
  r.v[8] = (int32_t)(a[7] >> 16);
  return r;
}
// 9 x 30-bit non-negative limbs (value < 2^256) -> 8 x 32-bit
IBFT_HD void s30_to_u32x8(const s30& a, uint32_t* r) {
  const uint32_t* v = reinterpret_cast<const uint32_t*>(a.v);
  r[0] = v[0] | (v[1] << 30);
  r[1] = (v[1] >> 2) | (v[2] << 28);
  r[2] = (v[2] >> 4) | (v[3] << 26);
  r[3] = (v[3] >> 6) | (v[4] << 24);
  r[4] = (v[4] >> 8) | (v[5] << 22);
  r[5] = (v[5] >> 10) | (v[6] << 20);
  r[6] = (v[6] >> 12) | (v[7] << 18);
  r[7] = (v[7] >> 14) | (v[8] << 16);
}

IBFT_HD int ctz32_nz(uint32_t x) {
#if defined(__CUDA_ARCH__)
  return __ffs((int)x) - 1;
#else
  return __builtin_ctz(x);
#endif
}

struct trans2x2 {
  int32_t u, v, q, r;
};

// 30 divsteps on the low bits of f (odd) and g; eta = -delta.  Returns the new eta and the transition matrix
// (scaled by 2^30).
IBFT_HD int32_t divsteps_30_var(int32_t eta, uint32_t f0, uint32_t g0, trans2x2& t) {
  uint32_t u = 1, v = 0, q = 0, r = 1;
  uint32_t f = f0, g = g0;
  int i = 30;
  for (;;) {
    // a sentinel bit bounds the zero count by the number of divsteps left
    int zeros = ctz32_nz(g | (0xFFFFFFFFu << i));
    g >>= zeros;
    u <<= zeros;
    v <<= zeros;
    eta -= zeros;
    i -= zeros;
    if (i == 0) break;
    if (eta < 0) {
      uint32_t tmp;
      eta = -eta;
      tmp = f; f = g; g = 0u - tmp;
      tmp = u; u = q; q = 0u - tmp;
      tmp = v; v = r; r = 0u - tmp;
    }
    // cancel up to min(eta+1, i, 8) low bits of g with a multiple of f
    int limit = (eta + 1) > i ? i : (eta + 1);
    uint32_t m = (0xFFFFFFFFu >> (32 - limit)) & 255u;
    // -f^-1 mod 2^8 by Newton iteration (f odd): x = f is correct mod 8, two steps give 12 bits
    uint32_t x = f;
    x *= 2u - f * x;
    x *= 2u - f * x;
    uint32_t w = (g * (0u - x)) & m;
    g += f * w;
    q += u * w;
    r += v * w;
  }
  t.u = (int32_t)u;
  t.v = (int32_t)v;
  t.q = (int32_t)q;
  t.r = (int32_t)r;
  return eta;
}

// (d, e) <- t * (d, e) / 2^30 mod m, limbs stay in (-2^30, 2^30), values in (-2m, m)
IBFT_HD void update_de_30(s30& d, s30& e, const trans2x2& t, const modinfo30& mi) {
  const int32_t M30 = 0x3FFFFFFF;
  const int32_t u = t.u, v = t.v, q = t.q, r = t.r;
  int32_t sd = d.v[8] >> 31, se = e.v[8] >> 31;
  int32_t md = (u & sd) + (v & se);
  int32_t me = (q & sd) + (r & se);
  int32_t di = d.v[0], ei = e.v[0];
  int64_t cd = (int64_t)u * di + (int64_t)v * ei;
  int64_t ce = (int64_t)q * di + (int64_t)r * ei;
  // choose md, me so that the low 30 bits of t*[d,e] + m*[md,me] vanish
  md -= (int32_t)((mi.minv30 * (uint32_t)cd + (uint32_t)md) & (uint32_t)M30);
  me -= (int32_t)((mi.minv30 * (uint32_t)ce + (uint32_t)me) & (uint32_t)M30);
  cd += (int64_t)mi.m[0] * md;
  ce += (int64_t)mi.m[0] * me;
  cd >>= 30;
  ce >>= 30;
#pragma unroll
  for (int i = 1; i < 9; i++) {
    di = d.v[i];
    ei = e.v[i];
    cd += (int64_t)u * di + (int64_t)v * ei;
    ce += (int64_t)q * di + (int64_t)r * ei;
    cd += (int64_t)mi.m[i] * md;
    ce += (int64_t)mi.m[i] * me;
    d.v[i - 1] = (int32_t)cd & M30;
    cd >>= 30;
    e.v[i - 1] = (int32_t)ce & M30;
    ce >>= 30;
  }
  d.v[8] = (int32_t)cd;
  e.v[8] = (int32_t)ce;
}

// (f, g) <- t * (f, g) / 2^30 (exact)
IBFT_HD void update_fg_30(s30& f, s30& g, const trans2x2& t) {
  const int32_t M30 = 0x3FFFFFFF;
  const int32_t u = t.u, v = t.v, q = t.q, r = t.r;
  int32_t fi = f.v[0], gi = g.v[0];
  int64_t cf = (int64_t)u * fi + (int64_t)v * gi;
  int64_t cg = (int64_t)q * fi + (int64_t)r * gi;
  cf >>= 30;
  cg >>= 30;
#pragma unroll
  for (int i = 1; i < 9; i++) {
    fi = f.v[i];
    gi = g.v[i];
    cf += (int64_t)u * fi + (int64_t)v * gi;
    cg += (int64_t)q * fi + (int64_t)r * gi;
    f.v[i - 1] = (int32_t)cf & M30;
    cf >>= 30;
    g.v[i - 1] = (int32_t)cg & M30;
    cg >>= 30;
  }
  f.v[8] = (int32_t)cf;
  g.v[8] = (int32_t)cg;
}

// bring d from (-2m, m) to [0, m), negating first when sign < 0
IBFT_HD void normalize_30(s30& r, int32_t sign, const modinfo30& mi) {
  const int32_t M30 = 0x3FFFFFFF;
  int32_t cond_add = r.v[8] >> 31;
#pragma unroll
  for (int i = 0; i < 9; i++) r.v[i] += mi.m[i] & cond_add;
  int32_t cond_negate = sign >> 31;
#pragma unroll
  for (int i = 0; i < 9; i++) r.v[i] = (r.v[i] ^ cond_negate) - cond_negate;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    r.v[i + 1] += r.v[i] >> 30;
    r.v[i] &= M30;
  }
  cond_add = r.v[8] >> 31;
#pragma unroll
  for (int i = 0; i < 9; i++) r.v[i] += mi.m[i] & cond_add;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    r.v[i + 1] += r.v[i] >> 30;
    r.v[i] &= M30;
  }
}

// x^-1 mod m for x in [0, m) given as 8 x 32-bit limbs; 0 -> 0.
IBFT_HD void modinv30_var(uint32_t* out8, const uint32_t* x8, const modinfo30& mi) {
  s30 d, e, f, g;
#pragma unroll
  for (int i = 0; i < 9; i++) {
    d.v[i] = 0;
    e.v[i] = 0;
    f.v[i] = mi.m[i];
  }
  e.v[0] = 1;
  g = s30_from_u32x8(x8);
  int32_t eta = -1;
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int it = 0; it < 40; it++) {  // 25 iterations suffice for 256-bit inputs; the bound only guards against misuse
    IBFT_OPCOUNT(IBFT_OP_INV_ITER);
    trans2x2 t;
    eta = divsteps_30_var(eta, (uint32_t)f.v[0], (uint32_t)g.v[0], t);
    update_de_30(d, e, t, mi);
    update_fg_30(f, g, t);
    int32_t any = 0;
#pragma unroll
    for (int i = 0; i < 9; i++) any |= g.v[i];
    if (any == 0) break;
  }
  // f = +/- gcd = +/- 1 (or +/- m when x = 0, in which case d = 0): its sign lives in the top limb
  // (limbs 0..7 are non-negative, so f < 0 exactly when the top limb is negative)
  normalize_30(d, f.v[8], mi);
  s30_to_u32x8(d, out8);
}

IBFT_FN fe fe_inv_safegcd(fe a) {
  IBFT_OPCOUNT(IBFT_OP_FE_INV);
  fe n = fe_normalize(a), r;
  modinv30_var(r.v, n.v, modinfo_p());
  return r;
}
IBFT_FN sc sc_inv_safegcd(sc a) {  // a in [0, n)
  IBFT_OPCOUNT(IBFT_OP_SC_INV);
  sc r;
  modinv30_var(r.v, a.v, modinfo_n());
  return r;
}

}  // namespace ibft
