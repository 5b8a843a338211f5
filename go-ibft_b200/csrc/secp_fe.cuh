// secp_fe.cuh -- arithmetic in GF(p), p = 2^256 - 2^32 - 977 (secp256k1 base field), 8 x 32-bit limbs.
//
// Part of the hot path behind core.Verifier.IsValidValidator / IsValidCommittedSeal
// (reference core/backend.go:41-45, :53-55): the reference ships no arithmetic, so there is no
// reference code to mirror here -- the design follows the GPU's integer pipe:
//   * saturated 32-bit limbs, because the sm_90a integer multiplier is the 32x32+64 IMAD.WIDE(.X)
//     (tools/imad_peak.cu measures its rate): a 256x256 product is 64 of them;
//   * products accumulate in two interleaved carry chains ("even"/"odd" columns) so that every
//     mad.lo.cc/madc.hi.cc pair fuses into ONE IMAD.WIDE.U32.X and two independent chains are always in
//     flight (the pipe needs ILP 2 per warp);
//   * values are kept only weakly reduced (< 2^256); p's special form folds the high half with 8 more
//     wide MACs.  Canonical form is produced only where bytes leave the field (fe_normalize).
//
// The same source compiles for the host (plain C++ path below) so that the whole per-signature pipeline
// can be checked against the oracle on a CPU-only box (tests/emul); on the device the PTX path is used.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define IBFT_HD __host__ __device__ __forceinline__
#else
#define IBFT_HD inline
#endif

// Code-size control.  The recover kernel is I-cache bound when everything is inlined (hundreds of KB of SASS,
// most stalls waiting for instructions), so the multiplier / squarer -- and optionally the adders --
// are real device functions, passed BY VALUE so that the ABI keeps every operand in registers (no stack traffic).
#if defined(__CUDACC__) && !defined(IBFT_INLINE_FE)
#define IBFT_FN __host__ __device__ __noinline__
#else
#define IBFT_FN IBFT_HD
#endif
#if defined(__CUDACC__) && defined(IBFT_NOINLINE_ADD)
#define IBFT_FN_ADD __host__ __device__ __noinline__
#else
#define IBFT_FN_ADD IBFT_HD
#endif

// Development instrumentation (tools/stage_clocks.cu): thread 0 of CTA 0 stamps clock64() at the pipeline's stage borders.
// Never defined in the product build.
#if defined(IBFT_STAGE_CLOCKS) && defined(__CUDACC__)
__device__ unsigned long long g_stage_clk[16];
#if defined(__CUDA_ARCH__)
#define IBFT_STAGE(i) do { if (blockIdx.x == 0 && threadIdx.x == 0) g_stage_clk[i] = clock64(); } while (0)
#else
#define IBFT_STAGE(i) do { } while (0)
#endif
#else
#define IBFT_STAGE(i) do { } while (0)
#endif

// Test instrumentation (tests/emul): counts the exceptional branches of the group law (IBFT_BR_*), so that the emulation tests
// can show that their crafted signatures reach them.  tests/emul defines IBFT_BRANCH before including the headers; everywhere
// else it expands to nothing.
#define IBFT_BR_ADD_DBL 0      // jac_add_affine: P + P (doubling)
#define IBFT_BR_ADD_NEG 1      // jac_add_affine: P + (-P) (infinity)
#define IBFT_BR_ADD_INF 2      // jac_add_affine: accumulator at infinity
#define IBFT_BR_XADD_DBL 3     // xyzz_add_x: P + P
#define IBFT_BR_XADD_NEG 4     // xyzz_add_x: P + (-P)
#define IBFT_BR_XADD_INF 5     // xyzz_add_x: accumulator at infinity
#define IBFT_BR_COUNT 6
// the rare cases of the one-thread recovery's final A + B (verify_core.cuh recover_final): ids past the 2 * IBFT_BR_COUNT
// overall and final-add counters of the emulation
#define IBFT_BR_REC_DBL 12     // A = B: the sum is a doubling
#define IBFT_BR_REC_NEG 13     // A = -B: the sum is the point at infinity
#define IBFT_BR_REC_B_INF 14   // u1 * G is the point at infinity (u1 = 0)
#define IBFT_BR_REC_NONRES 15  // r^3 + 7 is a non-residue: r is not an abscissa
#ifndef IBFT_BRANCH
#define IBFT_BRANCH(i) do { } while (0)
#endif

// Test instrumentation (tests/emul/opcount.cpp, read by tools/fma_budget.py): dynamic operation counts of one recovery
// (IBFT_OP_*), which the FMA-pipe ledger multiplies by the per-routine instruction counts of the SASS.  Expands to nothing
// everywhere else, the plain host emulation (tests/emul/emul.cpp) included.
#define IBFT_OP_MUL_BODY 0     // field multiplications (inlined multiplier bodies, wherever they run)
#define IBFT_OP_SQR_BODY 1     // field squarings (inlined squarer bodies, wherever they run)
#define IBFT_OP_MUL_CALL 2     // calls of the out-of-line multiplier fe_mul
#define IBFT_OP_SQR_CALL 3     // calls of the out-of-line squarer fe_sqr
#define IBFT_OP_SQRN_CALL 4    // calls of fe_sqrn
#define IBFT_OP_SQRN_ITER 5    // squarings inside fe_sqrn
#define IBFT_OP_DBL_FRONT 6    // calls of jac_dbl_front (doubling: A, B, C)
#define IBFT_OP_FE_INV 7       // field inversions (safegcd)
#define IBFT_OP_SC_INV 8       // scalar inversions (safegcd)
#define IBFT_OP_INV_ITER 9     // safegcd iterations (30 divsteps each), both kinds
#define IBFT_OP_WIN 10         // window-loop iterations
#define IBFT_OP_WIN_DBL 11     // doublings inside the window loop
#define IBFT_OP_WIN_ADD 12     // mixed additions inside the window loop
#define IBFT_OP_COUNT 13       // the counters above (emul_op_counts)
#define IBFT_OP_COMB_ADD 13    // mixed additions of the u1 * G comb (ecmult_gen_comb)
#define IBFT_OP_REC_FINAL 14   // final steps of the one-thread recovery (A + B, root and inverse, affine)
#define IBFT_OP_COUNT_ALL 15
#ifndef IBFT_OPCOUNT
#define IBFT_OPCOUNT(k) do { } while (0)
#endif

#if defined(__CUDA_ARCH__) && !defined(IBFT_PORTABLE_FE)
#define IBFT_PTX 1
#else
#define IBFT_PTX 0
#endif

namespace ibft {

struct fe {
  uint32_t v[8];  // little-endian limbs, value < 2^256 (not necessarily < p)
};

#define IBFT_P0 0xFFFFFC2Fu
#define IBFT_P1 0xFFFFFFFEu
#define IBFT_PC 977u  // 2^256 - p = 2^32 + 977

IBFT_HD fe fe_zero() {
  fe r;
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = 0;
  return r;
}
IBFT_HD fe fe_from_u32(uint32_t x) {
  fe r = fe_zero();
  r.v[0] = x;
  return r;
}
// big-endian 32 bytes -> limbs (no reduction)
IBFT_HD fe fe_from_be(const uint8_t* b) {
  fe r;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    const uint8_t* q = b + 4 * (7 - i);
    r.v[i] = ((uint32_t)q[0] << 24) | ((uint32_t)q[1] << 16) | ((uint32_t)q[2] << 8) | (uint32_t)q[3];
  }
  return r;
}
IBFT_HD void fe_to_be(const fe& a, uint8_t* b) {
#pragma unroll
  for (int i = 0; i < 8; i++) {
    uint8_t* q = b + 4 * (7 - i);
    q[0] = (uint8_t)(a.v[i] >> 24);
    q[1] = (uint8_t)(a.v[i] >> 16);
    q[2] = (uint8_t)(a.v[i] >> 8);
    q[3] = (uint8_t)(a.v[i]);
  }
}

// ------------------------------------------------------------------------------------------------
// add / sub
// ------------------------------------------------------------------------------------------------
IBFT_FN_ADD fe fe_add(fe a, fe b) {
  fe r;
#if IBFT_PTX
  uint32_t c;
  asm("add.cc.u32 %0,%9,%17;\n\taddc.cc.u32 %1,%10,%18;\n\taddc.cc.u32 %2,%11,%19;\n\taddc.cc.u32 %3,%12,%20;\n\t"
      "addc.cc.u32 %4,%13,%21;\n\taddc.cc.u32 %5,%14,%22;\n\taddc.cc.u32 %6,%15,%23;\n\taddc.cc.u32 %7,%16,%24;\n\t"
      "addc.u32 %8,0,0;"
      : "=r"(r.v[0]), "=r"(r.v[1]), "=r"(r.v[2]), "=r"(r.v[3]), "=r"(r.v[4]), "=r"(r.v[5]), "=r"(r.v[6]), "=r"(r.v[7]),
        "=r"(c)
      : "r"(a.v[0]), "r"(a.v[1]), "r"(a.v[2]), "r"(a.v[3]), "r"(a.v[4]), "r"(a.v[5]), "r"(a.v[6]), "r"(a.v[7]),
        "r"(b.v[0]), "r"(b.v[1]), "r"(b.v[2]), "r"(b.v[3]), "r"(b.v[4]), "r"(b.v[5]), "r"(b.v[6]), "r"(b.v[7]));
  // fold the carry: 2^256 = 2^32 + 977 (mod p)
  uint32_t k = c * IBFT_PC, c2;
  asm("add.cc.u32 %0,%0,%9;\n\taddc.cc.u32 %1,%1,%10;\n\taddc.cc.u32 %2,%2,0;\n\taddc.cc.u32 %3,%3,0;\n\t"
      "addc.cc.u32 %4,%4,0;\n\taddc.cc.u32 %5,%5,0;\n\taddc.cc.u32 %6,%6,0;\n\taddc.cc.u32 %7,%7,0;\n\t"
      "addc.u32 %8,0,0;"
      : "+r"(r.v[0]), "+r"(r.v[1]), "+r"(r.v[2]), "+r"(r.v[3]), "+r"(r.v[4]), "+r"(r.v[5]), "+r"(r.v[6]), "+r"(r.v[7]),
        "=r"(c2)
      : "r"(k), "r"(c));
  // a second wrap leaves a value < 2^34, so the last fold cannot ripple past limb 2
  uint32_t k2 = c2 * IBFT_PC;
  asm("add.cc.u32 %0,%0,%3;\n\taddc.cc.u32 %1,%1,%4;\n\taddc.u32 %2,%2,0;"
      : "+r"(r.v[0]), "+r"(r.v[1]), "+r"(r.v[2])
      : "r"(k2), "r"(c2));
#else
  uint64_t c = 0;
  for (int i = 0; i < 8; i++) {
    c += (uint64_t)a.v[i] + b.v[i];
    r.v[i] = (uint32_t)c;
    c >>= 32;
  }
  uint32_t k = (uint32_t)c;
  uint64_t d = (uint64_t)r.v[0] + k * IBFT_PC;
  r.v[0] = (uint32_t)d;
  d >>= 32;
  d += (uint64_t)r.v[1] + k;
  r.v[1] = (uint32_t)d;
  d >>= 32;
  for (int i = 2; i < 8; i++) {
    d += r.v[i];
    r.v[i] = (uint32_t)d;
    d >>= 32;
  }
  uint32_t k2 = (uint32_t)d;
  d = (uint64_t)r.v[0] + k2 * IBFT_PC;
  r.v[0] = (uint32_t)d;
  d >>= 32;
  d += (uint64_t)r.v[1] + k2;
  r.v[1] = (uint32_t)d;
  d >>= 32;
  r.v[2] += (uint32_t)d;
#endif
  return r;
}

IBFT_FN_ADD fe fe_sub(fe a, fe b) {
  fe r;
#if IBFT_PTX
  uint32_t c;
  asm("sub.cc.u32 %0,%9,%17;\n\tsubc.cc.u32 %1,%10,%18;\n\tsubc.cc.u32 %2,%11,%19;\n\tsubc.cc.u32 %3,%12,%20;\n\t"
      "subc.cc.u32 %4,%13,%21;\n\tsubc.cc.u32 %5,%14,%22;\n\tsubc.cc.u32 %6,%15,%23;\n\tsubc.cc.u32 %7,%16,%24;\n\t"
      "subc.u32 %8,0,0;"
      : "=r"(r.v[0]), "=r"(r.v[1]), "=r"(r.v[2]), "=r"(r.v[3]), "=r"(r.v[4]), "=r"(r.v[5]), "=r"(r.v[6]), "=r"(r.v[7]),
        "=r"(c)
      : "r"(a.v[0]), "r"(a.v[1]), "r"(a.v[2]), "r"(a.v[3]), "r"(a.v[4]), "r"(a.v[5]), "r"(a.v[6]), "r"(a.v[7]),
        "r"(b.v[0]), "r"(b.v[1]), "r"(b.v[2]), "r"(b.v[3]), "r"(b.v[4]), "r"(b.v[5]), "r"(b.v[6]), "r"(b.v[7]));
  // c = 0 or 0xFFFFFFFF (borrow).  a-b+2^256 = a-b+C (mod p)  =>  subtract C on borrow.
  uint32_t m = c & 1u, k = m * IBFT_PC, c2;
  asm("sub.cc.u32 %0,%0,%9;\n\tsubc.cc.u32 %1,%1,%10;\n\tsubc.cc.u32 %2,%2,0;\n\tsubc.cc.u32 %3,%3,0;\n\t"
      "subc.cc.u32 %4,%4,0;\n\tsubc.cc.u32 %5,%5,0;\n\tsubc.cc.u32 %6,%6,0;\n\tsubc.cc.u32 %7,%7,0;\n\t"
      "subc.u32 %8,0,0;"
      : "+r"(r.v[0]), "+r"(r.v[1]), "+r"(r.v[2]), "+r"(r.v[3]), "+r"(r.v[4]), "+r"(r.v[5]), "+r"(r.v[6]), "+r"(r.v[7]),
        "=r"(c2)
      : "r"(k), "r"(m));
  // a second borrow leaves a value >= 2^256 - 2^34: subtracting C again cannot ripple past limb 2
  uint32_t m2 = c2 & 1u, k2 = m2 * IBFT_PC;
  asm("sub.cc.u32 %0,%0,%3;\n\tsubc.cc.u32 %1,%1,%4;\n\tsubc.u32 %2,%2,0;"
      : "+r"(r.v[0]), "+r"(r.v[1]), "+r"(r.v[2])
      : "r"(k2), "r"(m2));
#else
  int64_t c = 0;
  for (int i = 0; i < 8; i++) {
    c += (int64_t)a.v[i] - (int64_t)b.v[i];
    r.v[i] = (uint32_t)c;
    c >>= 32;  // arithmetic shift: 0 or -1
  }
  uint32_t m = (uint32_t)(-c);
  int64_t d = (int64_t)r.v[0] - (int64_t)(m * IBFT_PC);
  r.v[0] = (uint32_t)d;
  d >>= 32;
  d += (int64_t)r.v[1] - (int64_t)m;
  r.v[1] = (uint32_t)d;
  d >>= 32;
  for (int i = 2; i < 8; i++) {
    d += (int64_t)r.v[i];
    r.v[i] = (uint32_t)d;
    d >>= 32;
  }
  uint32_t m2 = (uint32_t)(-d);
  d = (int64_t)r.v[0] - (int64_t)(m2 * IBFT_PC);
  r.v[0] = (uint32_t)d;
  d >>= 32;
  d += (int64_t)r.v[1] - (int64_t)m2;
  r.v[1] = (uint32_t)d;
  d >>= 32;
  r.v[2] += (uint32_t)d;
#endif
  return r;
}

IBFT_HD fe fe_neg(const fe& a) { return fe_sub(fe_zero(), a); }
IBFT_HD fe fe_dbl(const fe& a) { return fe_add(a, a); }

// canonical representative in [0, p)
IBFT_HD fe fe_normalize(const fe& a) {
  // a < 2^256 < 2p, so at most one subtraction of p.  a >= p  <=>  a + C overflows 2^256.
  fe t;
  uint64_t c = (uint64_t)a.v[0] + IBFT_PC;
  t.v[0] = (uint32_t)c;
  c >>= 32;
  c += (uint64_t)a.v[1] + 1u;
  t.v[1] = (uint32_t)c;
  c >>= 32;
#pragma unroll
  for (int i = 2; i < 8; i++) {
    c += a.v[i];
    t.v[i] = (uint32_t)c;
    c >>= 32;
  }
  // if carry out, a >= p and a - p = a + C - 2^256 = t
  fe r;
  uint32_t ge = (uint32_t)c;
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = ge ? t.v[i] : a.v[i];
  return r;
}

IBFT_HD bool fe_is_zero(const fe& a) {
  // zero mod p: a == 0 or a == p
  uint32_t z = a.v[0] | a.v[1] | a.v[2] | a.v[3] | a.v[4] | a.v[5] | a.v[6] | a.v[7];
  uint32_t q = (a.v[0] ^ IBFT_P0) | (a.v[1] ^ IBFT_P1) | ~a.v[2] | ~a.v[3] | ~a.v[4] | ~a.v[5] | ~a.v[6] | ~a.v[7];
  return z == 0 || q == 0;
}
IBFT_HD bool fe_equal(const fe& a, const fe& b) { return fe_is_zero(fe_sub(a, b)); }
IBFT_HD bool fe_is_odd(const fe& a) { return fe_normalize(a).v[0] & 1u; }

// ------------------------------------------------------------------------------------------------
// 256 x 256 -> 512 product
// ------------------------------------------------------------------------------------------------
#if IBFT_PTX
// acc pairs (p0,p1),(p2,p3),(p4,p5),(p6,p7) += x0*y, x1*y, x2*y, x3*y as one carry chain; returns carry out.
__device__ __forceinline__ uint32_t mad_chain4(uint32_t& p0, uint32_t& p1, uint32_t& p2, uint32_t& p3, uint32_t& p4,
                                               uint32_t& p5, uint32_t& p6, uint32_t& p7, uint32_t x0, uint32_t x1,
                                               uint32_t x2, uint32_t x3, uint32_t y) {
  uint32_t co;
  asm("mad.lo.cc.u32 %0,%9,%13,%0;\n\tmadc.hi.cc.u32 %1,%9,%13,%1;\n\t"
      "madc.lo.cc.u32 %2,%10,%13,%2;\n\tmadc.hi.cc.u32 %3,%10,%13,%3;\n\t"
      "madc.lo.cc.u32 %4,%11,%13,%4;\n\tmadc.hi.cc.u32 %5,%11,%13,%5;\n\t"
      "madc.lo.cc.u32 %6,%12,%13,%6;\n\tmadc.hi.cc.u32 %7,%12,%13,%7;\n\t"
      "addc.u32 %8,0,0;"
      : "+r"(p0), "+r"(p1), "+r"(p2), "+r"(p3), "+r"(p4), "+r"(p5), "+r"(p6), "+r"(p7), "=r"(co)
      : "r"(x0), "r"(x1), "r"(x2), "r"(x3), "r"(y));
  return co;
}
// same, when the top pair is known to hold only a 0/1 carry: the chain cannot carry out.
__device__ __forceinline__ void mad_chain4_nc(uint32_t& p0, uint32_t& p1, uint32_t& p2, uint32_t& p3, uint32_t& p4,
                                              uint32_t& p5, uint32_t& p6, uint32_t& p7, uint32_t x0, uint32_t x1,
                                              uint32_t x2, uint32_t x3, uint32_t y) {
  asm("mad.lo.cc.u32 %0,%8,%12,%0;\n\tmadc.hi.cc.u32 %1,%8,%12,%1;\n\t"
      "madc.lo.cc.u32 %2,%9,%12,%2;\n\tmadc.hi.cc.u32 %3,%9,%12,%3;\n\t"
      "madc.lo.cc.u32 %4,%10,%12,%4;\n\tmadc.hi.cc.u32 %5,%10,%12,%5;\n\t"
      "madc.lo.cc.u32 %6,%11,%12,%6;\n\tmadc.hi.u32 %7,%11,%12,%7;"
      : "+r"(p0), "+r"(p1), "+r"(p2), "+r"(p3), "+r"(p4), "+r"(p5), "+r"(p6), "+r"(p7)
      : "r"(x0), "r"(x1), "r"(x2), "r"(x3), "r"(y));
}
// both halves of the top pair are fresh: they are written with literal-zero addends, so no register has to be
// zero-initialised beforehand (moves on the FMA pipe, which is the busy one)
__device__ __forceinline__ void mad_chain4_nczz(uint32_t& p0, uint32_t& p1, uint32_t& p2, uint32_t& p3, uint32_t& p4,
                                                uint32_t& p5, uint32_t& p6_out, uint32_t& p7_out, uint32_t x0, uint32_t x1,
                                                uint32_t x2, uint32_t x3, uint32_t y) {
  asm("mad.lo.cc.u32 %0,%8,%12,%0;\n\tmadc.hi.cc.u32 %1,%8,%12,%1;\n\t"
      "madc.lo.cc.u32 %2,%9,%12,%2;\n\tmadc.hi.cc.u32 %3,%9,%12,%3;\n\t"
      "madc.lo.cc.u32 %4,%10,%12,%4;\n\tmadc.hi.cc.u32 %5,%10,%12,%5;\n\t"
      "madc.lo.cc.u32 %6,%11,%12,0;\n\tmadc.hi.u32 %7,%11,%12,0;"
      : "+r"(p0), "+r"(p1), "+r"(p2), "+r"(p3), "+r"(p4), "+r"(p5), "=r"(p6_out), "=r"(p7_out)
      : "r"(x0), "r"(x1), "r"(x2), "r"(x3), "r"(y));
}
// acc pairs (p0,p1),(p2,p3),(p4,p5),(p6,p7) += x0*y, x1*y, x2*y, x3*y, the carry out rippled into (p8, p9), which the caller
// guarantees cannot carry out.  Used where the pair above the chain has already been written by a later row: a carry never
// has to sit in a register pair whose other half is a materialised zero (an IMAD.MOV on the FMA pipe).
__device__ __forceinline__ void mad_chain4_r2(uint32_t& p0, uint32_t& p1, uint32_t& p2, uint32_t& p3, uint32_t& p4, uint32_t& p5,
                                              uint32_t& p6, uint32_t& p7, uint32_t& p8, uint32_t& p9, uint32_t x0, uint32_t x1,
                                              uint32_t x2, uint32_t x3, uint32_t y) {
  asm("mad.lo.cc.u32 %0,%10,%14,%0;\n\tmadc.hi.cc.u32 %1,%10,%14,%1;\n\t"
      "madc.lo.cc.u32 %2,%11,%14,%2;\n\tmadc.hi.cc.u32 %3,%11,%14,%3;\n\t"
      "madc.lo.cc.u32 %4,%12,%14,%4;\n\tmadc.hi.cc.u32 %5,%12,%14,%5;\n\t"
      "madc.lo.cc.u32 %6,%13,%14,%6;\n\tmadc.hi.cc.u32 %7,%13,%14,%7;\n\t"
      "addc.cc.u32 %8,%8,0;\n\taddc.u32 %9,%9,0;"
      : "+r"(p0), "+r"(p1), "+r"(p2), "+r"(p3), "+r"(p4), "+r"(p5), "+r"(p6), "+r"(p7), "+r"(p8), "+r"(p9)
      : "r"(x0), "r"(x1), "r"(x2), "r"(x3), "r"(y));
}
__device__ __forceinline__ void mulw(uint32_t& lo, uint32_t& hi, uint32_t x, uint32_t y) {
  asm("mul.lo.u32 %0,%2,%3;\n\tmul.hi.u32 %1,%2,%3;" : "=r"(lo), "=r"(hi) : "r"(x), "r"(y));
}
#endif

#if IBFT_PTX
// ---- 4x4-limb product with the even/odd carry-chain layout; "fresh" accumulator halves use literal-zero addends
__device__ __forceinline__ void mul4x4(uint32_t* R, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                       uint32_t b1, uint32_t b2, uint32_t b3) {
  uint32_t E0, E1, E2, E3, E4, E5, E6, E7, O0, O1, O2, O3, O4, O5, O6;
  // row 0
  mulw(E0, E1, a0, b0); mulw(E2, E3, a2, b0);
  mulw(O0, O1, a1, b0); mulw(O2, O3, a3, b0);
  // row 1: O idx 0,2 (x = a0,a2) carry -> O4 ; E idx 2,4 (x = a1,a3), (E4,E5) fresh
  asm("mad.lo.cc.u32 %0,%5,%7,%0;\n\tmadc.hi.cc.u32 %1,%5,%7,%1;\n\tmadc.lo.cc.u32 %2,%6,%7,%2;\n\tmadc.hi.cc.u32 %3,%6,%7,%3;\n\t"
      "addc.u32 %4,0,0;"
      : "+r"(O0), "+r"(O1), "+r"(O2), "+r"(O3), "=r"(O4) : "r"(a0), "r"(a2), "r"(b1));
  asm("mad.lo.cc.u32 %0,%4,%6,%0;\n\tmadc.hi.cc.u32 %1,%4,%6,%1;\n\tmadc.lo.cc.u32 %2,%5,%6,0;\n\tmadc.hi.u32 %3,%5,%6,0;"
      : "+r"(E2), "+r"(E3), "=r"(E4), "=r"(E5) : "r"(a1), "r"(a3), "r"(b1));
  // row 2: E idx 2,4 (x = a0,a2) carry -> E6 ; O idx 2,4 (x = a1,a3), (O4,O5) = (carry, fresh)
  asm("mad.lo.cc.u32 %0,%5,%7,%0;\n\tmadc.hi.cc.u32 %1,%5,%7,%1;\n\tmadc.lo.cc.u32 %2,%6,%7,%2;\n\tmadc.hi.cc.u32 %3,%6,%7,%3;\n\t"
      "addc.u32 %4,0,0;"
      : "+r"(E2), "+r"(E3), "+r"(E4), "+r"(E5), "=r"(E6) : "r"(a0), "r"(a2), "r"(b2));
  asm("mad.lo.cc.u32 %0,%4,%6,%0;\n\tmadc.hi.cc.u32 %1,%4,%6,%1;\n\tmadc.lo.cc.u32 %2,%5,%6,%2;\n\tmadc.hi.u32 %3,%5,%6,0;"
      : "+r"(O2), "+r"(O3), "+r"(O4), "=r"(O5) : "r"(a1), "r"(a3), "r"(b2));
  // row 3: O idx 2,4 (x = a0,a2) carry -> O6 ; E idx 4,6 (x = a1,a3), (E6,E7) = (carry, fresh)
  asm("mad.lo.cc.u32 %0,%5,%7,%0;\n\tmadc.hi.cc.u32 %1,%5,%7,%1;\n\tmadc.lo.cc.u32 %2,%6,%7,%2;\n\tmadc.hi.cc.u32 %3,%6,%7,%3;\n\t"
      "addc.u32 %4,0,0;"
      : "+r"(O2), "+r"(O3), "+r"(O4), "+r"(O5), "=r"(O6) : "r"(a0), "r"(a2), "r"(b3));
  asm("mad.lo.cc.u32 %0,%4,%6,%0;\n\tmadc.hi.cc.u32 %1,%4,%6,%1;\n\tmadc.lo.cc.u32 %2,%5,%6,%2;\n\tmadc.hi.u32 %3,%5,%6,0;"
      : "+r"(E4), "+r"(E5), "+r"(E6), "=r"(E7) : "r"(a1), "r"(a3), "r"(b3));
  // R = E + (O << 32)
  R[0] = E0;
  asm("add.cc.u32 %0,%7,%14;\n\taddc.cc.u32 %1,%8,%15;\n\taddc.cc.u32 %2,%9,%16;\n\taddc.cc.u32 %3,%10,%17;\n\t"
      "addc.cc.u32 %4,%11,%18;\n\taddc.cc.u32 %5,%12,%19;\n\taddc.u32 %6,%13,%20;"
      : "=r"(R[1]), "=r"(R[2]), "=r"(R[3]), "=r"(R[4]), "=r"(R[5]), "=r"(R[6]), "=r"(R[7])
      : "r"(E1), "r"(E2), "r"(E3), "r"(E4), "r"(E5), "r"(E6), "r"(E7), "r"(O0), "r"(O1), "r"(O2), "r"(O3), "r"(O4), "r"(O5), "r"(O6));
}

// |x - y| for 4-limb operands; returns the sign mask (0xFFFFFFFF when x < y)
__device__ __forceinline__ uint32_t absdiff4(uint32_t* d, const uint32_t* x, const uint32_t* y) {
  uint32_t m;
  asm("sub.cc.u32 %0,%5,%9;\n\tsubc.cc.u32 %1,%6,%10;\n\tsubc.cc.u32 %2,%7,%11;\n\tsubc.cc.u32 %3,%8,%12;\n\tsubc.u32 %4,0,0;"
      : "=r"(d[0]), "=r"(d[1]), "=r"(d[2]), "=r"(d[3]), "=r"(m)
      : "r"(x[0]), "r"(x[1]), "r"(x[2]), "r"(x[3]), "r"(y[0]), "r"(y[1]), "r"(y[2]), "r"(y[3]));
  // conditional two's-complement negation: (d ^ m) - m
  uint32_t t0 = d[0] ^ m, t1 = d[1] ^ m, t2 = d[2] ^ m, t3 = d[3] ^ m;
  asm("sub.cc.u32 %0,%4,%8;\n\tsubc.cc.u32 %1,%5,%8;\n\tsubc.cc.u32 %2,%6,%8;\n\tsubc.u32 %3,%7,%8;"
      : "=r"(d[0]), "=r"(d[1]), "=r"(d[2]), "=r"(d[3]) : "r"(t0), "r"(t1), "r"(t2), "r"(t3), "r"(m));
  return m;
}
#endif

// R[0..15] = a * b
IBFT_HD void mul_wide_8x8(uint32_t* R, const uint32_t* a, const uint32_t* b) {
#if IBFT_PTX && defined(IBFT_KARATSUBA)
  // OPT-IN (slower in practice, see DESIGN.md): one level of (subtractive) Karatsuba, 48 wide MACs instead of 64.  The IMAD.WIDE pipe is the bottleneck of the whole
  // kernel (4 issue cycles per warp-instruction) while the ALU pipe that takes the ~70 extra add/xor instructions is
  // less than half used, so trading 16 MACs for carry-chain adds looks like a win on paper.
  //   a*b = z0 + (z0 + z2 + (a0-a1)(b1-b0)) 2^128 + z2 2^256
  uint32_t z0[8], z2[8], m[8], da[4], db[4];
  mul4x4(z0, a[0], a[1], a[2], a[3], b[0], b[1], b[2], b[3]);
  mul4x4(z2, a[4], a[5], a[6], a[7], b[4], b[5], b[6], b[7]);
  uint32_t sa = absdiff4(da, a, a + 4);      // a0 - a1
  uint32_t sb = absdiff4(db, b + 4, b);      // b1 - b0
  mul4x4(m, da[0], da[1], da[2], da[3], db[0], db[1], db[2], db[3]);
  uint32_t s = sa ^ sb;                      // all-ones: the cross term is negative
  // z1 = z0 + z2 (9 limbs)
  uint32_t z1[9];
  asm("add.cc.u32 %0,%9,%17;\n\taddc.cc.u32 %1,%10,%18;\n\taddc.cc.u32 %2,%11,%19;\n\taddc.cc.u32 %3,%12,%20;\n\t"
      "addc.cc.u32 %4,%13,%21;\n\taddc.cc.u32 %5,%14,%22;\n\taddc.cc.u32 %6,%15,%23;\n\taddc.cc.u32 %7,%16,%24;\n\t"
      "addc.u32 %8,0,0;"
      : "=r"(z1[0]), "=r"(z1[1]), "=r"(z1[2]), "=r"(z1[3]), "=r"(z1[4]), "=r"(z1[5]), "=r"(z1[6]), "=r"(z1[7]), "=r"(z1[8])
      : "r"(z0[0]), "r"(z0[1]), "r"(z0[2]), "r"(z0[3]), "r"(z0[4]), "r"(z0[5]), "r"(z0[6]), "r"(z0[7]), "r"(z2[0]), "r"(z2[1]),
        "r"(z2[2]), "r"(z2[3]), "r"(z2[4]), "r"(z2[5]), "r"(z2[6]), "r"(z2[7]));
  // z1 += (-1)^s m :  z1 + (m ^ s) + (s & 1), and the 2^256 that the complement adds is taken back from the top limb
  uint32_t x0 = m[0] ^ s, x1 = m[1] ^ s, x2 = m[2] ^ s, x3 = m[3] ^ s, x4 = m[4] ^ s, x5 = m[5] ^ s, x6 = m[6] ^ s, x7 = m[7] ^ s;
  uint32_t scr;
  asm("add.cc.u32 %9,%18,0xFFFFFFFF;\n\t"  // carry flag <- (s != 0)
      "addc.cc.u32 %0,%0,%10;\n\taddc.cc.u32 %1,%1,%11;\n\taddc.cc.u32 %2,%2,%12;\n\taddc.cc.u32 %3,%3,%13;\n\t"
      "addc.cc.u32 %4,%4,%14;\n\taddc.cc.u32 %5,%5,%15;\n\taddc.cc.u32 %6,%6,%16;\n\taddc.cc.u32 %7,%7,%17;\n\t"
      "addc.u32 %8,%8,%18;"  // top limb: + carry, and - 1 (adding 0xFFFFFFFF) when the term was subtracted
      : "+r"(z1[0]), "+r"(z1[1]), "+r"(z1[2]), "+r"(z1[3]), "+r"(z1[4]), "+r"(z1[5]), "+r"(z1[6]), "+r"(z1[7]), "+r"(z1[8]),
        "=&r"(scr)
      : "r"(x0), "r"(x1), "r"(x2), "r"(x3), "r"(x4), "r"(x5), "r"(x6), "r"(x7), "r"(s));
  // R = z0 + z1 2^128 + z2 2^256
  R[0] = z0[0]; R[1] = z0[1]; R[2] = z0[2]; R[3] = z0[3];
  asm("add.cc.u32 %0,%12,%24;\n\taddc.cc.u32 %1,%13,%25;\n\taddc.cc.u32 %2,%14,%26;\n\taddc.cc.u32 %3,%15,%27;\n\t"
      "addc.cc.u32 %4,%16,%28;\n\taddc.cc.u32 %5,%17,%29;\n\taddc.cc.u32 %6,%18,%30;\n\taddc.cc.u32 %7,%19,%31;\n\t"
      "addc.cc.u32 %8,%20,%32;\n\taddc.cc.u32 %9,%21,0;\n\taddc.cc.u32 %10,%22,0;\n\taddc.u32 %11,%23,0;"
      : "=r"(R[4]), "=r"(R[5]), "=r"(R[6]), "=r"(R[7]), "=r"(R[8]), "=r"(R[9]), "=r"(R[10]), "=r"(R[11]), "=r"(R[12]),
        "=r"(R[13]), "=r"(R[14]), "=r"(R[15])
      : "r"(z0[4]), "r"(z0[5]), "r"(z0[6]), "r"(z0[7]), "r"(z2[0]), "r"(z2[1]), "r"(z2[2]), "r"(z2[3]), "r"(z2[4]), "r"(z2[5]),
        "r"(z2[6]), "r"(z2[7]), "r"(z1[0]), "r"(z1[1]), "r"(z1[2]), "r"(z1[3]), "r"(z1[4]), "r"(z1[5]), "r"(z1[6]), "r"(z1[7]),
        "r"(z1[8]));
#elif IBFT_PTX
  // E[k] sits at limb position k, O[k] at position k+1 (see DESIGN.md "field multiplier").  No accumulator is ever
  // zero-initialised: fresh halves are produced by literal-zero addends, carries by addc.  Rows are taken in pairs so that no
  // carry word is ever paired with a materialised zero either: the LATER row's chain runs first and writes the top pair fresh,
  // then the earlier row's chain ripples its carry into that pair (every partial sum is a partial product: nothing overflows).
  uint32_t E[16], O[15];
  mulw(E[0], E[1], a[0], b[0]); mulw(E[2], E[3], a[2], b[0]); mulw(E[4], E[5], a[4], b[0]); mulw(E[6], E[7], a[6], b[0]);
  mulw(O[0], O[1], a[1], b[0]); mulw(O[2], O[3], a[3], b[0]); mulw(O[4], O[5], a[5], b[0]); mulw(O[6], O[7], a[7], b[0]);
  // row 1, E: indices 2..9 where (E[8], E[9]) are both fresh
  mad_chain4_nczz(E[2], E[3], E[4], E[5], E[6], E[7], E[8], E[9], a[1], a[3], a[5], a[7], b[1]);
#pragma unroll
  for (int i = 1; i < 7; i++) {
    if (i & 1) {  // O: row i+1 with (O[i+7], O[i+8]) fresh, then row i rippling into them
      mad_chain4_nczz(O[i + 1], O[i + 2], O[i + 3], O[i + 4], O[i + 5], O[i + 6], O[i + 7], O[i + 8], a[1], a[3], a[5], a[7], b[i + 1]);
      mad_chain4_r2(O[i - 1], O[i], O[i + 1], O[i + 2], O[i + 3], O[i + 4], O[i + 5], O[i + 6], O[i + 7], O[i + 8], a[0], a[2], a[4],
                    a[6], b[i]);
    } else {      // E: row i+1 with (E[i+8], E[i+9]) fresh, then row i rippling into them
      mad_chain4_nczz(E[i + 2], E[i + 3], E[i + 4], E[i + 5], E[i + 6], E[i + 7], E[i + 8], E[i + 9], a[1], a[3], a[5], a[7], b[i + 1]);
      mad_chain4_r2(E[i], E[i + 1], E[i + 2], E[i + 3], E[i + 4], E[i + 5], E[i + 6], E[i + 7], E[i + 8], E[i + 9], a[0], a[2], a[4],
                    a[6], b[i]);
    }
  }
  // row 7, O: indices 6..13, carry out -> O[14]
  O[14] = mad_chain4(O[6], O[7], O[8], O[9], O[10], O[11], O[12], O[13], a[0], a[2], a[4], a[6], b[7]);
  // R = E + (O << 32)
  R[0] = E[0];
  asm("add.cc.u32 %0,%15,%30;\n\taddc.cc.u32 %1,%16,%31;\n\taddc.cc.u32 %2,%17,%32;\n\taddc.cc.u32 %3,%18,%33;\n\t"
      "addc.cc.u32 %4,%19,%34;\n\taddc.cc.u32 %5,%20,%35;\n\taddc.cc.u32 %6,%21,%36;\n\taddc.cc.u32 %7,%22,%37;\n\t"
      "addc.cc.u32 %8,%23,%38;\n\taddc.cc.u32 %9,%24,%39;\n\taddc.cc.u32 %10,%25,%40;\n\taddc.cc.u32 %11,%26,%41;\n\t"
      "addc.cc.u32 %12,%27,%42;\n\taddc.cc.u32 %13,%28,%43;\n\taddc.u32 %14,%29,%44;"
      : "=r"(R[1]), "=r"(R[2]), "=r"(R[3]), "=r"(R[4]), "=r"(R[5]), "=r"(R[6]), "=r"(R[7]), "=r"(R[8]), "=r"(R[9]),
        "=r"(R[10]), "=r"(R[11]), "=r"(R[12]), "=r"(R[13]), "=r"(R[14]), "=r"(R[15])
      : "r"(E[1]), "r"(E[2]), "r"(E[3]), "r"(E[4]), "r"(E[5]), "r"(E[6]), "r"(E[7]), "r"(E[8]), "r"(E[9]), "r"(E[10]),
        "r"(E[11]), "r"(E[12]), "r"(E[13]), "r"(E[14]), "r"(E[15]), "r"(O[0]), "r"(O[1]), "r"(O[2]), "r"(O[3]), "r"(O[4]),
        "r"(O[5]), "r"(O[6]), "r"(O[7]), "r"(O[8]), "r"(O[9]), "r"(O[10]), "r"(O[11]), "r"(O[12]), "r"(O[13]), "r"(O[14]));
#else
  for (int i = 0; i < 16; i++) R[i] = 0;
  for (int i = 0; i < 8; i++) {
    uint64_t c = 0;
    for (int j = 0; j < 8; j++) {
      c += (uint64_t)a[j] * b[i] + R[i + j];
      R[i + j] = (uint32_t)c;
      c >>= 32;
    }
    R[i + 8] = (uint32_t)c;
  }
#endif
}

// R[0..15] -> value mod p (weakly reduced): L + H*(2^32 + 977)
IBFT_HD fe fe_reduce512(const uint32_t* R) {
  fe r;
#if IBFT_PTX
  uint32_t S[8], s8, s9;
#if defined(IBFT_REDUCE_SHIFT)
  // H*977 on the ALU pipe instead of 8 wide MACs on the (saturated) FMA pipe: 977 = 2^10 - 2^6 + 2^4 + 1, so
  // T = (H<<10) - (H<<6) + (H<<4) + H with funnel shifts and three carry chains (9 limbs, T[8] < 2^10).
  {
    const uint32_t* H = R + 8;
    uint32_t A[9], B6[9], B4[9];
    A[0] = H[0] << 10; B6[0] = H[0] << 6; B4[0] = H[0] << 4;
#pragma unroll
    for (int i = 1; i < 8; i++) {
      A[i] = __funnelshift_l(H[i - 1], H[i], 10);
      B6[i] = __funnelshift_l(H[i - 1], H[i], 6);
      B4[i] = __funnelshift_l(H[i - 1], H[i], 4);
    }
    A[8] = H[7] >> 22; B6[8] = H[7] >> 26; B4[8] = H[7] >> 28;
    uint32_t U[9];  // U = B4 + H
    asm("add.cc.u32 %0,%9,%18;\n\taddc.cc.u32 %1,%10,%19;\n\taddc.cc.u32 %2,%11,%20;\n\taddc.cc.u32 %3,%12,%21;\n\t"
        "addc.cc.u32 %4,%13,%22;\n\taddc.cc.u32 %5,%14,%23;\n\taddc.cc.u32 %6,%15,%24;\n\taddc.cc.u32 %7,%16,%25;\n\t"
        "addc.u32 %8,%17,0;"
        : "=r"(U[0]), "=r"(U[1]), "=r"(U[2]), "=r"(U[3]), "=r"(U[4]), "=r"(U[5]), "=r"(U[6]), "=r"(U[7]), "=r"(U[8])
        : "r"(B4[0]), "r"(B4[1]), "r"(B4[2]), "r"(B4[3]), "r"(B4[4]), "r"(B4[5]), "r"(B4[6]), "r"(B4[7]), "r"(B4[8]), "r"(H[0]), "r"(H[1]),
          "r"(H[2]), "r"(H[3]), "r"(H[4]), "r"(H[5]), "r"(H[6]), "r"(H[7]));
    // U = U + A - B6   (two chains; every partial result fits in 9 limbs and the final one is non-negative)
    asm("add.cc.u32 %0,%0,%9;\n\taddc.cc.u32 %1,%1,%10;\n\taddc.cc.u32 %2,%2,%11;\n\taddc.cc.u32 %3,%3,%12;\n\t"
        "addc.cc.u32 %4,%4,%13;\n\taddc.cc.u32 %5,%5,%14;\n\taddc.cc.u32 %6,%6,%15;\n\taddc.cc.u32 %7,%7,%16;\n\t"
        "addc.u32 %8,%8,%17;"
        : "+r"(U[0]), "+r"(U[1]), "+r"(U[2]), "+r"(U[3]), "+r"(U[4]), "+r"(U[5]), "+r"(U[6]), "+r"(U[7]), "+r"(U[8])
        : "r"(A[0]), "r"(A[1]), "r"(A[2]), "r"(A[3]), "r"(A[4]), "r"(A[5]), "r"(A[6]), "r"(A[7]), "r"(A[8]));
    asm("sub.cc.u32 %0,%0,%9;\n\tsubc.cc.u32 %1,%1,%10;\n\tsubc.cc.u32 %2,%2,%11;\n\tsubc.cc.u32 %3,%3,%12;\n\t"
        "subc.cc.u32 %4,%4,%13;\n\tsubc.cc.u32 %5,%5,%14;\n\tsubc.cc.u32 %6,%6,%15;\n\tsubc.cc.u32 %7,%7,%16;\n\t"
        "subc.u32 %8,%8,%17;"
        : "+r"(U[0]), "+r"(U[1]), "+r"(U[2]), "+r"(U[3]), "+r"(U[4]), "+r"(U[5]), "+r"(U[6]), "+r"(U[7]), "+r"(U[8])
        : "r"(B6[0]), "r"(B6[1]), "r"(B6[2]), "r"(B6[3]), "r"(B6[4]), "r"(B6[5]), "r"(B6[6]), "r"(B6[7]), "r"(B6[8]));
    // S = L + T[0..7], s8 = T[8] + carry
    asm("add.cc.u32 %0,%9,%17;\n\taddc.cc.u32 %1,%10,%18;\n\taddc.cc.u32 %2,%11,%19;\n\taddc.cc.u32 %3,%12,%20;\n\t"
        "addc.cc.u32 %4,%13,%21;\n\taddc.cc.u32 %5,%14,%22;\n\taddc.cc.u32 %6,%15,%23;\n\taddc.cc.u32 %7,%16,%24;\n\t"
        "addc.u32 %8,%25,0;"
        : "=r"(S[0]), "=r"(S[1]), "=r"(S[2]), "=r"(S[3]), "=r"(S[4]), "=r"(S[5]), "=r"(S[6]), "=r"(S[7]), "=r"(s8)
        : "r"(R[0]), "r"(R[1]), "r"(R[2]), "r"(R[3]), "r"(R[4]), "r"(R[5]), "r"(R[6]), "r"(R[7]), "r"(U[0]), "r"(U[1]), "r"(U[2]),
          "r"(U[3]), "r"(U[4]), "r"(U[5]), "r"(U[6]), "r"(U[7]), "r"(U[8]));
    s9 = 0;
  }
  // S[1..8] += H ; S[9] += carry
  asm("add.cc.u32 %0,%0,%9;\n\taddc.cc.u32 %1,%1,%10;\n\taddc.cc.u32 %2,%2,%11;\n\taddc.cc.u32 %3,%3,%12;\n\t"
      "addc.cc.u32 %4,%4,%13;\n\taddc.cc.u32 %5,%5,%14;\n\taddc.cc.u32 %6,%6,%15;\n\taddc.cc.u32 %7,%7,%16;\n\t"
      "addc.u32 %8,%8,0;"
      : "+r"(S[1]), "+r"(S[2]), "+r"(S[3]), "+r"(S[4]), "+r"(S[5]), "+r"(S[6]), "+r"(S[7]), "+r"(s8), "+r"(s9)
      : "r"(R[8]), "r"(R[9]), "r"(R[10]), "r"(R[11]), "r"(R[12]), "r"(R[13]), "r"(R[14]), "r"(R[15]));
#else
  // S = L + H*977 + (H << 32) in two accumulators whose 64-bit addends are exactly the limb pairs the product leaves behind,
  // (L0,L1), (L2,L3), ... and (H0,H1), (H2,H3), ..., so that no limb is re-paired (copied) between chains:
  //   even: (L0,L1) += H0*977, (L2,L3) += H2*977, ...   limbs 0..7, carry -> e8
  //   odd:  (H0,H1) += H1*977, (H2,H3) += H3*977, ...   limbs 1..8, carry -> o9
  // and one add chain S = even + (odd << 32).  Each accumulator is < 978 * 2^256, so s9:s8 < 2^34 as before.
  uint32_t e0 = R[0], e1 = R[1], e2 = R[2], e3 = R[3], e4 = R[4], e5 = R[5], e6 = R[6], e7 = R[7], e8;
  uint32_t o1 = R[8], o2 = R[9], o3 = R[10], o4 = R[11], o5 = R[12], o6 = R[13], o7 = R[14], o8 = R[15], o9;
  e8 = mad_chain4(e0, e1, e2, e3, e4, e5, e6, e7, R[8], R[10], R[12], R[14], IBFT_PC);
  o9 = mad_chain4(o1, o2, o3, o4, o5, o6, o7, o8, R[9], R[11], R[13], R[15], IBFT_PC);
  S[0] = e0;
  asm("add.cc.u32 %0,%9,%17;\n\taddc.cc.u32 %1,%10,%18;\n\taddc.cc.u32 %2,%11,%19;\n\taddc.cc.u32 %3,%12,%20;\n\t"
      "addc.cc.u32 %4,%13,%21;\n\taddc.cc.u32 %5,%14,%22;\n\taddc.cc.u32 %6,%15,%23;\n\taddc.cc.u32 %7,%16,%24;\n\t"
      "addc.u32 %8,%25,0;"
      : "=r"(S[1]), "=r"(S[2]), "=r"(S[3]), "=r"(S[4]), "=r"(S[5]), "=r"(S[6]), "=r"(S[7]), "=r"(s8), "=r"(s9)
      : "r"(e1), "r"(e2), "r"(e3), "r"(e4), "r"(e5), "r"(e6), "r"(e7), "r"(e8), "r"(o1), "r"(o2), "r"(o3), "r"(o4), "r"(o5),
        "r"(o6), "r"(o7), "r"(o8), "r"(o9));
#endif
  // e = s9:s8 (< 2^34); g = e * (2^32 + 977) (< 2^67) as three limbs
  uint64_t m = (uint64_t)s8 * IBFT_PC + (((uint64_t)(s9 * IBFT_PC)) << 32);
  uint64_t mid = (m >> 32) + s8;
  uint32_t g0 = (uint32_t)m, g1 = (uint32_t)mid, g2 = (uint32_t)(mid >> 32) + s9, k;
  asm("add.cc.u32 %0,%0,%9;\n\taddc.cc.u32 %1,%1,%10;\n\taddc.cc.u32 %2,%2,%11;\n\taddc.cc.u32 %3,%3,0;\n\t"
      "addc.cc.u32 %4,%4,0;\n\taddc.cc.u32 %5,%5,0;\n\taddc.cc.u32 %6,%6,0;\n\taddc.cc.u32 %7,%7,0;\n\t"
      "addc.u32 %8,0,0;"
      : "+r"(S[0]), "+r"(S[1]), "+r"(S[2]), "+r"(S[3]), "+r"(S[4]), "+r"(S[5]), "+r"(S[6]), "+r"(S[7]), "=r"(k)
      : "r"(g0), "r"(g1), "r"(g2));
  uint32_t kk = k * IBFT_PC;
  asm("add.cc.u32 %0,%0,%3;\n\taddc.cc.u32 %1,%1,%4;\n\taddc.u32 %2,%2,0;"
      : "+r"(S[0]), "+r"(S[1]), "+r"(S[2])
      : "r"(kk), "r"(k));
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = S[i];
#else
  uint32_t S[10];
  uint64_t c = 0;
  // S = L + H*977
  for (int i = 0; i < 8; i++) {
    c += (uint64_t)R[8 + i] * IBFT_PC + R[i];
    S[i] = (uint32_t)c;
    c >>= 32;
  }
  S[8] = (uint32_t)c;
  S[9] = 0;
  // S += H << 32
  c = 0;
  for (int i = 0; i < 8; i++) {
    c += (uint64_t)S[i + 1] + R[8 + i];
    S[i + 1] = (uint32_t)c;
    c >>= 32;
  }
  S[9] = (uint32_t)c;
  uint64_t e = (uint64_t)S[8] | ((uint64_t)S[9] << 32);  // < 2^34
  // g = e*(2^32+977) as three limbs
  uint64_t m = e * IBFT_PC;
  uint64_t mid = (m >> 32) + (uint32_t)e;
  uint32_t g0 = (uint32_t)m, g1 = (uint32_t)mid, g2 = (uint32_t)(mid >> 32) + (uint32_t)(e >> 32);
  c = (uint64_t)S[0] + g0;
  S[0] = (uint32_t)c;
  c >>= 32;
  c += (uint64_t)S[1] + g1;
  S[1] = (uint32_t)c;
  c >>= 32;
  c += (uint64_t)S[2] + g2;
  S[2] = (uint32_t)c;
  c >>= 32;
  for (int i = 3; i < 8; i++) {
    c += S[i];
    S[i] = (uint32_t)c;
    c >>= 32;
  }
  uint32_t k = (uint32_t)c;
  c = (uint64_t)S[0] + k * IBFT_PC;
  S[0] = (uint32_t)c;
  c >>= 32;
  c += (uint64_t)S[1] + k;
  S[1] = (uint32_t)c;
  c >>= 32;
  S[2] += (uint32_t)c;
  for (int i = 0; i < 8; i++) r.v[i] = S[i];
#endif
  return r;
}

// always-inline body (used inside the out-of-line point routines) and the out-of-line entry point (everything else)
IBFT_HD fe fe_mul_i(const fe& a, const fe& b) {
  IBFT_OPCOUNT(IBFT_OP_MUL_BODY);
  uint32_t R[16];
  mul_wide_8x8(R, a.v, b.v);
  return fe_reduce512(R);
}
#if defined(IBFT_BLIND_COPY) && defined(__CUDACC__)
__constant__ uint32_t ibft_c_zero;
#endif
#if defined(IBFT_BLIND_COPY) && defined(__CUDA_ARCH__)
// EXPERIMENT (tools/quick_bench.py variants): the copies that marshal by-value operands into the out-of-line multiplier's
// argument registers are emitted by ptxas as IMAD.MOV -- on the FMA-heavy pipe, which is the one that binds (80 % busy).  Passing
// every operand through "x ^ c" with c a __constant__ word that happens to be 0 turns the copy into a LOP3 (ALU pipe, 41 % busy)
// that ptxas cannot fold away and can place straight into the argument register.
__device__ __forceinline__ fe fe_blind(const fe& a) {
  fe r;
  const uint32_t z = ibft_c_zero;
#pragma unroll
  for (int i = 0; i < 8; i++) asm("xor.b32 %0, %1, %2;" : "=r"(r.v[i]) : "r"(a.v[i]), "r"(z));
  return r;
}
__device__ __noinline__ fe fe_mul_o(fe a, fe b) { return fe_mul_i(a, b); }
__device__ __forceinline__ fe fe_mul(const fe& a, const fe& b) {
#if IBFT_BLIND_COPY >= 2
  return fe_blind(fe_mul_o(fe_blind(a), fe_blind(b)));
#else
  return fe_mul_o(fe_blind(a), fe_blind(b));
#endif
}
#else
IBFT_FN fe fe_mul(fe a, fe b) {
  IBFT_OPCOUNT(IBFT_OP_MUL_CALL);
  return fe_mul_i(a, b);
}
#endif

#if IBFT_PTX
// shorter carry chains for the squaring triangle, in the two shapes of mul_wide_8x8: "_nczz" writes its top pair fresh
// (literal-zero addends), "_r2" ripples its carry out into the pair above it, which a later row has already written
__device__ __forceinline__ void mad_chain3_nczz(uint32_t& p0, uint32_t& p1, uint32_t& p2, uint32_t& p3, uint32_t& p4_out,
                                                uint32_t& p5_out, uint32_t x0, uint32_t x1, uint32_t x2, uint32_t y) {
  asm("mad.lo.cc.u32 %0,%6,%9,%0;\n\tmadc.hi.cc.u32 %1,%6,%9,%1;\n\t"
      "madc.lo.cc.u32 %2,%7,%9,%2;\n\tmadc.hi.cc.u32 %3,%7,%9,%3;\n\t"
      "madc.lo.cc.u32 %4,%8,%9,0;\n\tmadc.hi.u32 %5,%8,%9,0;"
      : "+r"(p0), "+r"(p1), "+r"(p2), "+r"(p3), "=r"(p4_out), "=r"(p5_out)
      : "r"(x0), "r"(x1), "r"(x2), "r"(y));
}
__device__ __forceinline__ void mad_chain3_r2(uint32_t& p0, uint32_t& p1, uint32_t& p2, uint32_t& p3, uint32_t& p4, uint32_t& p5,
                                              uint32_t& p6, uint32_t& p7, uint32_t x0, uint32_t x1, uint32_t x2, uint32_t y) {
  asm("mad.lo.cc.u32 %0,%8,%11,%0;\n\tmadc.hi.cc.u32 %1,%8,%11,%1;\n\t"
      "madc.lo.cc.u32 %2,%9,%11,%2;\n\tmadc.hi.cc.u32 %3,%9,%11,%3;\n\t"
      "madc.lo.cc.u32 %4,%10,%11,%4;\n\tmadc.hi.cc.u32 %5,%10,%11,%5;\n\t"
      "addc.cc.u32 %6,%6,0;\n\taddc.u32 %7,%7,0;"
      : "+r"(p0), "+r"(p1), "+r"(p2), "+r"(p3), "+r"(p4), "+r"(p5), "+r"(p6), "+r"(p7)
      : "r"(x0), "r"(x1), "r"(x2), "r"(y));
}
__device__ __forceinline__ void mad_chain2_nczz(uint32_t& p0, uint32_t& p1, uint32_t& p2_out, uint32_t& p3_out, uint32_t x0,
                                                uint32_t x1, uint32_t y) {
  asm("mad.lo.cc.u32 %0,%4,%6,%0;\n\tmadc.hi.cc.u32 %1,%4,%6,%1;\n\t"
      "madc.lo.cc.u32 %2,%5,%6,0;\n\tmadc.hi.u32 %3,%5,%6,0;"
      : "+r"(p0), "+r"(p1), "=r"(p2_out), "=r"(p3_out)
      : "r"(x0), "r"(x1), "r"(y));
}
__device__ __forceinline__ void mad_chain2_r2(uint32_t& p0, uint32_t& p1, uint32_t& p2, uint32_t& p3, uint32_t& p4, uint32_t& p5,
                                              uint32_t x0, uint32_t x1, uint32_t y) {
  asm("mad.lo.cc.u32 %0,%6,%8,%0;\n\tmadc.hi.cc.u32 %1,%6,%8,%1;\n\t"
      "madc.lo.cc.u32 %2,%7,%8,%2;\n\tmadc.hi.cc.u32 %3,%7,%8,%3;\n\t"
      "addc.cc.u32 %4,%4,0;\n\taddc.u32 %5,%5,0;"
      : "+r"(p0), "+r"(p1), "+r"(p2), "+r"(p3), "+r"(p4), "+r"(p5)
      : "r"(x0), "r"(x1), "r"(y));
}
__device__ __forceinline__ void mad_chain1_r2(uint32_t& p0, uint32_t& p1, uint32_t& p2, uint32_t& p3, uint32_t x0, uint32_t y) {
  asm("mad.lo.cc.u32 %0,%4,%5,%0;\n\tmadc.hi.cc.u32 %1,%4,%5,%1;\n\taddc.cc.u32 %2,%2,0;\n\taddc.u32 %3,%3,0;"
      : "+r"(p0), "+r"(p1), "+r"(p2), "+r"(p3)
      : "r"(x0), "r"(y));
}
#endif

// R[0..15] = a^2 : 28 off-diagonal wide MACs (E/O carry chains, as in mul_wide_8x8), doubled, + 8 diagonal MACs
IBFT_HD void sqr_wide_8(uint32_t* R, const uint32_t* a) {
#if IBFT_PTX && !defined(IBFT_SQR_VIA_MUL)
  // Same row pairing as mul_wide_8x8: the later row of each pair writes the top pair fresh, the earlier one ripples into it.
  uint32_t E[14], O[14];
  E[0] = 0; E[1] = 0;
  // row 0
  mulw(E[2], E[3], a[2], a[0]); mulw(E[4], E[5], a[4], a[0]); mulw(E[6], E[7], a[6], a[0]);
  mulw(O[0], O[1], a[1], a[0]); mulw(O[2], O[3], a[3], a[0]); mulw(O[4], O[5], a[5], a[0]); mulw(O[6], O[7], a[7], a[0]);
  // row 1, E: (E[8], E[9]) fresh
  mad_chain3_nczz(E[4], E[5], E[6], E[7], E[8], E[9], a[3], a[5], a[7], a[1]);
  // rows 2 then 1, O: (O[8], O[9])
  mad_chain3_nczz(O[4], O[5], O[6], O[7], O[8], O[9], a[3], a[5], a[7], a[2]);
  mad_chain3_r2(O[2], O[3], O[4], O[5], O[6], O[7], O[8], O[9], a[2], a[4], a[6], a[1]);
  // rows 3 then 2, E: (E[10], E[11])
  mad_chain2_nczz(E[8], E[9], E[10], E[11], a[5], a[7], a[3]);
  mad_chain2_r2(E[6], E[7], E[8], E[9], E[10], E[11], a[4], a[6], a[2]);
  // rows 4 then 3, O: (O[10], O[11])
  mad_chain2_nczz(O[8], O[9], O[10], O[11], a[5], a[7], a[4]);
  mad_chain2_r2(O[6], O[7], O[8], O[9], O[10], O[11], a[4], a[6], a[3]);
  // rows 5 then 4, E: (E[12], E[13])
  mulw(E[12], E[13], a[7], a[5]);
  mad_chain1_r2(E[10], E[11], E[12], E[13], a[6], a[4]);
  // rows 6 then 5, O: (O[12], O[13])
  mulw(O[12], O[13], a[7], a[6]);
  mad_chain1_r2(O[10], O[11], O[12], O[13], a[6], a[5]);
  // T = E + (O << 32)   (T[0] = 0, T[15] = 0)
  uint32_t T[16];
  T[0] = 0;
  asm("add.cc.u32 %0,%14,%28;\n\taddc.cc.u32 %1,%15,%29;\n\taddc.cc.u32 %2,%16,%30;\n\taddc.cc.u32 %3,%17,%31;\n\t"
      "addc.cc.u32 %4,%18,%32;\n\taddc.cc.u32 %5,%19,%33;\n\taddc.cc.u32 %6,%20,%34;\n\taddc.cc.u32 %7,%21,%35;\n\t"
      "addc.cc.u32 %8,%22,%36;\n\taddc.cc.u32 %9,%23,%37;\n\taddc.cc.u32 %10,%24,%38;\n\taddc.cc.u32 %11,%25,%39;\n\t"
      "addc.cc.u32 %12,%26,%40;\n\taddc.u32 %13,%27,%41;"
      : "=r"(T[1]), "=r"(T[2]), "=r"(T[3]), "=r"(T[4]), "=r"(T[5]), "=r"(T[6]), "=r"(T[7]), "=r"(T[8]), "=r"(T[9]),
        "=r"(T[10]), "=r"(T[11]), "=r"(T[12]), "=r"(T[13]), "=r"(T[14])
      : "r"(E[1]), "r"(E[2]), "r"(E[3]), "r"(E[4]), "r"(E[5]), "r"(E[6]), "r"(E[7]), "r"(E[8]), "r"(E[9]), "r"(E[10]),
        "r"(E[11]), "r"(E[12]), "r"(E[13]), "r"(0u), "r"(O[0]), "r"(O[1]), "r"(O[2]), "r"(O[3]), "r"(O[4]), "r"(O[5]),
        "r"(O[6]), "r"(O[7]), "r"(O[8]), "r"(O[9]), "r"(O[10]), "r"(O[11]), "r"(O[12]), "r"(O[13]));
  // R = 2*T
  asm("add.cc.u32 %0,%16,%16;\n\taddc.cc.u32 %1,%17,%17;\n\taddc.cc.u32 %2,%18,%18;\n\taddc.cc.u32 %3,%19,%19;\n\t"
      "addc.cc.u32 %4,%20,%20;\n\taddc.cc.u32 %5,%21,%21;\n\taddc.cc.u32 %6,%22,%22;\n\taddc.cc.u32 %7,%23,%23;\n\t"
      "addc.cc.u32 %8,%24,%24;\n\taddc.cc.u32 %9,%25,%25;\n\taddc.cc.u32 %10,%26,%26;\n\taddc.cc.u32 %11,%27,%27;\n\t"
      "addc.cc.u32 %12,%28,%28;\n\taddc.cc.u32 %13,%29,%29;\n\taddc.cc.u32 %14,%30,%30;\n\taddc.u32 %15,0,0;"
      : "=r"(R[0]), "=r"(R[1]), "=r"(R[2]), "=r"(R[3]), "=r"(R[4]), "=r"(R[5]), "=r"(R[6]), "=r"(R[7]), "=r"(R[8]),
        "=r"(R[9]), "=r"(R[10]), "=r"(R[11]), "=r"(R[12]), "=r"(R[13]), "=r"(R[14]), "=r"(R[15])
      : "r"(T[0]), "r"(T[1]), "r"(T[2]), "r"(T[3]), "r"(T[4]), "r"(T[5]), "r"(T[6]), "r"(T[7]), "r"(T[8]), "r"(T[9]),
        "r"(T[10]), "r"(T[11]), "r"(T[12]), "r"(T[13]), "r"(T[14]));
  // R += sum a_i^2 2^(64 i): one carry chain of 8 wide MACs (cannot carry out: the total is a^2 < 2^512)
  asm("mad.lo.cc.u32 %0,%16,%16,%0;\n\tmadc.hi.cc.u32 %1,%16,%16,%1;\n\t"
      "madc.lo.cc.u32 %2,%17,%17,%2;\n\tmadc.hi.cc.u32 %3,%17,%17,%3;\n\t"
      "madc.lo.cc.u32 %4,%18,%18,%4;\n\tmadc.hi.cc.u32 %5,%18,%18,%5;\n\t"
      "madc.lo.cc.u32 %6,%19,%19,%6;\n\tmadc.hi.cc.u32 %7,%19,%19,%7;\n\t"
      "madc.lo.cc.u32 %8,%20,%20,%8;\n\tmadc.hi.cc.u32 %9,%20,%20,%9;\n\t"
      "madc.lo.cc.u32 %10,%21,%21,%10;\n\tmadc.hi.cc.u32 %11,%21,%21,%11;\n\t"
      "madc.lo.cc.u32 %12,%22,%22,%12;\n\tmadc.hi.cc.u32 %13,%22,%22,%13;\n\t"
      "madc.lo.cc.u32 %14,%23,%23,%14;\n\tmadc.hi.u32 %15,%23,%23,%15;"
      : "+r"(R[0]), "+r"(R[1]), "+r"(R[2]), "+r"(R[3]), "+r"(R[4]), "+r"(R[5]), "+r"(R[6]), "+r"(R[7]), "+r"(R[8]),
        "+r"(R[9]), "+r"(R[10]), "+r"(R[11]), "+r"(R[12]), "+r"(R[13]), "+r"(R[14]), "+r"(R[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(a[4]), "r"(a[5]), "r"(a[6]), "r"(a[7]));
#else
  mul_wide_8x8(R, a, a);
#endif
}

IBFT_HD fe fe_sqr_i(const fe& a) {
  IBFT_OPCOUNT(IBFT_OP_SQR_BODY);
  uint32_t R[16];
  sqr_wide_8(R, a.v);
  return fe_reduce512(R);
}
#if defined(IBFT_BLIND_COPY) && defined(__CUDA_ARCH__)
__device__ __noinline__ fe fe_sqr_o(fe a) { return fe_sqr_i(a); }
__device__ __forceinline__ fe fe_sqr(const fe& a) {
#if IBFT_BLIND_COPY >= 2
  return fe_blind(fe_sqr_o(fe_blind(a)));
#else
  return fe_sqr_o(fe_blind(a));
#endif
}
#else
IBFT_FN fe fe_sqr(fe a) {
  IBFT_OPCOUNT(IBFT_OP_SQR_CALL);
  return fe_sqr_i(a);
}
#endif

// a^(2^n): out of line, with the squarer inlined in the loop (no per-iteration call marshalling)
IBFT_FN fe fe_sqrn(fe a, int n) {
  IBFT_OPCOUNT(IBFT_OP_SQRN_CALL);
#if IBFT_PTX
#pragma unroll 1
#endif
  for (int i = 0; i < n; i++) {
    IBFT_OPCOUNT(IBFT_OP_SQRN_ITER);
    a = fe_sqr_i(a);
  }
  return a;
}

// multiply by a small constant (<= 2^10): one 8-MAC chain + fold
IBFT_HD fe fe_mul_small(const fe& a, uint32_t k) {
  uint32_t S[9];
  uint64_t c = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    c += (uint64_t)a.v[i] * k;
    S[i] = (uint32_t)c;
    c >>= 32;
  }
  S[8] = (uint32_t)c;  // < 2^10
  // fold S[8] * (2^32 + 977)
  fe r;
  uint64_t m = (uint64_t)S[8] * IBFT_PC;  // < 2^20
  c = (uint64_t)S[0] + (uint32_t)m;
  r.v[0] = (uint32_t)c;
  c >>= 32;
  c += (uint64_t)S[1] + S[8];
  r.v[1] = (uint32_t)c;
  c >>= 32;
#pragma unroll
  for (int i = 2; i < 8; i++) {
    c += S[i];
    r.v[i] = (uint32_t)c;
    c >>= 32;
  }
  uint32_t k2 = (uint32_t)c;
  c = (uint64_t)r.v[0] + k2 * IBFT_PC;
  r.v[0] = (uint32_t)c;
  c >>= 32;
  c += (uint64_t)r.v[1] + k2;
  r.v[1] = (uint32_t)c;
  c >>= 32;
  r.v[2] += (uint32_t)c;
  return r;
}

// ------------------------------------------------------------------------------------------------
// exponentiations with fixed addition chains
// ------------------------------------------------------------------------------------------------
// Shared prefix: x2 = a^(2^2-1), x3, x6, x9, x11, x22, x44, x88, x176, x220, x223  (x_k = a^(2^k - 1))
struct fe_chain {
  fe x2, x3, x22, x223;
};
IBFT_HD fe_chain fe_chain_223(const fe& a) {
  fe_chain c;
  c.x2 = fe_mul(fe_sqr(a), a);
  c.x3 = fe_mul(fe_sqr(c.x2), a);
  fe x6 = fe_mul(fe_sqrn(c.x3, 3), c.x3);
  fe x9 = fe_mul(fe_sqrn(x6, 3), c.x3);
  fe x11 = fe_mul(fe_sqrn(x9, 2), c.x2);
  c.x22 = fe_mul(fe_sqrn(x11, 11), x11);
  fe x44 = fe_mul(fe_sqrn(c.x22, 22), c.x22);
  fe x88 = fe_mul(fe_sqrn(x44, 44), x44);
  fe x176 = fe_mul(fe_sqrn(x88, 88), x88);
  fe x220 = fe_mul(fe_sqrn(x176, 44), x44);
  c.x223 = fe_mul(fe_sqrn(x220, 3), c.x3);
  return c;
}

// a^((p+1)/4): the square root when a is a quadratic residue (p = 3 mod 4).
// (p+1)/4 = 2^254 - 2^30 - 244 = [223 ones][0][22 ones][0000][11][00]
IBFT_HD fe fe_sqrt_candidate(const fe& a) {
  fe_chain c = fe_chain_223(a);
  fe t = fe_sqrn(c.x223, 23);
  t = fe_mul(t, c.x22);
  t = fe_sqrn(t, 6);
  t = fe_mul(t, c.x2);
  t = fe_sqrn(t, 2);
  return t;
}

// The square root of c and the inverse of y V from ONE exponentiation (V != 0):
//   u = (c V^4)^((p-3)/4) = c^((p-3)/4) V^-2,   y = c V^2 u = c^((p+1)/4),   w = u V = c^((p-3)/4) / V,
// and y w V = c^((p-1)/2), so w = 1 / (y V) exactly when c is a residue (y^2 = c); the caller checks that.  Negating y negates
// 1 / (y V): the caller flips w with y.  (p-3)/4 = [223 ones][0][22 ones][0000][1][0][11]: the chain of fe_sqrt_candidate
// up to its last six bits, one multiplication more.  Out of line: the recovery calls it from its rare branches too.
struct fe_root_inv {
  fe y, w;
};
IBFT_FN fe_root_inv fe_sqrt_inv(fe c, fe V) {
  const fe v2 = fe_sqr(V);
  const fe a = fe_mul(c, fe_sqr(v2));
  fe_chain ch = fe_chain_223(a);
  fe t = fe_sqrn(ch.x223, 23);
  t = fe_mul(t, ch.x22);
  t = fe_sqrn(t, 5);
  t = fe_mul(t, a);
  t = fe_sqrn(t, 3);
  t = fe_mul(t, ch.x2);
  fe_root_inv o;
  o.y = fe_mul(fe_mul(c, v2), t);
  o.w = fe_mul(t, V);
  return o;
}

// a^(p-2) (Fermat inverse; 0 -> 0).  p-2 = [223 ones][0][22 ones][0000][1][0][11][0][1]
IBFT_HD fe fe_inv_fermat(const fe& a) {
  fe_chain c = fe_chain_223(a);
  fe t = fe_sqrn(c.x223, 23);
  t = fe_mul(t, c.x22);
  t = fe_sqrn(t, 5);
  t = fe_mul(t, a);
  t = fe_sqrn(t, 3);
  t = fe_mul(t, c.x2);
  t = fe_sqrn(t, 2);
  t = fe_mul(t, a);
  return t;
}

}  // namespace ibft
