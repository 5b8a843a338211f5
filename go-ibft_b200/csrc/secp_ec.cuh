// secp_ec.cuh -- secp256k1 group law (Jacobian coordinates, a = 0) and the double-scalar multiplication
// u1*G + u2*R that dominates public-key recovery.
//
// SIMT-first formulation (this is the part a CPU library would do differently):
//   * GLV: both scalars are split into two ~128-bit halves (secp_scalar.cuh), so one chain of 132 doublings
//     serves four digit streams;
//   * signed FIXED windows (Booth digits) instead of wNAF: every lane of a warp performs its additions at the
//     same loop positions, so a warp never executes an addition for a minority of its lanes (wNAF's
//     data-dependent digit positions would leave ~5/6 of the lanes idle in every addition);
//   * the generator table ({1..2^(WG-1)} * G, affine, with beta*x alongside) is staged in shared memory once per
//     CTA; the per-signature table {1..8} * R lives in thread-local memory;
//   * exceptional cases (P + P, P - P, infinity) are handled exactly -- adversarial signatures can reach them
//     and the verdict must be bit-exact with the oracle -- but by rarely-taken branches.
#pragma once
#include "secp_fe.cuh"
#include "secp_scalar.cuh"

namespace ibft {

struct jac {
  fe x, y, z;
  bool inf;
};
struct aff {
  fe x, y;
};

// beta: cube root of unity mod p with lambda*(x,y) = (beta*x, y)
IBFT_HD fe fe_beta() {
  fe b;
  const uint32_t v[8] = {0x719501EEu, 0xC1396C28u, 0x12F58995u, 0x9CF04975u, 0xAC3434E9u, 0x6E64479Eu, 0x657C0710u, 0x7AE96A2Bu};
#pragma unroll
  for (int i = 0; i < 8; i++) b.v[i] = v[i];
  return b;
}

// IBFT_POINT_INLINE: the two hot group-law routines become out-of-line functions (operands by reference) with the
// field multiplier INLINED inside them -- one call per point operation instead of one per field operation.
#if defined(IBFT_POINT_INLINE) && defined(__CUDACC__)
#define IBFT_PT __host__ __device__ __noinline__
#define PMUL fe_mul_i
#define PSQR fe_sqr_i
#else
#define IBFT_PT IBFT_HD
#define PMUL fe_mul
#define PSQR fe_sqr
#endif

#if defined(IBFT_DBL_INLINE)
#define DMUL fe_mul_i
#define DSQR fe_sqr_i
#else
#define DMUL PMUL
#define DSQR PSQR
#endif

// The doubling's first three products in ONE out-of-line call (each with its own inlined squarer body) instead of three calls
// and their operand copies, and the rarely taken P + P case of the mixed addition out of the window loop's code.  Nothing more is
// fused: the window loop and the routines it calls must stay within about 27 KB of SASS.  Larger groups (the front of the
// mixed addition, pairs of independent products) remove more FMA-pipe instructions but ran slower on an H100 (DESIGN.md §3.1),
// the same instruction-cache wall that whole inlined point routines hit (IBFT_POINT_BYVAL, IBFT_POINT_INLINE).
#if !defined(IBFT_POINT_INLINE) && !defined(IBFT_DBL_INLINE)
#define IBFT_DBL_FRONT 1
#endif
struct dbl_abc {
  fe a, b, c;
};
// doubling: A = X^2, B = Y^2, C = B^2
IBFT_FN dbl_abc jac_dbl_front(fe x, fe y) {
  IBFT_OPCOUNT(IBFT_OP_DBL_FRONT);
  dbl_abc r;
  r.a = fe_sqr_i(x);
  r.b = fe_sqr_i(y);
  r.c = fe_sqr_i(r.b);
  return r;
}

// dbl-2009-l: 2M + 5S
IBFT_PT jac jac_double_body(const jac& p) {
  jac r;
  // Y = 0 never happens on secp256k1 (no points of order 2), so no exceptional case besides infinity.
#if defined(IBFT_DBL_FRONT)
  const dbl_abc abc = jac_dbl_front(p.x, p.y);
  const fe a = abc.a, b = abc.b, c = abc.c;
#else
  fe a = DSQR(p.x);
  fe b = DSQR(p.y);
  fe c = DSQR(b);
#endif
  fe t = fe_add(p.x, b);
  t = DSQR(t);
  t = fe_sub(t, a);
  t = fe_sub(t, c);
  fe d = fe_dbl(t);
  fe e = fe_add(fe_dbl(a), a);
  fe f = DSQR(e);
  r.x = fe_sub(f, fe_dbl(d));
  fe c8 = fe_dbl(fe_dbl(fe_dbl(c)));
  r.y = fe_sub(DMUL(e, fe_sub(d, r.x)), c8);
  r.z = fe_dbl(DMUL(p.y, p.z));
  r.inf = p.inf;
  return r;
}

#if defined(IBFT_DBL_FRONT) && !(defined(IBFT_POINT_BYVAL) && defined(__CUDA_ARCH__))
// P + P inside the mixed addition, out of line (the point travels by value, in registers): inlined, this doubling sat in the
// window loop's code -- 440 instructions, 7 KB -- for a branch that only crafted signatures take.
struct jac_words {
  uint32_t w[24];
};
IBFT_FN jac_words jac_double_rare(jac_words in) {
  jac p;
#pragma unroll
  for (int i = 0; i < 8; i++) { p.x.v[i] = in.w[i]; p.y.v[i] = in.w[8 + i]; p.z.v[i] = in.w[16 + i]; }
  p.inf = false;
  const jac r = jac_double_body(p);
  jac_words o;
#pragma unroll
  for (int i = 0; i < 8; i++) { o.w[i] = r.x.v[i]; o.w[8 + i] = r.y.v[i]; o.w[16 + i] = r.z.v[i]; }
  return o;
}
IBFT_HD jac jac_double_ool(const jac& p) {
  jac_words in;
#pragma unroll
  for (int i = 0; i < 8; i++) { in.w[i] = p.x.v[i]; in.w[8 + i] = p.y.v[i]; in.w[16 + i] = p.z.v[i]; }
  const jac_words o = jac_double_rare(in);
  jac r;
#pragma unroll
  for (int i = 0; i < 8; i++) { r.x.v[i] = o.w[i]; r.y.v[i] = o.w[8 + i]; r.z.v[i] = o.w[16 + i]; }
  r.inf = p.inf;
  return r;
}
#endif

#if defined(IBFT_POINT_BYVAL) && defined(__CUDA_ARCH__)
// IBFT_POINT_BYVAL: the two hot group-law routines are out-of-line functions taking the point BY VALUE (the whole accumulator
// travels in registers, like the by-value fe operands of fe_mul) with the field multiplier inlined inside them: one call per
// point operation, no per-multiplication operand marshalling.
#undef DMUL
#undef DSQR
#undef PMUL
#undef PSQR
#define DMUL fe_mul_i
#define DSQR fe_sqr_i
#define PMUL fe_mul_i
#define PSQR fe_sqr_i
struct jac24 { uint32_t w[24]; };
__device__ __noinline__ jac24 jac_double_v(jac24 in) {
  jac p;
#pragma unroll
  for (int i = 0; i < 8; i++) { p.x.v[i] = in.w[i]; p.y.v[i] = in.w[8 + i]; p.z.v[i] = in.w[16 + i]; }
  p.inf = false;
  fe a = DSQR(p.x);
  fe b = DSQR(p.y);
  fe c = DSQR(b);
  fe t = fe_add(p.x, b);
  t = DSQR(t);
  t = fe_sub(t, a);
  t = fe_sub(t, c);
  fe d = fe_dbl(t);
  fe e = fe_add(fe_dbl(a), a);
  fe f = DSQR(e);
  fe rx = fe_sub(f, fe_dbl(d));
  fe c8 = fe_dbl(fe_dbl(fe_dbl(c)));
  fe ry = fe_sub(DMUL(e, fe_sub(d, rx)), c8);
  fe rz = fe_dbl(DMUL(p.y, p.z));
  jac24 o;
#pragma unroll
  for (int i = 0; i < 8; i++) { o.w[i] = rx.v[i]; o.w[8 + i] = ry.v[i]; o.w[16 + i] = rz.v[i]; }
  return o;
}
__device__ __forceinline__ jac jac_double(const jac& p) {
  jac24 in;
#pragma unroll
  for (int i = 0; i < 8; i++) { in.w[i] = p.x.v[i]; in.w[8 + i] = p.y.v[i]; in.w[16 + i] = p.z.v[i]; }
  jac24 o = jac_double_v(in);
  jac r;
#pragma unroll
  for (int i = 0; i < 8; i++) { r.x.v[i] = o.w[i]; r.y.v[i] = o.w[8 + i]; r.z.v[i] = o.w[16 + i]; }
  r.inf = p.inf;
  return r;
}
#else
IBFT_PT jac jac_double(const jac& p) { return jac_double_body(p); }
#endif

// p + (qx, qy) with q affine (never infinity): 8M + 3S.  h_out (optional): Z3 / Z1 of the generic case (= H), 1 otherwise.
// OPT-IN -DIBFT_MADD_7M4S: madd-2007-bl, 7M + 4S -- Z3 = (Z1 + H)^2 - Z1Z1 - HH = 2 Z1 H trades the multiplication Z1 H for a
// squaring, and X3, Y3 carry the matching factors 4 and 8 (I = 4 HH, r = 2 (S2 - Y1)); h_out is then 2H.  Slower on an H100
// (DESIGN.md §3.1): the seven extra additions cost more issue slots and code than the 28 wide MACs it saves.
#if defined(IBFT_POINT_BYVAL) && defined(__CUDA_ARCH__)
// generic case only; *flag = 0 generic result, 1 = P + P (caller doubles), 2 = P + (-P) (infinity)
struct jac33 { uint32_t w[33]; };
__device__ __noinline__ jac33 jac_madd_v(jac24 in, fe qx, fe qy) {
  jac p;
#pragma unroll
  for (int i = 0; i < 8; i++) { p.x.v[i] = in.w[i]; p.y.v[i] = in.w[8 + i]; p.z.v[i] = in.w[16 + i]; }
  fe z1z1 = PSQR(p.z);
  fe u2 = PMUL(qx, z1z1);
  fe s2 = PMUL(PMUL(qy, p.z), z1z1);
  fe h = fe_sub(u2, p.x);
  fe rr = fe_sub(s2, p.y);
  uint32_t flag = 0;
  if (fe_is_zero(h)) flag = fe_is_zero(rr) ? 1u : 2u;
  fe hh = PSQR(h);
#if defined(IBFT_MADD_7M4S)
  fe i4 = fe_dbl(fe_dbl(hh));
  fe j = PMUL(h, i4);
  fe r2 = fe_dbl(rr);
  fe v = PMUL(p.x, i4);
  fe rx = fe_sub(fe_sub(PSQR(r2), j), fe_dbl(v));
  fe ry = fe_sub(PMUL(r2, fe_sub(v, rx)), fe_dbl(PMUL(p.y, j)));
  fe rz = fe_sub(fe_sub(PSQR(fe_add(p.z, h)), z1z1), hh);
  fe h2 = fe_dbl(h);
#else
  fe hhh = PMUL(h, hh);
  fe v = PMUL(p.x, hh);
  fe rx = fe_sub(fe_sub(PSQR(rr), hhh), fe_dbl(v));
  fe ry = fe_sub(PMUL(rr, fe_sub(v, rx)), PMUL(p.y, hhh));
  fe rz = PMUL(p.z, h);
  fe h2 = h;
#endif
  jac33 o;
#pragma unroll
  for (int i = 0; i < 8; i++) { o.w[i] = rx.v[i]; o.w[8 + i] = ry.v[i]; o.w[16 + i] = rz.v[i]; o.w[24 + i] = h2.v[i]; }
  o.w[32] = flag;
  return o;
}
__device__ __forceinline__ jac jac_add_affine(const jac& p, const fe& qx, const fe& qy, fe* h_out = nullptr) {
  jac r;
  if (h_out) *h_out = fe_from_u32(1);
  if (p.inf) {
    r.x = qx;
    r.y = qy;
    r.z = fe_from_u32(1);
    r.inf = false;
    return r;
  }
  jac24 in;
#pragma unroll
  for (int i = 0; i < 8; i++) { in.w[i] = p.x.v[i]; in.w[8 + i] = p.y.v[i]; in.w[16 + i] = p.z.v[i]; }
  jac33 o = jac_madd_v(in, qx, qy);
  if (o.w[32] != 0) {
    if (o.w[32] == 1u) return jac_double(p);  // P + P
    r = p;
    r.inf = true;  // P + (-P)
    return r;
  }
#pragma unroll
  for (int i = 0; i < 8; i++) { r.x.v[i] = o.w[i]; r.y.v[i] = o.w[8 + i]; r.z.v[i] = o.w[16 + i]; }
  r.inf = false;
  if (h_out) {
#pragma unroll
    for (int i = 0; i < 8; i++) h_out->v[i] = o.w[24 + i];
  }
  return r;
}
#else
IBFT_PT jac jac_add_affine(const jac& p, const fe& qx, const fe& qy, fe* h_out = nullptr) {
  jac r;
  if (h_out) *h_out = fe_from_u32(1);
  if (p.inf) {
    IBFT_BRANCH(IBFT_BR_ADD_INF);
    r.x = qx;
    r.y = qy;
    r.z = fe_from_u32(1);
    r.inf = false;
    return r;
  }
  fe z1z1 = PSQR(p.z);
  fe u2 = PMUL(qx, z1z1);
  fe s2 = PMUL(PMUL(qy, p.z), z1z1);
  fe h = fe_sub(u2, p.x);
  fe rr = fe_sub(s2, p.y);
  if (fe_is_zero(h)) {
    if (fe_is_zero(rr)) {
      IBFT_BRANCH(IBFT_BR_ADD_DBL);
#if defined(IBFT_DBL_FRONT)
      return jac_double_ool(p);  // P + P (rare)
#else
      return jac_double(p);  // P + P (rare; kept inline so that `p` never has its address taken)
#endif
    }
    IBFT_BRANCH(IBFT_BR_ADD_NEG);
    r = p;
    r.inf = true;  // P + (-P)
    return r;
  }
  fe hh = PSQR(h);
#if defined(IBFT_MADD_7M4S)
  fe i4 = fe_dbl(fe_dbl(hh));  // I = (2H)^2
  fe j = PMUL(h, i4);          // J = H I
  fe r2 = fe_dbl(rr);          // r = 2 (S2 - Y1)
  fe v = PMUL(p.x, i4);        // V = X1 I
  r.x = fe_sub(fe_sub(PSQR(r2), j), fe_dbl(v));
  r.y = fe_sub(PMUL(r2, fe_sub(v, r.x)), fe_dbl(PMUL(p.y, j)));
  r.z = fe_sub(fe_sub(PSQR(fe_add(p.z, h)), z1z1), hh);
  r.inf = false;
  if (h_out) *h_out = fe_dbl(h);
#else
  fe hhh = PMUL(h, hh);
  fe v = PMUL(p.x, hh);
  r.x = fe_sub(fe_sub(PSQR(rr), hhh), fe_dbl(v));
  r.y = fe_sub(PMUL(rr, fe_sub(v, r.x)), PMUL(p.y, hhh));
  r.z = PMUL(p.z, h);
  r.inf = false;
  if (h_out) *h_out = h;
#endif
  return r;
}
#endif
#if defined(IBFT_POINT_BYVAL) && defined(__CUDA_ARCH__)
#undef DMUL
#undef DSQR
#undef PMUL
#undef PSQR
#define PMUL fe_mul
#define PSQR fe_sqr
#define DMUL fe_mul
#define DSQR fe_sqr
#endif

// ------------------------------------------------------------------------------------------------
// Lane executors.  The group law below is written as LEVELS of up to four independent field multiplications.
//   exec_serial  one thread per signature (throughput path): the products of a level are computed one after the other.
//   exec_quad    four lanes per signature (latency path, "several lanes per signature" of the north star): every lane keeps a
//                full copy of the state, lane q of the quad computes product q of the level, and the four results are
//                exchanged through shared memory.  On the XYZZ law below the critical path of a doubling is 3 multiplications, of
//                an addition 4 (one thread: 7 and 11 on the Jacobian law of the throughput path).
// ------------------------------------------------------------------------------------------------
struct exec_serial {
  IBFT_HD void mul4(const fe* a, const fe* b, int count, fe* out) const {
    for (int k = 0; k < count; k++) out[k] = fe_mul(a[k], b[k]);
  }
  IBFT_HD bool leader() const { return true; }
  IBFT_HD void sync() const {}
};

#if defined(__CUDACC__)
struct exec_quad {
  int role;       // lane & 3
  unsigned mask;  // the four lanes of this quad: quads of one warp may diverge from each other, never the lanes of a quad
  // operand of THIS lane's product: a two-level binary select on the role bits.  Written with selp so that the compiler
  // keeps the candidates in registers (the C ternary chain was turned into a role-indexed LOCAL-memory array: 550 cycles).
  __device__ __forceinline__ static uint32_t sel(uint32_t if_set, uint32_t if_clear, int bit) {
    uint32_t r;
    asm("{\n\t.reg .pred p;\n\tsetp.ne.s32 p, %3, 0;\n\tselp.u32 %0, %1, %2, p;\n\t}" : "=r"(r) : "r"(if_set), "r"(if_clear), "r"(bit));
    return r;
  }
  __device__ __forceinline__ static fe pick(int role, const fe* v, int count) {
    fe r;
    const int b0 = role & 1, b1 = role & 2;
#pragma unroll
    for (int i = 0; i < 8; i++) {
      uint32_t lo = count > 1 ? sel(v[1].v[i], v[0].v[i], b0) : v[0].v[i];
      uint32_t hi = count > 3 ? sel(v[3].v[i], v[2].v[i], b0) : (count > 2 ? v[2].v[i] : lo);
      r.v[i] = count > 2 ? sel(hi, lo, b1) : lo;
    }
    return r;
  }
  // exchange buffer in shared memory: two parities x two halves x one uint4 per thread of the CTA.  A warp shuffle costs ~10 cycles of issue on this
  // part (330 cycles for the 32 shuffles of a four-product level); two STS.128 + 2k LDS.128 + one quad-level sync are cheaper.
  uint4* xb;            // CTA-wide buffer, 4 * blockDim.x uint4
  mutable uint32_t par; // level parity: double buffering, so one sync per level suffices
  __device__ __forceinline__ void mul4(const fe* a, const fe* b, int count, fe* out) const {
    fe p = fe_mul(pick(role, a, count), pick(role, b, count));
    const uint32_t nt = blockDim.x * blockDim.y;
    const uint32_t t = threadIdx.y * blockDim.x + threadIdx.x;
    uint4* buf = xb + par * 2u * nt;
    par ^= 1u;
    // slot of (quad Q of the warp, product k) = 8k + ((Q + 2k) & 7): the eight quads reading product k hit eight different
    // 16-byte bank groups, and so do the eight lanes of every quarter-warp when they write (the plain layout "slot = lane"
    // makes the eight quads reading one product collide in the same bank group)
    const uint32_t wb = t & ~31u, Q = (t >> 2) & 7u;
    if (role < count) {
      const uint32_t sl = wb + 8u * (uint32_t)role + ((Q + 2u * (uint32_t)role) & 7u);
      buf[sl] = make_uint4(p.v[0], p.v[1], p.v[2], p.v[3]);
      buf[nt + sl] = make_uint4(p.v[4], p.v[5], p.v[6], p.v[7]);
    }
    __syncwarp(mask);
#pragma unroll
    for (int k = 0; k < 4; k++) {
      if (k < count) {
        const uint32_t sl = wb + 8u * k + ((Q + 2u * k) & 7u);
        uint4 lo = buf[sl], hi = buf[nt + sl];
        out[k].v[0] = lo.x; out[k].v[1] = lo.y; out[k].v[2] = lo.z; out[k].v[3] = lo.w;
        out[k].v[4] = hi.x; out[k].v[5] = hi.y; out[k].v[6] = hi.z; out[k].v[7] = hi.w;
      }
    }
  }
  __device__ __forceinline__ bool leader() const { return role == 0; }
  __device__ __forceinline__ void sync() const { __syncwarp(mask); }
};
#endif

// The latency path keeps its accumulator in XYZZ coordinates (x = X/ZZ, y = Y/ZZZ, ZZ^3 = ZZZ^2): with four products per
// level a doubling is 3 levels deep (9 products) and a FULL addition 4 levels (14 products) -- the same depth as a mixed
// addition -- so the per-signature table needs no normalisation (no batched inversion) and one adder serves both the
// R streams (XYZZ entries) and the generator stream (affine entries, ZZ = ZZZ = 1).  Jacobian dbl-2009-l / madd are 4 and 5
// levels deep.  Formulas: EFD dbl-2008-s-1 and add-2008-s for short Weierstrass curves with a = 0.
struct xyzz {
  fe x, y, zz, zzz;
  bool inf;
};

// levels: {U^2, X^2} -> {U*V, X*V, M^2, V*ZZ} -> {M*(S-X3), W*Y, W*ZZZ}        (U = 2Y, V = U^2, W = U*V, S = X*V, M = 3X^2)
template <class EX>
IBFT_HD xyzz xyzz_double_x(const EX& ex, const xyzz& p) {
  xyzz r;
  fe a[4], b[4], o[4];
  fe U = fe_dbl(p.y);
  a[0] = U; b[0] = U; a[1] = p.x; b[1] = p.x;
  ex.mul4(a, b, 2, o);
  fe V = o[0];
  fe M = fe_add(fe_dbl(o[1]), o[1]);
  a[0] = U; b[0] = V; a[1] = p.x; b[1] = V; a[2] = M; b[2] = M; a[3] = V; b[3] = p.zz;
  ex.mul4(a, b, 4, o);
  fe W = o[0], S = o[1];
  r.x = fe_sub(o[2], fe_dbl(S));
  r.zz = o[3];
  a[0] = M; b[0] = fe_sub(S, r.x); a[1] = W; b[1] = p.y; a[2] = W; b[2] = p.zzz;
  ex.mul4(a, b, 3, o);
  r.y = fe_sub(o[0], o[1]);
  r.zzz = o[2];
  r.inf = p.inf;
  return r;
}

// levels: {X1*ZZ2, X2*ZZ1, Y1*ZZZ2, Y2*ZZZ1} -> {P^2, R^2, ZZ1*ZZ2, ZZZ1*ZZZ2} -> {P*PP, U1*PP, ZZ12*PP}
//         -> {R*(Q-X3), S1*PPP, ZZZ12*PPP}.   q is never the point at infinity (zero digits are skipped by the caller).
template <class EX>
IBFT_HD xyzz xyzz_add_x(const EX& ex, const xyzz& p, const xyzz& q) {
  if (p.inf) {
    IBFT_BRANCH(IBFT_BR_XADD_INF);
    return q;
  }
  xyzz r;
  fe a[4], b[4], o[4];
  a[0] = p.x; b[0] = q.zz; a[1] = q.x; b[1] = p.zz; a[2] = p.y; b[2] = q.zzz; a[3] = q.y; b[3] = p.zzz;
  ex.mul4(a, b, 4, o);
  fe U1 = o[0], S1 = o[2];
  fe P = fe_sub(o[1], U1), R = fe_sub(o[3], S1);
  a[0] = P; b[0] = P; a[1] = R; b[1] = R; a[2] = p.zz; b[2] = q.zz; a[3] = p.zzz; b[3] = q.zzz;
  ex.mul4(a, b, 4, o);
  fe PP = o[0], RR = o[1], ZZ12 = o[2], ZZZ12 = o[3];
  a[0] = P; b[0] = PP; a[1] = U1; b[1] = PP; a[2] = ZZ12; b[2] = PP;
  ex.mul4(a, b, 3, o);
  fe PPP = o[0], Q = o[1];
  r.zz = o[2];
  r.x = fe_sub(fe_sub(RR, PPP), fe_dbl(Q));
  a[0] = R; b[0] = fe_sub(Q, r.x); a[1] = S1; b[1] = PPP; a[2] = ZZZ12; b[2] = PPP;
  ex.mul4(a, b, 3, o);
  r.y = fe_sub(o[0], o[1]);
  r.zzz = o[2];
  r.inf = false;
  // exceptional cases, tested last so that the zero tests overlap the generic computation: every lane of a quad holds the
  // same state, so the whole quad takes these (rare) branches together
  if (fe_is_zero(P)) {
    if (fe_is_zero(R)) {
      IBFT_BRANCH(IBFT_BR_XADD_DBL);
      return xyzz_double_x(ex, p);  // same point
    }
    IBFT_BRANCH(IBFT_BR_XADD_NEG);
    r.inf = true;                   // opposite points
  }
  return r;
}

// per-signature table {1..8}*R in XYZZ (32 words per entry), same thread-interleaved shared-memory layout as rtab_view
struct qtab_view {
  uint32_t* base;
  uint32_t stride;
  IBFT_HD void store(int entry, const xyzz& p) const {
#pragma unroll
    for (int i = 0; i < 8; i++) {
      base[(uint32_t)(entry * 32 + i) * stride] = p.x.v[i];
      base[(uint32_t)(entry * 32 + 8 + i) * stride] = p.y.v[i];
      base[(uint32_t)(entry * 32 + 16 + i) * stride] = p.zz.v[i];
      base[(uint32_t)(entry * 32 + 24 + i) * stride] = p.zzz.v[i];
    }
  }
  IBFT_HD xyzz load(int entry) const {
    xyzz p;
#pragma unroll
    for (int i = 0; i < 8; i++) {
      p.x.v[i] = base[(uint32_t)(entry * 32 + i) * stride];
      p.y.v[i] = base[(uint32_t)(entry * 32 + 8 + i) * stride];
      p.zz.v[i] = base[(uint32_t)(entry * 32 + 16 + i) * stride];
      p.zzz.v[i] = base[(uint32_t)(entry * 32 + 24 + i) * stride];
    }
    p.inf = false;
    return p;
  }
};
#define IBFT_QTAB_WORDS 256  // 8 entries x 32 words per signature

// ------------------------------------------------------------------------------------------------
// u1*G + u2*R
// ------------------------------------------------------------------------------------------------
#ifndef IBFT_WG
#define IBFT_WG 8  // generator window: 2^(WG-1) table entries of (x, y)
#endif
#define IBFT_WR 4  // per-signature window: table {1..8} * R
#define IBFT_GTAB_ENTRIES (1 << (IBFT_WG - 1))
#define IBFT_NWIN_R 33  // ceil(130 / 4)
#if IBFT_WC > 0
static_assert(IBFT_WC % IBFT_WR == 0 && IBFT_WC <= 12, "combined window must be a multiple of the R window");
#endif
static_assert(IBFT_WG % IBFT_WR == 0, "generator window must be a multiple of the R window");

// Optional COMBINED generator table (IBFT_WC = 8 or 12, 0 = off): entry (d1, d2), 0 <= d1 <= 2^(WC-1), |d2| <= 2^(WC-1), holds
// d1*G + d2*lambda*G (affine x, y), so the two generator digit streams cost ONE addition per window instead of two.  The
// other half of the (d1, d2) plane is reached by negating y.  (2^(WC-1)+1) * (2^WC+1) * 64 bytes: 2.1 MB for WC = 8
// (L2 resident), 537 MB for WC = 12 (HBM; 704 B of gathers per signature) -- built on the device at engine creation.
#ifndef IBFT_WC
#define IBFT_WC 8  // 2.1 MB, L2 resident; WC = 12 trades HBM gathers for fewer additions
#endif
#define IBFT_CTAB_D2 ((1 << IBFT_WC) + 1)
#define IBFT_CTAB_ENTRIES (((1 << (IBFT_WC - 1)) + 1) * IBFT_CTAB_D2)
#define IBFT_CTAB_POSITIONS ((IBFT_NWIN_R * IBFT_WR + IBFT_WC - 1) / IBFT_WC)  // comb positions covering the 132 window bits

// Generator table accessor: entry i (0-based) = (i+1)*G as 16 words x[8] y[8] (shared memory on the device).
#define IBFT_GTAB_ENTRY_WORDS 16
struct gtab_view {
  const uint32_t* base;
  const uint32_t* comb = nullptr;  // combined table (global memory) or nullptr
  IBFT_HD void load_comb(int d1, int d2, fe& x, fe& y) const {
    const uint32_t* e = comb + (size_t)IBFT_GTAB_ENTRY_WORDS * ((size_t)d1 * IBFT_CTAB_D2 + (size_t)(d2 + (1 << (IBFT_WC > 0 ? IBFT_WC - 1 : 0))));
#if defined(__CUDA_ARCH__)
    const uint4* q = reinterpret_cast<const uint4*>(e);
    uint4 a = __ldg(q), b = __ldg(q + 1), c = __ldg(q + 2), d = __ldg(q + 3);
    x.v[0] = a.x; x.v[1] = a.y; x.v[2] = a.z; x.v[3] = a.w; x.v[4] = b.x; x.v[5] = b.y; x.v[6] = b.z; x.v[7] = b.w;
    y.v[0] = c.x; y.v[1] = c.y; y.v[2] = c.z; y.v[3] = c.w; y.v[4] = d.x; y.v[5] = d.y; y.v[6] = d.z; y.v[7] = d.w;
#else
    for (int i = 0; i < 8; i++) { x.v[i] = e[i]; y.v[i] = e[8 + i]; }
#endif
  }
  // entry (d1, d2) of POSITION pos of the per-position comb tables: device = the table itself (positions are contiguous after
  // the combined table); the host emulation computes the entry through `host_pos` (a 36 MB table is not built there)
#if !defined(__CUDA_ARCH__)
  void (*host_pos)(int pos, int d1, int d2, uint32_t* xy16) = nullptr;
#endif
  IBFT_HD void load_comb_pos(int pos, int d1, int d2, fe& x, fe& y) const {
#if defined(__CUDA_ARCH__)
    gtab_view P = *this;
    P.comb = comb + (size_t)pos * IBFT_GTAB_ENTRY_WORDS * (size_t)IBFT_CTAB_ENTRIES;
    P.load_comb(d1, d2, x, y);
#else
    uint32_t e[16];
    host_pos(pos, d1, d2, e);
    for (int i = 0; i < 8; i++) { x.v[i] = e[i]; y.v[i] = e[8 + i]; }
#endif
  }
  // entry idx of a table in GLOBAL memory: four 16-byte read-only loads (the entries are 64-byte aligned)
  IBFT_HD void load_wide(int idx, fe& x, fe& y) const {
    const uint32_t* e = base + (size_t)IBFT_GTAB_ENTRY_WORDS * (size_t)idx;
#if defined(__CUDA_ARCH__)
    const uint4* q = reinterpret_cast<const uint4*>(e);
    uint4 a = __ldg(q), b = __ldg(q + 1), c = __ldg(q + 2), d = __ldg(q + 3);
    x.v[0] = a.x; x.v[1] = a.y; x.v[2] = a.z; x.v[3] = a.w; x.v[4] = b.x; x.v[5] = b.y; x.v[6] = b.z; x.v[7] = b.w;
    y.v[0] = c.x; y.v[1] = c.y; y.v[2] = c.z; y.v[3] = c.w; y.v[4] = d.x; y.v[5] = d.y; y.v[6] = d.z; y.v[7] = d.w;
#else
    for (int i = 0; i < 8; i++) { x.v[i] = e[i]; y.v[i] = e[8 + i]; }
#endif
  }
  IBFT_HD void load(int idx, fe& x, fe& y) const {
    const uint32_t* e = base + IBFT_GTAB_ENTRY_WORDS * idx;
#pragma unroll
    for (int i = 0; i < 8; i++) {
      x.v[i] = e[i];
      y.v[i] = e[8 + i];
    }
  }
};

// Per-signature table {1..8}*R (affine x, y; 16 words per entry).  On the device it lives in SHARED memory, interleaved
// across the CTA's threads -- word (entry*16 + limb) of thread t sits at base[(entry*16 + limb) * stride + t] -- so that
// every lane always hits its own bank whatever entry it selects (conflict-free), and none of it ever reaches HBM.  (Kept
// in thread-local memory, the tables were written back through L2 to DRAM: several times the algorithmic traffic.)  The host emulation passes a plain array with stride 1.
struct rtab_view {
  uint32_t* base;
  uint32_t stride;
  IBFT_HD void store(int entry, const fe& x, const fe& y) const {
#pragma unroll
    for (int i = 0; i < 8; i++) {
      base[(uint32_t)(entry * 16 + i) * stride] = x.v[i];
      base[(uint32_t)(entry * 16 + 8 + i) * stride] = y.v[i];
    }
  }
  IBFT_HD void load(int entry, fe& x, fe& y) const {
#pragma unroll
    for (int i = 0; i < 8; i++) {
      x.v[i] = base[(uint32_t)(entry * 16 + i) * stride];
      y.v[i] = base[(uint32_t)(entry * 16 + 8 + i) * stride];
    }
  }
};
#define IBFT_RTAB_WORDS 128  // 8 entries x 16 words per signature

// inversion used for the per-signature table; defined by the including translation unit (verify_core.cuh)
IBFT_HD fe fe_inv_for_table(const fe& a);

#if defined(__CUDA_ARCH__)
#define IBFT_ROLLED _Pragma("unroll 1")
#else
#define IBFT_ROLLED
#endif

// {1..8} * R into T: entry m holds (m+1)R; even multiples by doubling, odd ones by adding R.  The table is then made
// AFFINE with one shared inversion (Montgomery's trick over the seven Z's), so that every addition of the main loop
// is a mixed addition (8M+3S instead of 12M+4S) and the loop holds a single adder.
// Every loop below is deliberately ROLLED and each group-law routine appears exactly once in the instruction stream:
// the kernel is instruction-cache bound otherwise (see secp_fe.cuh, IBFT_FN).
IBFT_HD void ecmult_build_rtable(const aff& R, const rtab_view& T) {
  fe zs[8];  // Z of entry m
  T.store(0, R.x, R.y);
  zs[0] = fe_from_u32(1);
  IBFT_ROLLED
  for (int m = 1; m < 8; m++) {
    jac p, t;
    int src = (m & 1) ? ((m + 1) >> 1) - 1 : m - 1;
    T.load(src, p.x, p.y);
    p.z = zs[src]; p.inf = false;
    if (m & 1) t = jac_double(p);
    else t = jac_add_affine(p, R.x, R.y);
    T.store(m, t.x, t.y);
    zs[m] = t.z;
  }
  // prefix products pre[m] = Z_1 * ... * Z_m (Z_0 = 1), one inversion, then peel the inverses off backwards
  IBFT_STAGE(5);
  fe pre[8];
  pre[1] = zs[1];
  IBFT_ROLLED
  for (int m = 2; m < 8; m++) pre[m] = fe_mul(pre[m - 1], zs[m]);
  fe acc_inv = fe_inv_for_table(pre[7]);
  IBFT_STAGE(6);
  IBFT_ROLLED
  for (int m = 7; m >= 1; m--) {
    fe zi = m > 1 ? fe_mul(acc_inv, pre[m - 1]) : acc_inv;  // 1 / Z_m
    if (m > 1) acc_inv = fe_mul(acc_inv, zs[m]);
    fe zi2 = fe_sqr(zi);
    fe x, y;
    T.load(m, x, y);
    T.store(m, fe_mul(x, zi2), fe_mul(y, fe_mul(zi2, zi)));
  }
}

// The same table WITHOUT any inversion ("effective affine", as libsecp256k1's odd-multiples table does it): build
// 2R = dbl(R), (m+1)R = mR + R, so that every new Z is the previous one times a known ratio (2y for the doubling, H for a mixed
// addition); scale every entry up to the LAST entry's Z with those ratios -- (X f^2, Y f^3), f = Z_8 / Z_m -- and read the
// table as AFFINE points of the isomorphic curve Y^2 = X^3 + 7 Z_8^6.  The caller runs the window loop on that curve (the a = 0
// law never uses b) and multiplies the accumulator's Z by the returned Z_8 at the end.  Only usable when nothing else (no
// generator point of the original curve) is added inside the loop: the chain warps of k_recover_split and the one-thread
// recovery (verify_core.cuh recover_key), which add u1*G after the loop.
// 1 dbl + 6 madd + 6 M + 7 (1S + 3M), against 4 dbl + 3 madd + inversion + 6 M + 7 (1S + 5M) for ecmult_build_rtable.
IBFT_HD fe ecmult_build_rtable_globalz(const aff& R, const rtab_view& T) {
  fe zr[8];  // zr[m] = Z of entry m / Z of entry m-1
  jac t;
  t.x = R.x; t.y = R.y; t.z = fe_from_u32(1); t.inf = false;
  T.store(0, R.x, R.y);
  IBFT_ROLLED
  for (int m = 1; m < 8; m++) {
    fe h;
    if (m == 1) { t = jac_double(t); h = t.z; }  // Z of R is 1
    else t = jac_add_affine(t, R.x, R.y, &h);
    T.store(m, t.x, t.y);
    zr[m] = h;
  }
  fe f = zr[7];
  IBFT_ROLLED
  for (int m = 6; m >= 0; m--) {
    if (m < 6) f = fe_mul(f, zr[m + 1]);
    fe f2 = fe_sqr(f);
    fe x, y;
    T.load(m, x, y);
    T.store(m, fe_mul(x, f2), fe_mul(y, fe_mul(f2, f)));
  }
  return t.z;
}

// digit streams of one double-scalar multiplication: 0 = u2 half 1 (R), 1 = u2 half 2 (lambda R), 2 = u1 half 1 (G),
// 3 = u1 half 2 (lambda G); magnitudes < 2^129 in five limbs (+ one zero limb for the Booth window reads), signs apart
struct ecmult_digits {
  uint32_t ks[4][6];
  bool kneg[4];
};
IBFT_HD void ecmult_split_into(const sc& k, ecmult_digits& d, int first) {
  glv_half h1, h2;
  glv_split(k, h1, h2);
#pragma unroll
  for (int i = 0; i < 5; i++) { d.ks[first][i] = h1.k[i]; d.ks[first + 1][i] = h2.k[i]; }
  d.ks[first][5] = d.ks[first + 1][5] = 0;
  d.kneg[first] = h1.neg; d.kneg[first + 1] = h2.neg;
}

// The interleaved window loop over the affine table T (streams 0, 1) and -- when with_g -- the generator table(s).
IBFT_HD jac ecmult_streams(const ecmult_digits& dg, const gtab_view& G, const rtab_view& T, bool with_g) {
  const fe beta = fe_beta();
  jac acc;
  acc.x = fe_zero(); acc.y = fe_zero(); acc.z = fe_zero();
  acc.inf = true;
  IBFT_ROLLED
  for (int j = IBFT_NWIN_R - 1; j >= 0; j--) {
    IBFT_OPCOUNT(IBFT_OP_WIN);
    if (!acc.inf) {
      IBFT_ROLLED
      for (int t = 0; t < IBFT_WR; t++) {
        IBFT_OPCOUNT(IBFT_OP_WIN_DBL);
        acc = jac_double(acc);
      }
    }
    // streams 0,1: R and lambda*R every window; streams 2,3: G and lambda*G every (WG/WR)-th window -- or, with a combined
    // table, ONE stream for both generator halves every (WC/WR)-th window
#if IBFT_WC > 0
    const bool comb = G.comb != nullptr;
    const int ns = !with_g ? 2 : comb ? ((j % (IBFT_WC / IBFT_WR) == 0) ? 3 : 2) : ((j % (IBFT_WG / IBFT_WR) == 0) ? 4 : 2);
#else
    const int ns = !with_g ? 2 : (j % (IBFT_WG / IBFT_WR) == 0) ? 4 : 2;
#endif
    IBFT_ROLLED
    for (int s = 0; s < ns; s++) {
      fe x, y;
      bool neg, use_beta = false;
#if IBFT_WC > 0
      if (comb && s == 2) {
        int jg = j / (IBFT_WC / IBFT_WR);
        int d1 = booth_digit<IBFT_WC>(dg.ks[2], jg), d2 = booth_digit<IBFT_WC>(dg.ks[3], jg);
        if (dg.kneg[2]) d1 = -d1;
        if (dg.kneg[3]) d2 = -d2;
        if ((d1 | d2) == 0) continue;
        neg = d1 < 0 || (d1 == 0 && d2 < 0);
        if (neg) { d1 = -d1; d2 = -d2; }
        G.load_comb(d1, d2, x, y);
      } else
#endif
      {
        int d = s < 2 ? booth_digit<IBFT_WR>(dg.ks[s], j) : booth_digit<IBFT_WG>(dg.ks[s], j / (IBFT_WG / IBFT_WR));
        if (d == 0) continue;
        int idx = (d < 0 ? -d : d) - 1;
        if (s < 2) T.load(idx, x, y);
        else G.load(idx, x, y);
        use_beta = (s & 1) != 0;
        neg = (d < 0) != dg.kneg[s];
      }
      if (use_beta) x = fe_mul(x, beta);  // lambda * (x, y) = (beta x, y)
      if (neg) y = fe_neg(y);
      IBFT_OPCOUNT(IBFT_OP_WIN_ADD);
      acc = jac_add_affine(acc, x, y);
    }
  }
  return acc;
}

// Returns u1*G + u2*R (R affine, on the curve) as a Jacobian point.  u1, u2 in [0, n).
IBFT_HD jac ecmult_double(const sc& u1, const sc& u2, const aff& R, const gtab_view& G, const rtab_view& T) {
  ecmult_digits dg;
  ecmult_split_into(u2, dg, 0);
  ecmult_split_into(u1, dg, 2);
  IBFT_STAGE(4);
  ecmult_build_rtable(R, T);
  IBFT_STAGE(7);
  return ecmult_streams(dg, G, T, true);
}

#if IBFT_WC > 0
// u1*G + u2*Q for a KNOWN point Q.  Q comes with a per-validator COMB table (IBFT_KEYTAB_COMB = 1, the default): position j
// (0..16) holds m * 2^(8j) * Q for m = 1..128 (affine, same entry format as the generator table; global memory, 136 KiB per
// validator), so the whole double-scalar multiplication is 17 positions x at most three mixed additions -- Q, lambda Q (the
// same entry with x * beta), and the generator's per-position comb entry -- and NOT ONE DOUBLING: 51 additions against the
// 136 doublings + 51 additions of a windowed walk (2.4x fewer wide multiply-adds), no per-signature table, no square root.
// IBFT_KEYTAB_COMB = 0 keeps the round-1 layout (one position, {1..128} * Q, 8 KiB per validator; 17 rounds of 8 doublings)
// for A/B measurements.  dg: streams 0,1 = split of u2, streams 2,3 = split of u1.
#define IBFT_WQ 8
#ifndef IBFT_KEYTAB_COMB
#define IBFT_KEYTAB_COMB 1
#endif
#define IBFT_KEYTAB_ENTRIES (1 << (IBFT_WQ - 1))
#define IBFT_KEYTAB_POSITIONS (IBFT_KEYTAB_COMB ? IBFT_CTAB_POSITIONS : 1)
#define IBFT_KEYTAB_WORDS ((size_t)IBFT_KEYTAB_POSITIONS * IBFT_KEYTAB_ENTRIES * IBFT_GTAB_ENTRY_WORDS)  // per validator
static_assert(IBFT_WQ == IBFT_WC, "the key comb shares the generator comb's positions");
IBFT_HD jac ecmult_streams_known(const ecmult_digits& dg, const gtab_view& G, const gtab_view& Qt, bool with_g = true) {
  const fe beta = fe_beta();
  jac acc;
  acc.x = fe_zero(); acc.y = fe_zero(); acc.z = fe_zero();
  acc.inf = true;
  IBFT_ROLLED
  for (int jg = IBFT_CTAB_POSITIONS - 1; jg >= 0; jg--) {
#if !IBFT_KEYTAB_COMB
    if (!acc.inf) {
      IBFT_ROLLED
      for (int t = 0; t < IBFT_WQ; t++) acc = jac_double(acc);
    }
#endif
    IBFT_ROLLED
    for (int s = 0; s < (with_g ? 3 : 2); s++) {
      fe x, y;
      bool neg;
      if (s == 2) {
        int d1 = booth_digit<IBFT_WC>(dg.ks[2], jg), d2 = booth_digit<IBFT_WC>(dg.ks[3], jg);
        if (dg.kneg[2]) d1 = -d1;
        if (dg.kneg[3]) d2 = -d2;
        if ((d1 | d2) == 0) continue;
        neg = d1 < 0 || (d1 == 0 && d2 < 0);
        if (neg) { d1 = -d1; d2 = -d2; }
#if IBFT_KEYTAB_COMB
        G.load_comb_pos(jg, d1, d2, x, y);
#else
        G.load_comb(d1, d2, x, y);
#endif
      } else {
        int d = booth_digit<IBFT_WQ>(dg.ks[s], jg);
        if (d == 0) continue;
#if IBFT_KEYTAB_COMB
        Qt.load_wide(jg * IBFT_KEYTAB_ENTRIES + (d < 0 ? -d : d) - 1, x, y);
#else
        Qt.load((d < 0 ? -d : d) - 1, x, y);
#endif
        if (s == 1) x = fe_mul(x, beta);
        neg = (d < 0) != dg.kneg[s];
      }
      if (neg) y = fe_neg(y);
      acc = jac_add_affine(acc, x, y);
    }
  }
  return acc;
}
#endif

#if IBFT_WC > 0
// u1*G alone as a fixed-base COMB over per-position tables (no doublings): position j of the table holds
// d1 * 2^(WC j) * G + d2 * 2^(WC j) * lambda G for the same (d1, d2) index space as the combined table (position 0 IS the
// combined table).  Used by the helper warp of the split latency kernel, which adds the result to the chain warp's u2*R.
// dg.ks[2], dg.ks[3] / kneg[2], kneg[3] must hold the split of u1.
IBFT_HD jac ecmult_gen_comb(const ecmult_digits& dg, const gtab_view& G) {
  jac acc;
  acc.x = fe_zero(); acc.y = fe_zero(); acc.z = fe_zero();
  acc.inf = true;
  IBFT_ROLLED
  for (int jg = IBFT_CTAB_POSITIONS - 1; jg >= 0; jg--) {
    int d1 = booth_digit<IBFT_WC>(dg.ks[2], jg), d2 = booth_digit<IBFT_WC>(dg.ks[3], jg);
    if (dg.kneg[2]) d1 = -d1;
    if (dg.kneg[3]) d2 = -d2;
    if ((d1 | d2) == 0) continue;
    bool neg = d1 < 0 || (d1 == 0 && d2 < 0);
    if (neg) { d1 = -d1; d2 = -d2; }
    fe x, y;
    G.load_comb_pos(jg, d1, d2, x, y);
    if (neg) y = fe_neg(y);
    IBFT_OPCOUNT(IBFT_OP_COMB_ADD);
    acc = jac_add_affine(acc, x, y);
  }
  return acc;
}

// L2 prefetch of the comb entries ecmult_gen_comb is about to read: the 17 gathers are issued together instead of one per
// dependent addition (the per-position tables are 36 MB, so a random entry is rarely in L2 already)
IBFT_HD void ecmult_gen_comb_prefetch(const ecmult_digits& dg, const gtab_view& G) {
#if defined(__CUDA_ARCH__)
  IBFT_ROLLED
  for (int jg = IBFT_CTAB_POSITIONS - 1; jg >= 0; jg--) {
    int d1 = booth_digit<IBFT_WC>(dg.ks[2], jg), d2 = booth_digit<IBFT_WC>(dg.ks[3], jg);
    if (dg.kneg[2]) d1 = -d1;
    if (dg.kneg[3]) d2 = -d2;
    if (d1 < 0 || (d1 == 0 && d2 < 0)) { d1 = -d1; d2 = -d2; }
    const uint32_t* e = G.comb + (size_t)jg * IBFT_GTAB_ENTRY_WORDS * (size_t)IBFT_CTAB_ENTRIES +
                        (size_t)IBFT_GTAB_ENTRY_WORDS * ((size_t)d1 * IBFT_CTAB_D2 + (size_t)(d2 + (1 << (IBFT_WC - 1))));
    asm volatile("prefetch.global.L2 [%0];" ::"l"(e));
    asm volatile("prefetch.global.L2 [%0];" ::"l"(e + 8));
  }
#else
  (void)dg;
  (void)G;
#endif
}
#endif

// The same double-scalar multiplication on the latency path: level-structured XYZZ group law driven by a lane executor
// (exec_quad on the device; the serial executor in the host emulation).  Same digit streams as ecmult_double; the
// per-signature table stays projective.  Table writes are done by the quad's leader lane, with a quad-level sync around them.
template <class EX>
IBFT_HD void ecmult_build_qtable(const EX& ex, const aff& R, const qtab_view& T) {
  const fe one = fe_from_u32(1);
  xyzz e0;
  e0.x = R.x; e0.y = R.y; e0.zz = one; e0.zzz = one; e0.inf = false;
  if (ex.leader()) T.store(0, e0);
  ex.sync();
  IBFT_ROLLED
  for (int m = 1; m < 8; m++) {
    int src = (m & 1) ? ((m + 1) >> 1) - 1 : m - 1;
    xyzz p = T.load(src);
    xyzz t = (m & 1) ? xyzz_double_x(ex, p) : xyzz_add_x(ex, p, e0);
    if (ex.leader()) T.store(m, t);
    ex.sync();
  }
}

template <class EX>
IBFT_HD xyzz ecmult_streams_x(const EX& ex, const ecmult_digits& dg, const gtab_view& G, const qtab_view& T, bool with_g) {
  const fe beta = fe_beta();
  const fe one = fe_from_u32(1);
  xyzz acc;
  acc.x = fe_zero(); acc.y = fe_zero(); acc.zz = fe_zero(); acc.zzz = fe_zero();
  acc.inf = true;
  IBFT_ROLLED
  for (int j = IBFT_NWIN_R - 1; j >= 0; j--) {
    if (!acc.inf) {
      IBFT_ROLLED
      for (int t = 0; t < IBFT_WR; t++) acc = xyzz_double_x(ex, acc);
    }
#if IBFT_WC > 0
    const bool comb = G.comb != nullptr;
    const int ns = !with_g ? 2 : comb ? ((j % (IBFT_WC / IBFT_WR) == 0) ? 3 : 2) : ((j % (IBFT_WG / IBFT_WR) == 0) ? 4 : 2);
#else
    const int ns = !with_g ? 2 : (j % (IBFT_WG / IBFT_WR) == 0) ? 4 : 2;
#endif
    IBFT_ROLLED
    for (int s = 0; s < ns; s++) {
      xyzz q;
      bool neg, use_beta = false;
#if IBFT_WC > 0
      if (comb && s == 2) {
        int jg = j / (IBFT_WC / IBFT_WR);
        int d1 = booth_digit<IBFT_WC>(dg.ks[2], jg), d2 = booth_digit<IBFT_WC>(dg.ks[3], jg);
        if (dg.kneg[2]) d1 = -d1;
        if (dg.kneg[3]) d2 = -d2;
        if ((d1 | d2) == 0) continue;
        neg = d1 < 0 || (d1 == 0 && d2 < 0);
        if (neg) { d1 = -d1; d2 = -d2; }
        G.load_comb(d1, d2, q.x, q.y);
        q.zz = one; q.zzz = one; q.inf = false;
      } else
#endif
      {
        int d = s < 2 ? booth_digit<IBFT_WR>(dg.ks[s], j) : booth_digit<IBFT_WG>(dg.ks[s], j / (IBFT_WG / IBFT_WR));
        if (d == 0) continue;
        int idx = (d < 0 ? -d : d) - 1;
        if (s < 2) {
          q = T.load(idx);
        } else {
          G.load(idx, q.x, q.y);
          q.zz = one; q.zzz = one; q.inf = false;
        }
        use_beta = (s & 1) != 0;
        neg = (d < 0) != dg.kneg[s];
      }
      if (use_beta) q.x = fe_mul(q.x, beta);  // lambda * (x, y) = (beta x, y)
      if (neg) q.y = fe_neg(q.y);
      acc = xyzz_add_x(ex, acc, q);
    }
  }
  return acc;
}

template <class EX>
IBFT_HD xyzz ecmult_double_x(const EX& ex, const sc& u1, const sc& u2, const aff& R, const gtab_view& G, const qtab_view& T) {
  ecmult_digits dg;
  ecmult_split_into(u2, dg, 0);
  ecmult_split_into(u1, dg, 2);
  IBFT_STAGE(4);
  ecmult_build_qtable(ex, R, T);
  IBFT_STAGE(5);
  IBFT_STAGE(6);
  IBFT_STAGE(7);
  return ecmult_streams_x(ex, dg, G, T, true);
}

}  // namespace ibft
