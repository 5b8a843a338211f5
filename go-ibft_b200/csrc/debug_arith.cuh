// debug_arith.cuh -- the arithmetic parity hooks IBFT_DBG_FE_MUL_RAW .. IBFT_DBG_SC_DIGITS and IBFT_DBG_RFC6979 of
// include/ibft_verify.h (TEST ONLY).
//
// One body for the device (k_debug_op in engine.cu) and the host emulation (emul_debug_op in tests/emul/emul.cpp), so both run
// the very routines the kernels run, on the same operands, and hand back their raw limbs: the tests chain non-canonical values
// the way the kernels do and compare with big integers.
#pragma once
#include "../../include/ibft_verify.h"
#include "secp_ec.cuh"
#include "sha256.cuh"

namespace ibft {

// a, b: 32-byte big-endian operands; o: the op's output (see ibft_verify.h); c: the 64-byte third operand of IBFT_DBG_RFC6979.
// Returns false for an op it does not handle, and for IBFT_DBG_RFC6979 without c.
IBFT_HD bool debug_arith_op(int op, const uint8_t* a, const uint8_t* b, uint8_t* o, const uint8_t* c = nullptr) {
  switch (op) {
    case IBFT_DBG_FE_MUL_RAW: fe_to_be(fe_mul(fe_from_be(a), fe_from_be(b)), o); return true;
    case IBFT_DBG_FE_SQR_RAW: fe_to_be(fe_sqr(fe_from_be(a)), o); return true;
    case IBFT_DBG_FE_ADD_RAW: fe_to_be(fe_add(fe_from_be(a), fe_from_be(b)), o); return true;
    case IBFT_DBG_FE_SUB_RAW: fe_to_be(fe_sub(fe_from_be(a), fe_from_be(b)), o); return true;
    case IBFT_DBG_FE_NORMALIZE: fe_to_be(fe_normalize(fe_from_be(a)), o); return true;
    case IBFT_DBG_FE_EQUAL: o[0] = fe_equal(fe_from_be(a), fe_from_be(b)) ? 1 : 0; return true;
    case IBFT_DBG_FE_SQRN: fe_to_be(fe_sqrn(fe_from_be(a), b[31]), o); return true;
    case IBFT_DBG_FE_SQRT_INV: {
      const fe_root_inv r = fe_sqrt_inv(fe_from_be(a), fe_from_be(b));
      fe_to_be(r.y, o);
      fe_to_be(r.w, o + 32);
      return true;
    }
    case IBFT_DBG_SC_ADD: sc_to_be(sc_add(sc_from_be(a), sc_from_be(b)), o); return true;
    case IBFT_DBG_SC_NEG: sc_to_be(sc_neg(sc_from_be(a)), o); return true;
    case IBFT_DBG_SC_REDUCE_ONCE: sc_to_be(sc_reduce_once(sc_from_be(a)), o); return true;
    case IBFT_DBG_SC_DIGITS: {  // the digits ecmult_streams (4-bit, R) and ecmult_gen_comb (8-bit, G) read from the halves
      ecmult_digits dg;
      ecmult_split_into(sc_from_be(a), dg, 0);
      for (int h = 0; h < 2; h++) {
        uint8_t* q = o + 128 * h;
        for (int i = 0; i < 128; i++) q[i] = 0;
        for (int i = 0; i < 6; i++)
          for (int j = 0; j < 4; j++) q[4 * i + j] = (uint8_t)(dg.ks[h][i] >> (8 * j));
        q[24] = dg.kneg[h] ? 1 : 0;
        for (int j = 0; j < IBFT_NWIN_R; j++) q[32 + j] = (uint8_t)(int8_t)booth_digit<4>(dg.ks[h], j);
        for (int j = 0; j < 17; j++) {
          const int d = booth_digit<8>(dg.ks[h], j);
          q[72 + 2 * j] = (uint8_t)(d & 0xFF);
          q[73 + 2 * j] = (uint8_t)((d >> 8) & 0xFF);
        }
      }
      return true;
    }
    case IBFT_DBG_RFC6979: {  // raw nonce candidate c[63] for the key a and the digest b
      if (c == nullptr) return false;
      uint8_t zm[32];
      sc_to_be(sc_reduce_once(sc_from_be(b)), zm);
      rfc6979_candidate(a, zm, c[63], o);
      return true;
    }
    case IBFT_DBG_FE_FUSED: {
      if (c == nullptr) return false;
      const fe x = fe_from_be(a), y = fe_from_be(b), z = fe_from_be(c);
      fe r;
      switch (c[63]) {
        case 0: r = fe_mul3(x); break;
        case 1: r = fe_sub_shl<1>(x, y); break;
        case 2: r = fe_sub_shl<3>(x, y); break;
        case 3: r = fe_sub_sub_dbl(x, y, z); break;
        case 4: r = fe_dbl_sub_sub(x, y, z); break;
        case 5: r = fe_sub_signed(x, y, false); break;
        case 6: r = fe_sub_signed(x, y, true); break;
        default: return false;
      }
      fe_to_be(r, o);
      return true;
    }
    default: return false;
  }
}

}  // namespace ibft
