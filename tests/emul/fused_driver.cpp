// The fused linear combinations of the group law (secp_fe.cuh: fe_mul3, fe_sub_shl, fe_sub_sub_dbl, fe_dbl_sub_sub,
// fe_sub_signed) on the host emulation (TEST ONLY), through the IBFT_DBG_FE_FUSED body the device runs.  Built on demand by
// tests/test_emul_fused_ops.py:
//   g++ -O2 -fPIC -std=c++17 -DEMUL_DIR=\"<tests/emul>\" -shared -o libibft_fused.so fused_driver.cpp -lpthread
#include "emul.cpp"

extern "C" {

// a, b, c: 32-byte big-endian operands; c[63] = the selector of IBFT_DBG_FE_FUSED.  Returns -1 for an unknown selector.
int emul_fe_fused(const uint8_t* a, const uint8_t* b, const uint8_t* c64, uint8_t* out) {
  return debug_arith_op(IBFT_DBG_FE_FUSED, a, b, out, c64) ? 0 : -1;
}
}
