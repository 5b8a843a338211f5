// key_matches_address (verify_core.cuh), the check k_adopt_peer_keys makes before a device of a multi-device engine takes a key
// another device learned, on the host emulation (TEST ONLY).  Built on demand by tests/test_emul_key_share.py:
//   g++ -O2 -fPIC -std=c++17 -DEMUL_DIR=\"<tests/emul>\" -shared -o libibft_key_share.so key_share_driver.cpp -lpthread
#include "emul.cpp"

extern "C" {

// 1 when the key (x, y: 32-byte big-endian, taken as given) may stand in the registry entry of addr20, else 0
int emul_key_matches_address(const uint8_t* x_be, const uint8_t* y_be, const uint8_t* addr20) {
  return key_matches_address(fe_from_be(x_be), fe_from_be(y_be), addr20) ? 1 : 0;
}
}
