// C entry points over go-ibft_b200/csrc/recover_plan.hpp (the recover step's kernel choice) for tests/test_recover_plan.py.
#include "../../go-ibft_b200/csrc/recover_plan.hpp"

extern "C" {

int rp_known(int key_cache, int want_recovered, int groups, int worklist, uint32_t cnt, uint32_t worklist_cap) {
  return ibft::known_key_ok(key_cache, want_recovered, groups, worklist, cnt, worklist_cap);
}

// first kernel * 16 + worklist kernel (ibft::sig_kernel values)
int rp_plan(int path, uint32_t cnt, size_t arena_len, uint32_t sms, int known, int wc) {
  const ibft::recover_plan p = ibft::plan_recover(path, cnt, arena_len, sms, known, wc);
  return p.first * 16 + p.worklist;
}

uint32_t rp_pieces(int path, uint32_t n, size_t arena_len, uint32_t sms, int known, int wc, int* piece_path) {
  const ibft::piece_plan p = ibft::plan_pieces(path, n, arena_len, sms, known, wc);
  *piece_path = p.path;
  return p.per;
}
}
