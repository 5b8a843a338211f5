// C entry points around go-ibft_b200/csrc/key_budget.hpp (the bounded key registry's table policy) for
// tests/test_key_budget_policy.py, which builds this file with g++ and compares it with a Python model of the ranking.
#include "../../go-ibft_b200/csrc/key_budget.hpp"

extern "C" {
void* kb_new() { return new ibft::key_budget(); }
void kb_free(void* h) { delete static_cast<ibft::key_budget*>(h); }
// one reclaim point; table_out[r] = entry r's slot afterwards (0xFFFFFFFF: none); returns the number of moves
uint32_t kb_reclaim(void* h, uint32_t n, const uint8_t* listed, const uint8_t* known, const uint8_t* used, const uint8_t* addr,
                    uint32_t new_max, uint32_t* table_out, uint32_t* n_evicted, uint32_t* n_admitted, uint32_t* n_retired) {
  auto* b = static_cast<ibft::key_budget*>(h);
  const ibft::key_budget::plan p = b->reclaim(n, listed, known, used, addr, new_max);
  for (uint32_t r = 0; r < n; r++) table_out[r] = b->table[r];
  *n_evicted = (uint32_t)p.evicted.size();
  *n_admitted = (uint32_t)p.admitted.size();
  *n_retired = (uint32_t)p.retired.size();
  for (const auto& m : p.moves)
    if (m.from < new_max || m.to >= new_max || b->table[m.entry] != m.to) return 0xFFFFFFFFu;
  return (uint32_t)p.moves.size();
}
uint32_t kb_take_free(void* h, uint32_t n, uint32_t r) {
  auto* b = static_cast<ibft::key_budget*>(h);
  b->ensure(n);
  return b->take_free(r);
}
uint32_t kb_live(void* h) { return static_cast<ibft::key_budget*>(h)->live(); }
}
