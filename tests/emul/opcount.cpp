// The host emulation of emul.cpp with operation counters (TEST / TOOL ONLY).
//
// IBFT_OPCOUNT(k) (secp_fe.cuh, IBFT_OP_*) expands to nothing in every other build; here it counts the calls into the
// multiplier, the squarer, the doubling front, fe_sqrn iterations, inversions and window-loop steps, so that
// tools/fma_budget.py can multiply the per-routine SASS counts of k_recover by how often each routine runs per recovery.
// Built on demand by tools/fma_budget.py and tests/test_emul_madd_7m4s.py:
//   g++ -O2 -fPIC -std=c++17 -DEMUL_DIR=\"<tests/emul>\" -shared -o libibft_opcount.so opcount.cpp -lpthread
#include <atomic>

// operation counts since the last emul_op_reset
static std::atomic<unsigned long long> g_ops[32];
#define IBFT_OPCOUNT(k) g_ops[k].fetch_add(1, std::memory_order_relaxed)

#include "emul.cpp"

extern "C" {

// out[k] = IBFT_OP_k since the last reset; returns IBFT_OP_COUNT
int emul_op_counts(unsigned long long* out /* IBFT_OP_COUNT */) {
  for (int i = 0; i < IBFT_OP_COUNT; i++) out[i] = g_ops[i].load();
  return IBFT_OP_COUNT;
}
void emul_op_reset() {
  for (auto& c : g_ops) c.store(0);
}

}  // extern "C"
