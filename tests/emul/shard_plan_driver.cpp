// C entry points over go-ibft_b200/csrc/shard_plan.hpp (the multi-device engine's shard planner) for tests/test_shard_plan.py.
#include "../../go-ibft_b200/csrc/shard_plan.hpp"

extern "C" {

uint32_t sp_devices(uint32_t n, uint32_t n_devices) { return ibft::shard_devices(n, n_devices); }

void sp_bounds(uint32_t n, uint32_t world, uint32_t rank, uint32_t* lo, uint32_t* hi) { ibft::shard_bounds(n, world, rank, lo, hi); }

// items[lo, hi) of a call over arena[0, arena_len) -> local[0, hi - lo) and local_arena; returns the shard arena's length
size_t sp_plan(const ibft_sig_item* items, uint32_t lo, uint32_t hi, const uint8_t* arena, size_t arena_len, ibft_sig_item* local,
               uint8_t* local_arena) {
  std::vector<ibft::arena_run> runs;
  const size_t len = ibft::plan_shard(items, lo, hi, arena_len, local, runs);
  ibft::copy_runs(arena, runs, local_arena);
  return len;
}
}
