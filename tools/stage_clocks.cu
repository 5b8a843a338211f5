// Development tool: per-stage clock64() stamps of ONE signature's serial chain (thread 0 of CTA 0), for the one-thread and the
// four-lane recover kernels.  Builds the whole engine translation unit with IBFT_STAGE_CLOCKS.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -diag-suppress 550 -I include tools/stage_clocks.cu -o tools/stage_clocks
//   tools/stage_clocks items.bin [n_items]      (items.bin: packed 128-byte tuples, e.g. dumped from tests/golden/config3.npz)
#define IBFT_STAGE_CLOCKS 1
#include "../go-ibft_b200/csrc/engine.cu"
#include <cstdio>
#include <vector>

int main(int argc, char** argv) {
  if (argc < 2) { fprintf(stderr, "usage: %s items.bin [n]\n", argv[0]); return 2; }
  FILE* f = fopen(argv[1], "rb");
  if (!f) { perror("items"); return 2; }
  std::vector<ibft_sig_item> items;
  ibft_sig_item it;
  while (fread(&it, sizeof it, 1, f) == 1) items.push_back(it);
  fclose(f);
  uint32_t n = argc > 2 ? (uint32_t)atoi(argv[2]) : 128u;
  if (n > items.size()) n = (uint32_t)items.size();
  ibft_engine_params p{};
  p.device = 0; p.max_items = 1 << 16; p.max_payload_bytes = 1 << 20; p.max_groups = 4; p.max_table_slots = 1; p.max_validators = 16;
  ibft_engine* e = nullptr;
  if (ibft_engine_create(&p, &e) != IBFT_OK) { fprintf(stderr, "create: %s\n", ibft_last_error()); return 1; }
  std::vector<uint32_t> bm((n + 31) / 32);
  uint8_t dummy = 0;
  static const char* names[] = {"digest(keccak)+checks", "sqrt / lift_x", "r^-1, u1, u2", "glv split", "table build (7 group ops)",
                                "table inversion", "table normalise", "main loop", "final inversion + affine", "keccak(address)"};
  for (int path = IBFT_PATH_THREAD; path <= IBFT_PATH_QUAD; path++) {  // (the split kernel has no single-thread chain to stamp)
    ibft_set_recover_path(e, path);
    for (int rep = 0; rep < 3; rep++)
      if (ibft_verify_batch(e, items.data(), n, &dummy, 0, nullptr, 0, bm.data(), nullptr, nullptr) != IBFT_OK) {
        fprintf(stderr, "verify: %s\n", ibft_last_error());
        return 1;
      }
    unsigned long long clk[16];
    cudaMemcpyFromSymbol(clk, g_stage_clk, sizeof clk);
    printf("path=%s n=%u bit0=%u total=%llu cycles\n", path == IBFT_PATH_THREAD ? "thread" : "quad", n, bm[0] & 1u, clk[10] - clk[0]);
    for (int i = 0; i < 10; i++) printf("  %-28s %8llu  %5.1f%%\n", names[i], clk[i + 1] - clk[i], 100.0 * (clk[i + 1] - clk[i]) / (clk[10] - clk[0]));
  }
  ibft_engine_destroy(e);
  return 0;
}
