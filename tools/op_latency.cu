// Development tool: dependent-chain latency (cycles per operation, one warp per SM sub-partition) of the field and group
// operations, serial and four-lane.   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -diag-suppress 550 -I include tools/op_latency.cu -o tools/op_latency
#include "../go-ibft_b200/csrc/engine.cu"
#include <cstdio>

struct fe2 { fe a, b; };
__device__ __noinline__ fe2 fe_mul2(fe a, fe b, fe c, fe d) {
  fe2 r;
  r.a = fe_mul_i(a, b);
  r.b = fe_mul_i(c, d);
  return r;
}
struct fe3 { fe a, b, c; };
__device__ __noinline__ fe3 fe_mul3(fe a, fe b, fe c, fe d, fe e, fe f) {
  fe3 r;
  r.a = fe_mul_i(a, b);
  r.b = fe_mul_i(c, d);
  r.c = fe_mul_i(e, f);
  return r;
}
__device__ __forceinline__ fe fe_xor(const fe& a, const fe& b) {
  fe r;
  for (int i = 0; i < 8; i++) r.v[i] = a.v[i] ^ b.v[i];
  return r;
}

__global__ void k_lat(unsigned long long* out, uint32_t* sink, int reps) {
  fe x = fe_from_u32(threadIdx.x + 3), y = fe_from_u32(0x12345 + (threadIdx.x >> 2));
  for (int i = 0; i < 8; i++) { x.v[i] ^= 0x9e3779b9u * (i + 1 + (threadIdx.x >> 2)); y.v[i] ^= 0x85ebca6bu * (i + 2); }
  exec_quad ex;
  ex.role = threadIdx.x & 3;
  ex.mask = 0xFu << (threadIdx.x & 28u);
  __shared__ uint4 s_xb[4 * 128];
  ex.xb = s_xb;
  ex.par = 0;
  unsigned long long t0, t1;
  int k = 0;
#define MEASURE(...)                                \
  __syncthreads();                                  \
  t0 = clock64();                                   \
  _Pragma("unroll 1") for (int i = 0; i < reps; i++) { __VA_ARGS__; } \
  t1 = clock64();                                   \
  if (threadIdx.x == 0) out[k] = (t1 - t0) / reps;  \
  k++;
  MEASURE(x = fe_mul(x, y))
  MEASURE(x = fe_sqr(x))
  MEASURE(x = fe_add(x, y))
  MEASURE(x = fe_sub(x, y))
  MEASURE(x = fe_dbl(x))
  {
    fe a[4], b[4], o[4];
    MEASURE(a[0] = x; b[0] = y; ex.mul4(a, b, 1, o); x = o[0])
    MEASURE(a[0] = x; b[0] = y; a[1] = y; b[1] = x; ex.mul4(a, b, 2, o); x = fe_add(o[0], o[1]))
    MEASURE(a[0] = x; b[0] = y; a[1] = y; b[1] = x; a[2] = x; b[2] = x; a[3] = y; b[3] = y; ex.mul4(a, b, 4, o); x = fe_add(fe_add(o[0], o[1]), fe_add(o[2], o[3])))
  }
  {
    xyzz p;
    p.x = x; p.y = y; p.zz = fe_sqr(y); p.zzz = fe_mul(p.zz, y); p.inf = false;
    xyzz q = p;
    q.x = fe_add(q.x, y);
    MEASURE(p = xyzz_double_x(ex, p))
    MEASURE(p = xyzz_add_x(ex, p, q))
    exec_serial es;
    MEASURE(p = xyzz_double_x(es, p))
    MEASURE(p = xyzz_add_x(es, p, q))
    x = fe_add(p.x, fe_add(p.y, fe_add(p.zz, p.zzz)));
  }
  {
    jac p;
    p.x = x; p.y = y; p.z = fe_sqr(y); p.inf = false;
    MEASURE(p = jac_double(p))
    MEASURE(p = jac_add_affine(p, x, y))
    x = fe_add(p.x, fe_add(p.y, p.z));
  }
  MEASURE(x = IBFT_FE_INV(x))
  MEASURE(fe2 r2 = fe_mul2(x, y, y, x); x = fe_xor(r2.a, r2.b))
  MEASURE(fe3 r3 = fe_mul3(x, y, y, x, x, x); x = fe_xor(r3.a, fe_xor(r3.b, r3.c)))
  {
    const int base = (int)(threadIdx.x & 31u) & ~3;
    MEASURE(fe o[4]; for (int kk = 0; kk < 4; kk++) for (int i = 0; i < 8; i++) o[kk].v[i] = __shfl_sync(ex.mask, x.v[i] + kk, base + kk);
            x = fe_xor(fe_xor(o[0], o[1]), fe_xor(o[2], o[3])))
    __shared__ uint4 s_x[128 * 2];
    MEASURE(s_x[threadIdx.x * 2] = make_uint4(x.v[0], x.v[1], x.v[2], x.v[3]); s_x[threadIdx.x * 2 + 1] = make_uint4(x.v[4], x.v[5], x.v[6], x.v[7]);
            __syncwarp(ex.mask);
            fe o[4];
            for (int kk = 0; kk < 4; kk++) {
              uint4 lo = s_x[((threadIdx.x & ~3u) + kk) * 2], hi = s_x[((threadIdx.x & ~3u) + kk) * 2 + 1];
              o[kk].v[0] = lo.x; o[kk].v[1] = lo.y; o[kk].v[2] = lo.z; o[kk].v[3] = lo.w; o[kk].v[4] = hi.x; o[kk].v[5] = hi.y; o[kk].v[6] = hi.z; o[kk].v[7] = hi.w;
            }
            __syncwarp(ex.mask);
            x = fe_xor(fe_xor(o[0], o[1]), fe_xor(o[2], o[3])))
    fe a[4];
    a[0] = x; a[1] = y; a[2] = fe_xor(x, y); a[3] = fe_dbl(y);
    MEASURE(a[0] = exec_quad::pick(ex.role, a, 4); a[0].v[0] += 1)
    x = a[0];
  }
  for (int i = 0; i < 8; i++) sink[threadIdx.x * 8 + i] = x.v[i];
}

int main() {
  unsigned long long* d_out;
  uint32_t* d_sink;
  cudaMalloc(&d_out, 32 * 8);
  cudaMalloc(&d_sink, 128 * 8 * 4);
  cudaMemset(d_out, 0, 32 * 8);
  for (int it = 0; it < 2; it++) k_lat<<<1, 128>>>(d_out, d_sink, 200);
  cudaError_t err = cudaDeviceSynchronize();
  if (err != cudaSuccess) { fprintf(stderr, "%s\n", cudaGetErrorString(err)); return 1; }
  unsigned long long h[32];
  cudaMemcpy(h, d_out, sizeof h, cudaMemcpyDeviceToHost);
  const char* names[] = {"fe_mul", "fe_sqr", "fe_add", "fe_sub", "fe_dbl", "quad mul4 x1", "quad mul4 x2 + add", "quad mul4 x4 + 3 add",
                         "xyzz_double quad", "xyzz_add quad", "xyzz_double serial", "xyzz_add serial", "jac_double serial", "jac_add_affine serial", "fe_inv (safegcd)", "fe_mul2 (dual, noinline)", "fe_mul3 (triple, noinline)", "shfl all-gather x4", "smem all-gather x4", "pick x4"};
  for (int i = 0; i < 20; i++) printf("%-26s %8llu cycles\n", names[i], h[i]);
  return 0;
}
