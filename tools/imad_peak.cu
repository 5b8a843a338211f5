// Integer-pipe micro-benchmark for sm_90a (H100): measures the issue-rate ceilings that bound the
// secp256k1 kernels (IMAD, IMAD.WIDE, IMAD.WIDE.X carry chains, IADD3, LOP3, SHF and mixes).
// Test/measurement tool only (not part of the product path). Build:
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o imad_peak imad_peak.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

#define CK(x) do{cudaError_t e=(x); if(e!=cudaSuccess){printf("CUDA error %s at %d\n",cudaGetErrorString(e),__LINE__); return 1;}}while(0)
constexpr int ITERS = 4096;
constexpr int UNROLL = 16;   // instructions per chain per iteration

// K independent chains per thread so latency is hidden; every variant does ITERS*UNROLL*K instrs/thread.
template<int K> __global__ void k_imad(uint32_t* out, uint32_t a, uint32_t b){
  uint32_t x[K]; for(int k=0;k<K;k++) x[k]=threadIdx.x+k;
  for(int i=0;i<ITERS;i++){
    #pragma unroll
    for(int u=0;u<UNROLL;u++){
      #pragma unroll
      for(int k=0;k<K;k++) asm volatile("mad.lo.u32 %0,%0,%1,%2;":"+r"(x[k]):"r"(a),"r"(b));
    }
  }
  uint32_t s=0; for(int k=0;k<K;k++) s^=x[k]; out[blockIdx.x*blockDim.x+threadIdx.x]=s;
}
template<int K> __global__ void k_imad_hi(uint32_t* out, uint32_t a, uint32_t b){
  uint32_t x[K]; for(int k=0;k<K;k++) x[k]=threadIdx.x+k;
  for(int i=0;i<ITERS;i++){
    #pragma unroll
    for(int u=0;u<UNROLL;u++){
      #pragma unroll
      for(int k=0;k<K;k++) asm volatile("mad.hi.u32 %0,%0,%1,%2;":"+r"(x[k]):"r"(a),"r"(b));
    }
  }
  uint32_t s=0; for(int k=0;k<K;k++) s^=x[k]; out[blockIdx.x*blockDim.x+threadIdx.x]=s;
}
template<int K> __global__ void k_imad_wide(uint32_t* out, uint32_t a, uint32_t b){
  uint64_t x[K]; for(int k=0;k<K;k++) x[k]=threadIdx.x+k;
  for(int i=0;i<ITERS;i++){
    #pragma unroll
    for(int u=0;u<UNROLL;u++){
      #pragma unroll
      for(int k=0;k<K;k++){ uint32_t lo=(uint32_t)x[k]; asm volatile("mad.wide.u32 %0,%1,%2,%0;":"+l"(x[k]):"r"(lo),"r"(b)); }
    }
  }
  uint64_t s=0; for(int k=0;k<K;k++) s^=x[k]; out[blockIdx.x*blockDim.x+threadIdx.x]=(uint32_t)(s^(s>>32));
}
// carry chain: 4 wide MACs chained through CC (mad.lo.cc/madc.hi.cc pairs -> IMAD.WIDE.U32.X)
template<int K> __global__ void k_imad_wide_x(uint32_t* out, uint32_t a, uint32_t b){
  uint32_t x[K][8]; for(int k=0;k<K;k++) for(int j=0;j<8;j++) x[k][j]=threadIdx.x+k+j;
  for(int i=0;i<ITERS;i++){
    #pragma unroll
    for(int u=0;u<UNROLL/4;u++){
      #pragma unroll
      for(int k=0;k<K;k++){
        asm volatile("mad.lo.cc.u32 %0,%8,%9,%0; madc.hi.cc.u32 %1,%8,%9,%1;"
                     "madc.lo.cc.u32 %2,%8,%9,%2; madc.hi.cc.u32 %3,%8,%9,%3;"
                     "madc.lo.cc.u32 %4,%8,%9,%4; madc.hi.cc.u32 %5,%8,%9,%5;"
                     "madc.lo.cc.u32 %6,%8,%9,%6; madc.hi.u32 %7,%8,%9,%7;"
                     :"+r"(x[k][0]),"+r"(x[k][1]),"+r"(x[k][2]),"+r"(x[k][3]),"+r"(x[k][4]),"+r"(x[k][5]),"+r"(x[k][6]),"+r"(x[k][7])
                     :"r"(a),"r"(b));
      }
    }
  }
  uint32_t s=0; for(int k=0;k<K;k++) for(int j=0;j<8;j++) s^=x[k][j]; out[blockIdx.x*blockDim.x+threadIdx.x]=s;
}
template<int K> __global__ void k_iadd3(uint32_t* out, uint32_t a, uint32_t b){
  uint32_t x[K]; for(int k=0;k<K;k++) x[k]=threadIdx.x+k;
  for(int i=0;i<ITERS;i++){
    #pragma unroll
    for(int u=0;u<UNROLL;u++){
      #pragma unroll
      for(int k=0;k<K;k++) asm volatile("add.u32 %0,%0,%1;":"+r"(x[k]):"r"(a));
    }
  }
  uint32_t s=0; for(int k=0;k<K;k++) s^=x[k]; out[blockIdx.x*blockDim.x+threadIdx.x]=s+b;
}
template<int K> __global__ void k_lop3(uint32_t* out, uint32_t a, uint32_t b){
  uint32_t x[K]; for(int k=0;k<K;k++) x[k]=threadIdx.x+k;
  for(int i=0;i<ITERS;i++){
    #pragma unroll
    for(int u=0;u<UNROLL;u++){
      #pragma unroll
      for(int k=0;k<K;k++) asm volatile("lop3.b32 %0,%0,%1,%2,0x96;":"+r"(x[k]):"r"(a),"r"(b));
    }
  }
  uint32_t s=0; for(int k=0;k<K;k++) s^=x[k]; out[blockIdx.x*blockDim.x+threadIdx.x]=s;
}
template<int K> __global__ void k_shf(uint32_t* out, uint32_t a, uint32_t b){
  uint32_t x[K]; for(int k=0;k<K;k++) x[k]=threadIdx.x+k;
  for(int i=0;i<ITERS;i++){
    #pragma unroll
    for(int u=0;u<UNROLL;u++){
      #pragma unroll
      for(int k=0;k<K;k++) asm volatile("shf.l.wrap.b32 %0,%0,%1,%2;":"+r"(x[k]):"r"(a),"r"(b));
    }
  }
  uint32_t s=0; for(int k=0;k<K;k++) s^=x[k]; out[blockIdx.x*blockDim.x+threadIdx.x]=s;
}
// mix: one IMAD.WIDE + one LOP3 per slot (do the two pipes dual-issue at 2x?)
template<int K> __global__ void k_mix(uint32_t* out, uint32_t a, uint32_t b){
  uint64_t x[K]; uint32_t y[K]; for(int k=0;k<K;k++){ x[k]=threadIdx.x+k; y[k]=k; }
  for(int i=0;i<ITERS;i++){
    #pragma unroll
    for(int u=0;u<UNROLL/2;u++){
      #pragma unroll
      for(int k=0;k<K;k++){
        { uint32_t lo=(uint32_t)x[k]; asm volatile("mad.wide.u32 %0,%1,%2,%0;":"+l"(x[k]):"r"(lo),"r"(b)); }
        asm volatile("lop3.b32 %0,%0,%1,%2,0x96;":"+r"(y[k]):"r"(a),"r"(b));
      }
    }
  }
  uint64_t s=0; for(int k=0;k<K;k++) s^=x[k]^y[k]; out[blockIdx.x*blockDim.x+threadIdx.x]=(uint32_t)(s^(s>>32));
}

template<typename F> int run(const char* name, F launch, double instr_per_thread, int blocks, int threads, int sms, int clk_khz){
  cudaEvent_t e0,e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  launch(); CK(cudaDeviceSynchronize());
  float best=1e30f;
  for(int r=0;r<5;r++){ CK(cudaEventRecord(e0)); launch(); CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1)); float ms; CK(cudaEventElapsedTime(&ms,e0,e1)); if(ms<best) best=ms; }
  double total = instr_per_thread*(double)blocks*threads;
  double per_s = total/(best*1e-3);
  printf("{\"bench\":\"%s\",\"ms\":%.4f,\"thread_instr_per_s\":%.4e,\"per_sm_per_clk_at_max\":%.2f}\n", name,best,per_s, per_s/sms/(clk_khz*1e3));
  return 0;
}

int main(){
  cudaDeviceProp p; CK(cudaGetDeviceProperties(&p,0));
  int clk_khz=0; CK(cudaDeviceGetAttribute(&clk_khz,cudaDevAttrClockRate,0));
  int sms=p.multiProcessorCount;
  printf("{\"device\":\"%s\",\"sms\":%d,\"clock_khz\":%d,\"cc\":\"%d.%d\"}\n",p.name,sms,clk_khz,p.major,p.minor);
  int threads=256, blocks=sms*8;
  uint32_t* out; CK(cudaMalloc(&out,(size_t)blocks*threads*4));
  double n=(double)ITERS*UNROLL;
  run("imad_lo_k4",[&]{k_imad<4><<<blocks,threads>>>(out,3,5);}, n*4,blocks,threads,sms,clk_khz);
  run("imad_lo_k8",[&]{k_imad<8><<<blocks,threads>>>(out,3,5);}, n*8,blocks,threads,sms,clk_khz);
  run("imad_hi_k8",[&]{k_imad_hi<8><<<blocks,threads>>>(out,3,5);}, n*8,blocks,threads,sms,clk_khz);
  run("imad_wide_k4",[&]{k_imad_wide<4><<<blocks,threads>>>(out,3,5);}, n*4,blocks,threads,sms,clk_khz);
  run("imad_wide_k8",[&]{k_imad_wide<8><<<blocks,threads>>>(out,3,5);}, n*8,blocks,threads,sms,clk_khz);
  run("imad_wide_x_chain_k2",[&]{k_imad_wide_x<2><<<blocks,threads>>>(out,3,5);}, n*2,blocks,threads,sms,clk_khz);
  run("imad_wide_x_chain_k4",[&]{k_imad_wide_x<4><<<blocks,threads>>>(out,3,5);}, n*4,blocks,threads,sms,clk_khz);
  run("iadd3_k8",[&]{k_iadd3<8><<<blocks,threads>>>(out,3,5);}, n*8,blocks,threads,sms,clk_khz);
  run("lop3_k8",[&]{k_lop3<8><<<blocks,threads>>>(out,3,5);}, n*8,blocks,threads,sms,clk_khz);
  run("shf_k8",[&]{k_shf<8><<<blocks,threads>>>(out,3,5);}, n*8,blocks,threads,sms,clk_khz);
  run("mix_wide_lop3_k4",[&]{k_mix<4><<<blocks,threads>>>(out,3,5);}, n*4,blocks,threads,sms,clk_khz);
  return 0;
}
