// Microbenchmark: latency/throughput of warp arg-max primitives on sm_90a with 1 vs 24 resident warps per SM.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o redux_bench redux_bench.cu
#include <cstdio>
#include <cuda_runtime.h>
__device__ __forceinline__ unsigned shfl_max(unsigned v) {
  #pragma unroll
  for (int o = 16; o > 0; o >>= 1) { unsigned u = __shfl_xor_sync(0xffffffffu, v, o); v = u > v ? u : v; }
  return v;
}
template <int MODE> __global__ void k(unsigned *out, long long *cyc, int iters) {
  unsigned x = threadIdx.x * 2654435761u;
  __syncthreads();
  long long t0 = clock64();
  for (int i = 0; i < iters; i++) {
    if (MODE == 0) x = __reduce_max_sync(0xffffffffu, x ^ i) + threadIdx.x;       // REDUX / CREDUX
    else if (MODE == 1) x = shfl_max(x ^ i) + threadIdx.x;                        // 5 x SHFL butterfly
    else if (MODE == 2) { unsigned b = __ballot_sync(0xffffffffu, (x ^ i) & 1); x = x * 3u + b; }   // VOTE
    else { x = x * 3u + i; __syncthreads(); }                                     // BAR.SYNC
  }
  long long t1 = clock64();
  if (threadIdx.x == 0 && blockIdx.x == 0) cyc[0] = t1 - t0;
  out[blockIdx.x * blockDim.x + threadIdx.x] = x;
}
int main() {
  unsigned *out; long long *cyc, h;
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);     // one CTA per SM
  cudaMalloc(&out, (size_t)sms * 1024 * 4); cudaMalloc(&cyc, 8);
  const int iters = 2000;
  const char *names[] = {"__reduce_max_sync (REDUX)", "shfl butterfly max", "ballot", "__syncthreads"};
  for (int threads : {32, 256, 768}) {
    for (int mode = 0; mode < 4; mode++) {
      for (int rep = 0; rep < 2; rep++) {
        if (mode == 0) k<0><<<sms, threads>>>(out, cyc, iters);
        if (mode == 1) k<1><<<sms, threads>>>(out, cyc, iters);
        if (mode == 2) k<2><<<sms, threads>>>(out, cyc, iters);
        if (mode == 3) k<3><<<sms, threads>>>(out, cyc, iters);
        cudaDeviceSynchronize();
      }
      cudaMemcpy(&h, cyc, 8, cudaMemcpyDeviceToHost);
      printf("threads/CTA %4d  %-28s %8.1f cycles per op (dependent chain, all warps at once)\n", threads, names[mode], (double)h / iters);
    }
  }
  return 0;
}
