// fp64_probe.cu -- latency of a dependent FP64 add chain on the device (what bounds the in-order sums of the
// MAD-tree build, tools/utils.h:55-73).  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -fmad=false scripts/fp64_probe.cu -o scripts/_bin/fp64_probe
#include <cstdio>
#include <cuda_runtime.h>
__global__ void chain1(const double* x, int n, double* out, long long* cyc) {
  __shared__ double tile[1024];
  double s = 0;
  long long t0 = clock64();
  for (int b = 0; b < n; b += 1024) {
    for (int i = threadIdx.x; i < 1024; i += blockDim.x) tile[i] = x[b + i];
    __syncthreads();
    if (threadIdx.x < 9) {
#pragma unroll 16
      for (int i = 0; i < 1024; ++i) s = __dadd_rn(s, __dmul_rn(tile[i], tile[(i + threadIdx.x) & 1023]));
    }
    __syncthreads();
  }
  if (threadIdx.x < 9) out[threadIdx.x] = s;
  if (threadIdx.x == 0) *cyc = clock64() - t0;
}
__global__ void chain_ilp(const double* x, int n, double* out, long long* cyc) {  // one thread, 9 chains
  double s[9] = {0};
  long long t0 = clock64();
  if (threadIdx.x == 0) {
    for (int i = 0; i < n; ++i) {
      const double v = x[i];
#pragma unroll
      for (int k = 0; k < 9; ++k) s[k] = __dadd_rn(s[k], __dmul_rn(v, v + k));
    }
    double t = 0;
    for (int k = 0; k < 9; ++k) t += s[k];
    out[0] = t;
    *cyc = clock64() - t0;
  }
}
int main() {
  const int n = 131072;
  double *x, *o; long long* c;
  cudaMalloc(&x, n * 8); cudaMalloc(&o, 128); cudaMalloc(&c, 8);
  double* h = new double[n];
  for (int i = 0; i < n; ++i) h[i] = 1.0 + 1e-3 * (i % 977);
  cudaMemcpy(x, h, n * 8, cudaMemcpyHostToDevice);
  long long hc;
  for (int rep = 0; rep < 2; ++rep) {
    chain1<<<1, 128>>>(x, n, o, c); cudaMemcpy(&hc, c, 8, cudaMemcpyDeviceToHost);
    printf("9 lanes, one chain each (smem tiles): %.2f cycles per element (n=%d, %lld cycles)\n", double(hc) / n, n, hc);
    chain_ilp<<<1, 32>>>(x, n, o, c); cudaMemcpy(&hc, c, 8, cudaMemcpyDeviceToHost);
    printf("1 thread, 9 chains ILP (global loads): %.2f cycles per element\n", double(hc) / n);
  }
  return 0;
}
