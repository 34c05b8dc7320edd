// Micro-probe of the register-resident Gauss-Jordan pivot loop of dspgn_solve.cuh (test tooling, not product):
// where do the cycles of one pivot go?  thread 0 accumulates clock64 deltas over the 71 pivots.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/probes/solve_probe tools/probes/solve_probe.cu && ./solve_probe
#include <cstdio>
#include <cuda_runtime.h>
constexpr int N = 71, NP = 72, STRIDE = 73;
__device__ __forceinline__ void bar96() { asm volatile("bar.sync 2, 96;" ::: "memory"); }
template <int VARIANT>
__global__ void __launch_bounds__(256) k_probe(const float* __restrict__ A, float* __restrict__ x, long long* clk) {
  __shared__ float As[N * STRIDE];
  __shared__ float4 bcast[2][NP / 4 + 1];
  const int tid = threadIdx.x;
  for (int i = tid; i < N * (N + 1); i += 256) { int r = i / (N + 1), c = i % (N + 1); As[r * STRIDE + c] = A[blockIdx.x * N * (N + 1) + i]; }
  __syncthreads();
  long long t_sts = 0, t_bar = 0, t_rcp = 0, t_fma = 0;
  const long long t00 = clock64();
  if (tid < 96) {
    float arow[NP];
    const int row = tid < N ? tid : N - 1;
#pragma unroll
    for (int j = 0; j < N; ++j) arow[j] = As[row * STRIDE + j];
    arow[N] = 0.f;
    float brow = As[row * STRIDE + N], mydiag = 1.f;
#pragma unroll 1
    for (int k = 0; k < N; ++k) {
      long long c0 = clock64();
      float4* buf = bcast[k & 1];
      if (tid == k) {
#pragma unroll
        for (int j = 0; j < NP; j += 4) buf[j >> 2] = make_float4(arow[j], arow[j + 1], arow[j + 2], arow[j + 3]);
        buf[NP / 4] = make_float4(brow, 0.f, 0.f, 0.f);
        mydiag = arow[0];
      }
      long long c1 = clock64();
      bar96();
      float pr[NP];
#pragma unroll
      for (int j = 0; j < NP; j += 4) { const float4 v = buf[j >> 2]; pr[j] = v.x; pr[j + 1] = v.y; pr[j + 2] = v.z; pr[j + 3] = v.w; }
      const float pb = buf[NP / 4].x;
      float sink = pr[0] + pr[71] + pb;
      asm volatile("" : "+f"(sink));
      long long c2 = clock64();
      const float l = (tid == k) ? 0.f : arow[0] * (VARIANT == 1 ? __frcp_rn(pr[0]) : __fdividef(1.f, pr[0]));
      float lsink = l;
      asm volatile("" : "+f"(lsink));
      long long c3 = clock64();
#pragma unroll
      for (int j = 1; j < NP; ++j) arow[j - 1] = fmaf(-l, pr[j], arow[j]);
      brow = fmaf(-l, pb, brow);
      float fs = arow[0] + arow[35] + arow[70] + brow;
      asm volatile("" : "+f"(fs));
      long long c4 = clock64();
      t_sts += c1 - c0; t_bar += c2 - c1; t_rcp += c3 - c2; t_fma += c4 - c3;
    }
    if (tid < N) x[blockIdx.x * N + tid] = brow / mydiag;
  }
  if (tid == 0 && blockIdx.x == 0) { clk[0] = t_sts; clk[1] = t_bar; clk[2] = t_rcp; clk[3] = t_fma; clk[4] = clock64() - t00; }
}
int main() {
  const int B = 32;
  float* hA = new float[B * N * (N + 1)];
  for (int b = 0; b < B; ++b)
    for (int i = 0; i < N; ++i)
      for (int j = 0; j <= N; ++j) hA[(b * N + i) * (N + 1) + j] = (j == N) ? 1.f : ((i == j) ? 80.f : 1.f / (1 + abs(i - j)));
  float *dA, *dx; long long* dc;
  cudaMalloc(&dA, sizeof(float) * B * N * (N + 1)); cudaMalloc(&dx, sizeof(float) * B * N); cudaMalloc(&dc, 64);
  cudaMemcpy(dA, hA, sizeof(float) * B * N * (N + 1), cudaMemcpyHostToDevice);
  for (int v = 0; v < 2; ++v) {
    for (int rep = 0; rep < 3; ++rep) { if (v) k_probe<1><<<B, 256>>>(dA, dx, dc); else k_probe<0><<<B, 256>>>(dA, dx, dc); }
    cudaDeviceSynchronize();
    long long c[5]; float x[4];
    cudaMemcpy(c, dc, 40, cudaMemcpyDeviceToHost); cudaMemcpy(x, dx, 16, cudaMemcpyDeviceToHost);
    printf("variant %d (%s): per pivot: sts %lld  bar+lds %lld  rcp %lld  fma %lld | loop total %lld cycles | x0..3 %g %g %g %g | err %s\n", v,
           v ? "__frcp_rn" : "fast rcp", c[0] / N, c[1] / N, c[2] / N, c[3] / N, c[4], x[0], x[1], x[2], x[3], cudaGetErrorString(cudaGetLastError()));
  }
  return 0;
}
