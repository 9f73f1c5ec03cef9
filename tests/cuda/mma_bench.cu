// Microbenchmark: cost of one wgmma.mma_async m64nNk16 (bf16 operands in shared memory, fp32 register accumulator)
// as a function of N, issued back to back by one warpgroup into the same accumulator -- the regime of the fused FFN
// kernels (N = 32..96).  Answers: is a narrow MMA paced by N, or by a per-instruction floor (operand fetch)?
// Build: make build/mma_bench     Run: build/mma_bench
#define SM3_GEMM_KERNEL_IMPL
#include "gemm_tc.cuh"
#include <cstdio>
#include <vector>

using namespace sm3;
using namespace sm3::gemm;

// mode 0: K-major x K-major, the 3-pass pattern (alo*bhi, ahi*blo, ahi*bhi) over `ksteps` k-steps per round
// mode 1: same operands every time (single descriptor pair)
// mode 2: MN-major x MN-major (the wgrad operands)
template <int N>
__global__ void __launch_bounds__(128, 1) mma_bench_kernel(int mode, int rounds, int ksteps, long long* out) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sb = (smem_u32(smem_raw) + 1023u) & ~1023u;
  for (uint32_t i = threadIdx.x; i < 160 * 1024 / 16; i += blockDim.x)
    asm volatile("st.shared.v4.b32 [%0], {%1, %1, %1, %1};" ::"r"(sb + i * 16), "r"(0x3C003C00u) : "memory");
  fence_proxy_async_smem();
  __syncthreads();
  float acc[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
  const bool mn = mode == 2;
  const uint32_t a0 = sb, b0 = sb + 64 * 1024;
  const uint64_t da = make_smem_desc(a0, mn), db = make_smem_desc(b0, mn);
  const uint64_t kstep = mn ? 128u : 2u, lo = 512u;
  const long long t0 = clock64();
  for (int r = 0; r < rounds; ++r) {
    wg::fence();
    for (int ks = 0; ks < ksteps; ++ks) {
      const int kb = (ks >> 1) % 3;           // wrap inside a 3 k-block operand (48 KB of A, <= 96 KB of B)
      const uint64_t a = da + (uint64_t)(ks & 1) * kstep + (uint64_t)kb * 1024u, b = db + (uint64_t)(ks & 1) * kstep + (uint64_t)kb * (mn ? 1024u : (uint64_t)N * 8u);
      if (mode == 1) {
        wg::mma<N, 0, 0>(acc, da, db, 1u); wg::mma<N, 0, 0>(acc, da, db, 1u); wg::mma<N, 0, 0>(acc, da, db, 1u);
      } else if (mode == 0) {
        wg::mma<N, 0, 0>(acc, a + lo, b, 1u);
        wg::mma<N, 0, 0>(acc, a, b + (uint64_t)N * 4u, 1u);
        wg::mma<N, 0, 0>(acc, a, b, 1u);
      } else {
        wg::mma<N, 1, 1>(acc, a + lo, b, 1u);
        wg::mma<N, 1, 1>(acc, a, b + lo, 1u);
        wg::mma<N, 1, 1>(acc, a, b, 1u);
      }
    }
    wg::commit();
    wg::wait<0>();
  }
  wg::fence_operand(acc);
  const long long t1 = clock64();
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < N / 2; ++i) s += acc[i];
  if (blockIdx.x == 0 && threadIdx.x == 0) { out[0] = t1 - t0; out[1] = (long long)s; }
}

template <int N>
static int run(int grid, int mode, int ksteps, long long* d) {
  const int smem = 161 * 1024 + 1024;
  cudaFuncSetAttribute(mma_bench_kernel<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  const int rounds = 400 / (ksteps / 6);
  mma_bench_kernel<N><<<grid, 128, smem>>>(mode, rounds, ksteps, d);
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) { printf("CUDA error %s\n", cudaGetErrorString(e)); return 1; }
  long long cyc[2]; cudaMemcpy(cyc, d, 16, cudaMemcpyDeviceToHost);
  const double per = (double)cyc[0] / ((double)rounds * ksteps * 3);
  printf("grid %3d mode %d N=%3d  %2d k-steps/commit: %7.1f cycles/MMA  round latency %.0f\n", grid, mode, N, ksteps, per,
         (double)cyc[0] / rounds);
  return 0;
}

int main() {
  long long* d; cudaMalloc(&d, 16);
  int sms = 0; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  printf("mode 0 = K-major 3-pass pattern, 1 = one descriptor pair repeated, 2 = MN-major 3-pass pattern; cycles per MMA (M=64,K=16)\n");
  for (int grid : {1, sms}) {
    for (int mode = 0; mode < 3; ++mode) {
      for (int ksteps : {6, 48}) {
        int rc = run<32>(grid, mode, ksteps, d) | run<64>(grid, mode, ksteps, d) | run<96>(grid, mode, ksteps, d) |
                 run<128>(grid, mode, ksteps, d);
        if (mode != 2) rc |= run<192>(grid, mode, ksteps, d) | run<256>(grid, mode, ksteps, d);   // MN-major test operand: 128 wide
        if (rc) return 1;
      }
    }
  }
  return 0;
}
