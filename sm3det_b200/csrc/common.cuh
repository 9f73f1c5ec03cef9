// Common helpers for the sm3det_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <cstdio>
#include "../../include/sm3det_b200.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900 || !defined(__CUDA_ARCH_FEAT_SM90_ALL))
#error "sm3det_b200 kernels are written for sm_90a only (wgmma, setmaxnreg)"
#endif

namespace sm3 {

// ---- error plumbing (thread-local message, C ABI returns negative codes) -------------------
// error codes: SM3_OK / SM3_ERR_* come from the public header

void set_last_error(const char* fmt, ...);
int check_launch(const char* what);   // cudaGetLastError() -> SM3_ERR_CUDA (+ message)

#define SM3_REQUIRE(cond, code, ...)                      \
  do {                                                    \
    if (!(cond)) {                                        \
      ::sm3::set_last_error(__VA_ARGS__);                 \
      return (code);                                      \
    }                                                     \
  } while (0)

int num_sms();  // cached per device
int persistent_grid_sms();  // num_sms() minus SM3_RESERVE_SMS (SMs left to concurrent NCCL kernels)

// ---- small device helpers ------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// exact-erf GELU and its derivative (matches torch.nn.GELU(approximate='none'))
__device__ __forceinline__ float gelu_erf(float x) {
  return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
}
__device__ __forceinline__ float gelu_erf_grad(float x) {
  const float cdf = 0.5f * (1.0f + erff(x * 0.70710678118654752440f));
  const float pdf = 0.39894228040143267794f * __expf(-0.5f * x * x);
  return cdf + x * pdf;
}

// Branch-free GELU / GELU' for the GEMM epilogues (the exact-erf pair above costs ~2x the instructions and the
// GELU-heavy epilogues are issue bound).  Phi(x) via Abramowitz-Stegun 7.1.26 (|error| <= 1.5e-7 absolute on erf,
// i.e. <= 1e-7 on Phi -- below the 1e-5 relative error of the split-bf16 products feeding it); exp(-x^2/2) is shared
// between Phi and the density term of the derivative.
__device__ __forceinline__ void phi_parts(float x, float& Phi, float& e) {
  const float z = fabsf(x) * 0.70710678118654752440f;
  float t;                                  // MUFU.RCP (1 ulp): __frcp_rn costs a Newton step + a slow-path call per element
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.0f)));
  float poly = fmaf(t, 1.061405429f, -1.453152027f);
  poly = fmaf(t, poly, 1.421413741f);
  poly = fmaf(t, poly, -0.284496736f);
  poly = fmaf(t, poly, 0.254829592f);
  poly *= t;
  e = __expf(-z * z);                       // = exp(-x^2/2)
  const float q = 0.5f * poly * e;          // upper-tail probability of |x|
  Phi = x >= 0.f ? 1.0f - q : q;
}
__device__ __forceinline__ float gelu_fast(float x) {
  float Phi, e;
  phi_parts(x, Phi, e);
  return x * Phi;
}
__device__ __forceinline__ float gelu_grad_fast(float x) {
  float Phi, e;
  phi_parts(x, Phi, e);
  return fmaf(x * 0.39894228040143267794f, e, Phi);
}

// Packed-FP32 pair: two adjacent fp32 values in one 64-bit register (low word first).  The kernels keep their
// operands as pairs (one LDS.64 feeds two FMAs); sm_90 has no packed-fp32 FMA, so ffma2 is two IEEE fmaf.
typedef unsigned long long f32x2_t;
__device__ __forceinline__ f32x2_t ffma2(f32x2_t a, f32x2_t b, f32x2_t c) {
  const float d0 = fmaf(__uint_as_float((uint32_t)a), __uint_as_float((uint32_t)b), __uint_as_float((uint32_t)c));
  const float d1 = fmaf(__uint_as_float((uint32_t)(a >> 32)), __uint_as_float((uint32_t)(b >> 32)), __uint_as_float((uint32_t)(c >> 32)));
  return (f32x2_t)__float_as_uint(d0) | ((f32x2_t)__float_as_uint(d1) << 32);
}

__device__ __forceinline__ float4 ldg_f4(const float* p) {
  return __ldg(reinterpret_cast<const float4*>(p));
}

// Counter-based dropout mask: element e of a tensor is kept when dropout_bits(seed, e) >= p * 2^32.  A pure function of
// (seed, flat element index), so every kernel that applies or differentiates the same dropout draws the same mask.
__device__ __forceinline__ uint32_t mix32(uint64_t z) {      // splitmix64 finaliser
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return (uint32_t)((z ^ (z >> 31)) >> 32);
}
__device__ __forceinline__ uint32_t dropout_bits(uint64_t seed, long long e) {
  const uint64_t base = seed ^ ((uint64_t)(e & ~3LL) * 0xD1342543DE82EF95ull);
  return mix32(base + (uint64_t)(e & 3) * 0x632BE59BD9B4E019ull);
}

}  // namespace sm3

// dispatch a kernel templated on V = C/32 (channels per lane)
#define SM3_V_DISPATCH(V_, ...)                                          \
  switch (V_) {                                                           \
    case 1: { constexpr int V = 1; __VA_ARGS__; } break;                         \
    case 2: { constexpr int V = 2; __VA_ARGS__; } break;                         \
    case 3: { constexpr int V = 3; __VA_ARGS__; } break;                         \
    case 4: { constexpr int V = 4; __VA_ARGS__; } break;                         \
    case 5: { constexpr int V = 5; __VA_ARGS__; } break;                         \
    case 6: { constexpr int V = 6; __VA_ARGS__; } break;                         \
    case 8: { constexpr int V = 8; __VA_ARGS__; } break;                         \
    case 10: { constexpr int V = 10; __VA_ARGS__; } break;                       \
    case 12: { constexpr int V = 12; __VA_ARGS__; } break;                       \
    case 16: { constexpr int V = 16; __VA_ARGS__; } break;                       \
    case 20: { constexpr int V = 20; __VA_ARGS__; } break;                       \
    case 24: { constexpr int V = 24; __VA_ARGS__; } break;                       \
    case 32: { constexpr int V = 32; __VA_ARGS__; } break;                       \
    default: ::sm3::set_last_error("unsupported channel count (C/32=%d)", V_); return SM3_ERR_UNSUPPORTED_SHAPE; \
  }

