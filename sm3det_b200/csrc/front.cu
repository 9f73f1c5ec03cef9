// Block front in one pass: 7x7 depthwise conv + bias + block LayerNorm (ConvNeXtBlock :347-351), NHWC fp32.
//
// Used by the activation-checkpointed blocks (functional.py, packs['checkpoint']): the forward asks only for what the
// FFN reads (fp32 v, or the fused FFN's K-major operand image) and the backward's recompute asks for u, stats and v.
// The results are bit-identical to dwconv7_tile_kernel followed by ln_fwd_kernel<V> (or ln_fwd_img_kernel<G> when
// the image is requested): the conv keeps the bias-first, taps-in-(i, j)-order fmaf chain of the tile kernel, and the
// normalisation keeps the LayerNorm kernels' lane-to-channel assignment, shuffle tree, `/ (float)C` and rsqrtf.
//
// A CTA owns a strip of TH x 16 tokens across all C channels.  It loops over 32-channel chunks, staging the
// (TH+6) x 22 halo with cp.async (double-buffered: chunk k+1 loads while chunk k computes), and keeps u for the whole
// strip in shared memory; then every warp normalises tokens of the strip straight from shared memory.
#include "common.cuh"
#include "kernels.h"

namespace sm3 {

constexpr int FW = 16;            // strip width (output columns)
constexpr int FWI = FW + 6;       // halo width
constexpr int FCC = 32;           // channels per conv chunk (lane = channel)
constexpr int FSEG = 4;           // output columns per warp work unit in the conv phase

struct FrontArgs {
  const float* x; const float* wt; const float* bias; const float* lnw; const float* lnb;
  float* u; float* stats; float* v; uint8_t* img;
  int H, W, C, TH, tiles_w, tiles_h, tiles;
  long long T, T_pad;
  float eps;
};

// cp.async the (TH+6) x 22 x 32-channel halo of one chunk (zero fill outside the image); commits, does not wait
__device__ __forceinline__ void front_load(float* xs, const FrontArgs& a, int n, int h0, int w0, int c0) {
  const int pixels = (a.TH + 6) * FWI;
  for (int idx = threadIdx.x; idx < pixels * 8; idx += blockDim.x) {
    const int q = idx & 7, pix = idx >> 3;
    const int py = pix / FWI, px = pix - py * FWI;
    const int hi = h0 + py - 3, wi = w0 + px - 3;
    const uint32_t dst = static_cast<uint32_t>(__cvta_generic_to_shared(xs + pix * FCC + q * 4));
    if (hi >= 0 && hi < a.H && wi >= 0 && wi < a.W) {
      const float* src = a.x + (((long long)n * a.H + hi) * a.W + wi) * a.C + c0 + q * 4;
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
    } else {
      asm volatile("st.shared.v4.f32 [%0], {%1, %1, %1, %1};" ::"r"(dst), "f"(0.f) : "memory");
    }
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
}

// conv phase: us[tok][C] = bias + sum_{i,j} taps * x for the strip's tokens (and u in global memory when requested)
__device__ __forceinline__ void front_conv(const FrontArgs& a, float* us, float* xs, int n, int h0, int w0) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int C = a.C, chunks = C / FCC, buf = (a.TH + 6) * FWI * FCC;
  const int units = a.TH * (FW / FSEG);
  front_load(xs, a, n, h0, w0, 0);
#pragma unroll 1
  for (int k = 0; k < chunks; ++k) {
    const float* cur = xs + (k & 1) * buf;
    if (k + 1 < chunks) {
      front_load(xs + ((k + 1) & 1) * buf, a, n, h0, w0, (k + 1) * FCC);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    const int c = k * FCC + lane;
    const float b = a.bias ? __ldg(a.bias + c) : 0.f;
    float wv[49];
#pragma unroll
    for (int i = 0; i < 49; ++i) wv[i] = __ldg(a.wt + i * C + c);
#pragma unroll 1
    for (int unit = warp; unit < units; unit += 8) {
      const int r = unit / (FW / FSEG), s0 = (unit % (FW / FSEG)) * FSEG;
      float acc[FSEG];
#pragma unroll
      for (int o = 0; o < FSEG; ++o) acc[o] = b;
#pragma unroll
      for (int i = 0; i < 7; ++i) {
        const float* xr = cur + ((r + i) * FWI + s0) * FCC + lane;
#pragma unroll
        for (int cc = 0; cc < FSEG + 6; ++cc) {
          const float xv = xr[cc * FCC];
#pragma unroll
          for (int j = 0; j < 7; ++j) {
            const int o = cc - j;
            if (o >= 0 && o < FSEG) acc[o] = fmaf(xv, wv[i * 7 + j], acc[o]);
          }
        }
      }
      const int h = h0 + r;
#pragma unroll
      for (int o = 0; o < FSEG; ++o) {
        const int w = w0 + s0 + o;
        us[(r * FW + s0 + o) * C + c] = acc[o];
        if (a.u && h < a.H && w < a.W) a.u[(((long long)n * a.H + h) * a.W + w) * C + c] = acc[o];
      }
    }
    __syncthreads();                              // chunk consumed before its buffer is refilled / us is read
  }
}

__device__ __forceinline__ bool front_tile(const FrontArgs& a, int& n, int& h0, int& w0) {
  if ((int)blockIdx.x >= a.tiles) return false;
  const int per_img = a.tiles_w * a.tiles_h;
  n = blockIdx.x / per_img;
  const int rem = blockIdx.x % per_img;
  h0 = (rem / a.tiles_w) * a.TH;
  w0 = (rem % a.tiles_w) * FW;
  return true;
}

// K-major bf16 hi|lo operand image entry of token t, 8-channel group g (the layout of ln_fwd_img_kernel / pack_act)
__device__ __forceinline__ uint8_t* front_img_dst(uint8_t* img, long long t, int g, int kblocks) {
  const long long rt = t >> 7;
  const uint32_t rr = (uint32_t)(t & 127), kb = (uint32_t)g >> 2, c = (uint32_t)g & 3u;
  return img + (rt * kblocks + kb) * 16384LL + ((rr >> 3) * 512u + (rr & 7u) * 64u + ((c ^ ((rr >> 1) & 3u)) << 4));
}

// LayerNorm with ln_fwd_kernel<V>'s arithmetic: one warp per token, lane holds channels lane, lane+32, ...
template <int V>
__global__ void __launch_bounds__(256) front_ln_kernel(const FrontArgs a) {
  extern __shared__ float smem[];
  int n, h0, w0;
  if (!front_tile(a, n, h0, w0)) return;
  const int C = a.C;
  float* us = smem;                               // [TH*16][C]
  float* xs = smem + a.TH * FW * C;               // [2][TH+6][22][32]
  front_conv(a, us, xs, n, h0, w0);
  if (!a.stats && !a.v) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll 1
  for (int tok = warp; tok < a.TH * FW; tok += 8) {
    const int h = h0 + tok / FW, w = w0 + tok % FW;
    if (h >= a.H || w >= a.W) continue;
    const long long t = ((long long)n * a.H + h) * a.W + w;
    const float* ur = us + tok * C;
    float v[V];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < V; ++i) { v[i] = ur[lane + 32 * i]; s += v[i]; }
    const float mean = warp_sum(s) / (float)C;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < V; ++i) { const float d = v[i] - mean; q += d * d; }
    const float rstd = rsqrtf(warp_sum(q) / (float)C + a.eps);
    if (a.stats && lane == 0) { a.stats[2 * t] = mean; a.stats[2 * t + 1] = rstd; }
    if (a.v) {
      float* yr = a.v + t * C;
#pragma unroll
      for (int i = 0; i < V; ++i) {
        const int c = lane + 32 * i;
        yr[c] = (v[i] - mean) * rstd * __ldg(a.lnw + c) + __ldg(a.lnb + c);
      }
    }
  }
}

// LayerNorm with ln_fwd_img_kernel<G>'s arithmetic, writing the operand image (+ optional fp32 v / stats).  The extra
// last CTA zeroes the image rows of the last 128-row tile beyond T.
template <int G>
__global__ void __launch_bounds__(256) front_img_kernel(const FrontArgs a) {
  extern __shared__ float smem[];
  const int C = a.C, chunks8 = C / 8, kblocks = C / 32;
  int n, h0, w0;
  if (!front_tile(a, n, h0, w0)) {
    for (long long idx = threadIdx.x; idx < (a.T_pad - a.T) * chunks8; idx += blockDim.x) {
      uint8_t* dst = front_img_dst(a.img, a.T + idx / chunks8, (int)(idx % chunks8), kblocks);
      *reinterpret_cast<uint4*>(dst) = make_uint4(0u, 0u, 0u, 0u);
      *reinterpret_cast<uint4*>(dst + 8192) = make_uint4(0u, 0u, 0u, 0u);
    }
    return;
  }
  float* us = smem;
  float* xs = smem + a.TH * FW * C;
  front_conv(a, us, xs, n, h0, w0);
  constexpr int TPW = 32 / G;                     // tokens per warp
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane % G;
  const bool act = g < chunks8;
#pragma unroll 1
  for (int base = warp * TPW; base < a.TH * FW; base += 8 * TPW) {
    const int tok = base + lane / G;
    const int h = h0 + tok / FW, w = w0 + tok % FW;
    const bool ok = h < a.H && w < a.W;
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = 0.f;
    if (act && ok) {
      const float4 p0 = *reinterpret_cast<const float4*>(us + tok * C + g * 8);
      const float4 p1 = *reinterpret_cast<const float4*>(us + tok * C + g * 8 + 4);
      v[0] = p0.x; v[1] = p0.y; v[2] = p0.z; v[3] = p0.w; v[4] = p1.x; v[5] = p1.y; v[6] = p1.z; v[7] = p1.w;
    }
    float s = 0.f;
#pragma unroll
    for (int e = 0; e < 8; ++e) s += v[e];
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s / (float)C;
    float q = 0.f;
    if (act) {
#pragma unroll
      for (int e = 0; e < 8; ++e) { const float d = v[e] - mean; q += d * d; }
    }
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float rstd = rsqrtf(q / (float)C + a.eps);
    if (!act || !ok) continue;
    const long long t = ((long long)n * a.H + h) * a.W + w;
    if (a.stats && g == 0) { a.stats[2 * t] = mean; a.stats[2 * t + 1] = rstd; }
    const float4 w0v = ldg_f4(a.lnw + g * 8), w1v = ldg_f4(a.lnw + g * 8 + 4);
    const float4 b0v = ldg_f4(a.lnb + g * 8), b1v = ldg_f4(a.lnb + g * 8 + 4);
    const float ww[8] = {w0v.x, w0v.y, w0v.z, w0v.w, w1v.x, w1v.y, w1v.z, w1v.w};
    const float bb[8] = {b0v.x, b0v.y, b0v.z, b0v.w, b1v.x, b1v.y, b1v.z, b1v.w};
    float o8[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) o8[e] = (v[e] - mean) * rstd * ww[e] + bb[e];
    if (a.v) {
      *reinterpret_cast<float4*>(a.v + t * C + g * 8) = make_float4(o8[0], o8[1], o8[2], o8[3]);
      *reinterpret_cast<float4*>(a.v + t * C + g * 8 + 4) = make_float4(o8[4], o8[5], o8[6], o8[7]);
    }
    uint32_t hi[4], lo[4];
#pragma unroll
    for (int e = 0; e < 8; e += 2) {
      const uint32_t u0 = __float_as_uint(o8[e]), u1 = __float_as_uint(o8[e + 1]);
      hi[e / 2] = __byte_perm(u0, u1, 0x7632);
      const uint32_t r0 = __float_as_uint(o8[e] - __uint_as_float(u0 & 0xFFFF0000u)) + 0x8000u;
      const uint32_t r1 = __float_as_uint(o8[e + 1] - __uint_as_float(u1 & 0xFFFF0000u)) + 0x8000u;
      lo[e / 2] = __byte_perm(r0, r1, 0x7632);
    }
    uint8_t* dst = front_img_dst(a.img, t, g, kblocks);
    *reinterpret_cast<uint4*>(dst) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
    *reinterpret_cast<uint4*>(dst + 8192) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
  }
}

int dwconv7_ln_fwd(const float* x, const float* wt, const float* bias, const float* lnw, const float* lnb, float* u,
                   float* stats, float* v, unsigned short* img, int N, int H, int W, int C, float eps, cudaStream_t stream) {
  SM3_REQUIRE(x && wt && lnw && lnb, SM3_ERR_INVALID_ARG, "dwconv7_ln_fwd: null argument");
  SM3_REQUIRE(N > 0 && H > 0 && W > 0, SM3_ERR_INVALID_ARG, "dwconv7_ln_fwd: empty tensor");
  SM3_REQUIRE(C % 32 == 0 && C <= 1024, SM3_ERR_UNSUPPORTED_SHAPE, "dwconv7_ln_fwd: C=%d must be a multiple of 32 <= 1024", C);
  SM3_REQUIRE(!img || C <= 256, SM3_ERR_UNSUPPORTED_SHAPE, "dwconv7_ln_fwd: the operand image needs C <= 256 (C=%d)", C);
  if (!u && !stats && !v && !img) return SM3_OK;
  FrontArgs a;
  a.x = x; a.wt = wt; a.bias = bias; a.lnw = lnw; a.lnb = lnb;
  a.u = u; a.stats = stats; a.v = v; a.img = reinterpret_cast<uint8_t*>(img);
  a.H = H; a.W = W; a.C = C; a.eps = eps;
  // strip height: u of the strip plus two halo buffers stay <= ~180 KB at C = 1024 and allow two CTAs per SM up to C = 384
  a.TH = C <= 64 ? 8 : C <= 192 ? 4 : 2;
  a.tiles_w = (W + FW - 1) / FW;
  a.tiles_h = (H + a.TH - 1) / a.TH;
  const long long tiles = (long long)N * a.tiles_w * a.tiles_h;
  SM3_REQUIRE(tiles < (1LL << 30), SM3_ERR_UNSUPPORTED_SHAPE, "dwconv7_ln_fwd: tensor too large");
  a.tiles = (int)tiles;
  a.T = (long long)N * H * W;
  a.T_pad = (a.T + 127) / 128 * 128;
  const size_t smem = ((size_t)a.TH * FW * C + 2 * (size_t)(a.TH + 6) * FWI * FCC) * sizeof(float);
  if (img) {
    const unsigned grid = (unsigned)(tiles + (a.T_pad > a.T ? 1 : 0));
    if (C <= 128) {
      cudaFuncSetAttribute(front_img_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      front_img_kernel<16><<<grid, 256, smem, stream>>>(a);
    } else {
      cudaFuncSetAttribute(front_img_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      front_img_kernel<32><<<grid, 256, smem, stream>>>(a);
    }
    return check_launch("dwconv7_ln_fwd(img)");
  }
  const int V_ = C / 32;
  SM3_V_DISPATCH(V_, {
    cudaFuncSetAttribute(front_ln_kernel<V>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    front_ln_kernel<V><<<(unsigned)tiles, 256, smem, stream>>>(a);
  });
  return check_launch("dwconv7_ln_fwd");
}

}  // namespace sm3
