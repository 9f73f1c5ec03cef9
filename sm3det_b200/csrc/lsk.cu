// Kernels of the LSKNet-MoE backbone (BASELINE config 5) that the ConvNeXt path does not already provide.
// All tensors NHWC fp32 ("tokens x channels").  Replaces, in reference mmrotate/models/backbones/lsk_moe.py:
//   dwconv_*            nn.Conv2d(groups=dim) of LSKblock.conv0 (5x5) :322, conv_spatial (7x7, dilation 3) :323 and
//                       DWConv (3x3) :583, + autograd's depthwise dgrad / wgrad
//   colstat / affine    BatchNorm2d (build_norm_layer BN / SyncBN) statistics, normalisation and its backward
//                       (Block.norm1/norm2 :369-374, OverlapPatchEmbed.norm :407-410), layer-scale + residual :388-395
//   lsk_agg/squeeze/mix channel mean / max, conv_squeeze(2->2, 7x7) + sigmoid, weighted sum (LSKblock.forward :336-341)
//   mul                 x * attn :343
//   im2col / col2im     OverlapPatchEmbed.proj (7x7/s4 stem, 3x3/s2 downsamples) :405-406 lowered to the wgmma GEMM
#include "common.cuh"
#include "kernels.h"

namespace sm3 {

// ------------------------------------------------------------------------------------------------
// Generic depthwise KSxKS convolution with dilation DIL ("same" padding DIL*(KS-1)/2), shared-memory tiled:
// a block owns a 16x16 output tile of 32 channels, lane = channel, a warp owns two output rows.
constexpr int GT = 16;
constexpr int GCC = 32;

template <int KS, int DIL>
struct DwGeom {
  static constexpr int R = DIL * (KS / 2);
  static constexpr int TI = GT + 2 * R;
};

template <int R, int TI>
__device__ __forceinline__ void dwg_load_tile(float* xs, const float* __restrict__ x, int n, int h0, int w0, int c0, int H,
                                              int W, int C) {
  for (int idx = threadIdx.x; idx < TI * TI * 8; idx += blockDim.x) {
    const int q = idx & 7, pix = idx >> 3;
    const int py = pix / TI, px = pix - py * TI;
    const int hi = h0 + py - R, wi = w0 + px - R;
    const uint32_t dst = static_cast<uint32_t>(__cvta_generic_to_shared(xs + pix * GCC + q * 4));
    if (hi >= 0 && hi < H && wi >= 0 && wi < W) {
      const float* src = x + (((long long)n * H + hi) * W + wi) * C + c0 + q * 4;
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
    } else {
      asm volatile("st.shared.v4.f32 [%0], {%1, %1, %1, %1};" ::"r"(dst), "f"(0.f) : "memory");
    }
  }
  asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
  __syncthreads();
}

// lane = (row selector l/16, channel pair l%16); ffma2 on channel pairs, as in stencil.cu's 7x7 kernel
template <int KS, int DIL>
__global__ void __launch_bounds__(256) dwconv_tile_kernel(const float* __restrict__ x, const float* __restrict__ wt,
                                                         const float* __restrict__ bias, const float* __restrict__ resid,
                                                         float* __restrict__ y, int H, int W, int C, int tiles_w) {
  constexpr int R = DwGeom<KS, DIL>::R, TI = DwGeom<KS, DIL>::TI;
  typedef unsigned long long f2;
  extern __shared__ float xs[];                           // [TI][TI][GCC]
  const int tw = blockIdx.x % tiles_w, th = blockIdx.x / tiles_w;
  const int cchunks = C / GCC;
  const int n = blockIdx.y / cchunks, c0 = (blockIdx.y % cchunks) * GCC;
  const int h0 = th * GT, w0 = tw * GT;
  dwg_load_tile<R, TI>(xs, x, n, h0, w0, c0, H, W, C);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int cp = lane & 15, r = warp * 2 + (lane >> 4);
  const int c = c0 + 2 * cp;
  const int h = h0 + r;
  if (h >= H) return;
  const f2 b2 = bias ? __ldg(reinterpret_cast<const f2*>(bias + c)) : 0ull;
  f2 acc[GT];
#pragma unroll
  for (int o = 0; o < GT; ++o) acc[o] = b2;
#pragma unroll 1
  for (int i = 0; i < KS; ++i) {
    f2 wv[KS];
#pragma unroll
    for (int j = 0; j < KS; ++j) wv[j] = __ldg(reinterpret_cast<const f2*>(wt + (i * KS + j) * C + c));
    const f2* xr = reinterpret_cast<const f2*>(xs + ((r + i * DIL) * TI) * GCC) + cp;
#pragma unroll
    for (int cc = 0; cc < TI; ++cc) {
      const f2 v = xr[cc * (GCC / 2)];
#pragma unroll
      for (int j = 0; j < KS; ++j) {
        const int o = cc - j * DIL;
        if (o >= 0 && o < GT) acc[o] = ffma2(v, wv[j], acc[o]);
      }
    }
  }
  const long long rowoff = (((long long)n * H + h) * W) * C + c;
#pragma unroll
  for (int o = 0; o < GT; ++o) {
    const int w = w0 + o;
    if (w < W) {
      float2 v = make_float2(__uint_as_float((uint32_t)acc[o]), __uint_as_float((uint32_t)(acc[o] >> 32)));
      if (resid) { const float2 rr = __ldg(reinterpret_cast<const float2*>(resid + rowoff + (long long)w * C)); v.x += rr.x; v.y += rr.y; }
      *reinterpret_cast<float2*>(y + rowoff + (long long)w * C) = v;
    }
  }
}

// wgrad: persistent blocks over the tiles of one 32-channel chunk; lane = channel keeps the KS*KS tap sums in registers
template <int KS, int DIL>
__global__ void __launch_bounds__(256) dwconv_wgrad_tile_kernel(const float* __restrict__ x, const float* __restrict__ dy,
                                                               float* __restrict__ dwt, float* __restrict__ dbias, int N,
                                                               int H, int W, int C, int tiles_w, int tiles_h,
                                                               int blocks_per_chunk) {
  constexpr int R = DwGeom<KS, DIL>::R, TI = DwGeom<KS, DIL>::TI, NT = KS * KS;
  extern __shared__ float smem[];
  float* xs = smem;                               // [TI][TI][GCC]
  float* ds = smem + TI * TI * GCC;               // [GT][GT][GCC]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c0 = blockIdx.y * GCC;
  float acc[NT];
#pragma unroll
  for (int i = 0; i < NT; ++i) acc[i] = 0.f;
  float accb = 0.f;
  const int tiles = N * tiles_h * tiles_w;
  for (int t = blockIdx.x; t < tiles; t += blocks_per_chunk) {
    const int n = t / (tiles_h * tiles_w), rem = t % (tiles_h * tiles_w);
    const int h0 = (rem / tiles_w) * GT, w0 = (rem % tiles_w) * GT;
    __syncthreads();
    for (int idx = threadIdx.x; idx < GT * GT * 8; idx += blockDim.x) {
      const int q = idx & 7, pix = idx >> 3;
      const int py = pix / GT, px = pix - py * GT;
      const int hi = h0 + py, wi = w0 + px;
      const uint32_t dst = static_cast<uint32_t>(__cvta_generic_to_shared(ds + pix * GCC + q * 4));
      if (hi < H && wi < W) {
        const float* src = dy + (((long long)n * H + hi) * W + wi) * C + c0 + q * 4;
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
      } else {
        asm volatile("st.shared.v4.f32 [%0], {%1, %1, %1, %1};" ::"r"(dst), "f"(0.f) : "memory");
      }
    }
    dwg_load_tile<R, TI>(xs, x, n, h0, w0, c0, H, W, C);
#pragma unroll 1
    for (int rr = 0; rr < 2; ++rr) {
      const int r = warp * 2 + rr;
      float d[GT];
#pragma unroll
      for (int o = 0; o < GT; ++o) { d[o] = ds[(r * GT + o) * GCC + lane]; accb += d[o]; }
#pragma unroll
      for (int i = 0; i < KS; ++i) {
        const float* xr = xs + ((r + i * DIL) * TI) * GCC + lane;
#pragma unroll
        for (int cc = 0; cc < TI; ++cc) {
          const float v = xr[cc * GCC];
#pragma unroll
          for (int j = 0; j < KS; ++j) {
            const int o = cc - j * DIL;
            if (o >= 0 && o < GT) acc[i * KS + j] = fmaf(v, d[o], acc[i * KS + j]);
          }
        }
      }
    }
  }
  __syncthreads();
  float* red = smem;                              // [8][NT+1][32]
#pragma unroll
  for (int i = 0; i < NT; ++i) red[(warp * (NT + 1) + i) * 32 + lane] = acc[i];
  red[(warp * (NT + 1) + NT) * 32 + lane] = accb;
  __syncthreads();
  for (int idx = threadIdx.x; idx < (NT + 1) * 32; idx += blockDim.x) {
    const int i = idx / 32, l = idx % 32;
    float sum = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) sum += red[(w * (NT + 1) + i) * 32 + l];
    if (i < NT) atomicAdd(dwt + i * C + c0 + l, sum);
    else if (dbias) atomicAdd(dbias + c0 + l, sum);
  }
}

template <int KS, int DIL>
static int dwconv_fwd_t(const float* x, const float* wt, const float* bias, const float* resid, float* y, int N, int H,
                        int W, int C, cudaStream_t stream) {
  constexpr int TI = DwGeom<KS, DIL>::TI;
  const int tiles_w = (W + GT - 1) / GT, tiles_h = (H + GT - 1) / GT;
  const size_t smem = (size_t)TI * TI * GCC * sizeof(float);
  cudaFuncSetAttribute(dwconv_tile_kernel<KS, DIL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  dim3 grid((unsigned)(tiles_w * tiles_h), (unsigned)(N * (C / GCC)));
  dwconv_tile_kernel<KS, DIL><<<grid, 256, smem, stream>>>(x, wt, bias, resid, y, H, W, C, tiles_w);
  return check_launch("dwconv_tile_kernel");
}

template <int KS, int DIL>
static int dwconv_wgrad_t(const float* x, const float* dy, float* dwt, float* dbias, int N, int H, int W, int C,
                          cudaStream_t stream) {
  constexpr int TI = DwGeom<KS, DIL>::TI;
  const int tiles_w = (W + GT - 1) / GT, tiles_h = (H + GT - 1) / GT;
  const int chunks = C / GCC;
  const long long tiles = (long long)N * tiles_w * tiles_h;
  int bpc = (num_sms() * 2 + chunks - 1) / chunks;
  if (bpc > tiles) bpc = (int)tiles;
  if (bpc < 1) bpc = 1;
  size_t smem = (size_t)(TI * TI + GT * GT) * GCC * sizeof(float);
  const size_t red = (size_t)8 * (KS * KS + 1) * 32 * sizeof(float);
  if (smem < red) smem = red;
  cudaFuncSetAttribute(dwconv_wgrad_tile_kernel<KS, DIL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  dim3 grid((unsigned)bpc, (unsigned)chunks);
  dwconv_wgrad_tile_kernel<KS, DIL><<<grid, 256, smem, stream>>>(x, dy, dwt, dbias, N, H, W, C, tiles_w, tiles_h, bpc);
  return check_launch("dwconv_wgrad_tile_kernel");
}

int dwconv_fwd(const float* x, const float* wt, const float* bias, const float* resid, float* y, int N, int H, int W, int C,
               int ks, int dil, cudaStream_t stream) {
  SM3_REQUIRE(x && wt && y, SM3_ERR_INVALID_ARG, "dwconv_fwd: null argument");
  SM3_REQUIRE(C % GCC == 0 && N > 0 && H > 0 && W > 0 && (long long)N * (C / GCC) < 65536, SM3_ERR_UNSUPPORTED_SHAPE,
              "dwconv_fwd: C=%d must be a multiple of 32 (N*C/32 < 65536)", C);
  if (ks == 3 && dil == 1) return dwconv_fwd_t<3, 1>(x, wt, bias, resid, y, N, H, W, C, stream);
  if (ks == 5 && dil == 1) return dwconv_fwd_t<5, 1>(x, wt, bias, resid, y, N, H, W, C, stream);
  if (ks == 7 && dil == 3) return dwconv_fwd_t<7, 3>(x, wt, bias, resid, y, N, H, W, C, stream);
  SM3_REQUIRE(false, SM3_ERR_UNSUPPORTED_SHAPE, "dwconv_fwd: kernel %dx%d dilation %d is not instantiated", ks, ks, dil);
}

int dwconv_wgrad(const float* x, const float* dy, float* dwt, float* dbias, int N, int H, int W, int C, int ks, int dil,
                 cudaStream_t stream) {
  SM3_REQUIRE(x && dy && dwt, SM3_ERR_INVALID_ARG, "dwconv_wgrad: null argument");
  SM3_REQUIRE(C % GCC == 0 && C / GCC < 65536, SM3_ERR_UNSUPPORTED_SHAPE, "dwconv_wgrad: C=%d must be a multiple of 32", C);
  if (ks == 3 && dil == 1) return dwconv_wgrad_t<3, 1>(x, dy, dwt, dbias, N, H, W, C, stream);
  if (ks == 5 && dil == 1) return dwconv_wgrad_t<5, 1>(x, dy, dwt, dbias, N, H, W, C, stream);
  if (ks == 7 && dil == 3) return dwconv_wgrad_t<7, 3>(x, dy, dwt, dbias, N, H, W, C, stream);
  SM3_REQUIRE(false, SM3_ERR_UNSUPPORTED_SHAPE, "dwconv_wgrad: kernel %dx%d dilation %d is not instantiated", ks, ks, dil);
}

// ------------------------------------------------------------------------------------------------
// Column statistics:  s1[c] += sum_r w * (x[r,c]-sh1[c]) ,  s2[c] += sum_r w * (x - sh1) * (y ? (y[r,c]-sh2[c])*sc2[c] : (x - sh1))
//   BatchNorm forward  : y = null, sh1 = running_mean (shifted-data variance, one pass)
//   BatchNorm backward : x = dy (sh1 = null), y = saved input, sh2 = mean, sc2 = rstd  ->  s1 = sum dy, s2 = sum dy*xhat
// block (32 channel quads, 8 row lanes); grid (C/128, row chunks)
__global__ void __launch_bounds__(256) colstat_kernel(const float* __restrict__ x, const float* __restrict__ sh1,
                                                     const float* __restrict__ y, const float* __restrict__ sh2,
                                                     const float* __restrict__ sc2, float* __restrict__ s1,
                                                     float* __restrict__ s2, long long rows, int C, long long rows_per_block) {
  __shared__ float4 red[2][8][32];
  const int ql = threadIdx.x & 31, rl = threadIdx.x >> 5;
  const int c = (blockIdx.x * 32 + ql) * 4;
  const bool ok = c < C;
  const long long r0 = (long long)blockIdx.y * rows_per_block, r1 = min(rows, r0 + rows_per_block);
  float4 a1 = make_float4(0.f, 0.f, 0.f, 0.f), a2 = a1;
  if (ok) {
    const float4 h1 = sh1 ? ldg_f4(sh1 + c) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 h2 = (y && sh2) ? ldg_f4(sh2 + c) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 k2 = (y && sc2) ? ldg_f4(sc2 + c) : make_float4(1.f, 1.f, 1.f, 1.f);
    for (long long r = r0 + rl; r < r1; r += 8) {
      float4 v = ldg_f4(x + r * C + c);
      v.x -= h1.x; v.y -= h1.y; v.z -= h1.z; v.w -= h1.w;
      float4 u = v;
      if (y) {
        u = ldg_f4(y + r * C + c);
        u.x = (u.x - h2.x) * k2.x; u.y = (u.y - h2.y) * k2.y; u.z = (u.z - h2.z) * k2.z; u.w = (u.w - h2.w) * k2.w;
      }
      a1.x += v.x; a1.y += v.y; a1.z += v.z; a1.w += v.w;
      a2.x = fmaf(v.x, u.x, a2.x); a2.y = fmaf(v.y, u.y, a2.y); a2.z = fmaf(v.z, u.z, a2.z); a2.w = fmaf(v.w, u.w, a2.w);
    }
  }
  red[0][rl][ql] = a1; red[1][rl][ql] = a2;
  __syncthreads();
  if (rl < 2 && ok) {
    float4 t = red[rl][0][ql];
#pragma unroll
    for (int i = 1; i < 8; ++i) { const float4 o = red[rl][i][ql]; t.x += o.x; t.y += o.y; t.z += o.z; t.w += o.w; }
    float* dst = (rl == 0 ? s1 : s2);
    if (dst) { atomicAdd(dst + c, t.x); atomicAdd(dst + c + 1, t.y); atomicAdd(dst + c + 2, t.z); atomicAdd(dst + c + 3, t.w); }
  }
}

int colstat(const float* x, const float* sh1, const float* y, const float* sh2, const float* sc2, float* s1, float* s2,
            long long rows, int C, cudaStream_t stream) {
  SM3_REQUIRE(x && (s1 || s2) && rows > 0 && C % 4 == 0, SM3_ERR_INVALID_ARG, "colstat: bad argument (C must be a multiple of 4)");
  const int gx = (C / 4 + 31) / 32;
  long long gy = (long long)num_sms() * 8 / gx;
  if (gy < 1) gy = 1;
  long long rpb = (rows + gy - 1) / gy;
  if (rpb < 32) rpb = 32;
  gy = (rows + rpb - 1) / rpb;
  dim3 grid((unsigned)gx, (unsigned)gy);
  colstat_kernel<<<grid, 256, 0, stream>>>(x, sh1, y, sh2, sc2, s1, s2, rows, C, rpb);
  return check_launch("colstat_kernel");
}

// out[r,c] = a1[c]*x1[r,c] + (x2 ? a2[c]*x2[r,c] : 0) + (b ? b[c] : 0) + (add ? add[r,c] : 0)     (a1 null = 1)
__global__ void __launch_bounds__(256) affine_kernel(const float* __restrict__ x1, const float* __restrict__ a1,
                                                    const float* __restrict__ x2, const float* __restrict__ a2,
                                                    const float* __restrict__ b, const float* __restrict__ add,
                                                    float* __restrict__ out, long long total, int C) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int Q = C >> 2;
  const int c = (int)(i % Q) * 4;
  const long long off = i * 4;
  float4 v = ldg_f4(x1 + off);
  if (a1) { const float4 s = ldg_f4(a1 + c); v.x *= s.x; v.y *= s.y; v.z *= s.z; v.w *= s.w; }
  if (x2) {
    const float4 u = ldg_f4(x2 + off), s = ldg_f4(a2 + c);
    v.x = fmaf(u.x, s.x, v.x); v.y = fmaf(u.y, s.y, v.y); v.z = fmaf(u.z, s.z, v.z); v.w = fmaf(u.w, s.w, v.w);
  }
  if (b) { const float4 s = ldg_f4(b + c); v.x += s.x; v.y += s.y; v.z += s.z; v.w += s.w; }
  if (add) { const float4 s = ldg_f4(add + off); v.x += s.x; v.y += s.y; v.z += s.z; v.w += s.w; }
  *reinterpret_cast<float4*>(out + off) = v;
}

int affine(const float* x1, const float* a1, const float* x2, const float* a2, const float* b, const float* add, float* out,
           long long rows, int C, cudaStream_t stream) {
  SM3_REQUIRE(x1 && out && C % 4 == 0 && (!x2 || a2), SM3_ERR_INVALID_ARG, "affine: bad argument");
  const long long total = rows * (C / 4);
  affine_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(x1, a1, x2, a2, b, add, out, total, C);
  return check_launch("affine_kernel");
}

// out = a * b (+ add)
__global__ void __launch_bounds__(256) mul_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                 const float* __restrict__ add, float* __restrict__ out, long long n4) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const float4 x = ldg_f4(a + i * 4), y = ldg_f4(b + i * 4);
  float4 v = make_float4(x.x * y.x, x.y * y.y, x.z * y.z, x.w * y.w);
  if (add) { const float4 s = ldg_f4(add + i * 4); v.x += s.x; v.y += s.y; v.z += s.z; v.w += s.w; }
  *reinterpret_cast<float4*>(out + i * 4) = v;
}

int mul(const float* a, const float* b, const float* add, float* out, long long n, cudaStream_t stream) {
  SM3_REQUIRE(a && b && out && n % 4 == 0, SM3_ERR_INVALID_ARG, "mul: bad argument");
  mul_kernel<<<(unsigned)((n / 4 + 255) / 256), 256, 0, stream>>>(a, b, add, out, n / 4);
  return check_launch("mul_kernel");
}

// Dropout with a counter-based mask (nn.Dropout of Mlp, lsk_moe.py:300,311,316): keep = hash(seed, element index) >= p,
// out = x * keep / (1 - p).  The same call with dy as input is the backward (the mask is recomputed, never stored), so
// dropout costs one read + one write instead of torch's rand / compare / scale / multiply passes and a saved mask.
__device__ __forceinline__ uint32_t mix32(uint64_t z) {      // splitmix64 finaliser
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return (uint32_t)((z ^ (z >> 31)) >> 32);
}
__global__ void __launch_bounds__(256) dropout_kernel(const float* __restrict__ x, float* __restrict__ out, long long n4,
                                                     uint32_t thresh, float scale, uint64_t seed,
                                                     const unsigned long long* __restrict__ seed_dev) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  if (seed_dev) seed = __ldg(seed_dev);      // CUDA-graph replay: the seed lives in device memory and changes between replays
  const float4 v = ldg_f4(x + i * 4);
  const uint64_t base = seed ^ ((uint64_t)i * 4ull * 0xD1342543DE82EF95ull);
  float4 o;
  o.x = mix32(base) >= thresh ? v.x * scale : 0.f;
  o.y = mix32(base + 0x632BE59BD9B4E019ull) >= thresh ? v.y * scale : 0.f;
  o.z = mix32(base + 2ull * 0x632BE59BD9B4E019ull) >= thresh ? v.z * scale : 0.f;
  o.w = mix32(base + 3ull * 0x632BE59BD9B4E019ull) >= thresh ? v.w * scale : 0.f;
  *reinterpret_cast<float4*>(out + i * 4) = o;
}

int dropout(const float* x, float* out, long long n, float p, unsigned long long seed, cudaStream_t stream) {
  SM3_REQUIRE(x && out && n % 4 == 0 && p >= 0.f && p < 1.f, SM3_ERR_INVALID_ARG, "dropout: bad argument");
  const uint32_t thresh = (uint32_t)((double)p * 4294967296.0);
  dropout_kernel<<<(unsigned)((n / 4 + 255) / 256), 256, 0, stream>>>(x, out, n / 4, thresh, 1.0f / (1.0f - p), seed, nullptr);
  return check_launch("dropout_kernel");
}

int dropout_dev(const float* x, float* out, long long n, float p, const unsigned long long* seed_dev, cudaStream_t stream) {
  SM3_REQUIRE(x && out && seed_dev && n % 4 == 0 && p >= 0.f && p < 1.f, SM3_ERR_INVALID_ARG, "dropout_dev: bad argument");
  const uint32_t thresh = (uint32_t)((double)p * 4294967296.0);
  dropout_kernel<<<(unsigned)((n / 4 + 255) / 256), 256, 0, stream>>>(x, out, n / 4, thresh, 1.0f / (1.0f - p), 0ull, seed_dev);
  return check_launch("dropout_kernel");
}

// ------------------------------------------------------------------------------------------------
// LSK spatial selection (LSKblock.forward :336-341).  a1, a2: [T, Ch].
// agg[t] = (mean, max) over the 2*Ch channels of cat(a1, a2); amax[t] = argmax channel (first on ties).
__global__ void __launch_bounds__(256) lsk_agg_kernel(const float* __restrict__ a1, const float* __restrict__ a2,
                                                     float* __restrict__ agg, int* __restrict__ amax, long long T, int Ch) {
  const long long t = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (t >= T) return;
  float s = 0.f, m = -INFINITY; int mi = 0;
  for (int c = lane; c < Ch; c += 32) { const float v = __ldg(a1 + t * Ch + c); s += v; if (v > m) { m = v; mi = c; } }
  for (int c = lane; c < Ch; c += 32) { const float v = __ldg(a2 + t * Ch + c); s += v; if (v > m) { m = v; mi = Ch + c; } }
  s = warp_sum(s);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, m, o);
    const int oi = __shfl_xor_sync(0xffffffffu, mi, o);
    if (om > m || (om == m && oi < mi)) { m = om; mi = oi; }
  }
  if (lane == 0) { agg[t * 2] = s / (float)(2 * Ch); agg[t * 2 + 1] = m; if (amax) amax[t] = mi; }
}

int lsk_agg(const float* a1, const float* a2, float* agg, int* amax, long long T, int Ch, cudaStream_t stream) {
  SM3_REQUIRE(a1 && a2 && agg && T > 0 && Ch > 0, SM3_ERR_INVALID_ARG, "lsk_agg: bad argument");
  lsk_agg_kernel<<<(unsigned)((T * 32 + 255) / 256), 256, 0, stream>>>(a1, a2, agg, amax, T, Ch);
  return check_launch("lsk_agg_kernel");
}

// y[n,h,w,co] = act( b[co] + sum_{ci,i,j} x[n,h+i-3,w+j-3,ci] * w[co,ci,i,j] ),  2 -> 2 channels, 7x7, pad 3.
// act: 0 none, 1 sigmoid.  Used for conv_squeeze forward and (with transposed + flipped weights) its dgrad.
__global__ void __launch_bounds__(256) conv7_c2_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                      const float* __restrict__ b, float* __restrict__ y, int N, int H, int W,
                                                      int act) {
  __shared__ float sw[196];
  if (threadIdx.x < 196) sw[threadIdx.x] = __ldg(w + threadIdx.x);
  __syncthreads();
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= (long long)N * H * W) return;
  const int wq = (int)(p % W); const long long r = p / W; const int h = (int)(r % H); const int n = (int)(r / H);
  float y0 = b ? __ldg(b) : 0.f, y1 = b ? __ldg(b + 1) : 0.f;
  for (int i = 0; i < 7; ++i) {
    const int hi = h + i - 3;
    if (hi < 0 || hi >= H) continue;
#pragma unroll
    for (int j = 0; j < 7; ++j) {
      const int wi = wq + j - 3;
      if (wi < 0 || wi >= W) continue;
      const float2 v = __ldg(reinterpret_cast<const float2*>(x) + ((long long)n * H + hi) * W + wi);
      y0 = fmaf(v.x, sw[0 * 98 + 0 * 49 + i * 7 + j], y0); y0 = fmaf(v.y, sw[0 * 98 + 1 * 49 + i * 7 + j], y0);
      y1 = fmaf(v.x, sw[1 * 98 + 0 * 49 + i * 7 + j], y1); y1 = fmaf(v.y, sw[1 * 98 + 1 * 49 + i * 7 + j], y1);
    }
  }
  if (act == 1) { y0 = 1.0f / (1.0f + expf(-y0)); y1 = 1.0f / (1.0f + expf(-y1)); }
  reinterpret_cast<float2*>(y)[p] = make_float2(y0, y1);
}

int conv7_c2(const float* x, const float* w, const float* b, float* y, int N, int H, int W, int act, cudaStream_t stream) {
  SM3_REQUIRE(x && w && y && N > 0 && H > 0 && W > 0, SM3_ERR_INVALID_ARG, "conv7_c2: bad argument");
  const long long total = (long long)N * H * W;
  conv7_c2_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(x, w, b, y, N, H, W, act);
  return check_launch("conv7_c2_kernel");
}

// dw[co,ci,i,j] += sum_p dpre[p,co] * x[p + (i-3, j-3), ci] ; db[co] += sum_p dpre[p,co].   thread = one of the 196 taps.
__global__ void __launch_bounds__(224) conv7_c2_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ dpre,
                                                            float* __restrict__ dw, float* __restrict__ db, int N, int H,
                                                            int W, long long px_per_block) {
  const int tid = threadIdx.x;
  const long long total = (long long)N * H * W;
  const long long p0 = (long long)blockIdx.x * px_per_block, p1 = min(total, p0 + px_per_block);
  if (tid < 196) {
    const int co = tid / 98, ci = (tid / 49) % 2, i = (tid % 49) / 7, j = tid % 7;
    float acc = 0.f;
    for (long long p = p0; p < p1; ++p) {
      const int wq = (int)(p % W); const long long r = p / W; const int h = (int)(r % H); const long long n = r / H;
      const int hi = h + i - 3, wi = wq + j - 3;
      if (hi < 0 || hi >= H || wi < 0 || wi >= W) continue;
      acc = fmaf(__ldg(dpre + p * 2 + co), __ldg(x + ((n * H + hi) * W + wi) * 2 + ci), acc);
    }
    atomicAdd(dw + tid, acc);
  } else if (tid < 198 && db) {
    const int co = tid - 196;
    float acc = 0.f;
    for (long long p = p0; p < p1; ++p) acc += __ldg(dpre + p * 2 + co);
    atomicAdd(db + co, acc);
  }
}

int conv7_c2_wgrad(const float* x, const float* dpre, float* dw, float* db, int N, int H, int W, cudaStream_t stream) {
  SM3_REQUIRE(x && dpre && dw, SM3_ERR_INVALID_ARG, "conv7_c2_wgrad: bad argument");
  const long long total = (long long)N * H * W;
  long long blocks = (long long)num_sms() * 8;
  long long ppb = (total + blocks - 1) / blocks;
  if (ppb < 64) ppb = 64;
  blocks = (total + ppb - 1) / ppb;
  conv7_c2_wgrad_kernel<<<(unsigned)blocks, 224, 0, stream>>>(x, dpre, dw, db, N, H, W, ppb);
  return check_launch("conv7_c2_wgrad_kernel");
}

// out[t,c] = a1[t,c]*sig[t,0] + a2[t,c]*sig[t,1]
__global__ void __launch_bounds__(256) lsk_mix_kernel(const float* __restrict__ a1, const float* __restrict__ a2,
                                                     const float* __restrict__ sig, float* __restrict__ out, long long total,
                                                     int Ch) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int Q = Ch >> 2;
  const long long t = i / Q;
  const float2 s = __ldg(reinterpret_cast<const float2*>(sig) + t);
  const float4 x = ldg_f4(a1 + i * 4), y = ldg_f4(a2 + i * 4);
  *reinterpret_cast<float4*>(out + i * 4) = make_float4(fmaf(x.x, s.x, y.x * s.y), fmaf(x.y, s.x, y.y * s.y),
                                                        fmaf(x.z, s.x, y.z * s.y), fmaf(x.w, s.x, y.w * s.y));
}

int lsk_mix(const float* a1, const float* a2, const float* sig, float* out, long long T, int Ch, cudaStream_t stream) {
  SM3_REQUIRE(a1 && a2 && sig && out && Ch % 4 == 0, SM3_ERR_INVALID_ARG, "lsk_mix: bad argument");
  const long long total = T * (Ch / 4);
  lsk_mix_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(a1, a2, sig, out, total, Ch);
  return check_launch("lsk_mix_kernel");
}

// dpre[t,s] = (sum_c dout[t,c] * a_s[t,c]) * sig_s * (1 - sig_s)        (backward of the weighted sum into the sigmoid input)
__global__ void __launch_bounds__(256) lsk_mix_bwd_sig_kernel(const float* __restrict__ dout, const float* __restrict__ a1,
                                                             const float* __restrict__ a2, const float* __restrict__ sig,
                                                             float* __restrict__ dpre, long long T, int Ch) {
  const long long t = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (t >= T) return;
  float d0 = 0.f, d1 = 0.f;
  for (int c = lane; c < Ch; c += 32) {
    const float d = __ldg(dout + t * Ch + c);
    d0 = fmaf(d, __ldg(a1 + t * Ch + c), d0);
    d1 = fmaf(d, __ldg(a2 + t * Ch + c), d1);
  }
  d0 = warp_sum(d0); d1 = warp_sum(d1);
  if (lane == 0) {
    const float s0 = __ldg(sig + t * 2), s1 = __ldg(sig + t * 2 + 1);
    dpre[t * 2] = d0 * s0 * (1.0f - s0);
    dpre[t * 2 + 1] = d1 * s1 * (1.0f - s1);
  }
}

int lsk_mix_bwd_sig(const float* dout, const float* a1, const float* a2, const float* sig, float* dpre, long long T, int Ch,
                    cudaStream_t stream) {
  SM3_REQUIRE(dout && a1 && a2 && sig && dpre, SM3_ERR_INVALID_ARG, "lsk_mix_bwd_sig: bad argument");
  lsk_mix_bwd_sig_kernel<<<(unsigned)((T * 32 + 255) / 256), 256, 0, stream>>>(dout, a1, a2, sig, dpre, T, Ch);
  return check_launch("lsk_mix_bwd_sig_kernel");
}

// da_s[t,c] = dout[t,c]*sig[t,s] + dagg[t,0]/(2Ch) + (amax[t] == s*Ch + c) * dagg[t,1]
__global__ void __launch_bounds__(256) lsk_mix_bwd_in_kernel(const float* __restrict__ dout, const float* __restrict__ sig,
                                                            const float* __restrict__ dagg, const int* __restrict__ amax,
                                                            float* __restrict__ da1, float* __restrict__ da2, long long total,
                                                            int Ch) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int Q = Ch >> 2;
  const long long t = i / Q;
  const int c = (int)(i % Q) * 4;
  const float2 s = __ldg(reinterpret_cast<const float2*>(sig) + t);
  const float2 g = __ldg(reinterpret_cast<const float2*>(dagg) + t);
  const int am = __ldg(amax + t);
  const float gm = g.x / (float)(2 * Ch);
  const float4 d = ldg_f4(dout + i * 4);
  float o1[4] = {fmaf(d.x, s.x, gm), fmaf(d.y, s.x, gm), fmaf(d.z, s.x, gm), fmaf(d.w, s.x, gm)};
  float o2[4] = {fmaf(d.x, s.y, gm), fmaf(d.y, s.y, gm), fmaf(d.z, s.y, gm), fmaf(d.w, s.y, gm)};
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    if (am == c + e) o1[e] += g.y;
    if (am == Ch + c + e) o2[e] += g.y;
  }
  *reinterpret_cast<float4*>(da1 + i * 4) = make_float4(o1[0], o1[1], o1[2], o1[3]);
  *reinterpret_cast<float4*>(da2 + i * 4) = make_float4(o2[0], o2[1], o2[2], o2[3]);
}

int lsk_mix_bwd_in(const float* dout, const float* sig, const float* dagg, const int* amax, float* da1, float* da2,
                   long long T, int Ch, cudaStream_t stream) {
  SM3_REQUIRE(dout && sig && dagg && amax && da1 && da2 && Ch % 4 == 0, SM3_ERR_INVALID_ARG, "lsk_mix_bwd_in: bad argument");
  const long long total = T * (Ch / 4);
  lsk_mix_bwd_in_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(dout, sig, dagg, amax, da1, da2, total, Ch);
  return check_launch("lsk_mix_bwd_in_kernel");
}

// ------------------------------------------------------------------------------------------------
// im2col for the patch-embedding convolutions: col[t_out, (kh*ks + kw)*Cin + ci] (zero padded to Kp columns).
// nchw = 1 reads the network input [N,Cin,H,W] (stem); otherwise x is NHWC.  One thread per col element quad.
__global__ void __launch_bounds__(256) im2col_kernel(const float* __restrict__ x, float* __restrict__ col, int N, int H, int W,
                                                    int Cin, int ks, int stride, int pad, int Ho, int Wo, int Kp, int nchw,
                                                    long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int Q = Kp >> 2;
  const long long t = i / Q;
  const int k0 = (int)(i % Q) * 4;
  const int wo = (int)(t % Wo); const long long r = t / Wo; const int ho = (int)(r % Ho); const long long n = r / Ho;
  float v[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const int k = k0 + e;
    float val = 0.f;
    if (k < ks * ks * Cin) {
      const int tap = k / Cin, ci = k - tap * Cin;
      const int hi = ho * stride - pad + tap / ks, wi = wo * stride - pad + tap % ks;
      if (hi >= 0 && hi < H && wi >= 0 && wi < W)
        val = nchw ? __ldg(x + ((n * Cin + ci) * H + hi) * W + wi) : __ldg(x + ((n * H + hi) * W + wi) * Cin + ci);
    }
    v[e] = val;
  }
  *reinterpret_cast<float4*>(col + t * Kp + k0) = make_float4(v[0], v[1], v[2], v[3]);
}

int im2col(const float* x, float* col, int N, int H, int W, int Cin, int ks, int stride, int pad, int Kp, int nchw,
           cudaStream_t stream) {
  SM3_REQUIRE(x && col && Kp % 4 == 0 && Kp >= ks * ks * Cin && stride >= 1, SM3_ERR_INVALID_ARG, "im2col: bad argument");
  const int Ho = (H + 2 * pad - ks) / stride + 1, Wo = (W + 2 * pad - ks) / stride + 1;
  const long long total = (long long)N * Ho * Wo * (Kp / 4);
  im2col_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(x, col, N, H, W, Cin, ks, stride, pad, Ho, Wo, Kp, nchw, total);
  return check_launch("im2col_kernel");
}

// dx[n,h,w,ci] = sum over taps (kh,kw) with (h + pad - kh) % stride == 0 of dcol[t_out, (kh*ks+kw)*Cin + ci]   (gather form)
// nchw = 1 writes dx as [N,Cin,H,W] (the previous stage's returned feature map is the conv input, lsk_moe.py:555-557).
__global__ void __launch_bounds__(256) col2im_kernel(const float* __restrict__ dcol, float* __restrict__ dx, int N, int H, int W,
                                                    int Cin, int ks, int stride, int pad, int Ho, int Wo, int Kp, int nchw,
                                                    long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  int c, w, h; long long n;
  if (nchw) {
    w = (int)(i % W); long long r = i / W; h = (int)(r % H); r /= H; c = (int)(r % Cin); n = r / Cin;
  } else {
    const int Q = Cin >> 2;
    c = (int)(i % Q) * 4;
    const long long p = i / Q;
    w = (int)(p % W); const long long r = p / W; h = (int)(r % H); n = r / H;
  }
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int kh = 0; kh < ks; ++kh) {
    const int hn = h + pad - kh;
    if (hn < 0 || hn % stride) continue;
    const int ho = hn / stride;
    if (ho >= Ho) continue;
    for (int kw = 0; kw < ks; ++kw) {
      const int wn = w + pad - kw;
      if (wn < 0 || wn % stride) continue;
      const int wo = wn / stride;
      if (wo >= Wo) continue;
      const float* src = dcol + ((n * Ho + ho) * Wo + wo) * Kp + (kh * ks + kw) * Cin + c;
      if (nchw) { acc.x += __ldg(src); }
      else { const float4 v = ldg_f4(src); acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w; }
    }
  }
  if (nchw) dx[i] = acc.x;
  else *reinterpret_cast<float4*>(dx + (((n * H + h) * W + w) * Cin) + c) = acc;
}

int col2im(const float* dcol, float* dx, int N, int H, int W, int Cin, int ks, int stride, int pad, int Kp, int nchw,
           cudaStream_t stream) {
  SM3_REQUIRE(dcol && dx && (nchw || Cin % 4 == 0) && Kp % 4 == 0, SM3_ERR_INVALID_ARG, "col2im: bad argument (NHWC needs Cin % 4 == 0)");
  const int Ho = (H + 2 * pad - ks) / stride + 1, Wo = (W + 2 * pad - ks) / stride + 1;
  const long long total = nchw ? (long long)N * Cin * H * W : (long long)N * H * W * (Cin / 4);
  col2im_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(dcol, dx, N, H, W, Cin, ks, stride, pad, Ho, Wo, Kp, nchw, total);
  return check_launch("col2im_kernel");
}

}  // namespace sm3
