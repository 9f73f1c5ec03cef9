// 7x7 depthwise convolution on NHWC fp32 tensors (padding 3, stride 1), forward / dgrad / wgrad.
//
// Replaces nn.Conv2d(C, C, 7, padding=3, groups=C) of ConvNeXtBlock (reference convnext_moe.py
// :311-312, applied :347) and autograd's depthwise dgrad/wgrad.  NHWC end-to-end removes the two
// full-tensor permute copies per block (:350, :358).  Taps are passed transposed as wt[49][C] so a
// warp reads 32 consecutive channel-quads (512 B) per tap.
//
// Forward: a thread owns 4 channels x WS consecutive output columns of one row, slides a
// (WS+6)-wide register window over the 7 input rows: 7*(WS+6) float4 loads for 49*WS*4 FMAs.
// dgrad is the same kernel on dy with the taps flipped (the caller passes wt_flipped).
#include "common.cuh"
#include "kernels.h"

namespace sm3 {

constexpr int DW_WS = 8;

__global__ void __launch_bounds__(256) dwconv7_fwd_kernel(const float* __restrict__ x, const float* __restrict__ wt,
                                                         const float* __restrict__ bias, const float* __restrict__ resid,
                                                         float* __restrict__ y, int N, int H, int W, int C, int strips,
                                                         long long total) {
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (tid >= total) return;
  const int Q = C >> 2;
  const int q = (int)(tid % Q);
  long long r = tid / Q;
  const int s = (int)(r % strips); r /= strips;
  const int h = (int)(r % H);
  const int n = (int)(r / H);
  const int w0 = s * DW_WS;
  const int c = q * 4;

  float4 acc[DW_WS];
  const float4 b = bias ? ldg_f4(bias + c) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int o = 0; o < DW_WS; ++o) acc[o] = b;

  const float* xn = x + (long long)n * H * W * C + c;
#pragma unroll 1
  for (int i = 0; i < 7; ++i) {
    const int hi = h + i - 3;
    if (hi < 0 || hi >= H) continue;
    float4 wv[7];
#pragma unroll
    for (int j = 0; j < 7; ++j) wv[j] = ldg_f4(wt + (i * 7 + j) * C + c);
    const float* xr = xn + (long long)hi * W * C;
#pragma unroll
    for (int jj = 0; jj < DW_WS + 6; ++jj) {
      const int wi = w0 + jj - 3;
      float4 xv = make_float4(0.f, 0.f, 0.f, 0.f);
      if (wi >= 0 && wi < W) xv = ldg_f4(xr + (long long)wi * C);
#pragma unroll
      for (int o = 0; o < DW_WS; ++o) {
        const int j = jj - o;
        if (j >= 0 && j < 7) {
          acc[o].x = fmaf(xv.x, wv[j].x, acc[o].x);
          acc[o].y = fmaf(xv.y, wv[j].y, acc[o].y);
          acc[o].z = fmaf(xv.z, wv[j].z, acc[o].z);
          acc[o].w = fmaf(xv.w, wv[j].w, acc[o].w);
        }
      }
    }
  }
  const long long rowoff = (((long long)n * H + h) * W) * C + c;
  float* yr = y + rowoff;
#pragma unroll
  for (int o = 0; o < DW_WS; ++o)
    if (w0 + o < W) {
      float4 v = acc[o];
      if (resid) { const float4 r = ldg_f4(resid + rowoff + (long long)(w0 + o) * C); v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w; }
      *reinterpret_cast<float4*>(yr + (long long)(w0 + o) * C) = v;
    }
}

// ------------------------------------------------------------------------------------------------
// Shared-memory tiled version (used when C % 32 == 0): a block owns a 16x16 output tile of 32 channels,
// stages the (16+6)^2 x 32 input halo tile with cp.async (zero fill outside the image), then every lane
// owns ONE channel (conflict-free stride-1 smem reads, its 7 taps of the current row in registers) and
// every warp two output rows: 22 LDS feed 16 outputs x 7 taps, so the kernel is FMA-issue bound
// (49 FMA : 9.6 LDS per output) and the input is read 1.9x instead of 12x.
constexpr int DT = 16;            // output tile edge
constexpr int DTI = DT + 6;       // input tile edge
constexpr int DCC = 32;           // channels per block

__device__ __forceinline__ void dw_load_tile(float* xs, const float* __restrict__ x, int n, int h0, int w0, int c0,
                                             int H, int W, int C) {
  // 22*22 pixels x 8 x 16-byte chunks
  for (int idx = threadIdx.x; idx < DTI * DTI * 8; idx += blockDim.x) {
    const int q = idx & 7, pix = idx >> 3;
    const int py = pix / DTI, px = pix - py * DTI;
    const int hi = h0 + py - 3, wi = w0 + px - 3;
    const uint32_t dst = static_cast<uint32_t>(__cvta_generic_to_shared(xs + pix * DCC + q * 4));
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

// Packed-FP32 helpers (ffma2 in common.cuh): a "pair" is two adjacent channels held in one 64-bit register, so every
// 64-bit shared-memory load feeds two FMAs of this issue-bound stencil.
__device__ __forceinline__ f32x2_t pack2(float lo, float hi) {
  return (f32x2_t)__float_as_uint(lo) | ((f32x2_t)__float_as_uint(hi) << 32);
}
__device__ __forceinline__ float2 unpack2(f32x2_t v) {
  return make_float2(__uint_as_float((uint32_t)v), __uint_as_float((uint32_t)(v >> 32)));
}

// lane = (row selector l/16, channel pair l%16): a half-warp owns one output row of the 16x16 tile and two channels per
// lane, so every LDS.64 does the work of two of the scalar version's loads.
__global__ void __launch_bounds__(256) dwconv7_tile_kernel(const float* __restrict__ x, const float* __restrict__ wt,
                                                          const float* __restrict__ bias, const float* __restrict__ resid,
                                                          float* __restrict__ y, int H, int W, int C, int tiles_w,
                                                          int tiles_h) {
  extern __shared__ float xs[];                           // [DTI][DTI][DCC]
  const int tw = blockIdx.x % tiles_w, th = blockIdx.x / tiles_w;
  const int cchunks = C / DCC;
  const int n = blockIdx.y / cchunks, c0 = (blockIdx.y % cchunks) * DCC;
  const int h0 = th * DT, w0 = tw * DT;
  dw_load_tile(xs, x, n, h0, w0, c0, H, W, C);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int cp = lane & 15, r = warp * 2 + (lane >> 4);
  const int c = c0 + 2 * cp;
  const int h = h0 + r;
  if (h >= H) return;
  const f32x2_t b2 = bias ? __ldg(reinterpret_cast<const f32x2_t*>(bias + c)) : 0ull;
  f32x2_t acc[DT];
#pragma unroll
  for (int o = 0; o < DT; ++o) acc[o] = b2;
#pragma unroll 1
  for (int i = 0; i < 7; ++i) {
    f32x2_t wv[7];
#pragma unroll
    for (int j = 0; j < 7; ++j) wv[j] = __ldg(reinterpret_cast<const f32x2_t*>(wt + (i * 7 + j) * C + c));
    const f32x2_t* xr = reinterpret_cast<const f32x2_t*>(xs + ((r + i) * DTI) * DCC) + cp;
#pragma unroll
    for (int cc = 0; cc < DTI; ++cc) {
      const f32x2_t v = xr[cc * (DCC / 2)];
#pragma unroll
      for (int j = 0; j < 7; ++j) {
        const int o = cc - j;
        if (o >= 0 && o < DT) acc[o] = ffma2(v, wv[j], acc[o]);
      }
    }
  }
  const long long rowoff = (((long long)n * H + h) * W) * C + c;
#pragma unroll
  for (int o = 0; o < DT; ++o) {
    const int w = w0 + o;
    if (w < W) {
      float2 v = unpack2(acc[o]);
      if (resid) { const float2 rr = __ldg(reinterpret_cast<const float2*>(resid + rowoff + (long long)w * C)); v.x += rr.x; v.y += rr.y; }
      *reinterpret_cast<float2*>(y + rowoff + (long long)w * C) = v;
    }
  }
}

int dwconv7_fwd(const float* x, const float* wt, const float* bias, const float* resid, float* y, int N, int H, int W,
                int C, cudaStream_t stream) {
  SM3_REQUIRE(x && wt && y, SM3_ERR_INVALID_ARG, "dwconv7_fwd: null argument");
  SM3_REQUIRE(C % 4 == 0 && N > 0 && H > 0 && W > 0, SM3_ERR_UNSUPPORTED_SHAPE, "dwconv7_fwd: C=%d must be a multiple of 4", C);
  if (C % DCC == 0) {
    const int tiles_w = (W + DT - 1) / DT, tiles_h = (H + DT - 1) / DT;
    const size_t smem = (size_t)DTI * DTI * DCC * sizeof(float);
    // per call: function attributes are per device, and the library may be driven from several devices of one process
    cudaFuncSetAttribute(dwconv7_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    SM3_REQUIRE((long long)N * (C / DCC) < 65536, SM3_ERR_UNSUPPORTED_SHAPE, "dwconv7_fwd: N*C/32 too large for grid.y");
    dim3 grid((unsigned)(tiles_w * tiles_h), (unsigned)(N * (C / DCC)));
    dwconv7_tile_kernel<<<grid, 256, smem, stream>>>(x, wt, bias, resid, y, H, W, C, tiles_w, tiles_h);
    return check_launch("dwconv7_tile_kernel");
  }
  const int strips = (W + DW_WS - 1) / DW_WS;
  const long long total = (long long)N * H * strips * (C / 4);
  const long long blocks = (total + 255) / 256;
  SM3_REQUIRE(blocks < (1LL << 31), SM3_ERR_UNSUPPORTED_SHAPE, "dwconv7_fwd: tensor too large");
  dwconv7_fwd_kernel<<<(unsigned)blocks, 256, 0, stream>>>(x, wt, bias, resid, y, N, H, W, C, strips, total);
  return check_launch("dwconv7_fwd");
}

// wgrad: dwt[i*7+j][c] += sum_{n,h,w} x[n,h+i-3,w+j-3,c] * dy[n,h,w,c] ; dbias[c] += sum dy
// Thread = (channel quad, tap row i) for a band of output rows; sliding 7-wide x window along w.
__global__ void __launch_bounds__(224) dwconv7_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ dy,
                                                           float* __restrict__ dwt, float* __restrict__ dbias, int N,
                                                           int H, int W, int C, int rows_per_band, int bands_per_img) {
  const int ql = threadIdx.x & 31;
  const int i = threadIdx.x >> 5;               // tap row 0..6
  const int q = blockIdx.y * 32 + ql;
  if (q * 4 >= C) return;
  const int c = q * 4;
  const int n = blockIdx.x / bands_per_img;
  const int h0 = (blockIdx.x % bands_per_img) * rows_per_band;
  const int h1 = min(H, h0 + rows_per_band);
  float4 acc[7];
#pragma unroll
  for (int j = 0; j < 7; ++j) acc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 accb = make_float4(0.f, 0.f, 0.f, 0.f);
  const float* xn = x + (long long)n * H * W * C + c;
  const float* dn = dy + (long long)n * H * W * C + c;
  for (int h = h0; h < h1; ++h) {
    const int hi = h + i - 3;
    if (hi < 0 || hi >= H) continue;       // (bias is accumulated by the i == 3 role, always in range)
    const float* xr = xn + (long long)hi * W * C;
    const float* dr = dn + (long long)h * W * C;
    float4 win[7];                          // x[hi, w-3 .. w+3]
#pragma unroll
    for (int j = 0; j < 7; ++j) {
      const int wi = j - 3;
      win[j] = (wi >= 0 && wi < W) ? ldg_f4(xr + (long long)wi * C) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    for (int w = 0; w < W; ++w) {
      const float4 d = ldg_f4(dr + (long long)w * C);
#pragma unroll
      for (int j = 0; j < 7; ++j) {
        acc[j].x = fmaf(win[j].x, d.x, acc[j].x); acc[j].y = fmaf(win[j].y, d.y, acc[j].y);
        acc[j].z = fmaf(win[j].z, d.z, acc[j].z); acc[j].w = fmaf(win[j].w, d.w, acc[j].w);
      }
      if (i == 3) { accb.x += d.x; accb.y += d.y; accb.z += d.z; accb.w += d.w; }
#pragma unroll
      for (int j = 0; j < 6; ++j) win[j] = win[j + 1];
      const int wn = w + 4;
      win[6] = (wn < W) ? ldg_f4(xr + (long long)wn * C) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
#pragma unroll
  for (int j = 0; j < 7; ++j) {
    float* p = dwt + (i * 7 + j) * C + c;
    atomicAdd(p, acc[j].x); atomicAdd(p + 1, acc[j].y); atomicAdd(p + 2, acc[j].z); atomicAdd(p + 3, acc[j].w);
  }
  if (i == 3 && dbias) {
    atomicAdd(dbias + c, accb.x); atomicAdd(dbias + c + 1, accb.y);
    atomicAdd(dbias + c + 2, accb.z); atomicAdd(dbias + c + 3, accb.w);
  }
}

// Tiled wgrad: persistent blocks loop over 16x16 tiles of one 32-channel chunk; lane = channel keeps the 49 tap
// sums (+ bias sum) in registers across all its tiles, so the cross-block reduction is one atomic per tap per block.
__global__ void __launch_bounds__(256) dwconv7_wgrad_tile_kernel(const float* __restrict__ x, const float* __restrict__ dy,
                                                                float* __restrict__ dwt, float* __restrict__ dbias, int N,
                                                                int H, int W, int C, int tiles_w, int tiles_h,
                                                                int blocks_per_chunk) {
  extern __shared__ float smem[];
  float* xs = smem;                               // [DTI][DTI][DCC]
  float* ds = smem + DTI * DTI * DCC;             // [DT][DT][DCC]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c0 = blockIdx.y * DCC;
  const int cp = lane & 15, half = lane >> 4;           // channel pair, row selector (two channels per lane)
  f32x2_t acc[49];
#pragma unroll
  for (int i = 0; i < 49; ++i) acc[i] = 0ull;
  float2 accb = make_float2(0.f, 0.f);
  const int tiles = N * tiles_h * tiles_w;
  for (int t = blockIdx.x; t < tiles; t += blocks_per_chunk) {
    const int n = t / (tiles_h * tiles_w), rem = t % (tiles_h * tiles_w);
    const int h0 = (rem / tiles_w) * DT, w0 = (rem % tiles_w) * DT;
    __syncthreads();                              // previous tile fully consumed
    for (int idx = threadIdx.x; idx < DT * DT * 8; idx += blockDim.x) {
      const int q = idx & 7, pix = idx >> 3;
      const int py = pix / DT, px = pix - py * DT;
      const int hi = h0 + py, wi = w0 + px;
      const uint32_t dst = static_cast<uint32_t>(__cvta_generic_to_shared(ds + pix * DCC + q * 4));
      if (hi < H && wi < W) {
        const float* src = dy + (((long long)n * H + hi) * W + wi) * C + c0 + q * 4;
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
      } else {
        asm volatile("st.shared.v4.f32 [%0], {%1, %1, %1, %1};" ::"r"(dst), "f"(0.f) : "memory");
      }
    }
    dw_load_tile(xs, x, n, h0, w0, c0, H, W, C);  // commits + waits for both tiles, then __syncthreads
    const int r = warp * 2 + half;
    f32x2_t d[DT];
#pragma unroll
    for (int o = 0; o < DT; ++o) {
      d[o] = reinterpret_cast<const f32x2_t*>(ds + (r * DT + o) * DCC)[cp];
      const float2 dv = unpack2(d[o]);
      accb.x += dv.x; accb.y += dv.y;
    }
#pragma unroll
    for (int i = 0; i < 7; ++i) {
      const f32x2_t* xr = reinterpret_cast<const f32x2_t*>(xs + ((r + i) * DTI) * DCC) + cp;
#pragma unroll
      for (int cc = 0; cc < DTI; ++cc) {
        const f32x2_t v = xr[cc * (DCC / 2)];
#pragma unroll
        for (int j = 0; j < 7; ++j) {
          const int o = cc - j;
          if (o >= 0 && o < DT) acc[i * 7 + j] = ffma2(v, d[o], acc[i * 7 + j]);
        }
      }
    }
  }
  // reduce the 16 half-warps of the block through shared memory, then one atomic per (tap, channel)
  __syncthreads();
  float* red = smem;                              // [16][50][32]
  const int hw = warp * 2 + half;
#pragma unroll
  for (int i = 0; i < 49; ++i) reinterpret_cast<f32x2_t*>(red + (hw * 50 + i) * 32)[cp] = acc[i];
  reinterpret_cast<float2*>(red + (hw * 50 + 49) * 32)[cp] = accb;
  __syncthreads();
  for (int idx = threadIdx.x; idx < 50 * 32; idx += blockDim.x) {
    const int i = idx / 32, l = idx % 32;
    float sum = 0.f;
#pragma unroll
    for (int w = 0; w < 16; ++w) sum += red[(w * 50 + i) * 32 + l];
    if (i < 49) atomicAdd(dwt + i * C + c0 + l, sum);
    else if (dbias) atomicAdd(dbias + c0 + l, sum);
  }
}

int dwconv7_wgrad(const float* x, const float* dy, float* dwt, float* dbias, int N, int H, int W, int C,
                  cudaStream_t stream) {
  SM3_REQUIRE(x && dy && dwt, SM3_ERR_INVALID_ARG, "dwconv7_wgrad: null argument");
  SM3_REQUIRE(C % 4 == 0, SM3_ERR_UNSUPPORTED_SHAPE, "dwconv7_wgrad: C=%d must be a multiple of 4", C);
  if (C % DCC == 0) {
    const int tiles_w = (W + DT - 1) / DT, tiles_h = (H + DT - 1) / DT;
    const int chunks = C / DCC;
    long long tiles = (long long)N * tiles_w * tiles_h;
    int bpc = (num_sms() * 2 + chunks - 1) / chunks;          // ~2 waves of blocks over all channel chunks
    if (bpc > tiles) bpc = (int)tiles;
    if (bpc < 1) bpc = 1;
    size_t smem = (size_t)(DTI * DTI + DT * DT) * DCC * sizeof(float);
    if (smem < (size_t)16 * 50 * 32 * sizeof(float)) smem = (size_t)16 * 50 * 32 * sizeof(float);   // final reduction buffer
    cudaFuncSetAttribute(dwconv7_wgrad_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    dim3 grid((unsigned)bpc, (unsigned)chunks);
    dwconv7_wgrad_tile_kernel<<<grid, 256, smem, stream>>>(x, dy, dwt, dbias, N, H, W, C, tiles_w, tiles_h, bpc);
    return check_launch("dwconv7_wgrad_tile_kernel");
  }
  const int gy = (C / 4 + 31) / 32;
  // enough bands to fill the GPU ~4x, at least 1 row per band
  long long want = (long long)num_sms() * 4 / gy;
  if (want < 1) want = 1;
  int bands_per_img = (int)((want + N - 1) / N);
  if (bands_per_img > H) bands_per_img = H;
  if (bands_per_img < 1) bands_per_img = 1;
  const int rows_per_band = (H + bands_per_img - 1) / bands_per_img;
  bands_per_img = (H + rows_per_band - 1) / rows_per_band;
  dim3 grid((unsigned)(N * bands_per_img), (unsigned)gy);
  dwconv7_wgrad_kernel<<<grid, 224, 0, stream>>>(x, dy, dwt, dbias, N, H, W, C, rows_per_band, bands_per_img);
  return check_launch("dwconv7_wgrad");
}

}  // namespace sm3
