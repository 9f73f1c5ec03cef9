// MultitaskFPN helpers (SURVEY.md 8(f) rank 1: the consumer of the backbone's 4-tuple).  The 1x1 lateral and 3x3 output
// convolutions run on the wgmma GEMM through im2col (lsk.cu); this file holds the two remaining data-movement kernels:
//   upsample_add      laterals[i-1] + F.interpolate(laterals[i], size=prev_shape, mode='nearest')
//                     (reference mmrotate/models/necks/Multitask_FPN.py:123-134) and its backward,
//   transpose_batched NHWC <-> NCHW conversion of the returned pyramid levels (the reference is NCHW end to end),
//   fpn_export_pool   mmdet FPN's top level to NCHW together with its max-pool extra levels, and its backward.
#include "common.cuh"
#include "kernels.h"

namespace sm3 {

// out[n,y,x,:] = a[n,y,x,:] + b[n, (y*h)/H, (x*w)/W, :]      (nearest; exact for integer ratios, which is all the FPN uses)
__global__ void __launch_bounds__(256) upsample_add_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                          float* __restrict__ out, int H, int W, int h, int w, int C,
                                                          long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int Q = C >> 2;
  const int c = (int)(i % Q) * 4;
  long long p = i / Q;
  const int x = (int)(p % W); p /= W;
  const int y = (int)(p % H); const long long n = p / H;
  const int ys = (int)(((long long)y * h) / H), xs = (int)(((long long)x * w) / W);
  const float4 u = ldg_f4(a + i * 4);
  const float4 v = ldg_f4(b + ((n * h + ys) * w + xs) * C + c);
  *reinterpret_cast<float4*>(out + i * 4) = make_float4(u.x + v.x, u.y + v.y, u.z + v.z, u.w + v.w);
}

// db[n,ys,xs,:] = sum of d over the destination pixels that read (ys,xs)
__global__ void __launch_bounds__(256) upsample_add_bwd_kernel(const float* __restrict__ d, float* __restrict__ db, int H, int W,
                                                              int h, int w, int C, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int Q = C >> 2;
  const int c = (int)(i % Q) * 4;
  long long p = i / Q;
  const int xs = (int)(p % w); p /= w;
  const int ys = (int)(p % h); const long long n = p / h;
  // destination rows y with (y*h)/H == ys  <=>  y in [ceil(ys*H/h), ceil((ys+1)*H/h))
  const int y0 = (int)(((long long)ys * H + h - 1) / h), y1 = (int)((((long long)ys + 1) * H + h - 1) / h);
  const int x0 = (int)(((long long)xs * W + w - 1) / w), x1 = (int)((((long long)xs + 1) * W + w - 1) / w);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int y = y0; y < y1 && y < H; ++y)
    for (int x = x0; x < x1 && x < W; ++x) {
      const float4 v = ldg_f4(d + ((n * H + y) * W + x) * C + c);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
  *reinterpret_cast<float4*>(db + i * 4) = acc;
}

int upsample_add(const float* a, const float* b, float* out, int N, int H, int W, int h, int w, int C, cudaStream_t stream) {
  SM3_REQUIRE(a && b && out && C % 4 == 0 && H >= h && W >= w && h > 0 && w > 0, SM3_ERR_INVALID_ARG, "upsample_add: bad argument");
  const long long total = (long long)N * H * W * (C / 4);
  upsample_add_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(a, b, out, H, W, h, w, C, total);
  return check_launch("upsample_add_kernel");
}

int upsample_add_bwd(const float* d, float* db, int N, int H, int W, int h, int w, int C, cudaStream_t stream) {
  SM3_REQUIRE(d && db && C % 4 == 0 && H >= h && W >= w && h > 0 && w > 0, SM3_ERR_INVALID_ARG, "upsample_add_bwd: bad argument");
  const long long total = (long long)N * h * w * (C / 4);
  upsample_add_bwd_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(d, db, H, W, h, w, C, total);
  return check_launch("upsample_add_bwd_kernel");
}

// out[b, c, r] = in[b, r, c]   (32x32 tiles through shared memory, both sides coalesced)
__global__ void __launch_bounds__(256) transpose_batched_kernel(const float* __restrict__ in, float* __restrict__ out, int R, int Cc) {
  __shared__ float tile[32][33];
  const long long b = blockIdx.z;
  const int r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const float* src = in + b * (long long)R * Cc;
  float* dst = out + b * (long long)R * Cc;
  for (int j = ty; j < 32; j += 8) {
    const int r = r0 + j, c = c0 + tx;
    tile[j][tx] = (r < R && c < Cc) ? __ldg(src + (long long)r * Cc + c) : 0.f;
  }
  __syncthreads();
  for (int j = ty; j < 32; j += 8) {
    const int c = c0 + j, r = r0 + tx;
    if (c < Cc && r < R) dst[(long long)c * R + r] = tile[tx][j];
  }
}

int transpose_batched(const float* in, float* out, int B, int R, int Cc, cudaStream_t stream) {
  SM3_REQUIRE(in && out && B > 0 && R > 0 && Cc > 0 && B < 65536, SM3_ERR_INVALID_ARG, "transpose_batched: bad argument");
  const unsigned gy = (unsigned)((R + 31) / 32);
  SM3_REQUIRE(gy < 65536, SM3_ERR_UNSUPPORTED_SHAPE, "transpose_batched: too many rows (%d)", R);
  dim3 grid((unsigned)((Cc + 31) / 32), gy, (unsigned)B);
  transpose_batched_kernel<<<grid, 256, 0, stream>>>(in, out, R, Cc);
  return check_launch("transpose_batched_kernel");
}

// ---- mmdet FPN: the top output level and its max-pool extra levels -------------------------------------------------
// With add_extra_convs=False, mmdet's FPN appends F.max_pool2d(outs[-1], 1, stride=2) L times: level k is
// [N, C, H_k, W_k], H_k = ceil(H_{k-1} / 2), and level k[y, x] = P_top[y << k, x << k].  One kernel exports P_top from
// NHWC to NCHW and writes every level from the same shared-memory tile; the backward folds the L+1 upstream gradients
// back into one NHWC gradient.
struct FpnLevels {
  float* p[SM3_FPN_MAX_POOL_LEVELS + 1];   // p[0] = P_top, p[k] = pool level k (all NCHW)
};

// deepest pool level pixel (y, x) feeds: the largest k <= L with 2^k | y and 2^k | x
__device__ __forceinline__ int fpn_pool_depth(int y, int x, int L) {
  const int yx = y | x;
  return yx == 0 ? L : min(L, __ffs(yx) - 1);
}

// grid (pixel tiles, channel tiles, N); a 32-pixel x 32-channel tile is read coalesced along C and written coalesced
// along the pixels of P_top.  The pool levels take the tile's pixels whose coordinates are multiples of 2^k: runs of
// 32 / 2^k consecutive words per warp.
__global__ void __launch_bounds__(256) fpn_export_pool_kernel(const float* __restrict__ in, FpnLevels o, int H, int W, int C,
                                                             int L) {
  __shared__ float tile[32][33];
  const int R = H * W;
  const long long n = blockIdx.z;
  const int r0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const float* src = in + n * R * C;
  for (int j = ty; j < 32; j += 8) {
    const int r = r0 + j, c = c0 + tx;
    tile[j][tx] = (r < R && c < C) ? __ldg(src + (long long)r * C + c) : 0.f;
  }
  __syncthreads();
  const int r = r0 + tx;
  if (r >= R) return;
  const int y = r / W, x = r - y * W;
  const int depth = fpn_pool_depth(y, x, L);
  for (int j = ty; j < 32; j += 8) {
    const int c = c0 + j;
    if (c >= C) break;
    const float v = tile[tx][j];
    const long long nc = n * C + c;
    o.p[0][nc * R + r] = v;
    int hk = H, wk = W;
#pragma unroll
    for (int k = 1; k <= SM3_FPN_MAX_POOL_LEVELS; ++k) {     // unrolled: o.p stays in the parameter bank
      if (k > depth) break;
      hk = (hk + 1) >> 1; wk = (wk + 1) >> 1;
      o.p[k][(nc * hk + (y >> k)) * wk + (x >> k)] = v;
    }
  }
}

// din[n, y, x, c] = dP_top[n, c, y, x] + sum over k = 1..L, in that order, of [2^k | y, 2^k | x] dP_k[n, c, y>>k, x>>k].
// Each output element is summed by one thread: no atomics, the same bits every run.
__global__ void __launch_bounds__(256) fpn_export_pool_bwd_kernel(FpnLevels g, float* __restrict__ din, int H, int W, int C,
                                                                 int L) {
  __shared__ float tile[32][33];
  const int R = H * W;
  const long long n = blockIdx.z;
  const int r0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int r = r0 + tx;
  const int y = r / W, x = r - y * W;
  const int depth = r < R ? fpn_pool_depth(y, x, L) : 0;
  for (int j = ty; j < 32; j += 8) {
    const int c = c0 + j;
    float v = 0.f;
    if (r < R && c < C) {
      const long long nc = n * C + c;
      v = __ldg(g.p[0] + nc * R + r);
      int hk = H, wk = W;
#pragma unroll
      for (int k = 1; k <= SM3_FPN_MAX_POOL_LEVELS; ++k) {
        if (k > depth) break;
        hk = (hk + 1) >> 1; wk = (wk + 1) >> 1;
        v += __ldg(g.p[k] + (nc * hk + (y >> k)) * wk + (x >> k));
      }
    }
    tile[j][tx] = v;
  }
  __syncthreads();
  float* dst = din + n * R * C;
  for (int j = ty; j < 32; j += 8) {
    const int rr = r0 + j, c = c0 + tx;
    if (rr < R && c < C) dst[(long long)rr * C + c] = tile[tx][j];
  }
}

static int fpn_pool_grid(int N, int H, int W, int C, int L, dim3* grid, const char* what) {
  SM3_REQUIRE(N > 0 && N < 65536 && H > 0 && W > 0 && C > 0 && L >= 1 && L <= SM3_FPN_MAX_POOL_LEVELS,
              SM3_ERR_INVALID_ARG, "%s: bad argument (N=%d H=%d W=%d C=%d L=%d)", what, N, H, W, C, L);
  SM3_REQUIRE((long long)H * W <= 0x7fffffe0LL && (C + 31) / 32 < 65536, SM3_ERR_UNSUPPORTED_SHAPE,
              "%s: level too large (H=%d W=%d C=%d)", what, H, W, C);
  *grid = dim3((unsigned)(((long long)H * W + 31) / 32), (unsigned)((C + 31) / 32), (unsigned)N);
  return SM3_OK;
}

int fpn_export_pool(const float* in, float* const* outs, int N, int H, int W, int C, int L, cudaStream_t stream) {
  dim3 grid;
  if (int rc = fpn_pool_grid(N, H, W, C, L, &grid, "fpn_export_pool")) return rc;
  SM3_REQUIRE(in && outs, SM3_ERR_INVALID_ARG, "fpn_export_pool: null pointer");
  FpnLevels o{};
  for (int k = 0; k <= L; ++k) {
    SM3_REQUIRE(outs[k], SM3_ERR_INVALID_ARG, "fpn_export_pool: output level %d is null", k);
    o.p[k] = outs[k];
  }
  fpn_export_pool_kernel<<<grid, 256, 0, stream>>>(in, o, H, W, C, L);
  return check_launch("fpn_export_pool_kernel");
}

int fpn_export_pool_bwd(const float* const* douts, float* din, int N, int H, int W, int C, int L, cudaStream_t stream) {
  dim3 grid;
  if (int rc = fpn_pool_grid(N, H, W, C, L, &grid, "fpn_export_pool_bwd")) return rc;
  SM3_REQUIRE(douts && din, SM3_ERR_INVALID_ARG, "fpn_export_pool_bwd: null pointer");
  FpnLevels g{};
  for (int k = 0; k <= L; ++k) {
    SM3_REQUIRE(douts[k], SM3_ERR_INVALID_ARG, "fpn_export_pool_bwd: gradient level %d is null", k);
    g.p[k] = const_cast<float*>(douts[k]);
  }
  fpn_export_pool_bwd_kernel<<<grid, 256, 0, stream>>>(g, din, H, W, C, L);
  return check_launch("fpn_export_pool_bwd_kernel");
}

}  // namespace sm3
