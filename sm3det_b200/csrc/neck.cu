// MultitaskFPN helpers (SURVEY.md 8(f) rank 1: the consumer of the backbone's 4-tuple).  The 1x1 lateral and 3x3 output
// convolutions run on the wgmma GEMM through im2col (lsk.cu); this file holds the two remaining data-movement kernels:
//   upsample_add      laterals[i-1] + F.interpolate(laterals[i], size=prev_shape, mode='nearest')
//                     (reference mmrotate/models/necks/Multitask_FPN.py:123-134) and its backward,
//   transpose_batched NHWC <-> NCHW conversion of the returned pyramid levels (the reference is NCHW end to end).
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

}  // namespace sm3
