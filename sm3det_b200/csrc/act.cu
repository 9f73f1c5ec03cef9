// Fused activation + operand pre-split ("act_pack").
//
// The FFN hidden tensor h = W1 v + b1 is the largest activation of a block ([rows, 4C]).  Evaluating GELU / GELU'
// in the GEMM epilogue (256 threads per SM) is instruction-issue bound,
// so the GEMM only stores h and this HBM-bound elementwise kernel -- full occupancy, 8 elements per thread -- applies
// the activation AND writes the result directly as the pre-split bf16 hi/lo tile images the next GEMMs bulk-copy:
//   mode 0  y = gelu(h)            forward:  A operand of GEMM2 (K-major image);  backward: B operand of wgrad2 (MN image)
//   mode 1  y = da * gelu'(h)      backward: A operand of dgrad1 (K-major) and of wgrad1 (MN-major), + column sums (db1)
//   mode 2  y = h                  plain pack of both images in one pass
// One thread owns one 16-byte chunk of both images: 8 consecutive columns of one row are 8 consecutive k of the
// K-major image and 8 consecutive mn of the MN-major image, so fp32 `a` / `dh` never touch HBM.
// Replaces nn.GELU() at reference convnext_moe.py:390,400 and autograd's GELU backward.
#include "common.cuh"
#include "gemm_tc.cuh"
#include "kernels.h"

namespace sm3 {

__device__ __forceinline__ void split8(const float (&v)[8], uint4& hi, uint4& lo) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int e = 0; e < 8; e += 2) {
    const uint32_t u0 = __float_as_uint(v[e]), u1 = __float_as_uint(v[e + 1]);
    h[e / 2] = __byte_perm(u0, u1, 0x7632);
    const uint32_t r0 = __float_as_uint(v[e] - __uint_as_float(u0 & 0xFFFF0000u)) + 0x8000u;
    const uint32_t r1 = __float_as_uint(v[e + 1] - __uint_as_float(u1 & 0xFFFF0000u)) + 0x8000u;
    l[e / 2] = __byte_perm(r0, r1, 0x7632);
  }
  hi = make_uint4(h[0], h[1], h[2], h[3]);
  lo = make_uint4(l[0], l[1], l[2], l[3]);
}

// grid: (column-chunk groups of CLW, row bands); block 256 = CLW chunk lanes x 256/CLW row lanes.  CLW = 16 when the row has
// an odd number of 16-chunk groups (W = 384: 48 chunks would leave half of the second 32-lane column idle).
template <int MODE, bool CS, int CLW>
__global__ void __launch_bounds__(256, 3) act_pack_kernel(const ActPackArgs a, int rows_per_band) {
  constexpr int RL = 256 / CLW;                      // row lanes
  __shared__ float s_cs[RL][CLW * 8 + 8];
  const int cl = threadIdx.x & (CLW - 1), rlane = threadIdx.x / CLW;
  const int chunk = blockIdx.x * CLW + cl;           // 8-column chunk index
  const int col = chunk * 8;
  const bool col_ok = col < a.W;
  const long long R_pad = (a.R + 31) / 32 * 32;      // images are padded to whole 32-row k-blocks
  const long long live = a.live_tiles ? (long long)__ldg(a.live_tiles) * 128 : a.R;   // rows worth reading
  const long long r_begin = (long long)blockIdx.y * rows_per_band;
  const long long r_end = min(R_pad, r_begin + rows_per_band);
  const int kblocks_k = (a.W + 31) / 32;
  const long long kblocks_mn = R_pad / 32;
  const uint32_t pb_mn = gemm::plane_bytes(a.mn_tile > 0 ? a.mn_tile : 128, true);
  float cs[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) cs[e] = 0.f;
  int cur_group = -1;
  // Software-pipelined over rows: the loads of row r+8 are in flight while row r is evaluated and stored (one row =
  // 32-64 B per thread is not enough memory-level parallelism to cover HBM latency at 4 blocks / SM).
  auto row_live = [&](long long r) { return col_ok && r < a.R && r < live; };
  float4 nh0 = make_float4(0.f, 0.f, 0.f, 0.f), nh1 = nh0, nd0 = nh0, nd1 = nh0;
  auto load_row = [&](long long r) {
    if (r < r_end && row_live(r)) {
      nh0 = ldg_f4(a.h + r * a.W + col); nh1 = ldg_f4(a.h + r * a.W + col + 4);
      if (MODE == 1 || MODE == 3) { nd0 = ldg_f4(a.da + r * a.W + col); nd1 = ldg_f4(a.da + r * a.W + col + 4); }
    }
  };
  load_row(r_begin + rlane);
  for (long long r = r_begin + rlane; r < r_end; r += RL) {
    float y[8], y2[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) { y[e] = 0.f; y2[e] = 0.f; }
    const bool row_ok = row_live(r);
    const float4 h0 = nh0, h1 = nh1, d0 = nd0, d1 = nd1;
    load_row(r + RL);
    if (row_ok) {
      const float hv[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
      if (MODE == 0) {
#pragma unroll
        for (int e = 0; e < 8; ++e) y[e] = gelu_fast(hv[e]);
      } else if (MODE == 1) {
        const float dv[8] = {d0.x, d0.y, d0.z, d0.w, d1.x, d1.y, d1.z, d1.w};
#pragma unroll
        for (int e = 0; e < 8; ++e) y[e] = dv[e] * gelu_grad_fast(hv[e]);
      } else if (MODE == 3) {
        const float dv[8] = {d0.x, d0.y, d0.z, d0.w, d1.x, d1.y, d1.z, d1.w};
#pragma unroll
        for (int e = 0; e < 8; ++e) {          // Phi and exp(-x^2/2) shared by gelu and gelu'
          float Phi, ex;
          phi_parts(hv[e], Phi, ex);
          y2[e] = hv[e] * Phi;
          y[e] = dv[e] * fmaf(hv[e] * 0.39894228040143267794f, ex, Phi);
        }
      } else {
#pragma unroll
        for (int e = 0; e < 8; ++e) y[e] = hv[e];
      }
    }
    if (CS) {
      // per-group sums (expert bias gradients): rows of one 128-row tile share a group; flush when it changes
      const int g = (a.tile_group && r < live) ? __ldg(a.tile_group + (int)(r >> 7)) : 0;
      if (g != cur_group) {
        if (cur_group >= 0 && col_ok) {
#pragma unroll
          for (int e = 0; e < 8; ++e) if (cs[e] != 0.f) atomicAdd(a.colsum + (long long)cur_group * a.W + col + e, cs[e]);
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) cs[e] = 0.f;
        cur_group = g;
      }
      if (row_ok) {
#pragma unroll
        for (int e = 0; e < 8; ++e) cs[e] += y[e];
      }
    }
    if (!col_ok) continue;
    if (a.out_f32 && r < a.R) {
      *reinterpret_cast<float4*>(a.out_f32 + r * a.W + col) = make_float4(y[0], y[1], y[2], y[3]);
      *reinterpret_cast<float4*>(a.out_f32 + r * a.W + col + 4) = make_float4(y[4], y[5], y[6], y[7]);
    }
    uint4 hi, lo;
    split8(y, hi, lo);
    if (a.pack_k) {           // K-major image, 128-row tiles: chunk (row r, k = col .. col+7)
      const long long rt = r >> 7; const uint32_t rr = (uint32_t)(r & 127);
      const int kb = chunk >> 2; const uint32_t c = (uint32_t)chunk & 3u;
      uint8_t* img = reinterpret_cast<uint8_t*>(a.pack_k) + (rt * kblocks_k + kb) * 16384LL;
      const uint32_t o = gemm::kmajor_sw64_offset(rr, c);
      *reinterpret_cast<uint4*>(img + o) = hi;
      *reinterpret_cast<uint4*>(img + 8192 + o) = lo;
    }
    if (a.pack_mn) {          // MN-major image (reduction index = row): chunk (k = r, mn = col .. col+7)
      const int mt = col / a.mn_tile; const uint32_t mc = (uint32_t)((col % a.mn_tile) >> 3);
      uint8_t* img = reinterpret_cast<uint8_t*>(a.pack_mn) + ((long long)mt * kblocks_mn + (r >> 5)) * (2LL * pb_mn);
      const uint32_t o = gemm::mnmajor_sw128_offset((uint32_t)(r & 31), mc);
      *reinterpret_cast<uint4*>(img + o) = hi;
      *reinterpret_cast<uint4*>(img + pb_mn + o) = lo;
    }
    if (MODE == 3) {          // second MN-major image: gelu(h), tile width mn_tile2
      uint4 hi2, lo2;
      split8(y2, hi2, lo2);
      const uint32_t pb2 = gemm::plane_bytes(a.mn_tile2, true);
      const int mt = col / a.mn_tile2; const uint32_t mc = (uint32_t)((col % a.mn_tile2) >> 3);
      uint8_t* img = reinterpret_cast<uint8_t*>(a.pack_mn2) + ((long long)mt * kblocks_mn + (r >> 5)) * (2LL * pb2);
      const uint32_t o = gemm::mnmajor_sw128_offset((uint32_t)(r & 31), mc);
      *reinterpret_cast<uint4*>(img + o) = hi2;
      *reinterpret_cast<uint4*>(img + pb2 + o) = lo2;
    }
  }
  if (CS) {
    // combine the 8 row lanes of the block (same group at the end of the band in all but pathological cases:
    // each lane flushes its own group, so correctness does not depend on it)
    if (cur_group >= 0 && col_ok) {
      if (a.tile_group) {
#pragma unroll
        for (int e = 0; e < 8; ++e) if (cs[e] != 0.f) atomicAdd(a.colsum + (long long)cur_group * a.W + col + e, cs[e]);
      } else {
#pragma unroll
        for (int e = 0; e < 8; ++e) s_cs[rlane][cl * 8 + e] = cs[e];
      }
    }
    if (!a.tile_group) {
      __syncthreads();
      if (rlane == 0 && col_ok) {
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          float t = 0.f;
#pragma unroll
          for (int w = 0; w < RL; ++w) t += s_cs[w][cl * 8 + e];
          atomicAdd(a.colsum + col + e, t);
        }
      }
    }
  }
}

int act_pack(const ActPackArgs& a, cudaStream_t stream) {
  SM3_REQUIRE(a.h && a.R > 0 && a.W > 0 && a.W % 8 == 0, SM3_ERR_INVALID_ARG, "act_pack: bad argument (W must be a multiple of 8)");
  SM3_REQUIRE(a.mode >= 0 && a.mode <= 3 && ((a.mode != 1 && a.mode != 3) || a.da), SM3_ERR_INVALID_ARG, "act_pack: mode/da");
  SM3_REQUIRE(a.mode != 3 || (a.pack_mn2 && a.mn_tile2 >= 32 && a.mn_tile2 <= 256 && a.mn_tile2 % 32 == 0), SM3_ERR_INVALID_ARG,
              "act_pack: mode 3 needs pack_mn2 / mn_tile2");
  SM3_REQUIRE(!a.pack_mn || (a.mn_tile >= 32 && a.mn_tile <= 256 && a.mn_tile % 32 == 0), SM3_ERR_INVALID_ARG, "act_pack: mn_tile");
  SM3_REQUIRE(a.pack_k || a.pack_mn || a.out_f32 || a.colsum, SM3_ERR_INVALID_ARG, "act_pack: no output requested");
  const long long R_pad = (a.R + 31) / 32 * 32;
  const int chunks_w = a.W / 8;
  const int clw = (chunks_w % 32 != 0 && chunks_w % 16 == 0) ? 16 : 32;
  const int gx = (chunks_w + clw - 1) / clw;
  long long bands = (long long)num_sms() * 8 / gx;
  if (bands < 1) bands = 1;
  long long rpb = (R_pad + bands - 1) / bands;
  rpb = (rpb + 127) / 128 * 128;                   // whole tiles per band keeps a band inside few groups
  bands = (R_pad + rpb - 1) / rpb;
  dim3 grid((unsigned)gx, (unsigned)bands);
  const bool cs = a.colsum != nullptr;
#define SM3_ACT_LAUNCH2(M, C_, W_) act_pack_kernel<M, C_, W_><<<grid, 256, 0, stream>>>(a, (int)rpb)
#define SM3_ACT_LAUNCH(M)                                                          \
  do {                                                                             \
    if (clw == 16) { if (cs) SM3_ACT_LAUNCH2(M, true, 16); else SM3_ACT_LAUNCH2(M, false, 16); }   \
    else { if (cs) SM3_ACT_LAUNCH2(M, true, 32); else SM3_ACT_LAUNCH2(M, false, 32); }             \
  } while (0)
  if (a.mode == 0) SM3_ACT_LAUNCH(0);
  else if (a.mode == 1) SM3_ACT_LAUNCH(1);
  else if (a.mode == 3) SM3_ACT_LAUNCH(3);
  else SM3_ACT_LAUNCH(2);
#undef SM3_ACT_LAUNCH2
#undef SM3_ACT_LAUNCH
  return check_launch("act_pack_kernel");
}

}  // namespace sm3
