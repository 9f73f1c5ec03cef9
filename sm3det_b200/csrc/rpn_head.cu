// OrientedRPNHead (mmrotate/models/dense_heads/oriented_rpn_head.py:18-24, rotated_rpn_head.py:43-49) on sm_90a:
//   rpn_conv (3x3, C_in -> 256, pad 1) -> ReLU -> rpn_cls (1x1, 256 -> ncls) and rpn_reg (1x1, 256 -> nreg), every level.
//
// rpn_conv_kernel<NHWC=false, HEAD=true> is the forward: an implicit-GEMM 3x3 conv (K = 9 taps x C_in, no im2col buffer:
// the operand rows are gathered per tap straight from the NCHW level maps, zero outside the map) whose 128 x 256 output
// tile gets bias + ReLU, is split into the bf16 hi/lo K-major image of a second wgmma GEMM in shared memory and multiplied
// there by the concatenated [rpn_cls; rpn_reg] weight; the epilogue writes cls / reg in NCHW.  Every pyramid level runs in
// the same launch: the level table is a __grid_constant__ parameter and each level owns a contiguous range of 128-row
// tiles.  rpn_conv_kernel<NHWC=true, HEAD=false> is the same main loop on the row-major gradient dpre [rows, 256] with the
// weight flipped 180 degrees and in/out-transposed (the caller packs it): dx, stored NCHW.  rpn_mid_bwd_kernel is the
// backward of the two 1x1 heads and the ReLU (fp32 FMAs, fixed order); rpn_tap_index_kernel writes the row gathers the
// per-tap weight-gradient GEMMs (sm3_gemm split-K) read.
//
// Row space: level l owns tiles [tile0_l, tile0_l + ceil(N H W / 128)) and rows [128 tile0_l, ...); position (n, y, x) of
// the level is row 128 tile0_l + (n H + y) W + x.  The saved ReLU output h, dpre and the NHWC copy of the input all use it.
#define SM3_GEMM_KERNEL_IMPL
#include "gemm_tc.cuh"
#include "kernels.h"

namespace sm3 {
namespace rpn {
using namespace gemm;

constexpr int THREADS = 256;                 // two consumer warpgroups; every thread also loads operands
constexpr int HID = 256;                     // feat_channels: one tile holds the whole hidden row
constexpr int NHP = 32;                      // head rows (ncls + nreg) padded to one wgmma N
constexpr int NSTAGE = 3;
constexpr uint32_t ST_A = 16384;             // A hi | lo planes, 128 rows x 32 k each
constexpr uint32_t ST_B = 32768;             // B hi | lo planes, 256 rows x 32 k each (pack_b image of one k-block, tile 256)
constexpr uint32_t STAGE = ST_A + ST_B;
constexpr uint32_t OFF_HID = 0;              // hidden image (8 k-blocks x 16 KB) reuses the stages once GEMM-a is done
constexpr uint32_t OFF_HEAD = NSTAGE * STAGE;
constexpr uint32_t HEAD_BYTES = (HID / 32) * NHP * 128;
constexpr uint32_t SMEM_FWD = OFF_HEAD + HEAD_BYTES + 1024;
constexpr uint32_t SMEM_DX = NSTAGE * STAGE + 1024;
static_assert(8 * 16384 <= NSTAGE * STAGE, "hidden image must fit in the stage ring");

struct Level {
  const float* in;   // NCHW level map (forward) or the dpre row buffer (dx)
  float* out0;       // cls (forward) / dx (dx)
  float* out1;       // reg (forward)
  int N, H, W, tile0;
};
struct Params {
  Level lv[SM3_RPN_MAX_LEVELS];
  int L, tiles;
  int Cg;              // gathered channels: K = 9 Cg, tap-major (k = tap * Cg + c)
  int Nout;            // stored GEMM-a columns (dx: C_in)
  const uint16_t* wimg;   // GEMM-a weight, pack_b image with tile 256: [k-block]{hi[256 x 32] | lo[256 x 32]}
  const float* bconv;
  const uint16_t* himg;   // [rpn_cls; rpn_reg] padded to 32 rows, pack_b image with tile 32
  const float* bhead;
  int ncls, nreg;
  float* h_out;        // ReLU output [rows, 256] for the backward (null in eval / no_grad)
  int passes;
};

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

__device__ __forceinline__ Level pick_level(const Params& p, int t) {
  Level lv = p.lv[0];
#pragma unroll
  for (int i = 1; i < SM3_RPN_MAX_LEVELS; ++i)
    if (i < p.L && t >= p.lv[i].tile0) lv = p.lv[i];
  return lv;
}

template <int N, bool A_MN>
__device__ __forceinline__ void mma_k16(float (&d)[N / 2], uint64_t ahi, uint64_t alo, uint64_t bhi, uint64_t blo,
                                        uint32_t accum, int passes) {
  if (passes == 1) {
    wg::mma<N, A_MN, 0>(d, ahi, bhi, accum);
  } else {
    wg::mma<N, A_MN, 0>(d, alo, bhi, accum);
    wg::mma<N, A_MN, 0>(d, ahi, blo, 1u);
    wg::mma<N, A_MN, 0>(d, ahi, bhi, 1u);
  }
}

template <bool NHWC, bool HEAD>
__global__ void __launch_bounds__(THREADS, 1) rpn_conv_kernel(const __grid_constant__ Params p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sb0 = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = warp >> 2, wq = warp & 3, rl = lane >> 2;
  const int kbc = p.Cg / 32, nkb = 9 * kbc;
  const uint8_t* wimg = reinterpret_cast<const uint8_t*>(p.wimg);

  if (HEAD) {   // the head weight image stays resident for all of the CTA's tiles
    for (int i = tid; i < (int)(HEAD_BYTES / 16); i += THREADS)
      cp_async16(sb0 + OFF_HEAD + 16u * i, reinterpret_cast<const uint8_t*>(p.himg) + 16 * i);
    cp_async_commit();
  }

  float acc[HID / 2];
  for (int t = blockIdx.x; t < p.tiles; t += gridDim.x) {
    const Level lv = pick_level(p, t);
    const int HW = lv.H * lv.W, M = lv.N * HW;
    const int m0 = (t - lv.tile0) * 128;           // first position of the tile inside its level

    // ---- per-thread gather rows.  NCHW (MN-major A): 8 consecutive positions 8*(tid&15)..+7, k-rows tid>>4 and +16.
    // NHWC (K-major A): rows (tid>>2) and +64, 8-channel chunk tid&3.
    constexpr int NP = NHWC ? 2 : 8;
    int off[NP], ph[NP], pw[NP];
#pragma unroll
    for (int j = 0; j < NP; ++j) {
      const int r = NHWC ? (tid >> 2) + 64 * j : 8 * (tid & 15) + j;
      const int pos = m0 + r;
      ph[j] = -0x40000000; pw[j] = 0; off[j] = 0;
      if (pos < M) {
        const int n = pos / HW, hw = pos - n * HW;
        ph[j] = hw / lv.W; pw[j] = hw - ph[j] * lv.W;
        off[j] = NHWC ? lv.tile0 * 128 + n * HW : n * p.Cg * HW + hw;
      }
    }
    float4 ra[4];   // this thread's share of one A k-block: 16 values
    auto load_a = [&](int kb) {
      const int tap = kb / kbc, c0 = (kb - tap * kbc) * 32;
      const int dy = tap / 3 - 1, dx = tap % 3 - 1;
      if (NHWC) {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int y = ph[j] + dy, x = pw[j] + dx;
          ra[2 * j] = ra[2 * j + 1] = make_float4(0.f, 0.f, 0.f, 0.f);
          if ((unsigned)y < (unsigned)lv.H && (unsigned)x < (unsigned)lv.W) {
            const float* src = lv.in + (long long)(off[j] + y * lv.W + x) * p.Cg + c0 + 8 * (tid & 3);
            ra[2 * j] = ldg_f4(src); ra[2 * j + 1] = ldg_f4(src + 4);
          }
        }
      } else {
        const int sh = dy * lv.W + dx;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const float* base = lv.in + (long long)(c0 + (tid >> 4) + 16 * i) * HW + sh;
          float v[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int y = ph[j] + dy, x = pw[j] + dx;
            v[j] = ((unsigned)y < (unsigned)lv.H && (unsigned)x < (unsigned)lv.W) ? __ldg(base + off[j]) : 0.f;
          }
          ra[2 * i] = make_float4(v[0], v[1], v[2], v[3]);
          ra[2 * i + 1] = make_float4(v[4], v[5], v[6], v[7]);
        }
      }
    };
    auto store_a = [&](int s) {
      const uint32_t st = sb0 + s * STAGE;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        uint4 hi, lo;
        split4(ra[2 * i], hi.x, hi.y, lo.x, lo.y);
        split4(ra[2 * i + 1], hi.z, hi.w, lo.z, lo.w);
        const uint32_t o = NHWC ? kmajor_sw64_offset((uint32_t)((tid >> 2) + 64 * i), (uint32_t)(tid & 3))
                                : mnmajor_sw128_offset((uint32_t)((tid >> 4) + 16 * i), (uint32_t)(tid & 15));
        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(st + o), "r"(hi.x), "r"(hi.y), "r"(hi.z), "r"(hi.w) : "memory");
        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(st + 8192u + o), "r"(lo.x), "r"(lo.y), "r"(lo.z), "r"(lo.w) : "memory");
      }
    };
    auto issue_b = [&](int kb, int s) {
      const uint8_t* src = wimg + (long long)kb * ST_B;
#pragma unroll
      for (int j = 0; j < (int)(ST_B / 16 / THREADS); ++j)
        cp_async16(sb0 + s * STAGE + ST_A + 16u * (tid + THREADS * j), src + 16 * (tid + THREADS * j));
      cp_async_commit();
    };

    // ---- GEMM-a: 3-stage ring, one barrier per k-block.  Stage (kb+1)%3 is refilled while MMA(kb) runs: its last reader,
    // MMA(kb-2), was waited for (wait<1> of iteration kb-1) by every thread before the barrier of iteration kb.
    issue_b(0, 0);
    load_a(0);
    store_a(0);
    cp_async_wait_all();
    fence_proxy_async_smem();
    int s = 0;
    for (int kb = 0; kb < nkb; ++kb) {
      __syncthreads();
      wg::fence();
      const uint32_t st = sb0 + s * STAGE;
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const uint32_t a = st + (uint32_t)g * WG_A_BYTES + j * (NHWC ? 32u : 2u * MN_SBO_BYTES);
        mma_k16<HID, !NHWC>(acc, make_smem_desc(a, !NHWC), make_smem_desc(a + 8192u, !NHWC), make_smem_desc(st + ST_A + 32u * j, false),
                            make_smem_desc(st + ST_A + 16384u + 32u * j, false), (kb > 0 || j > 0) ? 1u : 0u, p.passes);
      }
      wg::commit();
      const int s1 = s == NSTAGE - 1 ? 0 : s + 1;
      if (kb + 1 < nkb) { issue_b(kb + 1, s1); load_a(kb + 1); }
      wg::wait<1>();
      if (kb + 1 < nkb) { store_a(s1); cp_async_wait_all(); fence_proxy_async_smem(); }
      s = s1;
    }
    wg::wait<0>();
    wg::fence_operand(acc);
    __syncthreads();                                  // every warpgroup is done with the stages

    const int r_lo = g * 64 + wq * 16 + rl;           // tile rows of this thread's fragment: r_lo, r_lo + 8
    int on[2], ohw[2];
    bool ok[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int pos = m0 + r_lo + 8 * h;
      ok[h] = pos < M;
      on[h] = ok[h] ? pos / HW : 0;
      ohw[h] = pos - on[h] * HW;
    }
    if constexpr (!HEAD) {
      // dx: plain NCHW store of the first Nout columns
#pragma unroll
      for (int q = 0; q < HID / 8; ++q)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = 8 * q + 2 * (lane & 3) + e;
          if (col >= p.Nout) continue;
#pragma unroll
          for (int h = 0; h < 2; ++h)
            if (ok[h]) lv.out0[((long long)on[h] * p.Nout + col) * HW + ohw[h]] = acc[4 * q + 2 * h + e];
        }
    } else {
    // ---- middle stage: h = relu(acc + b), saved for the backward when asked, split into GEMM-b's K-major A image
#pragma unroll
    for (int q = 0; q < HID / 8; ++q) {
      const int col = 8 * q + 2 * (lane & 3);
      const float2 bv = __ldg(reinterpret_cast<const float2*>(p.bconv + col));
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = r_lo + 8 * h;
        const float x0 = fmaxf(acc[4 * q + 2 * h] + bv.x, 0.f), x1 = fmaxf(acc[4 * q + 2 * h + 1] + bv.y, 0.f);
        if (p.h_out && ok[h]) *reinterpret_cast<float2*>(p.h_out + ((long long)t * 128 + r) * HID + col) = make_float2(x0, x1);
        const uint32_t u0 = __float_as_uint(x0), u1 = __float_as_uint(x1);
        const uint32_t hi = __byte_perm(u0, u1, 0x7632);
        const uint32_t lo = __byte_perm(__float_as_uint(x0 - __uint_as_float(u0 & 0xFFFF0000u)) + 0x8000u,
                                        __float_as_uint(x1 - __uint_as_float(u1 & 0xFFFF0000u)) + 0x8000u, 0x7632);
        const uint32_t o = sb0 + OFF_HID + (uint32_t)(col >> 5) * 16384u + kmajor_sw64_offset((uint32_t)r, (uint32_t)((col & 31) >> 3)) +
                           (uint32_t)(col & 7) * 2u;
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(o), "r"(hi) : "memory");
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(o + 8192u), "r"(lo) : "memory");
      }
    }
    fence_proxy_async_smem();
    asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory");   // this warpgroup's 64 hidden rows are complete

    // ---- GEMM-b: [cls | reg] = h . [Wc; Wr]^T over K = 256, on chip
    float acc2[NHP / 2];
    wg::fence();
#pragma unroll
    for (int kb = 0; kb < HID / 32; ++kb)
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const uint32_t a = sb0 + OFF_HID + kb * 16384u + (uint32_t)g * WG_A_BYTES + 32u * j;
        const uint32_t b = sb0 + OFF_HEAD + kb * (NHP * 128u) + 32u * j;
        mma_k16<NHP, false>(acc2, make_smem_desc(a, false), make_smem_desc(a + 8192u, false), make_smem_desc(b, false),
                            make_smem_desc(b + NHP * 64u, false), (kb > 0 || j > 0) ? 1u : 0u, p.passes);
      }
    wg::commit();
    wg::wait<0>();
    wg::fence_operand(acc2);
    const int nh = p.ncls + p.nreg;
#pragma unroll
    for (int q = 0; q < NHP / 8; ++q)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = 8 * q + 2 * (lane & 3) + e;
        if (col >= nh) continue;
        const float b = __ldg(p.bhead + col);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (!ok[h]) continue;
          const float v = acc2[4 * q + 2 * h + e] + b;
          if (col < p.ncls) lv.out0[((long long)on[h] * p.ncls + col) * HW + ohw[h]] = v;
          else lv.out1[((long long)on[h] * p.nreg + (col - p.ncls)) * HW + ohw[h]] = v;
        }
      }
    __syncthreads();                                  // the hidden image is read by GEMM-b before the next tile's stages
    }
  }
}

// ---- backward of the heads and the ReLU --------------------------------------------------------------------------------
// Thread j owns hidden column j: dpre[row, j] = (sum_o dout[row, o] Wh[o, j]) * [h[row, j] > 0], written for every row of
// the row space (0 on the padding rows), summed in a fixed order; the weight / bias gradients are per-CTA partials added
// with one atomic per element at the end.
struct MidParams {
  Level lv[SM3_RPN_MAX_LEVELS];   // in = unused, out0 = dcls, out1 = dreg (read)
  int L, tiles;
  const float* h; const float* whead; int ncls, nreg;
  float* dpre; float* dwhead; float* dbhead; float* dbconv;
};

__device__ __forceinline__ Level pick_level_mid(const MidParams& p, int t) {
  Level lv = p.lv[0];
#pragma unroll
  for (int i = 1; i < SM3_RPN_MAX_LEVELS; ++i)
    if (i < p.L && t >= p.lv[i].tile0) lv = p.lv[i];
  return lv;
}

__global__ void __launch_bounds__(256, 1) rpn_mid_bwd_kernel(const __grid_constant__ MidParams p) {
  __shared__ float sd[NHP][129];
  const int j = threadIdx.x;
  const int nh = p.ncls + p.nreg;
  float w[NHP], dw[NHP];
#pragma unroll
  for (int o = 0; o < NHP; ++o) { w[o] = o < nh ? __ldg(p.whead + o * HID + j) : 0.f; dw[o] = 0.f; }
  float dbc = 0.f, dbh = 0.f;
  for (int t = blockIdx.x; t < p.tiles; t += gridDim.x) {
    const Level lv = pick_level_mid(p, t);
    const int HW = lv.H * lv.W, M = lv.N * HW, m0 = (t - lv.tile0) * 128;
    __syncthreads();
    for (int i = j; i < NHP * 128; i += 256) {
      const int o = i >> 7, r = i & 127, pos = m0 + r;
      float v = 0.f;
      if (pos < M && o < nh) {
        const int n = pos / HW, hw = pos - n * HW;
        v = o < p.ncls ? __ldg(lv.out0 + ((long long)n * p.ncls + o) * HW + hw)
                       : __ldg(lv.out1 + ((long long)n * p.nreg + (o - p.ncls)) * HW + hw);
      }
      sd[o][r] = v;
    }
    __syncthreads();
    const int rows = min(128, M - m0);
    for (int r = 0; r < 128; ++r) {
      const long long row = (long long)t * 128 + r;
      float dp = 0.f;
      if (r < rows) {
        const float hv = __ldg(p.h + row * HID + j);
        float d = 0.f;
#pragma unroll
        for (int o = 0; o < NHP; ++o) {
          const float g = sd[o][r];
          d = fmaf(g, w[o], d);
          dw[o] = fmaf(g, hv, dw[o]);
        }
        dp = hv > 0.f ? d : 0.f;
      }
      p.dpre[row * HID + j] = dp;
      dbc += dp;
    }
    if (j < nh)
      for (int r = 0; r < rows; ++r) dbh += sd[j][r];
  }
#pragma unroll
  for (int o = 0; o < NHP; ++o)
    if (o < nh) atomicAdd(p.dwhead + o * HID + j, dw[o]);
  atomicAdd(p.dbconv + j, dbc);
  if (j < nh) atomicAdd(p.dbhead + j, dbh);
}

// idx[tap][row] = row of the neighbour (y + ky - 1, x + kx - 1) of row's position, -1 outside the map or on padding rows
__global__ void __launch_bounds__(256) rpn_tap_index_kernel(const __grid_constant__ MidParams p, int* __restrict__ idx, long long R) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 9 * R) return;
  const int tap = (int)(i / R);
  const long long row = i - (long long)tap * R;
  const Level lv = pick_level_mid(p, (int)(row >> 7));
  const int HW = lv.H * lv.W, M = lv.N * HW;
  const long long pos = row - 128LL * lv.tile0;
  int v = -1;
  if (pos < M) {
    const int n = (int)(pos / HW), hw = (int)(pos - (long long)n * HW);
    const int y = hw / lv.W + tap / 3 - 1, x = hw % lv.W + tap % 3 - 1;
    if ((unsigned)y < (unsigned)lv.H && (unsigned)x < (unsigned)lv.W) v = lv.tile0 * 128 + n * HW + y * lv.W + x;
  }
  idx[i] = v;
}

// ---- host side ---------------------------------------------------------------------------------------------------------
// shapes: host [L][3] = (N, H, W).  Fills tile0 / N / H / W, returns the number of 128-row tiles (< 0: error).
static int level_table(const int* shapes, int L, int C, Level* lv, const char* what) {
  SM3_REQUIRE(shapes && L >= 1 && L <= SM3_RPN_MAX_LEVELS, SM3_ERR_INVALID_ARG, "%s: 1 <= levels <= %d, got %d", what,
              SM3_RPN_MAX_LEVELS, L);
  long long tiles = 0;
  for (int l = 0; l < L; ++l) {
    const int N = shapes[3 * l], H = shapes[3 * l + 1], W = shapes[3 * l + 2];
    SM3_REQUIRE(N >= 1 && H >= 1 && W >= 1, SM3_ERR_INVALID_ARG, "%s: level %d has shape N=%d H=%d W=%d", what, l, N, H, W);
    SM3_REQUIRE((long long)N * H * W * (C > HID ? C : HID) < (1LL << 31), SM3_ERR_UNSUPPORTED_SHAPE,
                "%s: level %d too large (N=%d H=%d W=%d)", what, l, N, H, W);
    lv[l].N = N; lv[l].H = H; lv[l].W = W; lv[l].tile0 = (int)tiles;
    tiles += ((long long)N * H * W + 127) / 128;
  }
  SM3_REQUIRE(tiles * 128 < (1LL << 31), SM3_ERR_UNSUPPORTED_SHAPE, "%s: too many positions", what);
  return (int)tiles;
}

long long rows(const int* shapes, int L) {
  Level lv[SM3_RPN_MAX_LEVELS];
  const int t = level_table(shapes, L, 0, lv, "rpn_head_rows");
  return t < 0 ? t : 128LL * t;
}

static bool aligned16(const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15u) == 0; }

int conv_fwd(const float* const* x, float* const* cls, float* const* reg, const int* shapes, int L, int Cin,
             const uint16_t* wimg, const float* bconv, const uint16_t* himg, const float* bhead, int ncls, int nreg,
             float* h_out, int passes, cudaStream_t stream) {
  Params p{};
  const int tiles = level_table(shapes, L, Cin, p.lv, "rpn_head_fwd");
  if (tiles < 0) return tiles;
  SM3_REQUIRE(Cin % 32 == 0 && Cin >= 32 && Cin <= 256, SM3_ERR_UNSUPPORTED_SHAPE,
              "rpn_head_fwd: in_channels must be a multiple of 32 in [32, 256], got %d", Cin);
  SM3_REQUIRE(ncls >= 1 && nreg >= 1 && ncls + nreg <= NHP, SM3_ERR_UNSUPPORTED_SHAPE,
              "rpn_head_fwd: combined head width must be <= %d (cls %d + reg %d)", NHP, ncls, nreg);
  SM3_REQUIRE(x && cls && reg && wimg && bconv && himg && bhead, SM3_ERR_INVALID_ARG, "rpn_head_fwd: null pointer");
  SM3_REQUIRE(aligned16(wimg) && aligned16(himg) && (reinterpret_cast<uintptr_t>(bconv) & 7u) == 0 && (!h_out || aligned16(h_out)),
              SM3_ERR_INVALID_ARG, "rpn_head_fwd: weight images / h_out must be 16-byte aligned, bconv 8-byte aligned");
  for (int l = 0; l < L; ++l) {
    SM3_REQUIRE(x[l] && cls[l] && reg[l], SM3_ERR_INVALID_ARG, "rpn_head_fwd: level %d has a null pointer", l);
    p.lv[l].in = x[l]; p.lv[l].out0 = cls[l]; p.lv[l].out1 = reg[l];
  }
  p.L = L; p.tiles = tiles; p.Cg = Cin; p.Nout = HID;
  p.wimg = wimg; p.bconv = bconv; p.himg = himg; p.bhead = bhead; p.ncls = ncls; p.nreg = nreg; p.h_out = h_out;
  p.passes = passes == 1 ? 1 : 3;
  int grid = persistent_grid_sms();
  if (grid > tiles) grid = tiles;
  cudaFuncSetAttribute(rpn_conv_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_FWD);
  rpn_conv_kernel<false, true><<<grid, THREADS, SMEM_FWD, stream>>>(p);
  return check_launch("rpn_conv_kernel<fwd>");
}

int conv_dx(const float* dpre, float* const* dx, const int* shapes, int L, int Cin, const uint16_t* wimg, int passes,
            cudaStream_t stream) {
  Params p{};
  const int tiles = level_table(shapes, L, Cin, p.lv, "rpn_head_dx");
  if (tiles < 0) return tiles;
  SM3_REQUIRE(Cin % 32 == 0 && Cin >= 32 && Cin <= 256, SM3_ERR_UNSUPPORTED_SHAPE,
              "rpn_head_dx: in_channels must be a multiple of 32 in [32, 256], got %d", Cin);
  SM3_REQUIRE(dpre && dx && wimg && aligned16(dpre) && aligned16(wimg), SM3_ERR_INVALID_ARG,
              "rpn_head_dx: null or misaligned pointer");
  for (int l = 0; l < L; ++l) {
    SM3_REQUIRE(dx[l], SM3_ERR_INVALID_ARG, "rpn_head_dx: level %d has a null pointer", l);
    p.lv[l].in = dpre; p.lv[l].out0 = dx[l];
  }
  p.L = L; p.tiles = tiles; p.Cg = HID; p.Nout = Cin; p.wimg = wimg;
  p.passes = passes == 1 ? 1 : 3;
  int grid = persistent_grid_sms();
  if (grid > tiles) grid = tiles;
  cudaFuncSetAttribute(rpn_conv_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_DX);
  rpn_conv_kernel<true, false><<<grid, THREADS, SMEM_DX, stream>>>(p);
  return check_launch("rpn_conv_kernel<dx>");
}

int mid_bwd(const float* h, const float* const* dcls, const float* const* dreg, const int* shapes, int L, const float* whead,
            int ncls, int nreg, float* dpre, float* dwhead, float* dbhead, float* dbconv, cudaStream_t stream) {
  MidParams p{};
  const int tiles = level_table(shapes, L, 0, p.lv, "rpn_head_mid_bwd");
  if (tiles < 0) return tiles;
  SM3_REQUIRE(ncls >= 1 && nreg >= 1 && ncls + nreg <= NHP, SM3_ERR_UNSUPPORTED_SHAPE,
              "rpn_head_mid_bwd: combined head width must be <= %d (cls %d + reg %d)", NHP, ncls, nreg);
  SM3_REQUIRE(h && dcls && dreg && whead && dpre && dwhead && dbhead && dbconv, SM3_ERR_INVALID_ARG, "rpn_head_mid_bwd: null pointer");
  for (int l = 0; l < L; ++l) {
    SM3_REQUIRE(dcls[l] && dreg[l], SM3_ERR_INVALID_ARG, "rpn_head_mid_bwd: level %d has a null pointer", l);
    p.lv[l].out0 = const_cast<float*>(dcls[l]); p.lv[l].out1 = const_cast<float*>(dreg[l]);
  }
  p.L = L; p.tiles = tiles; p.h = h; p.whead = whead; p.ncls = ncls; p.nreg = nreg;
  p.dpre = dpre; p.dwhead = dwhead; p.dbhead = dbhead; p.dbconv = dbconv;
  int grid = 2 * num_sms();
  if (grid > tiles) grid = tiles;
  rpn_mid_bwd_kernel<<<grid, 256, 0, stream>>>(p);
  return check_launch("rpn_mid_bwd_kernel");
}

int tap_index(const int* shapes, int L, int* idx, cudaStream_t stream) {
  MidParams p{};
  const int tiles = level_table(shapes, L, 0, p.lv, "rpn_head_tap_index");
  if (tiles < 0) return tiles;
  SM3_REQUIRE(idx, SM3_ERR_INVALID_ARG, "rpn_head_tap_index: null pointer");
  p.L = L; p.tiles = tiles;
  const long long R = 128LL * tiles;
  rpn_tap_index_kernel<<<(unsigned)((9 * R + 255) / 256), 256, 0, stream>>>(p, idx, R);
  return check_launch("rpn_tap_index_kernel");
}

}  // namespace rpn
}  // namespace sm3
