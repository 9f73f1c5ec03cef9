// Fused dense-FFN kernels (see ffn_fused.cuh for the what and why).  sm_90a only: wgmma.mma_async with register
// accumulators, cp.async.bulk (TMA bulk copies) completing on mbarriers, one persistent CTA per SM.
#define SM3_GEMM_KERNEL_IMPL
#include "gemm_tc.cuh"
#include "ffn_fused.cuh"
#include "kernels.h"

namespace sm3 {
namespace ffn {
using namespace gemm;

// 12 warps: 0 A/Wa producer, 1 Wb producer, 2-3 idle; 4-7 and 8-11 are the two consumer warpgroups, each owning 64 of
// the tile's 128 token rows through GEMM-a, the middle stage, GEMM-b and the final epilogue.
constexpr int THREADS = 384;
constexpr int W_PROD_A = 0, W_PROD_B = 1, EPI0 = 4, NE = 8;
constexpr int CONS_REGS = 232, PROD_REGS = 40;         // setmaxnreg: acc_o alone is up to 128 registers (C = 256)
constexpr uint32_t SMEM_LIMIT = 232448u - 1024u;      // 227 KB opt-in maximum minus the 1 KB alignment slack
constexpr uint32_t STAGING = NE * EPI_STAGE_BYTES;    // per-warp transpose staging of the final epilogue
constexpr uint32_t BARS = 256;

// shared-memory carve-up, computed on the host and passed by value
struct Layout {
  uint32_t a, ones, a2, wa, wb, act, act2, stage, cs, bar, total;
  uint32_t a_tile, wa_chunk, wa_stage, wb_stage, act_bytes;
  int sa, sb;
};

struct ChainK { ChainParams p; Layout L; int m_tiles, nch; };

__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void sts128(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}

// split 2 fp32 into one bf16x2 of the hi plane and one of the lo plane
__device__ __forceinline__ void split2(float v0, float v1, uint32_t& hi, uint32_t& lo) {
  const uint32_t u0 = __float_as_uint(v0), u1 = __float_as_uint(v1);
  hi = __byte_perm(u0, u1, 0x7632);
  const uint32_t r0 = __float_as_uint(v0 - __uint_as_float(u0 & 0xFFFF0000u)) + 0x8000u;
  const uint32_t r1 = __float_as_uint(v1 - __uint_as_float(u1 & 0xFFFF0000u)) + 0x8000u;
  lo = __byte_perm(r0, r1, 0x7632);
}

// 3-pass (or 1-pass) split-bf16 product of one 16-k step:  D (+)= (Ahi + Alo)(Bhi + Blo) minus the lo*lo term
template <int N, int NA>
__device__ __forceinline__ void mma3(float (&d)[NA], uint64_t ahi, uint64_t alo, uint64_t bhi, uint64_t blo, uint32_t accum,
                                     int passes) {
  if (passes == 1) {
    wg::mma<N, 0, 0>(d, ahi, bhi, accum);
  } else {
    wg::mma<N, 0, 0>(d, alo, bhi, accum);
    wg::mma<N, 0, 0>(d, ahi, blo, 1u);
    wg::mma<N, 0, 0>(d, ahi, bhi, 1u);
  }
}

// butterfly column reduction over the 8 row lanes of a quad column (lane bits 2-4).  In: v[4] = this lane's sums for the
// columns (qq, e) = (0,0), (0,1), (1,0), (1,1) of a 16-column group; out: the warp's sum of column 8*bit4 + 2*(lane&3) + bit3,
// complete in the lanes with bit2 == 0 (and their bit2 partners).  4 shuffles instead of 12.
__device__ __forceinline__ float colsum16(const float (&v)[4], int lane) {
  const bool b4 = lane & 16, b3 = lane & 8;
  const float k0 = b4 ? v[2] : v[0], k1 = b4 ? v[3] : v[1];
  const float s0 = b4 ? v[0] : v[2], s1 = b4 ? v[1] : v[3];
  const float u0 = k0 + __shfl_xor_sync(0xffffffffu, s0, 16), u1 = k1 + __shfl_xor_sync(0xffffffffu, s1, 16);
  const float w = (b3 ? u1 : u0) + __shfl_xor_sync(0xffffffffu, b3 ? u0 : u1, 8);
  return w + __shfl_xor_sync(0xffffffffu, w, 4);
}

// ================================================================================================================
template <int MODE, int HC, int C>
__global__ void __launch_bounds__(THREADS, 1) ffn_chain_kernel(const __grid_constant__ ChainK k) {
  const ChainParams& p = k.p;
  const Layout& L = k.L;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sb0 = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar = sb0 + L.bar;
  const uint32_t a_full = bar, a_empty = bar + 8;
  auto wa_full = [&](int s) { return bar + 16u + 8u * s; };
  auto wa_empty = [&](int s) { return bar + 32u + 8u * s; };
  auto wb_full = [&](int s) { return bar + 48u + 8u * s; };
  auto wb_empty = [&](int s) { return bar + 64u + 8u * s; };
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int NA = (MODE == 1 || MODE == 2) ? 2 : 1;
  constexpr bool WGRAD_IMG = MODE >= 2;          // modes 2 / 3 also emit the weight-gradient operand images and db1

  if (threadIdx.x == 0) {
    mbar_init(a_full, 1); mbar_init(a_empty, NE);
    for (int s = 0; s < 2; ++s) { mbar_init(wa_full(s), 1); mbar_init(wa_empty(s), NE); mbar_init(wb_full(s), 1); mbar_init(wb_empty(s), NE); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int nch = k.nch;
  constexpr int kbc = C / 32;

  if (warp < EPI0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(PROD_REGS));
    if (warp == W_PROD_A && lane == 0) {
      uint32_t n_t = 0, n_w = 0;
      for (int t = blockIdx.x; t < k.m_tiles; t += gridDim.x, ++n_t) {
        mbar_wait(a_empty, (n_t & 1u) ^ 1u);
        if ((p.debug & 8) && n_t > 0) { mbar_arrive(a_full); goto weights; }
        expect_tx(a_full, NA * L.a_tile);
        bulk_g2s(sb0 + L.a, reinterpret_cast<const uint8_t*>(MODE == 3 ? p.a2 : p.a1) + (long long)t * L.a_tile, L.a_tile, a_full);
        if (NA == 2) bulk_g2s(sb0 + L.a + L.a_tile, reinterpret_cast<const uint8_t*>(p.a2) + (long long)t * L.a_tile, L.a_tile, a_full);
      weights:
        for (int j = 0; j < nch; ++j, ++n_w) {
          const int s = n_w % L.sa;
          mbar_wait(wa_empty(s), ((n_w / L.sa) & 1u) ^ 1u);
          if ((p.debug & 4) && n_w >= (uint32_t)L.sa) { mbar_arrive(wa_full(s)); continue; }   // timing experiment: stale weights
          expect_tx(wa_full(s), L.wa_stage);
          const uint32_t dst = sb0 + L.wa + s * L.wa_stage;
          bulk_g2s(dst, reinterpret_cast<const uint8_t*>(MODE == 3 ? p.wa2 : p.wa1) + (long long)j * L.wa_chunk, L.wa_chunk, wa_full(s));
          if (NA == 2) bulk_g2s(dst + L.wa_chunk, reinterpret_cast<const uint8_t*>(p.wa2) + (long long)j * L.wa_chunk, L.wa_chunk, wa_full(s));
        }
      }
    } else if (warp == W_PROD_B && lane == 0) {
      uint32_t n = 0;
      for (int t = blockIdx.x; t < k.m_tiles; t += gridDim.x) {
        for (int j = 0; j < nch; ++j, ++n) {
          const int s = n % L.sb;
          mbar_wait(wb_empty(s), ((n / L.sb) & 1u) ^ 1u);
          if ((p.debug & 4) && n >= (uint32_t)L.sb) { mbar_arrive(wb_full(s)); continue; }
          expect_tx(wb_full(s), L.wb_stage);
          bulk_g2s(sb0 + L.wb + s * L.wb_stage, reinterpret_cast<const uint8_t*>(p.wb) + (long long)j * L.wb_stage, L.wb_stage, wb_full(s));
        }
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(CONS_REGS));
    // ------------------------------ consumers: GEMM-a, middle stage, GEMM-b, final epilogue -----------------------
    const int e = warp - EPI0, g = e >> 2, wq = warp & 3;
    const uint32_t slab = (uint32_t)g * WG_A_BYTES;              // this warpgroup's 64 rows inside a 128-row operand plane
    const uint32_t stage_base = sb0 + L.stage + (uint32_t)e * EPI_STAGE_BYTES;
    const int rl = lane >> 2, c4 = (lane & 3) * 4;
    const int r_lo = g * 64 + wq * 16 + rl;                      // tile rows of this thread's fragment: r_lo, r_lo + 8
    auto wg_bar = [&]() { asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory"); };
    float acc_h[HC / 2], acc_d[HC / 2], acc_o[C / 2];
    uint32_t n_c = 0, n_b = 0, n_t = 0;
    auto gemm_a = [&](uint32_t nc) {                              // acc_h (, acc_d) = A1 (, A2) . Wa_j^T over K = C
      const int s = nc % L.sa;
      mbar_wait(wa_full(s), (nc / L.sa) & 1u);
      const uint32_t wst = sb0 + L.wa + s * L.wa_stage;
#pragma unroll
      for (int q = 0; q < NA; ++q) {
        uint64_t da = make_smem_desc(sb0 + L.a + q * L.a_tile + slab, false), db = make_smem_desc(wst + q * L.wa_chunk, false);
        for (int kb = 0; kb < kbc; ++kb) {
          if (q == 0 && MODE != 3) {
            mma3<HC>(acc_h, da, da + 512u, db, db + HC * 4u, kb > 0 ? 1u : 0u, p.passes);
            mma3<HC>(acc_h, da + 2u, da + 514u, db + 2u, db + HC * 4u + 2u, 1u, p.passes);
          } else {
            mma3<HC>(acc_d, da, da + 512u, db, db + HC * 4u, kb > 0 ? 1u : 0u, p.passes);
            mma3<HC>(acc_d, da + 2u, da + 514u, db + 2u, db + HC * 4u + 2u, 1u, p.passes);
          }
          da += 1024u; db += HC * 8u;
        }
      }
    };
    const uint32_t cs_base = sb0 + L.cs;                         // modes 2 / 3: this CTA's db1 partials [H4]
    auto cons_bar = [&]() { asm volatile("bar.sync 3, 256;" ::: "memory"); };
    if constexpr (WGRAD_IMG) {
      for (int i = threadIdx.x - EPI0 * 32; i < p.H4; i += 256) asm volatile("st.shared.f32 [%0], %1;" ::"r"(cs_base + 4u * i), "f"(0.f) : "memory");
      cons_bar();
    }
    const long long R_pad = ((long long)p.M + 31) / 32 * 32;     // the MN-major images hold whole 32-row k-blocks
    for (int t = blockIdx.x; t < k.m_tiles; t += gridDim.x, ++n_t) {
      mbar_wait(a_full, n_t & 1u);
      wg::fence();
      gemm_a(n_c);
      wg::commit();
      for (int j = 0; j < nch; ++j, ++n_c) {
        if constexpr (MODE == 3) {
          // the saved pre-activation h (b1 included) straight into the fragment layout: a quad reads 32 contiguous bytes
#pragma unroll
          for (int q = 0; q < HC / 8; ++q)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const long long row = (long long)t * 128 + r_lo + 8 * h;
              const float2 x = row < p.M ? __ldg(reinterpret_cast<const float2*>(p.h_in + row * p.H4 + (long long)j * HC + 8 * q + 2 * (lane & 3)))
                                         : make_float2(0.f, 0.f);
              acc_h[4 * q + 2 * h] = x.x; acc_h[4 * q + 2 * h + 1] = x.y;
            }
        }
        // GEMM-a(j) and GEMM-b(j-1) are complete: hand their operand stages back
        wg::wait<0>();
        if constexpr (MODE != 3) wg::fence_operand(acc_h);
        if constexpr (MODE != 0) wg::fence_operand(acc_d);
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(wa_empty(n_c % L.sa));
          if (j > 0) mbar_arrive(wb_empty((n_b - 1) % L.sb));
          if (j == nch - 1) mbar_arrive(a_empty);
        }
        // middle: y = gelu(h) or dz-side * gelu'(h), split hi/lo into the K-major SWIZZLE_64B image of GEMM-b's A operand
        const float* b1 = p.bias1 + (long long)j * HC;
        if constexpr (WGRAD_IMG) {
          // dh = d * gelu'(h) -> GEMM-b's operand as in mode 1, and, through the warp's staging rows, dh and gelu(h) as
          // 16-byte chunks of the MN-major SWIZZLE_128B images of the two weight-gradient GEMMs (act_pack's layout);
          // db1 partials of dh per column into shared memory
          const long long wrow0 = (long long)t * 128 + g * 64 + wq * 16;
#pragma unroll
          for (int qp = 0; qp < HC / 16; ++qp) {
            float cs4[4];
#pragma unroll
            for (int qq = 0; qq < 2; ++qq) {
              const int q = 2 * qp + qq;
              const int kk = 8 * q + 2 * (lane & 3);
              const float2 bv = MODE == 3 ? make_float2(0.f, 0.f) : __ldg(reinterpret_cast<const float2*>(b1 + kk));   // mode 3: h holds b1
              cs4[2 * qq] = 0.f; cs4[2 * qq + 1] = 0.f;
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int r = r_lo + 8 * h;
                float y[2], a[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                  const float x = MODE == 3 ? acc_h[4 * q + 2 * h + e] : acc_h[4 * q + 2 * h + e] + (e ? bv.y : bv.x);
                  float Phi, ex;
                  phi_parts(x, Phi, ex);
                  a[e] = x * Phi;
                  y[e] = acc_d[4 * q + 2 * h + e] * fmaf(x * 0.39894228040143267794f, ex, Phi);
                }
                if (wrow0 + rl + 8 * h < p.M) { cs4[2 * qq] += y[0]; cs4[2 * qq + 1] += y[1]; }
                uint32_t hi, lo;
                split2(y[0], y[1], hi, lo);
                const uint32_t o = sb0 + L.act + (uint32_t)(kk >> 5) * 16384u + kmajor_sw64_offset((uint32_t)r, (uint32_t)((kk & 31) >> 3)) +
                                   (uint32_t)(kk & 7) * 2u;
                asm volatile("st.shared.b32 [%0], %1;" ::"r"(o), "r"(hi) : "memory");
                asm volatile("st.shared.b32 [%0], %1;" ::"r"(o + 8192u), "r"(lo) : "memory");
                const uint32_t so = stage_base + (uint32_t)((rl + 8 * h) * EPI_STAGE_ROW_FLOATS + 8 * qq + 2 * (lane & 3)) * 4u;
                asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(so), "f"(y[0]), "f"(y[1]) : "memory");
                asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(so + 16u * EPI_STAGE_ROW_FLOATS * 4u), "f"(a[0]), "f"(a[1]) : "memory");
              }
            }
            const float csum = colsum16(cs4, lane);
            const int col = j * HC + 16 * qp;                     // first hidden column of this 16-column group
            if ((lane & 4) == 0)
              asm volatile("red.shared.add.f32 [%0], %1;" ::"r"(cs_base + 4u * (uint32_t)(col + 8 * ((lane >> 4) & 1) + 2 * (lane & 3) + ((lane >> 3) & 1))),
                           "f"(csum) : "memory");
            __syncwarp();
            // lane -> token row wrow0 + lane/2, hidden columns col + 8*(lane&1) .. +7: one 16-byte chunk per image plane
            const int sr = lane >> 1, sc = 8 * (lane & 1);
            const long long row = wrow0 + sr;
            if (row < R_pad) {
              float dv8[8], av8[8];
              float4 x0, x1, z0, z1;
              const uint32_t ro = stage_base + (uint32_t)(sr * EPI_STAGE_ROW_FLOATS + sc) * 4u;
              asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(x0.x), "=f"(x0.y), "=f"(x0.z), "=f"(x0.w) : "r"(ro) : "memory");
              asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(x1.x), "=f"(x1.y), "=f"(x1.z), "=f"(x1.w) : "r"(ro + 16u) : "memory");
              asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(z0.x), "=f"(z0.y), "=f"(z0.z), "=f"(z0.w)
                           : "r"(ro + 16u * EPI_STAGE_ROW_FLOATS * 4u) : "memory");
              asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(z1.x), "=f"(z1.y), "=f"(z1.z), "=f"(z1.w)
                           : "r"(ro + 16u * EPI_STAGE_ROW_FLOATS * 4u + 16u) : "memory");
              const bool live = row < p.M;                        // rows M .. R_pad of both images are zero
              dv8[0] = x0.x; dv8[1] = x0.y; dv8[2] = x0.z; dv8[3] = x0.w; dv8[4] = x1.x; dv8[5] = x1.y; dv8[6] = x1.z; dv8[7] = x1.w;
              av8[0] = z0.x; av8[1] = z0.y; av8[2] = z0.z; av8[3] = z0.w; av8[4] = z1.x; av8[5] = z1.y; av8[6] = z1.z; av8[7] = z1.w;
              uint32_t dh_[4], dl_[4], ah_[4], al_[4];
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                split2(live ? dv8[2 * e] : 0.f, live ? dv8[2 * e + 1] : 0.f, dh_[e], dl_[e]);
                split2(live ? av8[2 * e] : 0.f, live ? av8[2 * e + 1] : 0.f, ah_[e], al_[e]);
              }
              constexpr uint32_t PB = 8192u;                      // plane_bytes(128, MN-major): both images use 128-column tiles
              const int n = col + sc;
              const long long blk = ((long long)(n >> 7) * (R_pad >> 5) + (row >> 5)) * (2LL * PB);
              const uint32_t o = mnmajor_sw128_offset((uint32_t)(row & 31), (uint32_t)((n & 127) >> 3));
              uint8_t* dimg = reinterpret_cast<uint8_t*>(p.dh_mn) + blk + o;
              uint8_t* aimg = reinterpret_cast<uint8_t*>(p.act_mn) + blk + o;
              *reinterpret_cast<uint4*>(dimg) = make_uint4(dh_[0], dh_[1], dh_[2], dh_[3]);
              *reinterpret_cast<uint4*>(dimg + PB) = make_uint4(dl_[0], dl_[1], dl_[2], dl_[3]);
              *reinterpret_cast<uint4*>(aimg) = make_uint4(ah_[0], ah_[1], ah_[2], ah_[3]);
              *reinterpret_cast<uint4*>(aimg + PB) = make_uint4(al_[0], al_[1], al_[2], al_[3]);
            }
            __syncwarp();                                         // staging rows are free for the next column group
          }
        } else {
#pragma unroll
          for (int q = 0; q < HC / 8; ++q) {
            const int kk = 8 * q + 2 * (lane & 3);
            const float2 bv = __ldg(reinterpret_cast<const float2*>(b1 + kk));
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int r = r_lo + 8 * h;
              const float x0 = acc_h[4 * q + 2 * h] + bv.x, x1 = acc_h[4 * q + 2 * h + 1] + bv.y;
              // training forward: the pre-activation h = A1 Wa1^T + b1 is stored once (fp32, row-major) for the GEMM-based backward
              if (MODE == 0 && p.h_out) {
                const long long row = (long long)t * 128 + r;
                if (row < p.M) *reinterpret_cast<float2*>(p.h_out + row * p.H4 + (long long)j * HC + kk) = make_float2(x0, x1);
              }
              float y0, y1;
              if (p.debug & 1) { y0 = x0; y1 = x1; }
              else if constexpr (MODE == 0) { y0 = gelu_fast(x0); y1 = gelu_fast(x1); }
              else { y0 = acc_d[4 * q + 2 * h] * gelu_grad_fast(x0); y1 = acc_d[4 * q + 2 * h + 1] * gelu_grad_fast(x1); }
              if (p.debug & 2) continue;
              uint32_t hi, lo;
              split2(y0, y1, hi, lo);
              const uint32_t o = sb0 + L.act + (uint32_t)(kk >> 5) * 16384u + kmajor_sw64_offset((uint32_t)r, (uint32_t)((kk & 31) >> 3)) +
                                 (uint32_t)(kk & 7) * 2u;
              asm volatile("st.shared.b32 [%0], %1;" ::"r"(o), "r"(hi) : "memory");
              asm volatile("st.shared.b32 [%0], %1;" ::"r"(o + 8192u), "r"(lo) : "memory");
            }
          }
        }
        fence_proxy_async_smem();
        wg_bar();                                                 // the warpgroup's 64 activation rows are complete
        // GEMM-b(j): acc_o += y . Wb_j^T over K = HC; GEMM-a(j+1) is issued behind it into the freed acc_h
        const int s = n_b % L.sb;
        mbar_wait(wb_full(s), (n_b / L.sb) & 1u);
        wg::fence();
        {
          uint64_t da = make_smem_desc(sb0 + L.act + slab, false), db = make_smem_desc(sb0 + L.wb + s * L.wb_stage, false);
          const uint64_t blo = (uint64_t)(C * 4);              // lo plane of a Wb k-block: C * 64 bytes behind the hi plane
#pragma unroll
          for (int kb = 0; kb < HC / 32; ++kb) {
            mma3<C>(acc_o, da, da + 512u, db, db + blo, (j > 0 || kb > 0) ? 1u : 0u, p.passes);
            mma3<C>(acc_o, da + 2u, da + 514u, db + 2u, db + blo + 2u, 1u, p.passes);
            da += 1024u; db += 2u * blo;
          }
        }
        ++n_b;
        if (j + 1 < nch) gemm_a(n_c + 1);
        wg::commit();
      }
      wg::wait<0>();
      wg::fence_operand(acc_o);
      __syncwarp();
      if (lane == 0) mbar_arrive(wb_empty((n_b - 1) % L.sb));
      // ---- final epilogue of the tile: registers -> per-warp smem transpose -> coalesced 64-byte row segments
      const long long row0 = (long long)t * 128 + g * 64 + wq * 16;
#pragma unroll
      for (int c = 0; c < C / 16; ++c) {
        const int n = c * 16 + c4;
        float4 rr[2];
#pragma unroll
        for (int it = 0; it < 2; ++it) {
          const long long row = row0 + it * 8 + rl;
          rr[it] = (p.resid && row < p.M) ? ldg_f4(p.resid + row * C + n) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        __syncwarp();                                    // the previous chunk's reads of the staging rows are done
#pragma unroll
        for (int qq = 0; qq < 2; ++qq)
#pragma unroll
          for (int h = 0; h < 2; ++h)
            asm volatile("st.shared.v2.f32 [%0], {%1, %2};"
                         ::"r"(stage_base + (uint32_t)((rl + 8 * h) * EPI_STAGE_ROW_FLOATS + 8 * qq + 2 * (lane & 3)) * 4u),
                           "f"(acc_o[8 * c + 4 * qq + 2 * h]), "f"(acc_o[8 * c + 4 * qq + 2 * h + 1]) : "memory");
        __syncwarp();
        float4 bv = make_float4(0.f, 0.f, 0.f, 0.f), sv = make_float4(1.f, 1.f, 1.f, 1.f);
        if (p.bias2) bv = ldg_f4(p.bias2 + n);
        if (p.col_scale) sv = ldg_f4(p.col_scale + n);
#pragma unroll
        for (int it = 0; it < 2; ++it) {
          const int rr_ = it * 8 + rl;
          const long long row = row0 + rr_;
          if (row >= p.M) continue;
          float4 x;
          asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(x.x), "=f"(x.y), "=f"(x.z), "=f"(x.w)
                       : "r"(stage_base + (uint32_t)(rr_ * EPI_STAGE_ROW_FLOATS + c4) * 4u) : "memory");
          x.x += bv.x; x.y += bv.y; x.z += bv.z; x.w += bv.w;
          if (p.aux_out) *reinterpret_cast<float4*>(p.aux_out + row * C + n) = x;
          x.x *= sv.x; x.y *= sv.y; x.z *= sv.z; x.w *= sv.w;
          if (p.row_scale) { const float rs = __ldg(p.row_scale + row); x.x *= rs; x.y *= rs; x.z *= rs; x.w *= rs; }
          x.x += rr[it].x; x.y += rr[it].y; x.z += rr[it].z; x.w += rr[it].w;
          *reinterpret_cast<float4*>(p.out + row * C + n) = x;
        }
      }
    }
    if constexpr (WGRAD_IMG) {                                   // one global atomic per db1 column per CTA
      cons_bar();
      for (int i = threadIdx.x - EPI0 * 32; i < p.H4; i += 256) {
        float v;
        asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(cs_base + 4u * i) : "memory");
        atomicAdd(p.db1 + i, v);
      }
    }
  }
}

// ================================================================================================================
static bool chain_layout(int mode, int C, int HC, int sa, int sb, Layout& L) {
  const uint32_t nA = (mode == 1 || mode == 2) ? 2 : 1;
  L.a_tile = (uint32_t)(C / 32) * 16384u;
  L.wa_chunk = (uint32_t)(C / 32) * HC * 128u;
  L.wa_stage = nA * L.wa_chunk;
  L.wb_stage = (uint32_t)(HC / 32) * C * 128u;
  L.act_bytes = (uint32_t)(HC / 32) * 16384u;
  L.sa = sa; L.sb = sb;
  uint32_t o = 0;
  L.a = o; o += nA * L.a_tile;
  L.ones = 0; L.a2 = L.a + L.a_tile;
  L.wa = o; o += sa * L.wa_stage;
  L.wb = o; o += sb * L.wb_stage;
  L.act = o; o += L.act_bytes;
  L.act2 = 0;
  L.stage = o; o += STAGING;
  L.cs = o; o += mode >= 2 ? (uint32_t)(4 * C) * 4u : 0u;
  L.bar = o; o += BARS;
  L.total = o + 1024u;
  return L.total <= SMEM_LIMIT + 1024u;
}

// HC_req > 0: only layouts with that chunk width (the caller packed its weights for it)
static bool pick_chain(int mode, int C, int HC_req, int& HC, Layout& L) {
  static const int cand[][3] = {{64, 2, 2}, {32, 2, 2}, {64, 2, 1}, {32, 2, 1}, {32, 1, 1}};
  if (C % 32 != 0 || C < 32 || C > 256) return false;
  // mode 2 recomputes h where v and dz tiles fit beside the weight chunks (C <= 128); mode 3 reads the saved h and is built
  // for the one wider dense stage ConvNeXt has, C = 192
  if ((mode == 2 && C > 128) || (mode == 3 && C != 192)) return false;
  for (auto& c : cand)
    if ((HC_req == 0 || c[0] == HC_req) && chain_layout(mode, C, c[0], c[1], c[2], L)) { HC = c[0]; return true; }
  return false;
}

int chain_chunk(int mode, int C) {
  int HC = 0; Layout L;
  return pick_chain(mode, C, 0, HC, L) ? HC : 0;
}

static bool aligned16(const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15u) == 0; }

int chain(const ChainParams& p, cudaStream_t stream) {
  SM3_REQUIRE(p.mode >= 0 && p.mode <= 3, SM3_ERR_INVALID_ARG, "ffn chain: mode");
  SM3_REQUIRE((p.mode == 3 || (p.a1 && p.wa1)) && p.wb && p.bias1 && p.out && (p.mode == 0 || (p.a2 && p.wa2)), SM3_ERR_INVALID_ARG,
              "ffn chain: null operand");
  SM3_REQUIRE(p.mode < 2 || (p.dh_mn && p.act_mn && p.db1 && (p.mode == 2 || p.h_in)), SM3_ERR_INVALID_ARG,
              "ffn chain: modes 2 / 3 need dh_mn, act_mn, db1 (and h_in in mode 3)");
  SM3_REQUIRE(p.M > 0 && p.H4 > 0 && p.C > 0, SM3_ERR_INVALID_ARG, "ffn chain: bad shape");
  ChainK k{};
  k.p = p;
  int HC = 0;
  SM3_REQUIRE(p.HC == 32 || p.HC == 64, SM3_ERR_INVALID_ARG, "ffn chain: chunk must be 32 or 64 (sm3_ffn_fused_chunk), got %d", p.HC);
  SM3_REQUIRE(pick_chain(p.mode, p.C, p.HC, HC, k.L), SM3_ERR_UNSUPPORTED_SHAPE, "ffn chain: C=%d with chunk %d does not fit shared memory (mode %d)", p.C, p.HC, p.mode);
  SM3_REQUIRE(p.H4 % HC == 0 && p.C % 16 == 0, SM3_ERR_UNSUPPORTED_SHAPE, "ffn chain: H4=%d not a multiple of the chunk %d", p.H4, HC);
  SM3_REQUIRE(p.mode < 2 || p.H4 % 128 == 0, SM3_ERR_UNSUPPORTED_SHAPE, "ffn chain: the MN-major images use 128-column tiles, H4=%d", p.H4);
  SM3_REQUIRE(aligned16(p.a1) && aligned16(p.wa1) && aligned16(p.wb) && aligned16(p.out) && aligned16(p.bias1) &&
              (!p.a2 || aligned16(p.a2)) && (!p.wa2 || aligned16(p.wa2)) && (!p.resid || aligned16(p.resid)) &&
              (!p.aux_out || aligned16(p.aux_out)) && (!p.bias2 || aligned16(p.bias2)) && (!p.col_scale || aligned16(p.col_scale)) &&
              (!p.dh_mn || aligned16(p.dh_mn)) && (!p.act_mn || aligned16(p.act_mn)) && (!p.h_in || aligned16(p.h_in)),
              SM3_ERR_INVALID_ARG, "ffn chain: pointers must be 16B aligned");
  k.p.passes = (p.passes == 1) ? 1 : 3;
  k.m_tiles = (p.M + 127) / 128;
  k.nch = p.H4 / HC;
  int grid = persistent_grid_sms();
  if (grid > k.m_tiles) grid = k.m_tiles;
#define SM3_CHAIN_LAUNCH(MODE_, HC_, C_)                                                                                    \
  do {                                                                                                                      \
    cudaFuncSetAttribute(ffn_chain_kernel<MODE_, HC_, C_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k.L.total);    \
    ffn_chain_kernel<MODE_, HC_, C_><<<grid, THREADS, k.L.total, stream>>>(k);                                              \
  } while (0)
  // the accumulator widths (HC for GEMM-a, C for GEMM-b) are wgmma shapes, i.e. template arguments
#define SM3_CHAIN_C(MODE_, HC_)                                                                                             \
  switch (p.C) {                                                                                                            \
    case 32: SM3_CHAIN_LAUNCH(MODE_, HC_, 32); break;   case 64: SM3_CHAIN_LAUNCH(MODE_, HC_, 64); break;                   \
    case 96: SM3_CHAIN_LAUNCH(MODE_, HC_, 96); break;   case 128: SM3_CHAIN_LAUNCH(MODE_, HC_, 128); break;                 \
    case 160: SM3_CHAIN_LAUNCH(MODE_, HC_, 160); break; case 192: SM3_CHAIN_LAUNCH(MODE_, HC_, 192); break;                 \
    case 224: SM3_CHAIN_LAUNCH(MODE_, HC_, 224); break; default: SM3_CHAIN_LAUNCH(MODE_, HC_, 256); break;                  \
  }
  if (p.mode == 0) { if (HC == 64) { SM3_CHAIN_C(0, 64) } else { SM3_CHAIN_C(0, 32) } }
  else if (p.mode == 1) { if (HC == 64) { SM3_CHAIN_C(1, 64) } else { SM3_CHAIN_C(1, 32) } }
  else if (p.mode == 2) {            // the layouts pick_chain admits: 64-column chunks up to C = 96, 32 up to C = 128
    if (HC == 64) {
      switch (p.C) { case 32: SM3_CHAIN_LAUNCH(2, 64, 32); break; case 64: SM3_CHAIN_LAUNCH(2, 64, 64); break; default: SM3_CHAIN_LAUNCH(2, 64, 96); break; }
    } else {
      switch (p.C) {
        case 32: SM3_CHAIN_LAUNCH(2, 32, 32); break;  case 64: SM3_CHAIN_LAUNCH(2, 32, 64); break;
        case 96: SM3_CHAIN_LAUNCH(2, 32, 96); break;  default: SM3_CHAIN_LAUNCH(2, 32, 128); break;
      }
    }
  } else SM3_CHAIN_LAUNCH(3, 32, 192);                         // pick_chain: mode 3 is C = 192 with 32-column chunks
#undef SM3_CHAIN_C
#undef SM3_CHAIN_LAUNCH
  return check_launch("ffn_chain_kernel");
}

}  // namespace ffn
}  // namespace sm3
