// Split-bf16 ("bf16x3") tensor-core GEMM for sm_90a: D[M,N] = epilogue( sum_k A(m,k) * B(n,k) ).
//
// fp32 operands live in HBM.  Producer warps load them (coalesced float4, optional row gather),
// split every value into bf16 hi + bf16 lo (a = hi + lo, |a-(hi+lo)| <= 2^-16 |a|), and store both
// planes straight into the wgmma canonical shared-memory layouts (K-major SWIZZLE_64B or MN-major
// SWIZZLE_128B).  Two consumer warpgroups (64 rows of the 128-row tile each) issue wgmma.mma_async
// three times per k-step (hi*hi + hi*lo + lo*hi) into fp32 register accumulators, so the product error
// is ~1e-5 relative (vs 5e-4 for single-pass TF32) at 3 bf16 MMAs per logical MAC.  The same warps
// then apply the fused epilogue (bias / GELU / GELU' / layer-scale / gate / residual / atomic split-K)
// while the producers already fill the ring with the next tile.
//
// Replaces, on the reference hot path (convnext_moe.py): nn.Linear pointwise_conv1/2 + GELU
// (:389-404), the per-expert Python loop (:244) incl. the gather x[_batch_index] (:265), and the
// 2x2/s2 downsample convs (:549-558); and autograd's dgrad/wgrad GEMMs for all of them.
#pragma once
#include <type_traits>
#include "common.cuh"

namespace sm3 {
namespace gemm {

constexpr int BM = 128;          // rows of D per tile (two m64 warpgroup MMAs)
constexpr int BK = 32;           // bf16 elements per k-block (2 wgmma k-steps of 16)
constexpr int MAX_BN = 128;      // the accumulator of a 64 x 128 slab is 64 registers per consumer thread
constexpr int STAGES = 6;
constexpr int NUM_CONS_WARPS = 8;                                    // warps 0-7: two consumer warpgroups
constexpr int NUM_PROD_WARPS = 8;
constexpr int FIRST_PROD_WARP = 8;                                   // warps 8-15: producers
constexpr int NUM_THREADS = (NUM_CONS_WARPS + NUM_PROD_WARPS) * 32;  // 512
constexpr int CONS_REGS = 144, PROD_REGS = 112;                       // setmaxnreg split of the 64K-entry register file
constexpr int MAX_UNITS = 4;     // producer units per warp per k-block: (128 + 128) / 8 / 8

constexpr uint32_t OFF_A_HI = 0;
constexpr uint32_t OFF_A_LO = 8192;
constexpr uint32_t OFF_B_HI = 16384;
constexpr uint32_t OFF_B_LO = 24576;
constexpr uint32_t STAGE_BYTES = 32768;
constexpr uint32_t WG_A_BYTES = 4096;     // offset of rows 64..127 in an A plane (both layouts): the second warpgroup's slab
constexpr int MAX_STAGES = 8;             // fully packed kernels use as many stages as fit (narrow tiles need less smem per stage)
constexpr uint32_t BAR_BYTES = 256;
constexpr int EPI_CW = 16;                                          // accumulator columns per epilogue pass
constexpr uint32_t EPI_STAGE_ROW_FLOATS = EPI_CW + 4;               // + 4 pad: conflict-free 16-byte accesses
constexpr uint32_t EPI_STAGE_BYTES = 32 * EPI_STAGE_ROW_FLOATS * 4;  // per epilogue warp
constexpr int MAX_EPI_WARPS = 8;
constexpr int COLSUM_SMEM_COLS = 3072;                              // EPI_COLSUM accumulates per CTA in smem when N fits
constexpr uint32_t SMEM_BYTES = STAGES * STAGE_BYTES + BAR_BYTES + MAX_EPI_WARPS * EPI_STAGE_BYTES + COLSUM_SMEM_COLS * 4 + 1024;  // +1024 alignment slack

enum Sched : int { SCHED_DENSE = 0, SCHED_GROUPED = 1, SCHED_SPLITK = 2 };

enum Epi : int {
  EPI_BIAS = 1,       // acc += bias[n]
  EPI_GELU = 2,       // (aux_out[m,n] = acc if aux_out) ; acc = gelu(acc)
  EPI_DGELU = 4,      // acc *= gelu'(aux_in[m,n])
  EPI_COLSCALE = 8,   // acc *= col_scale[n]
  EPI_ROWSCALE = 16,  // acc *= row_scale[m]
  EPI_RESID = 32,     // acc += resid[m,n]
  EPI_ATOMIC = 64,    // atomicAdd(D, acc) instead of store
  EPI_AUXSTORE = 128, // aux_out[m,n] = acc (after bias), e.g. the pre-layer-scale FFN output
  EPI_COLSUM = 256,   // colsum[group][n] += sum over the tile's rows of the final value (bias gradients)
};

struct Params {
  // operands: element (mn,k) at ptr + mn*s_mn + k*s_k ; exactly one stride must be 1
  const float* A; long long a_smn, a_sk;
  const float* B; long long b_smn, b_sk; long long b_group_stride;
  const int* a_row_index;   // optional gather of A rows (K-major A only); -1 -> zero row
  const int* b_k_index;     // optional gather of B along the reduction index (MN-major B only); -1 -> zero
  // pre-split weights (see pack_b): tile-ordered bf16 hi/lo images brought in with one cp.async.bulk per k-block
  const uint16_t* b_packed; long long b_packed_group_stride;   // stride in bf16 elements
  const uint16_t* a_packed;   // pre-split activation image (pack_a); with b_packed the whole main loop is bulk copies
  // Column tail: N need only be a multiple of 8.  When BN does not divide N the last N-tile is padded to BN columns: its
  // B rows past N load as zeros (the fp32 producers skip them, pack_b writes zero rows, pack_act zero columns) and the
  // epilogue masks every per-column access at n >= N (bias, col_scale, aux, resid, D, colsum).
  int M, N, K, BN;
  // schedule
  int sched;
  int num_tiles;            // DENSE / SPLITK: total tiles; GROUPED: upper bound (unused)
  int m_tiles, n_tiles, k_splits, num_groups;
  const int* tile_group;        // GROUPED: group id per m tile
  const int* num_m_tiles_dev;   // GROUPED: device scalar
  // SPLITK: per-group reduction range [seg_begin, seg_end) (device) or null => [0,K).  The fully packed path (a_packed)
  // bulk-copies whole 32-row k-blocks starting at k_begin / 32 and multiplies all of them, so it requires
  // seg_begin % 32 == 0 and the rows [seg_end, ceil32(seg_end)) zero in one of the two operand images; the other paths
  // mask k < seg_end.  The MoE, LSK and expert-parallel wgrads meet it: segments start at multiples of 128 and the rows
  // past each segment's end are zero in d_o / gathered -1 rows (tests/test_gemm_gpu.py).
  const int* seg_begin;
  const int* seg_end;
  // epilogue
  float* D; long long ldd; long long d_group_stride;
  const float* bias; long long bias_group_stride;
  int epi;
  float* aux_out; const float* aux_in; long long ld_aux;
  const float* col_scale; const float* row_scale;
  const float* resid; long long ld_resid;
  float* colsum; long long colsum_group_stride;
  int passes;   // 3 (default) or 1 (bf16 operands: only the hi*hi product)
  int nstages; unsigned stage_bytes;   // filled by launch(): smem ring depth / stride (4 x 48 KB unless fully packed)
  int debug;   // perf experiments only: bit0 skip A loads+stores, bit1 skip the packed-B bulk copy, bit2 skip MMAs
};

// ---------------------------------------------------------------------------------------------
// Canonical-layout offset functions (host+device so the CPU tests can check the mapping).
// K-major, SWIZZLE_64B: rows of 32 bf16 (64 B); atom = 8 rows (512 B); chunk = 8 bf16 (16 B).
__host__ __device__ inline uint32_t kmajor_sw64_offset(uint32_t row, uint32_t chunk) {
  return (row >> 3) * 512u + (row & 7u) * 64u + ((chunk ^ ((row >> 1) & 3u)) << 4);
}
// MN-major, SWIZZLE_128B: atom = 8 k-rows x 64 mn-elements (1024 B); atoms ordered (mn_group*4 + k_group).
__host__ __device__ inline uint32_t mnmajor_sw128_offset(uint32_t k, uint32_t mn_chunk /* mn/8 */) {
  const uint32_t g = mn_chunk >> 3, cc = mn_chunk & 7u;
  return (g * 4u + (k >> 3)) * 1024u + (k & 7u) * 128u + ((cc ^ (k & 7u)) << 4);
}
constexpr uint32_t MN_LBO_BYTES = 4096;  // stride between 64-element mn groups
constexpr uint32_t MN_SBO_BYTES = 1024;  // stride between 8-row k groups
constexpr uint32_t K_SBO_BYTES = 512;    // stride between 8-row groups (K-major SW64)
// bytes of one bf16 plane of a [width x 32] k-block tile in the two canonical layouts
__host__ __device__ inline uint32_t plane_bytes(int width, bool mn_major) {
  return mn_major ? (uint32_t)((width + 63) / 64) * 4096u : (uint32_t)width * 64u;
}

__host__ __device__ inline uint64_t make_smem_desc(uint32_t smem_addr, bool mn_major) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFFu);
  if (mn_major) {
    d |= (uint64_t)((MN_LBO_BYTES >> 4) & 0x3FFFu) << 16;
    d |= (uint64_t)((MN_SBO_BYTES >> 4) & 0x3FFFu) << 32;
    d |= (uint64_t)1 << 62;  // SWIZZLE_128B
  } else {
    d |= (uint64_t)1 << 16;  // LBO unused for swizzled K-major
    d |= (uint64_t)((K_SBO_BYTES >> 4) & 0x3FFFu) << 32;
    d |= (uint64_t)2 << 62;  // SWIZZLE_64B
  }
  return d;
}
#if defined(__CUDACC__) && defined(SM3_GEMM_KERNEL_IMPL)
}  // namespace gemm
}  // namespace sm3
#include "wgmma.cuh"
namespace sm3 {
namespace gemm {
// ---------------------------------------------------------------------------------------------
// PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
  return ok != 0;
}
// Bounded wait: a pipeline bug traps (launch failure) instead of hanging the GPU.  No printf here: a function call
// between wgmma issue and wait would make ptxas serialise the asynchronous MMAs.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 20000000000LL) __trap();  // ~10 s
  }
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// ---------------------------------------------------------------------------------------------
struct Tile {
  int m0, n0, group, k_begin, k_end;
  __device__ __forceinline__ int nkb() const { return (k_end - k_begin + BK - 1) / BK; }
};

__device__ __forceinline__ int total_tiles(const Params& p) {
  if (p.sched == SCHED_GROUPED) return __ldg(p.num_m_tiles_dev) * p.n_tiles;
  return p.num_tiles;
}

__device__ __forceinline__ Tile decode_tile(const Params& p, int t) {
  Tile tl;
  if (p.sched == SCHED_SPLITK) {
    const int s = t % p.k_splits;
    int rest = t / p.k_splits;
    const int nt = rest % p.n_tiles; rest /= p.n_tiles;
    const int mt = rest % p.m_tiles;
    tl.group = rest / p.m_tiles;
    tl.m0 = mt * BM; tl.n0 = nt * p.BN;
    int b = 0, e = p.K;
    if (p.seg_begin) { b = __ldg(p.seg_begin + tl.group); e = __ldg(p.seg_end + tl.group); }
    int len = e - b; if (len < 0) len = 0;
    int chunk = (len + p.k_splits - 1) / p.k_splits;
    chunk = (chunk + BK - 1) / BK * BK;
    tl.k_begin = b + s * chunk;
    tl.k_end = min(e, tl.k_begin + chunk);
    if (tl.k_end < tl.k_begin) tl.k_end = tl.k_begin;
  } else {
    const int mt = t / p.n_tiles, nt = t % p.n_tiles;
    tl.m0 = mt * BM; tl.n0 = nt * p.BN;
    tl.group = (p.sched == SCHED_GROUPED) ? __ldg(p.tile_group + mt) : 0;
    tl.k_begin = 0; tl.k_end = p.K;
  }
  return tl;
}

// split 4 fp32 -> 2 packed bf16x2 hi (truncated) + 2 packed bf16x2 lo (rounded residual)
__device__ __forceinline__ void split4(const float4& x, uint32_t& h01, uint32_t& h23, uint32_t& l01,
                                       uint32_t& l23) {
  const uint32_t u0 = __float_as_uint(x.x), u1 = __float_as_uint(x.y);
  const uint32_t u2 = __float_as_uint(x.z), u3 = __float_as_uint(x.w);
  h01 = __byte_perm(u0, u1, 0x7632);
  h23 = __byte_perm(u2, u3, 0x7632);
  const uint32_t r0 = __float_as_uint(x.x - __uint_as_float(u0 & 0xFFFF0000u)) + 0x8000u;
  const uint32_t r1 = __float_as_uint(x.y - __uint_as_float(u1 & 0xFFFF0000u)) + 0x8000u;
  const uint32_t r2 = __float_as_uint(x.z - __uint_as_float(u2 & 0xFFFF0000u)) + 0x8000u;
  const uint32_t r3 = __float_as_uint(x.w - __uint_as_float(u3 & 0xFFFF0000u)) + 0x8000u;
  l01 = __byte_perm(r0, r1, 0x7632);
  l23 = __byte_perm(r2, r3, 0x7632);
}

// ---------------------------------------------------------------------------------------------
// Kernel.  Warp roles: 0-7 consumers (warpgroup g = warp / 4 owns rows 64g..64g+63 of the tile: wgmma main loop,
// then the epilogue straight from its register accumulator), 8-15 producers.  A k-block of an operand is cut into
// "units" of 8 rows x 32 k (K-major) or 2 k-rows x 128 mn (MN-major); unit u of a k-block belongs to producer warp
// u % 8.  All per-tile address arithmetic is hoisted: a thread keeps one 32-bit element offset per (unit, half) and
// advances it by a constant per k-block.
// EPI_T >= 0: the epilogue flag set is a compile-time constant (the hot FFN / expert / wgrad variants: the epilogue
// is on the critical path of the HBM-bound GEMMs and the runtime flag branches cost issue slots there);
// EPI_T = -1: generic, flags read from Params.
template <bool A_MN, bool B_MN, bool B_PACKED, bool A_PACKED, int EPI_T>
__global__ void __launch_bounds__(NUM_THREADS, 1) gemm_bf16x3_kernel(const __grid_constant__ Params p) {
  const int EPI = (EPI_T >= 0) ? EPI_T : p.epi;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_base = smem_base + STAGES * STAGE_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 64u + 8u * s; };
  const int NST = p.nstages;
  const uint32_t STB = p.stage_bytes;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < NST; ++s) { mbar_init(full_bar(s), A_PACKED ? 1 : NUM_PROD_WARPS + (B_PACKED ? 1 : 0)); mbar_init(empty_bar(s), NUM_CONS_WARPS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int ntiles = total_tiles(p);

  if (warp < NUM_CONS_WARPS) {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(CONS_REGS));
    // ============================== CONSUMERS: MMA + EPILOGUE ===============================
    constexpr int NE = NUM_CONS_WARPS;
    const int wg = warp >> 2;
    const int nchunks = p.BN / EPI_CW;
    const uint32_t stage_base = bar_base + BAR_BYTES + (uint32_t)warp * EPI_STAGE_BYTES;
    const int rl = lane >> 2, c4 = (lane & 3) * 4;      // this lane's row-in-group-of-8 and first column of 4
    // EPI_COLSUM: column sums are accumulated per CTA in shared memory across all its tiles of one group and
    // flushed with one global atomic per column (instead of one per column per tile).
    const uint32_t cs_base = bar_base + BAR_BYTES + MAX_EPI_WARPS * EPI_STAGE_BYTES;
    const bool cs_smem = (EPI & EPI_COLSUM) && p.N <= COLSUM_SMEM_COLS;
    int cs_group = -1;
    const int e_tid = warp * 32 + lane;
    auto epi_bar = []() { asm volatile("bar.sync 1, %0;" ::"n"(NE * 32) : "memory"); };
    auto cs_flush = [&](int group) {
      epi_bar();
      if (group >= 0) {
        float* cd = p.colsum + (long long)group * p.colsum_group_stride;
        for (int n = e_tid; n < p.N; n += NE * 32) {
          float sv;
          asm volatile("ld.shared.f32 %0, [%1];" : "=f"(sv) : "r"(cs_base + 4u * n) : "memory");
          if (sv != 0.f) atomicAdd(cd + n, sv);
        }
      }
      for (int n = e_tid; n < p.N; n += NE * 32)
        asm volatile("st.shared.f32 [%0], %1;" ::"r"(cs_base + 4u * n), "f"(0.f) : "memory");
      epi_bar();
    };
    if (cs_smem) cs_flush(-1);
    int stage = 0; uint32_t phase = 0;
    constexpr uint32_t a_kstep = A_MN ? 2u * MN_SBO_BYTES : 32u;   // advance 16 k per wgmma
    constexpr uint32_t b_kstep = B_MN ? 2u * MN_SBO_BYTES : 32u;
    const uint32_t b_lo_off = B_PACKED ? OFF_B_HI + plane_bytes(p.BN, B_MN) : OFF_B_LO;   // packed: lo follows hi
    float acc[MAX_BN / 2];
    for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
      const Tile tl = decode_tile(p, t);
      const int nkb = tl.nkb();
      if (nkb == 0) continue;
      if (cs_smem && tl.group != cs_group) { if (cs_group >= 0) cs_flush(cs_group); cs_group = tl.group; }
      const int row0 = tl.m0 + wg * 64 + (warp & 3) * 16;
      // residual (shortcut) rows of the first chunk are fetched before the main loop and the next chunk's while the
      // current one is written out, so the epilogue does not stall a full HBM round trip per 16 x 16 block
      float4 rr[2], rn[2];
      auto load_resid = [&](int c_, float4 (&dst)[2]) {
        const int n_ = tl.n0 + c_ * EPI_CW + c4;
#pragma unroll
        for (int it = 0; it < 2; ++it) {
          const int row = row0 + it * 8 + rl;
          dst[it] = (row < p.M && n_ < p.N) ? ldg_f4(p.resid + (long long)row * p.ld_resid + n_) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
      };
      if (EPI & EPI_RESID) load_resid(0, rr);

      // ---- main loop: one k-block's MMAs stay in flight while the previous stage is handed back to the producers.
      // The wgmma shape (N = BN) is a template argument of the whole loop, so ptxas sees a single accumulator shape.
      int prev = -1;
      auto mainloop = [&](auto bn_c) {
        constexpr int N = decltype(bn_c)::value;
        for (int kb = 0; kb < nkb; ++kb) {
          mbar_wait(full_bar(stage), phase);
          wg::fence();
          const uint32_t sb = smem_base + stage * STB + (uint32_t)wg * WG_A_BYTES;
          const uint32_t sbb = smem_base + stage * STB;
#pragma unroll
          for (int j = 0; j < BK / 16; ++j) {
            const uint64_t ahi = make_smem_desc(sb + OFF_A_HI + j * a_kstep, A_MN);
            const uint64_t alo = make_smem_desc(sb + OFF_A_LO + j * a_kstep, A_MN);
            const uint64_t bhi = make_smem_desc(sbb + OFF_B_HI + j * b_kstep, B_MN);
            const uint64_t blo = make_smem_desc(sbb + b_lo_off + j * b_kstep, B_MN);
            if (!(p.debug & 4)) {
              const uint32_t accum = (kb > 0 || j > 0) ? 1u : 0u;
              if (p.passes == 1) {
                wg::mma<N, A_MN, B_MN>(acc, ahi, bhi, accum);
              } else {
                wg::mma<N, A_MN, B_MN>(acc, alo, bhi, accum);
                wg::mma<N, A_MN, B_MN>(acc, ahi, blo, 1u);
                wg::mma<N, A_MN, B_MN>(acc, ahi, bhi, 1u);
              }
            }
          }
          wg::commit();
          if (prev >= 0) {
            wg::wait<1>();
            __syncwarp();
            if (lane == 0) mbar_arrive(empty_bar(prev));
          }
          prev = stage;
          if (++stage == NST) { stage = 0; phase ^= 1u; }
        }
      };
      switch (p.BN) {
        case 32: mainloop(std::integral_constant<int, 32>{}); break;
        case 64: mainloop(std::integral_constant<int, 64>{}); break;
        case 96: mainloop(std::integral_constant<int, 96>{}); break;
        default: mainloop(std::integral_constant<int, 128>{}); break;
      }
      wg::wait<0>();
      wg::fence_operand(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_bar(prev));
      if (p.debug & 4) {
#pragma unroll
        for (int i = 0; i < MAX_BN / 2; ++i) acc[i] = 0.f;
      }

      // ---- epilogue: registers (wgmma fragment: row 16w + lane/4 (+8), column pair 8q + 2(lane%4)) -> per-warp smem
      // transpose -> (lane = 4 columns) so that every global access (stores, residual / saved-activation loads,
      // atomics) is a coalesced row segment
      float* dbase = p.D + (long long)tl.group * p.d_group_stride;
      const float* bias = p.bias ? p.bias + (long long)tl.group * p.bias_group_stride : nullptr;
#pragma unroll
      for (int c = 0; c < MAX_BN / EPI_CW; ++c) {
        if (c >= nchunks) break;
        __syncwarp();                                     // previous chunk's reads of the stage are done
#pragma unroll
        for (int qq = 0; qq < 2; ++qq)
#pragma unroll
          for (int h = 0; h < 2; ++h)
            asm volatile("st.shared.v2.f32 [%0], {%1, %2};"
                         ::"r"(stage_base + (uint32_t)((rl + 8 * h) * EPI_STAGE_ROW_FLOATS + 8 * qq + 2 * (lane & 3)) * 4u),
                           "f"(acc[8 * c + 4 * qq + 2 * h]), "f"(acc[8 * c + 4 * qq + 2 * h + 1]) : "memory");
        if ((EPI & EPI_RESID) && c + 1 < nchunks) load_resid(c + 1, rn);
        __syncwarp();
        const int n = tl.n0 + c * EPI_CW + c4;
        const bool n_ok = n < p.N;           // column tail: N % 8 == 0, so a lane's 4 columns are all in or all out
        float4 bv = make_float4(0.f, 0.f, 0.f, 0.f), sv = make_float4(1.f, 1.f, 1.f, 1.f);
        if ((EPI & EPI_BIAS) && n_ok) bv = ldg_f4(bias + n);
        if ((EPI & EPI_COLSCALE) && n_ok) sv = ldg_f4(p.col_scale + n);
        float4 cs = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int it = 0; it < 2; ++it) {
          const int r = it * 8 + rl;
          const int row = row0 + r;
          if (row >= p.M || !n_ok) continue;
          float4 x;
          asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
                       : "=f"(x.x), "=f"(x.y), "=f"(x.z), "=f"(x.w)
                       : "r"(stage_base + (uint32_t)(r * EPI_STAGE_ROW_FLOATS + c4) * 4u) : "memory");
          x.x += bv.x; x.y += bv.y; x.z += bv.z; x.w += bv.w;
          if ((EPI & (EPI_AUXSTORE | EPI_GELU)) && p.aux_out)
            *reinterpret_cast<float4*>(p.aux_out + (long long)row * p.ld_aux + n) = x;
          if (EPI & EPI_GELU) { x.x = gelu_fast(x.x); x.y = gelu_fast(x.y); x.z = gelu_fast(x.z); x.w = gelu_fast(x.w); }
          if (EPI & EPI_DGELU) {
            const float4 h = ldg_f4(p.aux_in + (long long)row * p.ld_aux + n);
            x.x *= gelu_grad_fast(h.x); x.y *= gelu_grad_fast(h.y); x.z *= gelu_grad_fast(h.z); x.w *= gelu_grad_fast(h.w);
          }
          x.x *= sv.x; x.y *= sv.y; x.z *= sv.z; x.w *= sv.w;
          if (EPI & EPI_ROWSCALE) { const float rs = __ldg(p.row_scale + row); x.x *= rs; x.y *= rs; x.z *= rs; x.w *= rs; }
          if (EPI & EPI_RESID) { x.x += rr[it].x; x.y += rr[it].y; x.z += rr[it].z; x.w += rr[it].w; }
          cs.x += x.x; cs.y += x.y; cs.z += x.z; cs.w += x.w;
          float* dst = dbase + (long long)row * p.ldd + n;
          if (EPI & EPI_ATOMIC) {
            asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "f"(x.x), "f"(x.y), "f"(x.z), "f"(x.w) : "memory");
          } else {
            *reinterpret_cast<float4*>(dst) = x;
          }
        }
        if (EPI & EPI_RESID) {
#pragma unroll
          for (int it = 0; it < 2; ++it) rr[it] = rn[it];
        }
        if (EPI & EPI_COLSUM) {
          // lanes with the same (lane & 3) hold partial sums of the same 4 columns
#pragma unroll
          for (int o = 4; o < 32; o <<= 1) {
            cs.x += __shfl_xor_sync(0xffffffffu, cs.x, o); cs.y += __shfl_xor_sync(0xffffffffu, cs.y, o);
            cs.z += __shfl_xor_sync(0xffffffffu, cs.z, o); cs.w += __shfl_xor_sync(0xffffffffu, cs.w, o);
          }
          if (lane < 4 && n_ok) {
            if (cs_smem) {
              const uint32_t sa = cs_base + 4u * (uint32_t)n;
              asm volatile("red.shared.add.f32 [%0], %1;" ::"r"(sa), "f"(cs.x) : "memory");
              asm volatile("red.shared.add.f32 [%0], %1;" ::"r"(sa + 4u), "f"(cs.y) : "memory");
              asm volatile("red.shared.add.f32 [%0], %1;" ::"r"(sa + 8u), "f"(cs.z) : "memory");
              asm volatile("red.shared.add.f32 [%0], %1;" ::"r"(sa + 12u), "f"(cs.w) : "memory");
            } else {
              float* cd = p.colsum + (long long)tl.group * p.colsum_group_stride + n;
              asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(cd), "f"(cs.x), "f"(cs.y), "f"(cs.z), "f"(cs.w) : "memory");
            }
          }
        }
      }
    }
    if (cs_smem && cs_group >= 0) cs_flush(cs_group);
  } else {
    // ============================== PRODUCERS =============================================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(PROD_REGS));
    if (A_PACKED) {
      // Both operands are pre-split tile images: one thread streams them in with two cp.async.bulk per k-block.
      if (warp == FIRST_PROD_WARP && lane == 0) {
        const uint32_t a_bytes = 2u * plane_bytes(BM, A_MN), b_bytes = 2u * plane_bytes(p.BN, B_MN);
        const long long kblocks = (p.K + BK - 1) / BK;
        int stage = 0; uint32_t phase = 0;
        for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
          const Tile tl = decode_tile(p, t);
          const int nkb = tl.nkb();
          if (nkb == 0) continue;
          const long long kb0 = tl.k_begin / BK;
          const uint8_t* srcA = reinterpret_cast<const uint8_t*>(p.a_packed) + ((long long)(tl.m0 / BM) * kblocks + kb0) * a_bytes;
          const uint8_t* srcB = reinterpret_cast<const uint8_t*>(p.b_packed + (long long)tl.group * p.b_packed_group_stride) +
                                ((long long)(tl.n0 / p.BN) * kblocks + kb0) * b_bytes;
          for (int kb = 0; kb < nkb; ++kb) {
            mbar_wait(empty_bar(stage), phase ^ 1u);
            const uint32_t sb = smem_base + stage * STB;
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(full_bar(stage)), "r"(a_bytes + b_bytes) : "memory");
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         ::"r"(sb + OFF_A_HI), "l"(srcA + (long long)kb * a_bytes), "r"(a_bytes), "r"(full_bar(stage)) : "memory");
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         ::"r"(sb + OFF_B_HI), "l"(srcB + (long long)kb * b_bytes), "r"(b_bytes), "r"(full_bar(stage)) : "memory");
            if (++stage == NST) { stage = 0; phase ^= 1u; }
          }
        }
      }
    } else {
    // A k-block of an operand is cut into "units" a warp handles with two LDG.128 + two STS.128 per lane:
    //   K-major : 8 rows x 32 k  -- lane = (row l>>2, 16-byte chunk l&3 = 8 consecutive k)
    //   MN-major: 2 k-rows x 128 mn -- lane = (k-row l>>4, chunk l&15 = 8 consecutive mn)
    // Every lane owns a whole 8-element chunk, so hi/lo go out as one 16-byte store each with no shuffles;
    // a quarter-warp writes 128 contiguous (swizzled) bytes -> bank-conflict free.
    const int wq = warp - FIRST_PROD_WARP;
    constexpr int units_a = 16;
    const int segs_b = (p.BN + 127) / 128;
    const int units_b = B_PACKED ? 0 : (B_MN ? 16 * segs_b : p.BN / 8);
    const int units = units_a + units_b;
    // lane-constant parts of the shared-memory store offsets
    const uint32_t st_k = (uint32_t)((lane >> 2) * 64 + ((((uint32_t)lane & 3u) ^ (((uint32_t)lane >> 3) & 3u)) << 4));
    const uint32_t kr_lane = (uint32_t)lane >> 4, j_lane = (uint32_t)lane & 15u;

    // per-tile state
    constexpr int MU = B_PACKED ? (16 + NUM_PROD_WARPS - 1) / NUM_PROD_WARPS : MAX_UNITS;   // units per producer warp per k-block
    uint32_t off[MU];               // element offset of this lane's chunk from the operand base (A) / group base (B)
    uint32_t vmask = 0;             // bit i: row / mn range valid
    const float* baseB = p.B;
    const uint16_t* packB = nullptr;   // packed B image of the current tile's first k-block
    int t_cur = blockIdx.x - gridDim.x, kb_cur = 0, nkb_cur = 0, k_begin = 0, k_end = 0;
    const uint32_t adv_a = A_MN ? (uint32_t)(BK * p.a_sk) : (uint32_t)BK;
    const uint32_t adv_b = B_MN ? (uint32_t)(BK * p.b_sk) : (uint32_t)BK;
    const bool b_gather = B_MN && (p.b_k_index != nullptr);   // B rows come through an index (expert wgrad)

    auto setup_tile = [&](const Tile& tl) {
      k_begin = tl.k_begin; k_end = tl.k_end;
      baseB = p.B + (long long)tl.group * p.b_group_stride;
      if (B_PACKED) {
        const long long kblocks = (p.K + BK - 1) / BK;
        packB = p.b_packed + (long long)tl.group * p.b_packed_group_stride +
                ((long long)(tl.n0 / p.BN) * kblocks) * (2LL * p.BN * BK);
      }
      vmask = 0;
#pragma unroll
      for (int i = 0; i < MU; ++i) {
        const int u = wq + NUM_PROD_WARPS * i;
        off[i] = 0;
        if (u >= units) continue;
        const bool is_a = u < units_a;
        const int ul = is_a ? u : u - units_a;
        const int mn0 = is_a ? tl.m0 : tl.n0;
        const int mn_lim = is_a ? p.M : p.N;
        if (is_a ? !A_MN : !B_MN) {
          const long long s_mn = is_a ? p.a_smn : p.b_smn;
          const int row = mn0 + 8 * ul + (lane >> 2);
          if (row >= mn_lim) continue;
          long long ridx = row;
          if (is_a && p.a_row_index) { ridx = __ldg(p.a_row_index + row); if (ridx < 0) continue; }
          off[i] = (uint32_t)(ridx * s_mn + tl.k_begin + 8 * (lane & 3));
          vmask |= 1u << i;
        } else {
          const int segs = is_a ? 1 : segs_b;
          const int pi = (segs == 2) ? (ul >> 1) : ul, seg = (segs == 2) ? (ul & 1) : 0;
          const int mnl = seg * 128 + 8 * (int)j_lane;
          const int tile_w = is_a ? BM : p.BN;
          if (mnl + 8 > tile_w || mn0 + mnl + 8 > mn_lim) continue;     // tile widths / extents are multiples of 8
          const long long s_k = is_a ? p.a_sk : p.b_sk;
          const int koff = 2 * pi + (int)kr_lane;
          off[i] = (!is_a && b_gather) ? (uint32_t)(mn0 + mnl)
                                       : (uint32_t)((long long)(tl.k_begin + koff) * s_k + mn0 + mnl);
          vmask |= 1u << i;
        }
      }
    };
    // advance (t_cur, kb_cur) to the next k-block with work; returns false at the end
    auto advance = [&]() -> bool {
      if (kb_cur + 1 < nkb_cur) { ++kb_cur; return true; }
      for (t_cur += gridDim.x; t_cur < ntiles; t_cur += gridDim.x) {
        const Tile tl = decode_tile(p, t_cur);
        nkb_cur = tl.nkb();
        if (nkb_cur > 0) { kb_cur = 0; setup_tile(tl); return true; }
      }
      return false;
    };

    // issue the global loads of the current k-block, then step the offsets to the next one
    auto load_kb = [&](float4 (&r)[MU][2]) {
      const int k0 = k_begin + kb_cur * BK;
      const int kl = k0 + 8 * (lane & 3);                     // K-major operands: this lane's 8 k values
      const bool kin0 = (kl + 4 <= k_end), kin1 = (kl + 8 <= k_end);
#pragma unroll
      for (int i = 0; i < MU; ++i) {
        r[i][0] = make_float4(0.f, 0.f, 0.f, 0.f);
        r[i][1] = make_float4(0.f, 0.f, 0.f, 0.f);
        const int u = wq + NUM_PROD_WARPS * i;
        if (u >= units) continue;
        const bool is_a = u < units_a;
        const float* base = is_a ? p.A : baseB;
        const bool ok = (vmask >> i) & 1u;
        if (is_a ? !A_MN : !B_MN) {
          if (ok && kin0) r[i][0] = ldg_f4(base + off[i]);
          if (ok && kin1) r[i][1] = ldg_f4(base + off[i] + 4);
        } else {
          const int ul = is_a ? u : u - units_a;
          const int pi = (!is_a && segs_b == 2) ? (ul >> 1) : ul;
          const int k = k0 + 2 * pi + (int)kr_lane;
          if (ok && k < k_end) {
            const float* src = base + off[i];
            if (!is_a && b_gather) {
              const int kk = __ldg(p.b_k_index + k);
              src = (kk >= 0) ? base + (long long)kk * p.b_sk + off[i] : nullptr;
            }
            if (src) { r[i][0] = ldg_f4(src); r[i][1] = ldg_f4(src + 4); }
          }
        }
        off[i] += is_a ? adv_a : ((!is_a && b_gather) ? 0u : adv_b);
      }
    };

    // split + store one k-block into its smem stage
    auto store_kb = [&](const float4 (&r)[MU][2], uint32_t sb) {
#pragma unroll
      for (int i = 0; i < MU; ++i) {
        const int u = wq + NUM_PROD_WARPS * i;
        if (u >= units) continue;
        const bool is_a = u < units_a;
        const int ul = is_a ? u : u - units_a;
        uint4 hi, lo;
        split4(r[i][0], hi.x, hi.y, lo.x, lo.y);
        split4(r[i][1], hi.z, hi.w, lo.z, lo.w);
        uint32_t o;
        if (is_a ? !A_MN : !B_MN) {
          o = (uint32_t)ul * 512u + st_k;
        } else {
          const int segs = is_a ? 1 : segs_b;
          const uint32_t pi = (segs == 2) ? (uint32_t)(ul >> 1) : (uint32_t)ul;
          const uint32_t seg = (segs == 2) ? (uint32_t)(ul & 1) : 0u;
          const uint32_t k = 2u * pi + kr_lane;             // k-row inside the k-block
          const uint32_t mc = seg * 16u + j_lane;           // 8-element mn chunk inside the tile
          o = ((mc >> 3) * 4u + (k >> 3)) * 1024u + (k & 7u) * 128u + (((mc & 7u) ^ (k & 7u)) << 4);
        }
        const uint32_t dst_hi = sb + (is_a ? OFF_A_HI : OFF_B_HI) + o;
        const uint32_t dst_lo = sb + (is_a ? OFF_A_LO : OFF_B_LO) + o;
        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};"
                     ::"r"(dst_hi), "r"(hi.x), "r"(hi.y), "r"(hi.z), "r"(hi.w) : "memory");
        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};"
                     ::"r"(dst_lo), "r"(lo.x), "r"(lo.y), "r"(lo.z), "r"(lo.w) : "memory");
      }
    };

    int stage = 0; uint32_t phase = 0;
    const uint16_t* pub_src = nullptr; int pub_kb = 0;   // packed-B source of the k-block the next publish() stores
    auto publish = [&](const float4 (&r)[MU][2]) {
      mbar_wait(empty_bar(stage), phase ^ 1u);
      if (B_PACKED && wq == 0 && lane == 0 && (p.debug & 2)) {
        mbar_arrive(full_bar(stage));
      } else if (B_PACKED && wq == 0 && lane == 0) {
        // one thread: arm the stage barrier with the byte count and start the bulk copy of B's hi|lo image
        const uint32_t bytes = (uint32_t)p.BN * 128u;
        const uint16_t* src = pub_src + (long long)pub_kb * (2LL * p.BN * BK);
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(full_bar(stage)), "r"(bytes) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(smem_base + stage * STB + OFF_B_HI), "l"(src), "r"(bytes), "r"(full_bar(stage)) : "memory");
      }
      if (p.debug & 8) {            // loads only: consume the registers without the split / stores
#pragma unroll
        for (int i = 0; i < MU; ++i) asm volatile("" ::"f"(r[i][0].x), "f"(r[i][1].w));
      } else if (!(p.debug & 1)) store_kb(r, smem_base + stage * STB);
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) mbar_arrive(full_bar(stage));
      if (++stage == NST) { stage = 0; phase ^= 1u; }
    };

    // PF k-blocks of global loads are kept in flight per thread (register ring, statically indexed): one
    // k-block (16 KB of A per SM) in flight is latency-bound at ~14 GB/s/SM -- measured 3x slower than the MMAs.
    constexpr int PF = B_PACKED ? 4 : 2;
    float4 r[PF][MU][2];
    if (p.debug & 16) {
#pragma unroll
      for (int d = 0; d < PF; ++d)
#pragma unroll
        for (int i = 0; i < MU; ++i) { r[d][i][0] = make_float4(1.f, 2.f, 3.f, 4.f); r[d][i][1] = r[d][i][0]; }
    }
    const uint16_t* q_src[PF]; int q_kb[PF]; bool q_ok[PF];
    const bool dbg_noload = p.debug & (1 | 16);   // bit4: stores of zeros without loads
#pragma unroll
    for (int d = 0; d < PF; ++d) {
      q_ok[d] = advance();
      q_src[d] = packB; q_kb[d] = kb_cur;
      if (q_ok[d] && !dbg_noload) load_kb(r[d]);
    }
    bool done = !q_ok[0];
    while (!done) {
#pragma unroll
      for (int d = 0; d < PF; ++d) {
        if (!q_ok[d]) { done = true; break; }
        pub_src = q_src[d]; pub_kb = q_kb[d];
        publish(r[d]);
        q_ok[d] = advance();
        q_src[d] = packB; q_kb[d] = kb_cur;
        if (q_ok[d] && !dbg_noload) load_kb(r[d]);
      }
    }
    }  // !A_PACKED
  }

}
#endif  // __CUDACC__ && SM3_GEMM_KERNEL_IMPL

// Pre-split a weight operand B(n,k) (element at ptr + n*s_mn + k*s_k, `groups` matrices `group_stride` apart) into
// the tile-ordered bf16 image the kernel bulk-copies: [group][n_tile][k_block]{ hi[BN x 32] | lo[BN x 32] } with
// each plane in the K-major SWIZZLE_64B canonical layout.  packed_elems(N, K) bf16 elements per group: N is padded to
// whole tiles of pick_bn(N) rows, and the padding rows are written as zeros.
long long packed_elems(int N, int K);
// `tile` > 0 overrides the tile width (the fused FFN kernels stream weight chunks of their own width).
int pack_b(const float* B, long long s_mn, long long s_k, long long group_stride, int groups, int N, int K,
           uint16_t* out, cudaStream_t stream, int tile = 0);
// Pre-split an ACTIVATION operand.  mn_major = 0: X[rows, K] row-major (optional row gather, -1 = zero row) ->
// K-major tiles of `tile` rows (128 for the A operand).  mn_major = 1: X[R, W] row-major where the ROW index is the
// reduction index (wgrad operands; optional row gather) -> MN-major tiles of `tile` columns (128 for A, BN for B).
long long packed_act_elems(long long rows, int cols, int mn_major, int tile);
int pack_act(const float* X, long long ld, const int* row_index, long long rows, int cols, int mn_major, int tile,
             uint16_t* out, cudaStream_t stream);
// Host-side launcher (gemm_tc.cu): validates shapes, fills derived fields, launches on `stream`.
int launch(Params p, cudaStream_t stream);
// Tile width of an N-column output: the largest of {128, 96, 64, 32} that divides N; for other N % 8 == 0 (column
// tail) the one with the fewest tiles, then the least padding; 0 if N % 8 != 0.
int pick_bn(int N);

}  // namespace gemm
}  // namespace sm3
