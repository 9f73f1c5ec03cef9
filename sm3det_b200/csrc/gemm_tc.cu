// Host launcher for the split-bf16 wgmma GEMM (see gemm_tc.cuh).
#define SM3_GEMM_KERNEL_IMPL
#include "gemm_tc.cuh"
#include <mutex>

namespace sm3 {
const char* last_error();
namespace gemm {

int pick_bn(int N) {
  static const int cand[] = {128, 96, 64, 32};   // MAX_BN = 128
  for (int bn : cand)
    if (N % bn == 0) return bn;
  if (N <= 0 || N % 8) return 0;
  // column tail: the last N-tile runs padded and masked.  Fewest tiles, then the least padding (N = 16 -> 32, 80 -> 96).
  int best = 0, best_tiles = 0;
  for (int bn : cand) {
    const int tiles = (N + bn - 1) / bn;
    if (!best || tiles < best_tiles || (tiles == best_tiles && tiles * bn < best_tiles * best)) { best = bn; best_tiles = tiles; }
  }
  return best;
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

long long packed_elems(int N, int K) {
  const long long kblocks = (K + BK - 1) / BK;
  const int bn = pick_bn(N);
  const long long rows = bn > 0 ? (long long)(N + bn - 1) / bn * bn : N;   // N padded to whole tiles (column tail)
  return rows * kblocks * BK * 2;             // hi + lo planes, K padded to a multiple of 32
}

// one thread per 16-byte chunk (8 k-values of one row); rows [N, rows) of the last tile are written as zeros
__global__ void __launch_bounds__(256) pack_b_kernel(const float* __restrict__ B, long long s_mn, long long s_k,
                                                    long long group_stride, int N, int rows, int K, int BN,
                                                    uint16_t* __restrict__ out, long long out_group_stride,
                                                    long long chunks_per_group) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= chunks_per_group) return;
  const int g = blockIdx.y;
  const int kblocks = (K + BK - 1) / BK;
  // chunk index -> (row n fastest, then chunk c, then k-block): consecutive threads read consecutive rows
  const int n = (int)(i % rows);
  const long long r = i / rows;
  const int c = (int)(r % 4), kb = (int)(r / 4);
  const bool live = n < N;
  const float* src = B + (long long)g * group_stride + (long long)n * s_mn;
  uint32_t hi[4], lo[4];
#pragma unroll
  for (int e = 0; e < 8; e += 2) {
    float v[2];
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int k = kb * BK + c * 8 + e + q;
      v[q] = (live && k < K) ? __ldg(src + (long long)k * s_k) : 0.f;
    }
    const uint32_t u0 = __float_as_uint(v[0]), u1 = __float_as_uint(v[1]);
    hi[e / 2] = __byte_perm(u0, u1, 0x7632);
    const uint32_t r0 = __float_as_uint(v[0] - __uint_as_float(u0 & 0xFFFF0000u)) + 0x8000u;
    const uint32_t r1 = __float_as_uint(v[1] - __uint_as_float(u1 & 0xFFFF0000u)) + 0x8000u;
    lo[e / 2] = __byte_perm(r0, r1, 0x7632);
  }
  const int nt = n / BN, row = n % BN;
  uint8_t* tile = reinterpret_cast<uint8_t*>(out + (long long)g * out_group_stride) +
                  ((long long)nt * kblocks + kb) * ((long long)BN * 128);
  const uint32_t o = kmajor_sw64_offset((uint32_t)row, (uint32_t)c);
  *reinterpret_cast<uint4*>(tile + o) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
  *reinterpret_cast<uint4*>(tile + (long long)BN * 64 + o) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
}

int pack_b(const float* B, long long s_mn, long long s_k, long long group_stride, int groups, int N, int K,
           uint16_t* out, cudaStream_t stream, int tile) {
  SM3_REQUIRE(B && out && N > 0 && K > 0 && groups >= 1, SM3_ERR_INVALID_ARG, "gemm pack: bad argument");
  const int BN = tile > 0 ? tile : pick_bn(N);
  // an explicit tile must divide N; the default tile may leave a column tail, whose image rows are padded with zeros
  SM3_REQUIRE(BN > 0 && BN % 8 == 0 && BN <= 256 && (tile > 0 ? N % BN == 0 : N % 8 == 0), SM3_ERR_UNSUPPORTED_SHAPE,
              "gemm pack: N=%d has no tile width (tile=%d)", N, tile);
  SM3_REQUIRE((reinterpret_cast<uintptr_t>(out) & 15u) == 0, SM3_ERR_INVALID_ARG, "gemm pack: output must be 16B aligned");
  const long long kblocks = (K + BK - 1) / BK;
  const int rows = (N + BN - 1) / BN * BN;
  const long long chunks = (long long)rows * kblocks * 4;
  dim3 grid((unsigned)((chunks + 255) / 256), (unsigned)groups);
  pack_b_kernel<<<grid, 256, 0, stream>>>(B, s_mn, s_k, group_stride, N, rows, K, BN, out, packed_elems(N, K), chunks);
  return check_launch("pack_b_kernel");
}

long long packed_act_elems(long long rows, int cols, int mn_major, int tile) {
  if (!mn_major) {     // [rows, K=cols] -> ceil(rows/tile) row tiles x ceil(K/32) k-blocks x 2 planes of tile x 32
    const long long rt = (rows + tile - 1) / tile, kb = (cols + BK - 1) / BK;
    return rt * kb * 2 * (long long)tile * BK;
  }
  const long long ct = (cols + tile - 1) / tile, kb = (rows + BK - 1) / BK;
  return ct * kb * 2 * (long long)(plane_bytes(tile, true) / 2);
}

// K-major activation pack: one thread per 16-byte chunk (8 k of one row); rows beyond `rows` / gathered -1 -> zeros
__global__ void __launch_bounds__(256) pack_act_k_kernel(const float* __restrict__ X, long long ld, const int* __restrict__ row_index,
                                                        long long rows, int K, int tile, uint16_t* __restrict__ out,
                                                        long long chunks) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= chunks) return;
  const int kblocks = (K + BK - 1) / BK;
  // consecutive threads -> consecutive chunks of one row (coalesced 32 B each), then rows
  const int cpr = kblocks * 4;
  const long long row = i / cpr;
  const int cc = (int)(i % cpr), kb = cc >> 2, c = cc & 3;
  long long src_row = row < rows ? row : -1;
  if (src_row >= 0 && row_index) src_row = __ldg(row_index + row);
  float v[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) v[e] = 0.f;
  if (src_row >= 0) {
    const int k = kb * BK + c * 8;
    const float* src = X + src_row * ld + k;
    if (k + 8 <= K) { const float4 a = ldg_f4(src), b = ldg_f4(src + 4); v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w; }
    else { for (int e = 0; e < 8; ++e) if (k + e < K) v[e] = __ldg(src + e); }
  }
  uint32_t hi[4], lo[4];
#pragma unroll
  for (int e = 0; e < 8; e += 2) {
    const uint32_t u0 = __float_as_uint(v[e]), u1 = __float_as_uint(v[e + 1]);
    hi[e / 2] = __byte_perm(u0, u1, 0x7632);
    const uint32_t r0 = __float_as_uint(v[e] - __uint_as_float(u0 & 0xFFFF0000u)) + 0x8000u;
    const uint32_t r1 = __float_as_uint(v[e + 1] - __uint_as_float(u1 & 0xFFFF0000u)) + 0x8000u;
    lo[e / 2] = __byte_perm(r0, r1, 0x7632);
  }
  const long long rt = row / tile; const int rr = (int)(row % tile);
  uint8_t* img = reinterpret_cast<uint8_t*>(out) + (rt * kblocks + kb) * ((long long)tile * 128);
  const uint32_t o = kmajor_sw64_offset((uint32_t)rr, (uint32_t)c);
  *reinterpret_cast<uint4*>(img + o) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
  *reinterpret_cast<uint4*>(img + (long long)tile * 64 + o) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
}

// MN-major activation pack: chunk = 8 consecutive columns of one (reduction) row
__global__ void __launch_bounds__(256) pack_act_mn_kernel(const float* __restrict__ X, long long ld, const int* __restrict__ row_index,
                                                         long long rows, int W, int tile, uint16_t* __restrict__ out,
                                                         long long chunks, long long rows_pad) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= chunks) return;
  const int ct = (W + tile - 1) / tile;
  const int cpr = ct * (tile / 8);                 // chunks per (padded) row, including tile padding columns
  const long long r = i / cpr;
  const int cc = (int)(i % cpr);
  const int mt = cc / (tile / 8), mc = cc % (tile / 8);
  const int col = mt * tile + mc * 8;
  long long src_row = r < rows ? r : -1;
  if (src_row >= 0 && row_index) src_row = __ldg(row_index + r);
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
  if (src_row >= 0 && col + 8 <= W) { const float* src = X + src_row * ld + col; a = ldg_f4(src); b = ldg_f4(src + 4); }
  const float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
  uint32_t hi[4], lo[4];
#pragma unroll
  for (int e = 0; e < 8; e += 2) {
    const uint32_t u0 = __float_as_uint(v[e]), u1 = __float_as_uint(v[e + 1]);
    hi[e / 2] = __byte_perm(u0, u1, 0x7632);
    const uint32_t r0 = __float_as_uint(v[e] - __uint_as_float(u0 & 0xFFFF0000u)) + 0x8000u;
    const uint32_t r1 = __float_as_uint(v[e + 1] - __uint_as_float(u1 & 0xFFFF0000u)) + 0x8000u;
    lo[e / 2] = __byte_perm(r0, r1, 0x7632);
  }
  const long long kblocks = rows_pad / BK;
  const long long kb = r / BK; const uint32_t k = (uint32_t)(r % BK);
  const uint32_t pb = plane_bytes(tile, true);
  uint8_t* img = reinterpret_cast<uint8_t*>(out) + ((long long)mt * kblocks + kb) * (2LL * pb);
  const uint32_t o = mnmajor_sw128_offset(k, (uint32_t)mc);
  *reinterpret_cast<uint4*>(img + o) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
  *reinterpret_cast<uint4*>(img + pb + o) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
}

int pack_act(const float* X, long long ld, const int* row_index, long long rows, int cols, int mn_major, int tile,
             uint16_t* out, cudaStream_t stream) {
  SM3_REQUIRE(X && out && rows > 0 && cols > 0, SM3_ERR_INVALID_ARG, "gemm pack_act: bad argument");
  SM3_REQUIRE(tile >= 32 && tile <= 256 && tile % 32 == 0, SM3_ERR_INVALID_ARG, "gemm pack_act: tile=%d", tile);
  SM3_REQUIRE(aligned16(X) && aligned16(out) && ld % 4 == 0 && cols % 4 == 0, SM3_ERR_INVALID_ARG, "gemm pack_act: alignment");
  if (!mn_major) {
    const long long rt = (rows + tile - 1) / tile, kb = (cols + BK - 1) / BK;
    const long long chunks = rt * tile * kb * 4;
    pack_act_k_kernel<<<(unsigned)((chunks + 255) / 256), 256, 0, stream>>>(X, ld, row_index, rows, cols, tile, out, chunks);
  } else {
    SM3_REQUIRE(cols % 8 == 0, SM3_ERR_UNSUPPORTED_SHAPE, "gemm pack_act: MN-major needs cols%%8==0");
    const long long rows_pad = (rows + BK - 1) / BK * BK;
    const long long ct = (cols + tile - 1) / tile;
    const long long chunks = rows_pad * ct * (tile / 8);
    // plane padding beyond tile/64 groups (tile = 96 or 160...) is never read by the MMA (N = tile columns)
    pack_act_mn_kernel<<<(unsigned)((chunks + 255) / 256), 256, 0, stream>>>(X, ld, row_index, rows, cols, tile, out, chunks, rows_pad);
  }
  return check_launch("pack_act");
}

int launch(Params p, cudaStream_t stream) {
  if (p.b_packed && !p.B) p.B = reinterpret_cast<const float*>(p.b_packed);   // B itself is not read in packed mode
  if (p.a_packed && !p.A) p.A = reinterpret_cast<const float*>(p.a_packed);
  SM3_REQUIRE(p.A && p.B && p.D, SM3_ERR_INVALID_ARG, "gemm: null operand");
  SM3_REQUIRE(p.M > 0 && p.N > 0 && p.K >= 0, SM3_ERR_INVALID_ARG, "gemm: bad shape %d %d %d", p.M, p.N, p.K);
  SM3_REQUIRE((p.a_smn == 1) != (p.a_sk == 1) || (p.a_smn == 1 && p.M == 1), SM3_ERR_INVALID_ARG,
              "gemm: A needs exactly one unit stride");
  const bool packed = p.b_packed != nullptr;
  const bool apacked = p.a_packed != nullptr;
  if (packed && !apacked) { p.b_smn = p.K; p.b_sk = 1; }     // weights-only packing: the image is always K-major
  if (apacked) {                                             // fully packed: B's image has A's majorness
    const bool amn = (p.a_smn == 1 && p.a_sk != 1);
    if (amn) { p.b_smn = 1; p.b_sk = p.N; } else { p.b_smn = p.K; p.b_sk = 1; }
  }
  SM3_REQUIRE((p.b_smn == 1) != (p.b_sk == 1), SM3_ERR_INVALID_ARG, "gemm: B needs exactly one unit stride");
  const bool a_mn = (p.a_smn == 1 && p.a_sk != 1), b_mn = (p.b_smn == 1 && p.b_sk != 1);
  if (p.BN == 0) p.BN = pick_bn(p.N);
  SM3_REQUIRE(p.BN >= 32 && p.BN <= MAX_BN && p.BN % 32 == 0 && p.N % 8 == 0, SM3_ERR_UNSUPPORTED_SHAPE,
              "gemm: N=%d has no tile width (N a multiple of 8, tile width a multiple of 32 <= 128)", p.N);
  SM3_REQUIRE(aligned16(p.A) && aligned16(p.B) && aligned16(p.D), SM3_ERR_INVALID_ARG, "gemm: pointers must be 16B aligned");
  if (!a_mn) SM3_REQUIRE(p.a_smn % 4 == 0 && p.K % 4 == 0, SM3_ERR_UNSUPPORTED_SHAPE, "gemm: K-major A needs K%%4==0, lda%%4==0");
  else       SM3_REQUIRE(p.a_sk % 4 == 0 && p.M % 8 == 0, SM3_ERR_UNSUPPORTED_SHAPE, "gemm: MN-major A needs M%%8==0, lda%%4==0");
  if (!b_mn) SM3_REQUIRE(p.b_smn % 4 == 0 && p.K % 4 == 0, SM3_ERR_UNSUPPORTED_SHAPE, "gemm: K-major B needs K%%4==0, ldb%%4==0");
  else       SM3_REQUIRE(p.b_sk % 4 == 0, SM3_ERR_UNSUPPORTED_SHAPE, "gemm: MN-major B needs ldb%%4==0");
  SM3_REQUIRE(!(p.a_row_index && a_mn), SM3_ERR_INVALID_ARG, "gemm: row gather needs K-major A");
  SM3_REQUIRE(!(p.b_k_index && !b_mn), SM3_ERR_INVALID_ARG, "gemm: k gather needs MN-major B");
  SM3_REQUIRE(p.ldd % 4 == 0, SM3_ERR_UNSUPPORTED_SHAPE, "gemm: ldd%%4");
  if (p.epi & (EPI_GELU | EPI_AUXSTORE)) SM3_REQUIRE(!p.aux_out || (aligned16(p.aux_out) && p.ld_aux % 4 == 0), SM3_ERR_INVALID_ARG, "gemm: aux_out");
  if (p.epi & EPI_DGELU) SM3_REQUIRE(p.aux_in && aligned16(p.aux_in) && p.ld_aux % 4 == 0, SM3_ERR_INVALID_ARG, "gemm: aux_in");
  if (p.epi & EPI_BIAS) SM3_REQUIRE(p.bias && aligned16(p.bias) && p.bias_group_stride % 4 == 0, SM3_ERR_INVALID_ARG, "gemm: bias");
  if (p.epi & EPI_COLSCALE) SM3_REQUIRE(p.col_scale && aligned16(p.col_scale), SM3_ERR_INVALID_ARG, "gemm: col_scale");
  if (p.epi & EPI_ROWSCALE) SM3_REQUIRE(p.row_scale, SM3_ERR_INVALID_ARG, "gemm: row_scale");
  if (p.epi & EPI_COLSUM) SM3_REQUIRE(p.colsum && aligned16(p.colsum) && p.colsum_group_stride % 4 == 0, SM3_ERR_INVALID_ARG, "gemm: colsum");
  if (p.epi & EPI_RESID) SM3_REQUIRE(p.resid && aligned16(p.resid) && p.ld_resid % 4 == 0, SM3_ERR_INVALID_ARG, "gemm: resid");

  p.n_tiles = (p.N + p.BN - 1) / p.BN;      // a column tail runs as one more, padded and masked, tile
  p.m_tiles = (p.M + BM - 1) / BM;
  if (p.sched == SCHED_DENSE) {
    p.k_splits = 1; p.num_groups = 1;
    p.num_tiles = p.m_tiles * p.n_tiles;
  } else if (p.sched == SCHED_GROUPED) {
    SM3_REQUIRE(p.tile_group && p.num_m_tiles_dev, SM3_ERR_INVALID_ARG, "gemm: grouped schedule needs tile map");
    p.k_splits = 1;
    p.num_tiles = p.m_tiles * p.n_tiles;  // upper bound; the device scalar decides
  } else if (p.sched == SCHED_SPLITK) {
    SM3_REQUIRE(p.k_splits >= 1 && p.num_groups >= 1, SM3_ERR_INVALID_ARG, "gemm: split-K needs k_splits/num_groups");
    SM3_REQUIRE((p.epi & EPI_ATOMIC) || p.k_splits == 1, SM3_ERR_INVALID_ARG, "gemm: split-K>1 needs EPI_ATOMIC");
    p.num_tiles = p.num_groups * p.m_tiles * p.n_tiles * p.k_splits;
  } else {
    SM3_REQUIRE(false, SM3_ERR_INVALID_ARG, "gemm: bad schedule %d", p.sched);
  }
  // 32-bit element offsets inside the kernel: every operand must span < 2^32 floats (16 GiB)
  {
    const long long a_ext = apacked ? 0 : a_mn ? (long long)p.K * p.a_sk : (long long)(p.a_row_index ? (1LL << 31) / (p.a_smn ? p.a_smn : 1) : p.M) * p.a_smn;
    const long long b_ext = packed ? 0 : b_mn ? (long long)(p.b_k_index ? 1 : p.K) * p.b_sk + p.N : (long long)p.N * p.b_smn;
    SM3_REQUIRE(a_ext < (1LL << 32) && b_ext < (1LL << 32), SM3_ERR_UNSUPPORTED_SHAPE, "gemm: operand larger than 2^32 elements");
  }
  // smem ring: 6 stages of 32 KB when the producer warps write the stage; fully packed operands only need
  // 16 KB (A) + the two B planes per stage, so narrow tiles get a deeper ring (more bytes in flight per SM -- the
  // narrow GEMMs of stages 0/1 are HBM-bound streams of the packed A image).
  p.nstages = STAGES; p.stage_bytes = STAGE_BYTES;
  if (apacked) {
    const unsigned sb = (16384u + 2u * plane_bytes(p.BN, b_mn) + 1023u) & ~1023u;
    int ns = (int)((unsigned)(STAGES * STAGE_BYTES) / sb);
    if (ns > MAX_STAGES) ns = MAX_STAGES;
    if (ns >= STAGES) { p.nstages = ns; p.stage_bytes = sb; }
  }
  int grid = persistent_grid_sms();
  if (grid > p.num_tiles) grid = p.num_tiles;
  if (grid < 1) grid = 1;
#define SM3_GEMM_LAUNCH_E(AMN, BMN, BPK, APK, EPIT)                                                                             \
  do {                                                                                                                          \
    cudaFuncSetAttribute(gemm_bf16x3_kernel<AMN, BMN, BPK, APK, EPIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES); \
    gemm_bf16x3_kernel<AMN, BMN, BPK, APK, EPIT><<<grid, NUM_THREADS, SMEM_BYTES, stream>>>(p);                                     \
  } while (0)
#define SM3_GEMM_LAUNCH(AMN, BMN, BPK, APK) SM3_GEMM_LAUNCH_E(AMN, BMN, BPK, APK, -1)
  if (apacked) {
    SM3_REQUIRE(packed && a_mn == b_mn && p.BN == pick_bn(p.N) && !p.a_row_index && !p.b_k_index, SM3_ERR_INVALID_ARG,
                "gemm: packed A needs packed B of the same majorness (gathers are applied by the pack kernels)");
    SM3_REQUIRE(aligned16(p.a_packed) && aligned16(p.b_packed) && (p.b_packed_group_stride % 8) == 0, SM3_ERR_INVALID_ARG,
                "gemm: packed operands must be 16B aligned");
    // the flag sets of the hot launches get their own instantiation (compile-time epilogue)
    constexpr int E_FFN2_TRAIN = EPI_BIAS | EPI_COLSCALE | EPI_RESID | EPI_AUXSTORE, E_FFN2_EVAL = EPI_BIAS | EPI_COLSCALE | EPI_RESID;
    if (a_mn) {
      if (p.epi == EPI_ATOMIC) SM3_GEMM_LAUNCH_E(true, true, true, true, EPI_ATOMIC);
      else if (p.epi == (EPI_ATOMIC | EPI_ROWSCALE)) SM3_GEMM_LAUNCH_E(true, true, true, true, EPI_ATOMIC | EPI_ROWSCALE);
      else SM3_GEMM_LAUNCH(true, true, true, true);
    } else {
      if (p.epi == 0) SM3_GEMM_LAUNCH_E(false, false, true, true, 0);
      else if (p.epi == EPI_BIAS) SM3_GEMM_LAUNCH_E(false, false, true, true, EPI_BIAS);
      else if (p.epi == E_FFN2_TRAIN) SM3_GEMM_LAUNCH_E(false, false, true, true, E_FFN2_TRAIN);
      else if (p.epi == E_FFN2_EVAL) SM3_GEMM_LAUNCH_E(false, false, true, true, E_FFN2_EVAL);
      else SM3_GEMM_LAUNCH(false, false, true, true);
    }
  }
  else if (packed) {
    SM3_REQUIRE(!a_mn && p.sched != SCHED_SPLITK && p.BN == pick_bn(p.N), SM3_ERR_INVALID_ARG,
                "gemm: packed B needs K-major A, a dense/grouped schedule and the default tile width");
    SM3_REQUIRE((reinterpret_cast<uintptr_t>(p.b_packed) & 15u) == 0 && (p.b_packed_group_stride % 8) == 0,
                SM3_ERR_INVALID_ARG, "gemm: packed B must be 16B aligned");
    SM3_GEMM_LAUNCH(false, false, true, false);
  }
  else if (!a_mn && !b_mn) SM3_GEMM_LAUNCH(false, false, false, false);
  else if (!a_mn && b_mn) SM3_GEMM_LAUNCH(false, true, false, false);
  else if (a_mn && b_mn) SM3_GEMM_LAUNCH(true, true, false, false);
  else SM3_REQUIRE(false, SM3_ERR_UNSUPPORTED_SHAPE, "gemm: MN-major A with K-major B is not instantiated");
#undef SM3_GEMM_LAUNCH_E
#undef SM3_GEMM_LAUNCH
  return check_launch("gemm_bf16x3_kernel");
}

}  // namespace gemm
}  // namespace sm3
