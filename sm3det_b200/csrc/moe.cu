// Grid-level sparse-MoE routing kernels: cosine top-k router, dispatch plan, slot assignment and
// deterministic combine.  No host synchronisation anywhere (the reference syncs twice per layer:
// torch.nonzero at convnext_moe.py:254 and .cpu().numpy() at :259).
//
// Replaces (reference convnext_moe.py): CosineTopKGate.forward :99-106, noisy_top_k_gating
// :194-223, _prob_in_top_k :152-174, cv_squared :140-147, the loss in MoE_layer.forward :234-238,
// SparseDispatcher.__init__ :252-262 (plan), dispatch :264-266 (fused into the expert GEMM's
// A-operand gather), combine :269-284 (moe_combine, fixed summation order instead of index_add).
#include "common.cuh"
#include "kernels.h"

namespace sm3 {

constexpr int RT = 64;        // tokens per router block
constexpr int R_KC = 32;      // k-chunk of the projection GEMM
constexpr int R_MAXE = 16;    // experts <= 16 (one lane per expert in the statistics)
constexpr int R_MAXK = 8;

int router_blocks(int T) { return (T + RT - 1) / RT; }

__device__ __forceinline__ float softplus_f(float x) { return x > 20.f ? x : log1pf(expf(x)); }
__device__ __forceinline__ float normal_cdf(float v) { return 0.5f * (1.0f + erff(v * 0.70710678118654752440f)); }

template <int PJ>  // padded projection width 32 * PJ >= a.P
__global__ void __launch_bounds__(256, 2) moe_router_kernel(const RouterArgs a, int soft_load) {
  extern __shared__ float smem[];
  const int P = 32 * PJ, PR = a.P, E = a.E, C = a.C, k = a.k;   // PR = real width; padding columns are zero
  float* s_p = smem;                         // [RT][P+1]   projected tokens
  float* s_sim = s_p + RT * (P + 1);         // [E][P+1]    column-normalised sim matrix
  float* s_a = s_sim + E * (P + 1);          // [R_KC][RT+2]  (8-byte aligned rows: token pairs are read as one LDS.64)
  s_a += ((RT + E) * (P + 1)) & 1;           // (RT+E)*(P+1) floats precede it: keep the pairs 8-byte aligned for odd E
  float* s_b = s_a + R_KC * (RT + 2);        // [R_KC][P+1]
  float* s_red = s_b + R_KC * (P + 1);       // [8][3*R_MAXE]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long t0 = (long long)blockIdx.x * RT;

  // ---- normalised sim matrix: S[:,e] / max(||S[:,e]||, 1e-12)   (F.normalize(dim=0), :103) -----
  for (int e = warp; e < E; e += 8) {
    float ss = 0.f;
    for (int p = lane; p < PR; p += 32) { const float s = __ldg(a.sim + p * E + e); ss += s * s; }
    const float inv = 1.0f / fmaxf(sqrtf(warp_sum(ss)), 1e-12f);
    for (int p = lane; p < P; p += 32) s_sim[e * (P + 1) + p] = (p < PR) ? __ldg(a.sim + p * E + e) * inv : 0.f;
  }

  // ---- projection: p[t, :] = Wp v[t] + bp  (fp32 FMA; thread tile 8 tokens x PJ outputs) --------
  unsigned long long acc2[4][PJ];            // (token 2i, token 2i+1) x output j
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < PJ; ++j) acc2[i][j] = 0ull;
  // Staging is software-pipelined: the global loads of k-chunk i+1 (8 KB of tokens + P x 128 B of Wp per block) are in
  // flight in registers while chunk i is multiplied -- the un-pipelined version spent most of its time in `long
  // scoreboard` at the staging stores.
  constexpr int NLD = 2 + PJ;                      // float4 per thread per chunk: (RT + 32*PJ) rows x 8 float4 / 256 threads
  float4 pre[NLD];
  auto gload = [&](int k0) {
#pragma unroll
    for (int q = 0; q < NLD; ++q) {
      const int idx = tid + 256 * q, row = idx >> 3, c4 = (idx & 7) * 4;
      float4 v4 = make_float4(0.f, 0.f, 0.f, 0.f);
      if (row < RT) {
        const long long t = t0 + row;
        if (t < a.T) v4 = ldg_f4(a.v + t * C + k0 + c4);
      } else if (row - RT < PR) {
        v4 = ldg_f4(a.wp + (long long)(row - RT) * C + k0 + c4);
      }
      pre[q] = v4;
    }
  };
  auto sstore = [&]() {
#pragma unroll
    for (int q = 0; q < NLD; ++q) {
      const int idx = tid + 256 * q, row = idx >> 3, c4 = (idx & 7) * 4;
      const float e4[4] = {pre[q].x, pre[q].y, pre[q].z, pre[q].w};
      if (row < RT) {
#pragma unroll
        for (int e = 0; e < 4; ++e) s_a[(c4 + e) * (RT + 2) + row] = e4[e];
      } else {
#pragma unroll
        for (int e = 0; e < 4; ++e) s_b[(c4 + e) * (P + 1) + row - RT] = e4[e];
      }
    }
  };
  gload(0);
  for (int k0 = 0; k0 < C; k0 += R_KC) {
    __syncthreads();                                // previous chunk fully consumed
    sstore();
    __syncthreads();
    if (k0 + R_KC < C) gload(k0 + R_KC);
    // accumulators are token pairs (ffma2: two IEEE fp32 FMAs on a 64-bit pair)
#pragma unroll 4
    for (int kk = 0; kk < R_KC; ++kk) {
      unsigned long long av2[4], bv2[PJ];
#pragma unroll
      for (int i = 0; i < 4; ++i) av2[i] = *reinterpret_cast<const unsigned long long*>(s_a + kk * (RT + 2) + warp * 8 + 2 * i);
#pragma unroll
      for (int j = 0; j < PJ; ++j) {
        const unsigned int b = __float_as_uint(s_b[kk * (P + 1) + lane + 32 * j]);
        bv2[j] = (unsigned long long)b | ((unsigned long long)b << 32);
      }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < PJ; ++j)
          acc2[i][j] = ffma2(av2[i], bv2[j], acc2[i][j]);
    }
  }
#pragma unroll
  for (int j = 0; j < PJ; ++j) {
    const bool pin = lane + 32 * j < PR;
    const float bj = pin ? __ldg(a.bp + lane + 32 * j) : 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float acc_ij = __uint_as_float((unsigned int)(acc2[i >> 1][j] >> ((i & 1) * 32)));
      const float pv = pin ? acc_ij + bj : 0.f;
      s_p[(warp * 8 + i) * (P + 1) + lane + 32 * j] = pv;
      const long long t = t0 + warp * 8 + i;
      if (a.p_out && pin && t < a.T) a.p_out[t * PR + lane + 32 * j] = pv;
    }
  }
  __syncthreads();

  // ---- per-token gating (warp per token; every lane ends up holding all E logits) --------------
  const float tau = __ldg(a.temperature);
  const float scale = expf(fminf(tau, 4.605170185988092f /* log(1/0.01), :96 */));
  const int m = min(k + 1, E);
  float imp = 0.f, ld = 0.f, cnt = 0.f;   // lane e accumulates expert e
  for (int i = 0; i < 8; ++i) {
    const int tt = warp * 8 + i;
    const long long t = t0 + tt;
    if (t >= a.T) break;
    float pv[PJ];
    float ss = 0.f;
#pragma unroll
    for (int j = 0; j < PJ; ++j) { pv[j] = s_p[tt * (P + 1) + lane + 32 * j]; ss += pv[j] * pv[j]; }
    const float inv = 1.0f / fmaxf(sqrtf(warp_sum(ss)), 1e-12f);
#pragma unroll
    for (int j = 0; j < PJ; ++j) pv[j] *= inv;
    float clean[R_MAXE], sel[R_MAXE], sig[R_MAXE];
#pragma unroll
    for (int e = 0; e < R_MAXE; ++e) {
      if (e < E) {
        float d = 0.f;
#pragma unroll
        for (int j = 0; j < PJ; ++j) d = fmaf(pv[j], s_sim[e * (P + 1) + lane + 32 * j], d);
        clean[e] = warp_sum(d) * scale;
        sel[e] = clean[e];
        sig[e] = 1.f;
      }
    }
    if (a.noise) {   // noisy logits :200-204   (softplus(x @ w_noise) + 1e-2) * randn
      const float* vr = a.v + t * C;
#pragma unroll
      for (int e = 0; e < R_MAXE; ++e) {
        if (e < E) {
          float d = 0.f;
          for (int c = lane; c < C; c += 32) d = fmaf(__ldg(vr + c), __ldg(a.w_noise + (long long)c * E + e), d);
          sig[e] = softplus_f(warp_sum(d)) + 1e-2f;
          sel[e] = clean[e] + __ldg(a.noise + t * E + e) * sig[e];
        }
      }
    }
    if (a.logits && lane < E) {
      float cv = 0.f, sv = 1.f;
#pragma unroll
      for (int e = 0; e < R_MAXE; ++e) if (e == lane) { cv = clean[e]; sv = sig[e]; }
      a.logits[t * E + lane] = cv;
      if (a.sigma) a.sigma[t * E + lane] = sv;
    }
    // top-(k+1), ties -> lowest expert id
    int idx[R_MAXK + 1]; float val[R_MAXK + 1];
    unsigned taken = 0;
#pragma unroll
    for (int r = 0; r < R_MAXK + 1; ++r) {
      if (r < m) {
        float best = -INFINITY; int bi = 0;
#pragma unroll
        for (int e = 0; e < R_MAXE; ++e)
          if (e < E && !((taken >> e) & 1u) && sel[e] > best) { best = sel[e]; bi = e; }
        // all-(-inf)/NaN rows: keep first free expert
        if (best == -INFINITY) { for (int e = 0; e < E; ++e) if (!((taken >> e) & 1u)) { bi = e; break; } }
        taken |= 1u << bi; idx[r] = bi; val[r] = best;
      }
    }
    float g[R_MAXK]; float den = 0.f;
#pragma unroll
    for (int j = 0; j < R_MAXK; ++j) if (j < k) { g[j] = expf(val[j] - val[0]); den += g[j]; }
#pragma unroll
    for (int j = 0; j < R_MAXK; ++j) if (j < k) g[j] = g[j] / den;
    if (lane == 0) {
#pragma unroll
      for (int j = 0; j < R_MAXK; ++j) if (j < k) {
        a.top_idx[t * k + j] = g[j] > 0.f ? idx[j] : -1;     // dispatch is defined by gates > 0 (:254,259)
        a.top_gate[t * k + j] = g[j];
      }
      if (a.top_vals) {
#pragma unroll
        for (int r = 0; r < R_MAXK + 1; ++r) if (r < m) a.top_vals[t * m + r] = val[r];
      }
      if (a.top_idx_m) {
#pragma unroll
        for (int r = 0; r < R_MAXK + 1; ++r) if (r < m) a.top_idx_m[t * m + r] = idx[r];
      }
    }
    // statistics for expert e = lane
    if (lane < E) {
      float myg = 0.f;
#pragma unroll
      for (int j = 0; j < R_MAXK; ++j) if (j < k && idx[j] == lane) myg = g[j];
      imp += myg;
      if (myg > 0.f) cnt += 1.f;
      if (soft_load) {   // _prob_in_top_k :152-174
        float c_e = 0.f, n_e = 0.f, s_e = 1.f;
#pragma unroll
        for (int e = 0; e < R_MAXE; ++e) if (e == lane) { c_e = clean[e]; n_e = sel[e]; s_e = sig[e]; }
        const float thr_in = val[k], thr_out = val[k - 1];
        const bool is_in = n_e > thr_in;
        ld += normal_cdf((c_e - (is_in ? thr_in : thr_out)) / s_e);
      } else if (myg > 0.f) {
        ld += 1.f;
      }
    }
  }
  if (lane < E) { s_red[warp * 3 * R_MAXE + lane] = imp; s_red[warp * 3 * R_MAXE + R_MAXE + lane] = ld;
                  s_red[warp * 3 * R_MAXE + 2 * R_MAXE + lane] = cnt; }
  __syncthreads();
  if (tid < E) {
    float si = 0.f, sl = 0.f, sc = 0.f;
    for (int w = 0; w < 8; ++w) { si += s_red[w * 3 * R_MAXE + tid]; sl += s_red[w * 3 * R_MAXE + R_MAXE + tid];
                                  sc += s_red[w * 3 * R_MAXE + 2 * R_MAXE + tid]; }
    float* out = a.partials + (long long)blockIdx.x * 3 * E;
    out[tid] = si; out[E + tid] = sl; out[2 * E + tid] = sc;
  }
}

int moe_router(const RouterArgs& a, cudaStream_t stream) {
  SM3_REQUIRE(a.v && a.wp && a.bp && a.sim && a.temperature && a.top_idx && a.top_gate && a.partials,
              SM3_ERR_INVALID_ARG, "moe_router: null argument");
  SM3_REQUIRE(a.E >= 1 && a.E <= R_MAXE && a.k >= 1 && a.k <= R_MAXK && a.k <= a.E, SM3_ERR_UNSUPPORTED_SHAPE,
              "moe_router: E=%d k=%d unsupported (E<=16, k<=8, k<=E)", a.E, a.k);
  SM3_REQUIRE(a.P % 4 == 0 && a.P >= 4 && a.P <= 256 && a.C % R_KC == 0, SM3_ERR_UNSUPPORTED_SHAPE,
              "moe_router: P=%d C=%d unsupported (P multiple of 4 <= 256, C multiple of 32)", a.P, a.C);
  SM3_REQUIRE(!a.noise || a.w_noise, SM3_ERR_INVALID_ARG, "moe_router: noise needs w_noise");
  const int soft = (a.noise && a.k < a.E) ? 1 : 0;
  const int P = (a.P + 31) / 32 * 32, E = a.E;
  const size_t smem = sizeof(float) * ((size_t)RT * (P + 1) + (size_t)E * (P + 1) + R_KC * (RT + 2) + 1 + (size_t)R_KC * (P + 1) + 8 * 3 * R_MAXE);
  const int blocks = router_blocks(a.T);
#define SM3_ROUTER_CASE(PJ)                                                                                   \
  case PJ:                                                                                                    \
    cudaFuncSetAttribute(moe_router_kernel<PJ>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);      \
    moe_router_kernel<PJ><<<blocks, 256, smem, stream>>>(a, soft);                                            \
    break;
  switch (P / 32) {
    SM3_ROUTER_CASE(1) SM3_ROUTER_CASE(2) SM3_ROUTER_CASE(3) SM3_ROUTER_CASE(4)
    SM3_ROUTER_CASE(5) SM3_ROUTER_CASE(6) SM3_ROUTER_CASE(7) SM3_ROUTER_CASE(8)
    default: SM3_REQUIRE(false, SM3_ERR_UNSUPPORTED_SHAPE, "moe_router: P=%d", P);
  }
#undef SM3_ROUTER_CASE
  return check_launch("moe_router");
}

// ------------------------------------------------------------------------------------------------
// Plan: reduce the per-block partials in a fixed order, emit the load-balance loss and the padded
// expert segments (each expert's slot range starts at a multiple of 128 = GEMM tile rows).
__global__ void __launch_bounds__(1024) moe_plan_kernel(const PlanArgs a) {
  __shared__ float s_imp[R_MAXE], s_load[R_MAXE];
  __shared__ int s_cnt[R_MAXE];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (warp < a.E) {
    float si = 0.f, sl = 0.f, sc = 0.f;
    for (int b = lane; b < a.nblocks; b += 32) {
      const float* pb = a.partials + (long long)b * 3 * a.E;
      si += pb[warp]; sl += pb[a.E + warp]; sc += pb[2 * a.E + warp];
    }
    si = warp_sum(si); sl = warp_sum(sl); sc = warp_sum(sc);
    if (lane == 0) { s_imp[warp] = si; s_load[warp] = sl; s_cnt[warp] = (int)(sc + 0.5f); }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const int E = a.E;
    float cv[2] = {0.f, 0.f};
    if (E > 1) {
      for (int which = 0; which < 2; ++which) {
        const float* z = which ? s_load : s_imp;
        float mean = 0.f;
        for (int e = 0; e < E; ++e) mean += z[e];
        mean /= (float)E;
        float var = 0.f;
        for (int e = 0; e < E; ++e) { const float d = z[e] - mean; var += d * d; }
        var /= (float)(E - 1);
        cv[which] = var / (mean * mean + 1e-10f);
      }
    }
    *a.loss = (cv[0] + cv[1]) * 1e-2f;
    int pos = 0, tile = 0;
    for (int e = 0; e < E; ++e) {
      a.importance[e] = s_imp[e]; a.load[e] = s_load[e];
      const int c = s_cnt[e];
      a.counts[e] = c; a.seg_begin[e] = pos; a.seg_end[e] = pos + c; a.cursor[e] = 0;
      const int nt = (c + 127) / 128;
      for (int i = 0; i < nt && tile < a.max_m_tiles; ++i) a.tile_group[tile++] = e;
      pos += nt * 128;
    }
    *a.num_m_tiles = tile;
  }
}

int moe_plan(const PlanArgs& a, cudaStream_t stream) {
  SM3_REQUIRE(a.partials && a.importance && a.load && a.loss && a.counts && a.seg_begin && a.seg_end && a.cursor &&
              a.tile_group && a.num_m_tiles, SM3_ERR_INVALID_ARG, "moe_plan: null argument");
  SM3_REQUIRE(a.E >= 1 && a.E <= R_MAXE, SM3_ERR_UNSUPPORTED_SHAPE, "moe_plan: E=%d", a.E);
  SM3_REQUIRE(a.max_m_tiles >= (a.T * (long long)a.k + 127) / 128 + a.E, SM3_ERR_WORKSPACE,
              "moe_plan: tile map too small (%d)", a.max_m_tiles);
  moe_plan_kernel<<<1, 1024, 0, stream>>>(a);
  return check_launch("moe_plan");
}

// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) moe_assign_kernel(const int* __restrict__ top_idx, int npairs, int k, int E,
                                                        const int* __restrict__ seg_begin, int* __restrict__ cursor,
                                                        int* __restrict__ slot_of, int* __restrict__ pair_token) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  const int e = (p < npairs) ? __ldg(top_idx + p) : -1;
  int slot = -1;
  for (int e2 = 0; e2 < E; ++e2) {
    const unsigned mask = __ballot_sync(0xffffffffu, e == e2);
    if (mask == 0) continue;
    const int leader = __ffs(mask) - 1;
    int base = 0;
    if (lane == leader) base = atomicAdd(cursor + e2, __popc(mask));
    base = __shfl_sync(0xffffffffu, base, leader);
    if (e == e2) slot = __ldg(seg_begin + e2) + base + __popc(mask & ((1u << lane) - 1u));
  }
  if (p < npairs) {
    slot_of[p] = slot;
    if (slot >= 0) pair_token[slot] = p / k;
  }
}

int moe_assign(const int* top_idx, int T, int k, int E, const int* seg_begin, int* cursor, int* slot_of,
               int* pair_token, cudaStream_t stream) {
  SM3_REQUIRE(top_idx && seg_begin && cursor && slot_of && pair_token, SM3_ERR_INVALID_ARG, "moe_assign: null argument");
  const long long np = (long long)T * k;
  SM3_REQUIRE(np < (1LL << 31), SM3_ERR_UNSUPPORTED_SHAPE, "moe_assign: too many pairs");
  moe_assign_kernel<<<(unsigned)((np + 255) / 256), 256, 0, stream>>>(top_idx, (int)np, k, E, seg_begin, cursor, slot_of, pair_token);
  return check_launch("moe_assign");
}

// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) moe_combine_kernel(const float* __restrict__ o, const int* __restrict__ slot_of,
                                                         const int* __restrict__ top_idx,
                                                         const float* __restrict__ gate, const float* __restrict__ gamma,
                                                         const float* __restrict__ resid, const float* __restrict__ row_scale,
                                                         float* __restrict__ out, float* __restrict__ y_opt, long long total,
                                                         int C, int k) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int Q = C >> 2;
  const long long t = i / Q;
  const int c = (int)(i % Q) * 4;
  float4 y = make_float4(0.f, 0.f, 0.f, 0.f);
  // ascending expert id = the order the reference's expert-major index_add visits a token's pairs (:283)
  int last = -1;
  for (int r = 0; r < k; ++r) {
    int bj = -1, be = 0x7fffffff;
    for (int j = 0; j < k; ++j) {
      const int e = __ldg(top_idx + t * k + j);
      if (e > last && e < be) { be = e; bj = j; }
    }
    if (bj < 0) break;
    last = be;
    const int s = __ldg(slot_of + t * k + bj);
    if (s < 0) continue;
    const float g = __ldg(gate + t * k + bj);
    const float4 v = ldg_f4(o + (long long)s * C + c);
    y.x = __fadd_rn(y.x, __fmul_rn(g, v.x)); y.y = __fadd_rn(y.y, __fmul_rn(g, v.y));
    y.z = __fadd_rn(y.z, __fmul_rn(g, v.z)); y.w = __fadd_rn(y.w, __fmul_rn(g, v.w));
  }
  if (y_opt) *reinterpret_cast<float4*>(y_opt + t * C + c) = y;
  const float4 gm = gamma ? ldg_f4(gamma + c) : make_float4(1.f, 1.f, 1.f, 1.f);
  const float rs = row_scale ? __ldg(row_scale + t) : 1.0f;
  const float4 r = resid ? ldg_f4(resid + t * C + c) : make_float4(0.f, 0.f, 0.f, 0.f);
  float4 res;
  res.x = __fadd_rn(r.x, __fmul_rn(__fmul_rn(y.x, gm.x), rs)); res.y = __fadd_rn(r.y, __fmul_rn(__fmul_rn(y.y, gm.y), rs));
  res.z = __fadd_rn(r.z, __fmul_rn(__fmul_rn(y.z, gm.z), rs)); res.w = __fadd_rn(r.w, __fmul_rn(__fmul_rn(y.w, gm.w), rs));
  *reinterpret_cast<float4*>(out + t * C + c) = res;
}

int moe_combine(const float* o, const int* slot_of, const int* top_idx, const float* gate, const float* gamma, const float* resid,
                const float* row_scale, float* out, float* y_opt, int T, int C, int k, cudaStream_t stream) {
  SM3_REQUIRE(o && slot_of && top_idx && gate && out, SM3_ERR_INVALID_ARG, "moe_combine: null argument");   // gamma / resid optional (LSK fc1)
  SM3_REQUIRE(C % 4 == 0, SM3_ERR_UNSUPPORTED_SHAPE, "moe_combine: C=%d", C);
  const long long total = (long long)T * (C / 4);
  moe_combine_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(o, slot_of, top_idx, gate, gamma, resid, row_scale, out, y_opt, total, C, k);
  return check_launch("moe_combine");
}

// ------------------------------------------------------------------------------------------------
// Backward of combine (+ layer scale + drop-path):  out = resid + rs*gamma*y,  y[t] = sum_j g_j o[s_j]
//   dY = gamma*rs*dout ; d_o[s_j] = g_j*dY ; dgate[t,j] = <o[s_j], dY> ; dgamma += rs*dout*y
// Warp per token, lane owns channels lane+32i; dgamma partials live in registers across the warp's
// tokens and are flushed with one atomic per channel per warp.
template <int V>
__global__ void __launch_bounds__(256) moe_combine_bwd_kernel(const float* __restrict__ dout, const float* __restrict__ o,
                                                             const int* __restrict__ slot_of, const float* __restrict__ gate,
                                                             const float* __restrict__ gamma, const float* __restrict__ row_scale,
                                                             float* __restrict__ d_o, float* __restrict__ dgate,
                                                             float* __restrict__ dgamma, int T, int C, int k,
                                                             int tokens_per_warp) {
  const int gwarp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  float gm[V], adg[V];
#pragma unroll
  for (int i = 0; i < V; ++i) { gm[i] = __ldg(gamma + lane + 32 * i); adg[i] = 0.f; }
  const long long tb = (long long)gwarp * tokens_per_warp;
  for (int q = 0; q < tokens_per_warp; ++q) {
    const long long t = tb + q;
    if (t >= T) break;
    const float rs = row_scale ? __ldg(row_scale + t) : 1.0f;
    float dz[V], dy[V], y[V];
#pragma unroll
    for (int i = 0; i < V; ++i) { dz[i] = __ldg(dout + t * C + lane + 32 * i) * rs; dy[i] = dz[i] * gm[i]; y[i] = 0.f; }
    for (int j = 0; j < k; ++j) {
      const int s = __ldg(slot_of + t * k + j);
      if (s < 0) { if (lane == 0) dgate[t * k + j] = 0.f; continue; }
      const float g = __ldg(gate + t * k + j);
      float dot = 0.f;
#pragma unroll
      for (int i = 0; i < V; ++i) {
        const float ov = __ldg(o + (long long)s * C + lane + 32 * i);
        dot = fmaf(ov, dy[i], dot);
        y[i] = fmaf(g, ov, y[i]);
        d_o[(long long)s * C + lane + 32 * i] = g * dy[i];
      }
      dot = warp_sum(dot);
      if (lane == 0) dgate[t * k + j] = dot;
    }
#pragma unroll
    for (int i = 0; i < V; ++i) adg[i] = fmaf(dz[i], y[i], adg[i]);
  }
#pragma unroll
  for (int i = 0; i < V; ++i) atomicAdd(dgamma + lane + 32 * i, adg[i]);
}

// Any C (multiple of 4), optional gamma: warp per token, lanes stride over float4 channel quads; dgamma (if requested) is
// accumulated with one atomic per channel per token-group -- used by the LSKNet MoE layers whose output width is the MLP
// hidden size (up to 2048) and which have no layer scale of their own (lsk_moe.py:195-228).
__global__ void __launch_bounds__(256) moe_combine_bwd_generic_kernel(const float* __restrict__ dout, const float* __restrict__ o,
                                                                     const int* __restrict__ slot_of, const float* __restrict__ gate,
                                                                     const float* __restrict__ gamma, const float* __restrict__ row_scale,
                                                                     float* __restrict__ d_o, float* __restrict__ dgate,
                                                                     float* __restrict__ dgamma, int T, int C, int k) {
  const long long t = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (t >= T) return;
  const float rs = row_scale ? __ldg(row_scale + t) : 1.0f;
  for (int j = 0; j < k; ++j) {
    const int s = __ldg(slot_of + t * k + j);
    if (s < 0) { if (lane == 0) dgate[t * k + j] = 0.f; continue; }
    const float g = __ldg(gate + t * k + j);
    float dot = 0.f;
    for (int c = lane * 4; c < C; c += 128) {
      float4 dy = ldg_f4(dout + t * C + c);
      dy.x *= rs; dy.y *= rs; dy.z *= rs; dy.w *= rs;
      if (gamma) { const float4 gm = ldg_f4(gamma + c); dy.x *= gm.x; dy.y *= gm.y; dy.z *= gm.z; dy.w *= gm.w; }
      const float4 ov = ldg_f4(o + (long long)s * C + c);
      dot = fmaf(ov.x, dy.x, fmaf(ov.y, dy.y, fmaf(ov.z, dy.z, fmaf(ov.w, dy.w, dot))));
      *reinterpret_cast<float4*>(d_o + (long long)s * C + c) = make_float4(g * dy.x, g * dy.y, g * dy.z, g * dy.w);
    }
    dot = warp_sum(dot);
    if (lane == 0) dgate[t * k + j] = dot;
  }
  if (dgamma) {
    for (int c = lane * 4; c < C; c += 128) {
      float4 y = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int j = 0; j < k; ++j) {
        const int s = __ldg(slot_of + t * k + j);
        if (s < 0) continue;
        const float g = __ldg(gate + t * k + j);
        const float4 ov = ldg_f4(o + (long long)s * C + c);
        y.x = fmaf(g, ov.x, y.x); y.y = fmaf(g, ov.y, y.y); y.z = fmaf(g, ov.z, y.z); y.w = fmaf(g, ov.w, y.w);
      }
      const float4 dz = ldg_f4(dout + t * C + c);
      atomicAdd(dgamma + c, dz.x * rs * y.x); atomicAdd(dgamma + c + 1, dz.y * rs * y.y);
      atomicAdd(dgamma + c + 2, dz.z * rs * y.z); atomicAdd(dgamma + c + 3, dz.w * rs * y.w);
    }
  }
}

int moe_combine_bwd(const float* dout, const float* o, const int* slot_of, const int* top_idx, const float* gate,
                    const float* gamma, const float* row_scale, float* d_o, float* dgate, float* dgamma, int T, int C,
                    int k, cudaStream_t stream) {
  (void)top_idx;
  SM3_REQUIRE(dout && o && slot_of && gate && d_o && dgate, SM3_ERR_INVALID_ARG, "moe_combine_bwd: null argument");
  SM3_REQUIRE((gamma == nullptr) == (dgamma == nullptr), SM3_ERR_INVALID_ARG, "moe_combine_bwd: gamma and dgamma go together");
  static const int vlist[] = {1, 2, 3, 4, 5, 6, 8, 10, 12, 16, 20, 24, 32};
  bool fast = gamma && C % 32 == 0;
  if (fast) { fast = false; for (int v : vlist) if (C / 32 == v) fast = true; }
  if (!fast) {
    SM3_REQUIRE(C % 4 == 0, SM3_ERR_UNSUPPORTED_SHAPE, "moe_combine_bwd: C=%d must be a multiple of 4", C);
    moe_combine_bwd_generic_kernel<<<(unsigned)(((long long)T * 32 + 255) / 256), 256, 0, stream>>>(
        dout, o, slot_of, gate, gamma, row_scale, d_o, dgate, dgamma, T, C, k);
    return check_launch("moe_combine_bwd_generic");
  }
  long long warps = (long long)num_sms() * 32;
  int tpw = (int)((T + warps - 1) / warps);
  if (tpw < 8) tpw = 8;
  warps = ((long long)T + tpw - 1) / tpw;
  const int blocks = (int)((warps + 7) / 8);
  const int V_ = C / 32;
  SM3_V_DISPATCH(V_, (moe_combine_bwd_kernel<V><<<blocks, 256, 0, stream>>>(dout, o, slot_of, gate, gamma, row_scale, d_o, dgate, dgamma, T, C, k, tpw)));
  return check_launch("moe_combine_bwd");
}

// ------------------------------------------------------------------------------------------------
// Router backward.  Lane e of the token's warp owns expert e.  Per token:
//   dG_j   = dgate_j + c_imp[idx_j]                    c_imp = up * 0.01 * dCV2/d importance
//   dval_j = g_j (dG_j - sum_i g_i dG_i)               softmax over the k kept (noisy) logits
//   noisy & k < E (soft load, _prob_in_top_k :152-174):  z_e = (l_e - thr_e) / sigma_e,
//       dz_e = c_load[e] * pdf(z_e);  dl_e += dz_e / sigma_e;  dthr_e = -dz_e / sigma_e (flows into the
//       (k+1)-th noisy value for experts inside the top-k, into the k-th for the others);
//       dsigma_e = -dz_e z_e / sigma_e + eps_e * dnoisy_e;  dr_e = dsigma_e * sigmoid(r_e)
//   dl_e  += dnoisy_e ; dcos_e = dl_e * scale ; dtau += dl_e * l_e (if tau <= ln 100)
//   dphat  = sum_e dcos_e Shat[:,e] ; dShat[:,e] += dcos_e phat ; dp = (dphat - phat <phat,dphat>) / ||p||
// dp [T,P] and dr [T,32] feed tensor-core GEMMs on the host side (dWp, dw_noise, dv) and a colsum (dbp).
__device__ __forceinline__ void cv2_grad(const float* z, int E, float up, float* out /*smem [E]*/) {
  float m = 0.f;
  for (int e = 0; e < E; ++e) m += __ldg(z + e);
  m /= (float)E;
  float s2 = 0.f;
  for (int e = 0; e < E; ++e) { const float d = __ldg(z + e) - m; s2 += d * d; }
  if (E > 1) s2 /= (float)(E - 1);
  const float den = m * m + 1e-10f;
  for (int e = 0; e < E; ++e) {
    float g = 0.f;
    if (E > 1) g = 2.f * (__ldg(z + e) - m) / ((float)(E - 1) * den) - 2.f * m * s2 / ((float)E * den * den);
    out[e] = up * 1e-2f * g;
  }
}

template <int PJ>
__global__ void __launch_bounds__(256) moe_router_bwd_kernel(const RouterBwdArgs a, int tokens_per_warp) {
  extern __shared__ float smem[];
  const int P = 32 * PJ, PR = a.P, E = a.E, k = a.k;
  float* s_sim = smem;                 // [E][P+1] normalised
  float* s_dsim = s_sim + E * (P + 1); // [E][P+1] block accumulator
  __shared__ float s_cimp[R_MAXE], s_cload[R_MAXE];
  __shared__ float s_dtau;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool noisy = a.noise != nullptr;
  const bool soft = noisy && (k < E);
  for (int e = warp; e < E; e += 8) {
    float ss = 0.f;
    for (int p = lane; p < PR; p += 32) { const float s = __ldg(a.sim + p * E + e); ss += s * s; }
    const float inv = 1.0f / fmaxf(sqrtf(warp_sum(ss)), 1e-12f);
    for (int p = lane; p < P; p += 32) { s_sim[e * (P + 1) + p] = (p < PR) ? __ldg(a.sim + p * E + e) * inv : 0.f; s_dsim[e * (P + 1) + p] = 0.f; }
  }
  if (tid == 0) {
    s_dtau = 0.f;
    const float up = a.loss_scale ? __ldg(a.loss_scale) : 0.f;
    cv2_grad(a.importance, E, up, s_cimp);
    if (soft) cv2_grad(a.load, E, up, s_cload);
    else for (int e = 0; e < E; ++e) s_cload[e] = 0.f;
  }
  __syncthreads();
  const float tau = __ldg(a.temperature);
  const bool unclamped = tau <= 4.605170185988092f;
  const float scale = expf(fminf(tau, 4.605170185988092f));
  const int m = min(k + 1, E);
  float dtau = 0.f;
  const long long tb = ((long long)blockIdx.x * 8 + warp) * tokens_per_warp;
  for (int q = 0; q < tokens_per_warp; ++q) {
    const long long t = tb + q;
    if (t >= a.T) break;
    float pv[PJ]; float ss = 0.f;
#pragma unroll
    for (int j = 0; j < PJ; ++j) { pv[j] = (lane + 32 * j < PR) ? __ldg(a.p + t * PR + lane + 32 * j) : 0.f; ss += pv[j] * pv[j]; }
    const float nrm = fmaxf(sqrtf(warp_sum(ss)), 1e-12f);
    const float inv = 1.0f / nrm;
#pragma unroll
    for (int j = 0; j < PJ; ++j) pv[j] *= inv;                 // phat
    // --- gradient w.r.t. the (noisy) logit of expert `lane`
    float g[R_MAXK], dG[R_MAXK]; int idx[R_MAXK];
    float sdot = 0.f;
    bool mine_in = false;
#pragma unroll
    for (int j = 0; j < R_MAXK; ++j) if (j < k) {
      idx[j] = a.top_idx_m ? __ldg(a.top_idx_m + t * m + j) : __ldg(a.top_idx + t * k + j);
      g[j] = __ldg(a.top_gate + t * k + j);
      dG[j] = __ldg(a.dgate + t * k + j) + s_cimp[idx[j] < 0 ? 0 : idx[j]];
      sdot += g[j] * dG[j];
      mine_in = mine_in || (idx[j] == lane);
    }
    float dnz = 0.f;
#pragma unroll
    for (int j = 0; j < R_MAXK; ++j) if (j < k && idx[j] == lane) dnz += g[j] * (dG[j] - sdot);
    const float l_e = (lane < E) ? __ldg(a.logits + t * E + lane) : 0.f;
    float dl = 0.f, dr = 0.f;
    if (noisy) {
      // the gates depend on the noise scale sigma = softplus(r) + 0.01 whenever noise was added (also for k == E, where
      // the load falls back to the hard count, :219-222); the soft-load terms exist only for k < E
      float dsig = 0.f, sg = 1.f, ep = 0.f;
      if (lane < E) {
        sg = __ldg(a.sigma + t * E + lane);
        ep = __ldg(a.noise + t * E + lane);
      }
      if (soft) {
        const int idx_k = __ldg(a.top_idx_m + t * m + k);           // the (k+1)-th expert
        const float thr_in = __ldg(a.top_vals + t * m + k), thr_out = __ldg(a.top_vals + t * m + k - 1);
        float dthr = 0.f;
        if (lane < E) {
          const float z = (l_e - (mine_in ? thr_in : thr_out)) / sg;
          const float dz = s_cload[lane] * 0.3989422804014327f * __expf(-0.5f * z * z);
          dl = dz / sg;
          dthr = -dz / sg;
          dsig = -dz * z / sg;
        }
        const float sum_in = warp_sum(mine_in ? dthr : 0.f);
        const float sum_out = warp_sum(mine_in ? 0.f : dthr);
        if (lane == idx_k) dnz += sum_in;
        if (lane == idx[k - 1]) dnz += sum_out;
      }
      if (lane < E) {
        dsig += ep * dnz;
        dr = dsig * (1.0f - __expf(-(sg - 1e-2f)));                // sigmoid(r) from softplus(r) = sigma - 0.01
      }
      if (a.dr) a.dr[t * 32 + lane] = (lane < E) ? dr : 0.f;
    }
    dl += dnz;
    if (lane < E) dtau += dl * l_e;
    // --- cosine-similarity backward
    float dph[PJ];
#pragma unroll
    for (int j = 0; j < PJ; ++j) dph[j] = 0.f;
    for (int e = 0; e < E; ++e) {
      const float dcos = __shfl_sync(0xffffffffu, dl, e) * scale;
      if (dcos == 0.f) continue;
#pragma unroll
      for (int i = 0; i < PJ; ++i) {
        dph[i] = fmaf(dcos, s_sim[e * (P + 1) + lane + 32 * i], dph[i]);
        atomicAdd(&s_dsim[e * (P + 1) + lane + 32 * i], dcos * pv[i]);
      }
    }
    float pd = 0.f;
#pragma unroll
    for (int i = 0; i < PJ; ++i) pd = fmaf(pv[i], dph[i], pd);
    pd = warp_sum(pd);
#pragma unroll
    for (int i = 0; i < PJ; ++i) if (lane + 32 * i < PR) a.dp[t * PR + lane + 32 * i] = (dph[i] - pv[i] * pd) * inv;
  }
  dtau = warp_sum(dtau);
  if (lane == 0 && unclamped) atomicAdd(&s_dtau, dtau);
  __syncthreads();
  for (int i = tid; i < E * P; i += 256) {
    const int e = i / P, p = i % P;
    if (p < PR) atomicAdd(a.dsim_hat + p * E + e, s_dsim[e * (P + 1) + p]);
  }
  if (tid == 0) atomicAdd(a.dtemperature, s_dtau);
}

int moe_router_bwd(const RouterBwdArgs& a, cudaStream_t stream) {
  SM3_REQUIRE(a.p && a.sim && a.temperature && a.top_idx && a.top_gate && a.dgate && a.logits && a.importance && a.dp &&
              a.dsim_hat && a.dtemperature, SM3_ERR_INVALID_ARG, "moe_router_bwd: null argument");
  if (a.noise)
    SM3_REQUIRE(a.sigma && a.dr, SM3_ERR_INVALID_ARG, "moe_router_bwd: noisy gating needs sigma and dr");
  if (a.noise && a.k < a.E)
    SM3_REQUIRE(a.top_vals && a.top_idx_m && a.load, SM3_ERR_INVALID_ARG,
                "moe_router_bwd: the soft load (noisy, k < E) needs top_vals, top_idx_m and load");
  SM3_REQUIRE(a.P % 4 == 0 && a.P <= 256 && a.E <= R_MAXE && a.k <= R_MAXK, SM3_ERR_UNSUPPORTED_SHAPE, "moe_router_bwd: shape");
  const int Ppad = (a.P + 31) / 32 * 32;
  const size_t smem = sizeof(float) * 2 * (size_t)a.E * (Ppad + 1);
  long long warps = (long long)num_sms() * 16;
  int tpw = (int)((a.T + warps - 1) / warps);
  if (tpw < 4) tpw = 4;
  warps = ((long long)a.T + tpw - 1) / tpw;
  const int blocks = (int)((warps + 7) / 8);
#define SM3_RB_CASE(PJ) case PJ: moe_router_bwd_kernel<PJ><<<blocks, 256, smem, stream>>>(a, tpw); break;
  switch (Ppad / 32) {
    SM3_RB_CASE(1) SM3_RB_CASE(2) SM3_RB_CASE(3) SM3_RB_CASE(4) SM3_RB_CASE(5) SM3_RB_CASE(6) SM3_RB_CASE(7) SM3_RB_CASE(8)
    default: SM3_REQUIRE(false, SM3_ERR_UNSUPPORTED_SHAPE, "moe_router_bwd: P=%d", a.P);
  }
#undef SM3_RB_CASE
  return check_launch("moe_router_bwd");
}

// dS[:,e] = (dShat_e - Shat_e <Shat_e, dShat_e>) / max(||S_e||, 1e-12)      (F.normalize(dim=0) backward)
__global__ void moe_router_bwd_finalize_kernel(const float* __restrict__ dsim_hat, const float* __restrict__ sim,
                                               float* __restrict__ dsim, int P, int E) {
  const int e = blockIdx.x, lane = threadIdx.x;
  float ss = 0.f, sd = 0.f;
  for (int p = lane; p < P; p += 32) { const float s = __ldg(sim + p * E + e); ss += s * s; }
  const float nrm = fmaxf(sqrtf(warp_sum(ss)), 1e-12f);
  for (int p = lane; p < P; p += 32) sd += (__ldg(sim + p * E + e) / nrm) * __ldg(dsim_hat + p * E + e);
  sd = warp_sum(sd);
  for (int p = lane; p < P; p += 32) {
    const float sh = __ldg(sim + p * E + e) / nrm;
    dsim[p * E + e] += (__ldg(dsim_hat + p * E + e) - sh * sd) / nrm;
  }
}

int moe_router_bwd_finalize(const float* dsim_hat, const float* sim, float* dsim, int P, int E, cudaStream_t stream) {
  SM3_REQUIRE(dsim_hat && sim && dsim, SM3_ERR_INVALID_ARG, "moe_router_bwd_finalize: null argument");
  moe_router_bwd_finalize_kernel<<<E, 32, 0, stream>>>(dsim_hat, sim, dsim, P, E);
  return check_launch("moe_router_bwd_finalize");
}

}  // namespace sm3
