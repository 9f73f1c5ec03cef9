/* sm3det_b200 -- C ABI of the H100 (sm_90a) kernel library behind SM3Det's ConvNeXt-MoE backbone.
 *
 * The reference hot path is pure Python/PyTorch (mmrotate/models/backbones/convnext_moe.py); it has
 * no FFI of its own.  The closest analogue of this boundary is the `mmcv._ext` extension built at
 * mmcv/setup.py:238-296, which the backbone never calls.  Each entry point below therefore cites the
 * reference *Python* call site(s) it replaces (file:line relative to the SM3Det tree) -- that is the
 * place where a maintainer binds it (see INTEGRATION.md for the ctypes stub).
 *
 * Conventions
 *  - every pointer is a DEVICE pointer owned by the caller (PyTorch); the library never allocates,
 *    frees or retains memory past the call; workspaces are passed in explicitly;
 *  - tensors are fp32, contiguous, NHWC ("tokens x channels") unless stated; indices are int32;
 *  - `stream` is a cudaStream_t passed as void*; calls are stream-ordered, never synchronise and
 *    never touch the default stream implicitly;
 *  - return 0 on success, a negative SM3_ERR_* otherwise; sm3_last_error() returns a thread-local
 *    message; no C++ exception or STL type crosses the boundary.
 */
#ifndef SM3DET_B200_H_
#define SM3DET_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SM3_ABI_VERSION 1

#define SM3_OK 0
#define SM3_ERR_INVALID_ARG (-1)
#define SM3_ERR_UNSUPPORTED_SHAPE (-2)
#define SM3_ERR_CUDA (-3)
#define SM3_ERR_WORKSPACE (-4)

int sm3_abi_version(void);
const char* sm3_last_error(void);
/* 1 if the current device is compute capability 10.x (the only supported target), else 0 */
int sm3_device_supported(void);

/* ---- tensor-core GEMM ------------------------------------------------------------------------
 * D[M,N] = epilogue( sum_k A(m,k) * B(n,k) ), fp32 in HBM, split-bf16 (hi+lo) operands on wgmma,
 * fp32 register accumulation (product error ~1e-5 relative).
 * Replaces: FFN.forward nn.Linear/GELU/nn.Linear (convnext_moe.py:397-405), the expert loop
 * (:244) with its gather x[_batch_index] (:265), the 2x2/s2 downsample Conv2d (:549-558), and the
 * dgrad / wgrad GEMMs autograd derives for them.
 * Element (mn,k) of an operand is at ptr + mn*stride_mn + k*stride_k; exactly one stride is 1.
 */
enum { SM3_SCHED_DENSE = 0, SM3_SCHED_GROUPED = 1, SM3_SCHED_SPLITK = 2 };
enum {
  SM3_EPI_BIAS = 1,      /* acc += bias[n] */
  SM3_EPI_GELU = 2,      /* aux_out[m,n] = acc (if aux_out); acc = gelu_erf(acc) */
  SM3_EPI_DGELU = 4,     /* acc *= gelu_erf'(aux_in[m,n]) */
  SM3_EPI_COLSCALE = 8,  /* acc *= col_scale[n]   (layer scale gamma) */
  SM3_EPI_ROWSCALE = 16, /* acc *= row_scale[m]   (drop-path / gate) */
  SM3_EPI_RESID = 32,    /* acc += resid[m,n]     (shortcut) */
  SM3_EPI_ATOMIC = 64,   /* atomicAdd into D (split-K) */
  SM3_EPI_AUXSTORE = 128,/* aux_out[m,n] = acc after bias (no activation) */
  SM3_EPI_COLSUM = 256   /* colsum[group][n] += column sums of the final values (bias gradient fused in dgrad) */
};
typedef struct sm3_gemm_args {
  const float* A; int64_t a_stride_mn, a_stride_k;
  const float* B; int64_t b_stride_mn, b_stride_k, b_group_stride;
  const int32_t* a_row_index;      /* optional row gather of A (K-major A); -1 = zero row */
  const int32_t* b_k_index;        /* optional gather of B along the reduction index (MN-major B) */
  const uint16_t* b_packed;        /* optional pre-split weight image from sm3_gemm_pack_b (then B may be NULL) */
  int64_t b_packed_group_stride;   /* bf16 elements between the packed images of consecutive groups */
  const uint16_t* a_packed;        /* optional pre-split activation image from sm3_gemm_pack_act (needs b_packed) */
  int32_t M, N, K;
  int32_t tile_n;                  /* 0 = auto */
  int32_t sched;
  int32_t k_splits, num_groups;    /* SPLITK */
  const int32_t* tile_group;       /* GROUPED: expert id of each 128-row tile (device) */
  const int32_t* num_m_tiles;      /* GROUPED: device scalar, number of live 128-row tiles */
  const int32_t* seg_begin;        /* SPLITK: per-group reduction range (device), or NULL = [0,K) */
  const int32_t* seg_end;
  float* D; int64_t ldd, d_group_stride;
  const float* bias; int64_t bias_group_stride;
  int32_t epilogue;
  float* aux_out; const float* aux_in; int64_t ld_aux;
  const float* col_scale; const float* row_scale;
  const float* resid; int64_t ld_resid;
  float* colsum; int64_t colsum_group_stride;
  int32_t mma_passes;              /* 0 or 3: hi*hi + hi*lo + lo*hi (fp32-accurate, default); 1: hi*hi only = plain bf16
                                      operands with fp32 accumulation (the mixed-precision recipe, SURVEY 8f rank 2) */
} sm3_gemm_args;
int sm3_gemm(const sm3_gemm_args* args, void* stream);
/* Weights are constant across the tokens of a step: split them into bf16 hi/lo ONCE per optimizer step, already
 * in the tile order / swizzle the kernel's shared-memory stages use, so the GEMM brings a whole k-block of B in
 * with a single cp.async.bulk.  B(n,k) is read at B + n*stride_mn + k*stride_k (any majorness: the forward uses
 * W[N,K], the dgrad the same storage as B(n=k', k=n')).  Output: sm3_gemm_packed_elems(N,K) bf16 per group; N is
 * padded to whole tiles of sm3_gemm_tile_n(N) rows and the padding rows are written as zeros. */
int64_t sm3_gemm_packed_elems(int32_t N, int32_t K);
int sm3_gemm_pack_b(const float* B, int64_t stride_mn, int64_t stride_k, int64_t group_stride, int32_t groups,
                    int32_t N, int32_t K, uint16_t* out, void* stream);
/* Activation operands.  mn_major = 0: X[rows, cols=K] row-major (optional row gather = the MoE dispatch, -1 =
 * zero row) -> K-major tiles of `tile` rows (128 for A).  mn_major = 1: X[rows, cols] row-major whose ROW index is
 * the reduction index (wgrad operands; optional row gather) -> MN-major tiles of `tile` columns (128 for A, the
 * GEMM's tile width for B).  With both operands packed the GEMM main loop is two cp.async.bulk per k-block. */
int64_t sm3_gemm_packed_act_elems(int64_t rows, int32_t cols, int32_t mn_major, int32_t tile);
int sm3_gemm_pack_act(const float* X, int64_t ld, const int32_t* row_index, int64_t rows, int32_t cols,
                      int32_t mn_major, int32_t tile, uint16_t* out, void* stream);
/* Tile width the GEMM uses for an N-column output: the largest of 128/96/64/32 dividing N; for any other N % 8 == 0 the
 * last tile is padded and masked (fewest tiles, then least padding); 0 if N % 8 != 0. */
int32_t sm3_gemm_tile_n(int32_t N);
/* Same image with an explicit tile width (N % tile == 0): the fused FFN kernels stream weight chunks of their own width. */
int sm3_gemm_pack_b_tile(const float* B, int64_t stride_mn, int64_t stride_k, int64_t group_stride, int32_t groups,
                         int32_t N, int32_t K, int32_t tile, uint16_t* out, void* stream);
/* Workspace contract (SURVEY 8b): every op works on caller-owned buffers only.  sm3_gemm itself needs no scratch memory
 * (operand images are explicit arguments sized by sm3_gemm_packed_elems / sm3_gemm_packed_act_elems), so this returns 0;
 * it exists so that callers can size allocations uniformly through the C ABI. */
size_t sm3_gemm_workspace_bytes(const sm3_gemm_args* args);

/* ---- fused dense FFN for the narrow stages (C <= 192 forward, C <= 128 backward into dv) ------------------------------
 * The [M, 4C] hidden tensor is produced and consumed on chip (GEMM1 -> +b1 -> GELU -> bf16 hi/lo split -> shared memory ->
 * GEMM2 with register accumulators).  Replaces FFN.forward (convnext_moe.py:397-405) + layer scale / drop-path /
 * shortcut (:367-370) of dense ConvNeXt blocks.
 *   mode 0 (forward)     out = resid + row_scale * col_scale * (gelu(A1 Wa1^T + b1) Wb^T + bias2);  aux_out = pre-scale value;
 *                        h_out (optional) = A1 Wa1^T + b1, stored once for the GEMM-based backward
 *                        A1 = v, Wa1 = W1 [4C,C], Wb = W2 [C,4C]
 *   mode 1 (backward dv) out = ((A2 Wa2^T) * gelu'(A1 Wa1^T + b1)) Wb^T      (the hidden pre-activation is recomputed)
 *                        A1 = v, A2 = dz, Wa1 = W1, Wa2 = (gamma W2)^T stored [4C,C], Wb = W1^T stored [C,4C]
 *   mode 2 (backward dv + weight-gradient operands, C <= 128) mode 1, and also dh_mn / act_mn = the MN-major images
 *                        (sm3_gemm_packed_act_elems(M, 4C, 1, 128) elements each) of dh = (A2 Wa2^T) * gelu'(h) and of
 *                        gelu(h), rows M .. ceil32(M) zero; db1 += column sums of dh
 *   mode 3 (as mode 2, C = 192)  h is read from h_in (the forward's h_out) instead of recomputed; a1 / wa1 are unused
 * a1 / a2: K-major images from sm3_gemm_pack_act(tile 128) or sm3_layernorm_fwd_img; wa1 / wa2: sm3_gemm_pack_b_tile(tile =
 * chunk) of the [4C,C] matrices; wb: sm3_gemm_pack_b_tile(tile = C) of the [C,4C] matrix; chunk = sm3_ffn_fused_chunk(mode, C). */
typedef struct sm3_ffn_args {
  const uint16_t* a1; const uint16_t* a2;
  const uint16_t* wa1; const uint16_t* wa2; const uint16_t* wb;
  const float* bias1;              /* [4C] */
  const float* bias2;              /* [C]  mode 0 */
  const float* col_scale;          /* [C]  mode 0: gamma (optional) */
  const float* row_scale;          /* [M]  mode 0: drop-path scale (optional) */
  const float* resid;              /* [M,C] mode 0: shortcut (optional) */
  float* out;                      /* [M,C] modes 0, 1 */
  float* aux_out;                  /* [M,C] mode 0, optional */
  float* h_out;                    /* [M,4C] mode 0, optional: hidden pre-activation, for the GEMM-based backward */
  int32_t M, C, H4, chunk, mma_passes, mode;
  uint16_t* dh_mn; uint16_t* act_mn;   /* modes 2, 3 */
  float* db1;                      /* [4C] modes 2, 3: accumulated into */
  const float* h_in;               /* [M,4C] mode 3 */
} sm3_ffn_args;
int32_t sm3_ffn_fused_chunk(int32_t mode, int32_t C);   /* hidden chunk width for (mode, C); 0 = shape not supported */
int sm3_ffn_fused(const sm3_ffn_args* args, void* stream);
size_t sm3_ffn_fused_workspace_bytes(const sm3_ffn_args* args);   /* 0: accumulators live in registers, operands in smem */

/* ---- LayerNorm over channels (F.layer_norm, eps inside rsqrt, biased variance) ---------------
 * Replaces LayerNorm2d.forward (convnext_moe.py:34-47) at :351 (block norm), :549-551 (downsample
 * norm, written directly in 2x2-patch order for the following GEMM) and :811-817 (output norm incl.
 * the NHWC->NCHW permute+contiguous).  stats (optional) receives (mean, rstd) per token.
 */
enum { SM3_LN_NHWC = 0, SM3_LN_PATCH2 = 1, SM3_LN_NCHW = 2 };
int sm3_layernorm_fwd(const float* x, const float* weight, const float* bias, float* y, float* stats,
                      int64_t tokens, int32_t C, float eps, int32_t out_mode, int32_t H, int32_t W, void* stream);
/* Block LayerNorm (:351) fused with the operand split of the following pointwise GEMM: writes the K-major bf16 hi|lo image
 * (sm3_gemm_packed_act_elems(T, C, 0, 128) elements) that sm3_ffn_fused / sm3_gemm bulk-copy; y (fp32 [T,C]) is optional. */
int sm3_layernorm_fwd_img(const float* x, const float* weight, const float* bias, uint16_t* img, float* y, float* stats,
                          int64_t T, int32_t C, float eps, void* stream);
int sm3_layernorm_bwd(const float* dy, const float* x, const float* stats, const float* weight, float* dx,
                      float* dweight, float* dbias, int64_t tokens, int32_t C, int32_t in_mode, int32_t H,
                      int32_t W, int32_t dx_accumulate, void* stream);

/* ---- stem: LN(conv ps x ps / stride ps) NCHW -> NHWC ------------------------------------------
 * Replaces dataset_stems['single'] + downsample_layers[0] (convnext_moe.py:783-791, :800-806) and
 * the plain-class stem (:532-536).  weight_t is the conv weight transposed to [Cin*ps*ps][C0].
 */
int sm3_stem_fwd(const float* x_nchw, const float* weight_t, const float* bias, const float* ln_weight,
                 const float* ln_bias, float* y, float* conv_out, float* stats, int32_t N, int32_t Cin,
                 int32_t H, int32_t W, int32_t ps, int32_t C0, float eps, void* stream);
int sm3_stem_wgrad(const float* x_nchw, const float* dconv, float* dweight_t, float* dbias, int32_t N,
                   int32_t Cin, int32_t H, int32_t W, int32_t ps, int32_t C0, void* stream);

/* ---- 7x7 depthwise conv, NHWC ------------------------------------------------------------------
 * Replaces ConvNeXtBlock.depthwise_conv (convnext_moe.py:311-312, :347).  weight_t = taps as
 * [49][C].  dgrad = the same call on dy with the taps flipped; wgrad accumulates into dweight_t.
 */
int sm3_dwconv7_fwd(const float* x, const float* weight_t, const float* bias, const float* resid, float* y,
                    int32_t N, int32_t H, int32_t W, int32_t C, void* stream);
int sm3_dwconv7_wgrad(const float* x, const float* dy, float* dweight_t, float* dbias, int32_t N, int32_t H,
                      int32_t W, int32_t C, void* stream);
/* Block front in one pass: u = dwconv7(x) + bias (taps as [49][C]) and the block LayerNorm of u (:347-351).  Each output is
 * written only when its pointer is non-null: u [T,C], stats (mean, rstd) [T,2], v [T,C] and img, the K-major bf16 hi|lo
 * operand image of sm3_layernorm_fwd_img (C <= 256; rows of the last 128-row tile beyond T are zero).  C is a multiple of
 * 32, at most 1024.  Bit-identical to sm3_dwconv7_fwd followed by sm3_layernorm_fwd, or by sm3_layernorm_fwd_img when
 * img is requested (v and stats then follow that kernel's reduction order). */
int sm3_dwconv7_ln_fwd(const float* x, const float* weight_t, const float* bias, const float* ln_weight,
                       const float* ln_bias, float* u, float* stats, float* v, uint16_t* img, int32_t N, int32_t H,
                       int32_t W, int32_t C, float eps, void* stream);

/* ---- MoE routing --------------------------------------------------------------------------------
 * sm3_moe_router : CosineTopKGate.forward :99-106 + noisy_top_k_gating :194-223 (+ _prob_in_top_k
 *                  :152-174 when `noise` is given and k < E); true fp32 FMA so top-k is exact.
 * sm3_moe_plan   : importance/load reduction, cv_squared :140-147 and the loss :234-238, plus the
 *                  expert-major slot layout that SparseDispatcher.__init__ :252-262 builds with two
 *                  host syncs -- here entirely on device; segments start at multiples of 128 rows.
 * sm3_moe_assign : pair (token, j) -> slot, and pair_token[slot] = token (caller pre-fills -1).
 * sm3_moe_combine: SparseDispatcher.combine :269-284 + layer scale :367-368 + shortcut/drop-path
 *                  :370: out = resid + row_scale * gamma * sum_j gate_j * o[slot_j]  (ascending
 *                  expert order, no atomics).  gamma / resid / row_scale may be NULL (LSKNet MoE fc1,
 *                  lsk_moe.py:243-263: plain gate-weighted sum).
 */
typedef struct sm3_router_args {
  const float* v; const float* proj_weight; const float* proj_bias; const float* sim_matrix;
  const float* temperature; const float* w_noise; const float* noise;
  int32_t T, C, P, E, k;
  int32_t* top_idx; float* top_gate; float* logits; float* top_vals; float* p_out;
  float* sigma; int32_t* top_idx_m;   /* optional, noisy gating: noise stddev [T,E], experts [T,min(k+1,E)] */
  float* partials;                 /* [sm3_moe_router_blocks(T)][3*E] workspace */
} sm3_router_args;
int sm3_moe_router_blocks(int32_t T);
int sm3_moe_router(const sm3_router_args* args, void* stream);
size_t sm3_moe_router_workspace_bytes(const sm3_router_args* args);   /* bytes of `partials` for args->T, args->E */

typedef struct sm3_plan_args {
  const float* partials; int32_t T, E, k, max_m_tiles;
  float* importance; float* load; float* loss;
  int32_t* counts; int32_t* seg_begin; int32_t* seg_end; int32_t* cursor;
  int32_t* tile_group; int32_t* num_m_tiles;
} sm3_plan_args;
int sm3_moe_plan(const sm3_plan_args* args, void* stream);
size_t sm3_moe_plan_workspace_bytes(const sm3_plan_args* args);       /* bytes of all plan outputs laid out back to back */
int sm3_moe_assign(const int32_t* top_idx, int32_t T, int32_t k, int32_t E, const int32_t* seg_begin,
                   int32_t* cursor, int32_t* slot_of, int32_t* pair_token, void* stream);
int sm3_moe_combine(const float* expert_out, const int32_t* slot_of, const int32_t* top_idx, const float* gate,
                    const float* gamma, const float* resid, const float* row_scale, float* out, float* y_opt,
                    int32_t T, int32_t C, int32_t k, void* stream);

/* ---- fused activation + operand pre-split ---------------------------------------------------------
 * y = gelu(h) (mode 0) | da * gelu'(h) (mode 1) | h (mode 2) | both (mode 3: the whole backward in one pass over h) for the FFN hidden tensor, written directly as
 * the bf16 hi/lo tile images the following GEMMs bulk-copy (K-major image = A operand of GEMM2 / dgrad1,
 * MN-major image = wgrad operands), optionally also as fp32 and with per-group column sums (bias gradients).
 * Replaces nn.GELU() (convnext_moe.py:390,400) and its autograd backward; fp32 a / dh never reach HBM. */
typedef struct sm3_act_pack_args {
  const float* h; const float* da; int64_t R; int32_t W; int32_t mode;
  const int32_t* live_tiles; const int32_t* tile_group;
  float* out_f32; uint16_t* pack_k; uint16_t* pack_mn; int32_t mn_tile; float* colsum;
  uint16_t* pack_mn2; int32_t mn_tile2;   /* mode 3 only: MN-major image of gelu(h) (wgrad2's B operand) */
} sm3_act_pack_args;
int sm3_act_pack(const sm3_act_pack_args* args, void* stream);

/* ---- backward-only helpers ------------------------------------------------------------------------
 * (autograd derives these in the reference; each cites the forward statement it differentiates)
 * sm3_moe_combine_bwd : backward of combine/layer-scale/shortcut (convnext_moe.py:269-284,:367-370)
 * sm3_moe_router_bwd  : backward of softmax-of-k, cosine logits and the importance loss
 *                       (:99-106, :208-217, :234-238) for clean gating -> dp [T,P], d sim_hat, d tau
 * sm3_colsum          : out[g][c] += sum_r a[r,c]*(b?b[r,c]:1)*(rs?rs[r]:1) over rows of segment g
 *                       (bias / gamma gradients)
 * sm3_gather_sum      : out[t] = add[t] + sum_j src[slot_of[t,j]]  (backward of x[_batch_index], :265)
 * sm3_scale_rows      : out = x * row_scale[r] * col_scale[c]
 */
int sm3_moe_combine_bwd(const float* dout, const float* expert_out, const int32_t* slot_of, const int32_t* top_idx,
                        const float* gate, const float* gamma, const float* row_scale, float* d_expert_out,
                        float* dgate, float* dgamma, int32_t T, int32_t C, int32_t k, void* stream);
typedef struct sm3_router_bwd_args {
  const float* p; const float* sim_matrix; const float* temperature;
  const int32_t* top_idx; const float* top_gate; const float* dgate; const float* logits;
  const float* importance; const float* loss_scale;
  int32_t T, P, E, k;
  float* dp; float* dsim_hat; float* dtemperature;
  /* noisy gating (all NULL for clean gating): backward of :200-204 and _prob_in_top_k :152-174 */
  const float* noise; const float* sigma; const float* top_vals; const int32_t* top_idx_m; const float* load;
  float* dr;                          /* [T,32]: d(v @ w_noise), zero padded */
} sm3_router_bwd_args;
int sm3_moe_router_bwd(const sm3_router_bwd_args* args, void* stream);
int sm3_moe_router_bwd_finalize(const float* dsim_hat, const float* sim_matrix, float* dsim, int32_t P, int32_t E,
                                void* stream);
int sm3_colsum(const float* a, const float* b, const float* row_scale, const int32_t* seg_begin,
               const int32_t* seg_end, int32_t groups, float* out, int64_t rows, int32_t C, void* stream);
int sm3_gather_sum(const float* src, const int32_t* slot_of, const float* add, float* out, int32_t T, int32_t C,
                   int32_t k, void* stream);
int sm3_scale_rows(const float* x, const float* row_scale, const float* col_scale, float* out, int64_t rows,
                   int32_t C, void* stream);

/* ---- expert parallelism over NVLink peer memory (BASELINE config 4; beyond the reference, SURVEY 8e) -----------
 * sm3_gather_rows_peer: out[r,:] = scale[r] * bases[src_rank[r]][row*C ..], row = src_row[r] or, when token_lists is
 * given, token_lists[src_rank[r]][src_row[r]].  `bases` / `token_lists` are DEVICE arrays of `world` device pointers
 * into P2P-mapped (symmetric) buffers of the peer GPUs: the dispatch and combine all-to-alls of SparseDispatcher
 * (convnext_moe.py:264-284) become direct NVLink loads -- no staging copy, no NCCL call on the data path.
 * src_rank < 0 or row < 0 -> zero row. */
int sm3_gather_rows_peer(const float* const* bases, const int32_t* const* token_lists, const int32_t* src_rank,
                         const int32_t* src_row, const float* scale, float* out, int64_t rows, int32_t C, void* stream);

/* Expert-parallel exchange plan on the device (no host sync): from the all-gathered [W][2][E] (pair count, segment start)
 * table, the calling rank's expert-side gather lists / grouped-GEMM schedule and its source-side combine lists.  Replaces
 * the index bookkeeping of SparseDispatcher.__init__ (convnext_moe.py:252-262) for the expert-sharded layout. */
typedef struct sm3_ep_plan_args {
  const int32_t* allm; const int32_t* tile_group_s; const int32_t* num_tiles_s; const int32_t* pair_token;
  int32_t W, me, E, R_s, cap;
  int32_t* src_rank; int32_t* src_slot; int32_t* tile_group; int32_t* num_tiles; int32_t* seg_begin; int32_t* seg_end;
  int32_t* comb_rank; int32_t* comb_row; int32_t* overflow;
} sm3_ep_plan_args;
int sm3_ep_plan(const sm3_ep_plan_args* args, void* stream);

/* ---- LSKNet-MoE backbone (BASELINE config 5; mmrotate/models/backbones/lsk_moe.py) -------------------
 * sm3_dwconv_fwd / _wgrad : depthwise ks x ks conv, dilation dil, "same" padding, NHWC; weight_t = taps as
 *                           [ks*ks][C].  Replaces LSKblock.conv0 (5x5) :322, conv_spatial (7x7 dil 3) :323 and
 *                           DWConv (3x3) :583; dgrad = the same call on dy with flipped taps (+ resid).
 *                           Instantiated (ks,dil): (3,1) (5,1) (7,3).
 * sm3_colstat             : s1[c] += sum_r (x-sh1), s2[c] += sum_r (x-sh1) * (y ? (y-sh2)*sc2 : (x-sh1)).
 *                           BatchNorm2d batch statistics (shifted by running_mean, one pass) and the two
 *                           reductions of its backward (sum dy, sum dy*xhat).  Block.norm1/2 :369-374.
 * sm3_affine              : out = a1[c]*x1 + a2[c]*x2 + b[c] + add  -- BN normalise, BN backward, layer-scale +
 *                           residual (:388-395); NULL operands are skipped (a1 NULL = 1).
 * sm3_mul                 : out = a*b (+ add)  -- x * attn :343 and its backward.
 * sm3_lsk_agg             : channel mean / max (+argmax) of cat(attn1, attn2) :336-338.
 * sm3_conv7_c2 / _wgrad   : conv_squeeze Conv2d(2,2,7,padding=3) (+ sigmoid when act=1) :339; dgrad = the same call
 *                           with transposed + flipped weights, act=0.
 * sm3_lsk_mix (+bwd)      : attn1*sig[:,0] + attn2*sig[:,1] :340 and its backward into the sigmoid input / attn1,2.
 * sm3_im2col / sm3_col2im : OverlapPatchEmbed.proj (7x7/s4 stem from NCHW, 3x3/s2 downsamples from NHWC) :405-406
 *                           lowered to sm3_gemm; columns ordered (kh, kw, ci), zero padded to Kp.
 */
int sm3_dwconv_fwd(const float* x, const float* weight_t, const float* bias, const float* resid, float* y, int32_t N,
                   int32_t H, int32_t W, int32_t C, int32_t ks, int32_t dil, void* stream);
int sm3_dwconv_wgrad(const float* x, const float* dy, float* dweight_t, float* dbias, int32_t N, int32_t H, int32_t W,
                     int32_t C, int32_t ks, int32_t dil, void* stream);
int sm3_colstat(const float* x, const float* sh1, const float* y, const float* sh2, const float* sc2, float* s1, float* s2,
                int64_t rows, int32_t C, void* stream);
int sm3_affine(const float* x1, const float* a1, const float* x2, const float* a2, const float* b, const float* add,
               float* out, int64_t rows, int32_t C, void* stream);
int sm3_mul(const float* a, const float* b, const float* add, float* out, int64_t n, void* stream);
/* nn.Dropout (lsk_moe.py:300,311,316) with a counter-based mask: out = x * keep(seed, index) / (1-p); the same call on dy is
 * the backward (mask recomputed from the seed, nothing saved). */
int sm3_dropout(const float* x, float* out, int64_t n, float p, uint64_t seed, void* stream);
/* Same mask function with the seed read from device memory (one uint64): a captured CUDA graph replays the launch while the
 * seed tensor is refreshed between replays, so every step still draws a new mask. */
int sm3_dropout_dev(const float* x, float* out, int64_t n, float p, const uint64_t* seed_dev, void* stream);
/* Mlp middle stage (Mlp.forward :307-311): a = drop(gelu(dwconv3x3(h) + bias)) on NHWC h [N,H,W,C], C % 32 == 0,
 * weight_t = the 3x3 taps as [9][C].  Bit-identical to sm3_dwconv_fwd(ks 3) -> sm3_act_pack(GELU) -> sm3_dropout / sm3_mul
 * with the same seed or mask; nothing but h is needed for the backward.  Dropout: mask != NULL multiplies by that
 * pre-scaled keep mask; else p > 0 applies the sm3_dropout mask of `seed` (of *seed_dev when seed_dev != NULL, as
 * sm3_dropout_dev); else none.
 * sm3_mlp_mid_bwd: dh (bit-identical to the dgrad of that sequence) and dweight_t / dbias ACCUMULATED (+=) from da in one
 * pass that recomputes gelu(dwconv(h)) from h. */
int sm3_mlp_mid_fwd(const float* h, const float* weight_t, const float* bias, const float* mask, float* a, int32_t N,
                    int32_t H, int32_t W, int32_t C, float p, uint64_t seed, const uint64_t* seed_dev, void* stream);
int sm3_mlp_mid_bwd(const float* h, const float* weight_t, const float* bias, const float* da, const float* mask, float* dh,
                    float* dweight_t, float* dbias, int32_t N, int32_t H, int32_t W, int32_t C, float p, uint64_t seed,
                    const uint64_t* seed_dev, void* stream);
int sm3_lsk_agg(const float* a1, const float* a2, float* agg, int32_t* amax, int64_t T, int32_t Ch, void* stream);
int sm3_conv7_c2(const float* x, const float* w, const float* b, float* y, int32_t N, int32_t H, int32_t W, int32_t act,
                 void* stream);
int sm3_conv7_c2_wgrad(const float* x, const float* dpre, float* dw, float* db, int32_t N, int32_t H, int32_t W, void* stream);
int sm3_lsk_mix(const float* a1, const float* a2, const float* sig, float* out, int64_t T, int32_t Ch, void* stream);
int sm3_lsk_mix_bwd_sig(const float* dout, const float* a1, const float* a2, const float* sig, float* dpre, int64_t T,
                        int32_t Ch, void* stream);
int sm3_lsk_mix_bwd_in(const float* dout, const float* sig, const float* dagg, const int32_t* amax, float* da1, float* da2,
                       int64_t T, int32_t Ch, void* stream);
int sm3_im2col(const float* x, float* col, int32_t N, int32_t H, int32_t W, int32_t Cin, int32_t ks, int32_t stride,
               int32_t pad, int32_t Kp, int32_t nchw, void* stream);
int sm3_col2im(const float* dcol, float* dx, int32_t N, int32_t H, int32_t W, int32_t Cin, int32_t ks, int32_t stride,
               int32_t pad, int32_t Kp, int32_t nchw, void* stream);

/* ---- MultitaskFPN (the consumer of the 4-tuple; mmrotate/models/necks/Multitask_FPN.py:108-162) -----------------
 * Lateral 1x1 / output 3x3 convolutions = sm3_im2col + sm3_gemm.  sm3_upsample_add: laterals[i-1] +
 * F.interpolate(laterals[i], size=prev_shape, mode='nearest') :123-134 (NHWC) and its backward into the coarse level.
 * sm3_transpose_batched: out[b,c,r] = in[b,r,c] -- NHWC <-> NCHW conversion of the returned levels. */
int sm3_upsample_add(const float* a, const float* b, float* out, int32_t N, int32_t H, int32_t W, int32_t h, int32_t w,
                     int32_t C, void* stream);
int sm3_upsample_add_bwd(const float* d, float* db, int32_t N, int32_t H, int32_t W, int32_t h, int32_t w, int32_t C,
                         void* stream);
int sm3_transpose_batched(const float* in, float* out, int32_t B, int32_t R, int32_t Cc, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SM3DET_B200_H_ */
