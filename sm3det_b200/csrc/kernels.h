// Internal C++ launcher declarations (one per kernel family).  The public C ABI in
// include/sm3det_b200.h (capi.cu) forwards to these.  All pointers are device pointers owned by
// the caller; every launcher is stream-ordered, never allocates and never synchronises.
#pragma once
#include <cuda_runtime.h>

namespace sm3 {

const char* last_error();

// norm.cu ----------------------------------------------------------------------------------------
int layernorm_fwd(const float* x, const float* w, const float* b, float* y, float* stats, long long T, int C,
                  float eps, int out_mode, int H, int W, cudaStream_t stream);
// LayerNorm -> K-major bf16 hi|lo operand image (128-row tiles, same layout as gemm::pack_act); y (fp32) optional
int layernorm_fwd_img(const float* x, const float* w, const float* b, unsigned short* img, float* y, float* stats, long long T,
                      int C, float eps, cudaStream_t stream);
int layernorm_bwd(const float* dy, const float* x, const float* stats, const float* w, float* dx, float* dw,
                  float* db, long long T, int C, int in_mode, int H, int W, int dx_accum, cudaStream_t stream);
int stem_fwd(const float* x, const float* wt, const float* bias, const float* lnw, const float* lnb, float* y,
             float* conv_out, float* stats, int N, int Cin, int H, int W, int ps, int C0, float eps,
             cudaStream_t stream);
int stem_wgrad(const float* x, const float* du, float* dwt, float* dbias, int N, int Cin, int H, int W, int ps,
               int C0, cudaStream_t stream);

// stencil.cu -------------------------------------------------------------------------------------
// wt: depthwise taps transposed to [49][C]
int dwconv7_fwd(const float* x, const float* wt, const float* bias, const float* resid, float* y, int N, int H, int W,
                int C, cudaStream_t stream);
// dx (+)= corr(dy, flipped taps); the forward kernel is reused with flipped taps by the caller.
int dwconv7_wgrad(const float* x, const float* dy, float* dwt, float* dbias, int N, int H, int W, int C,
                  cudaStream_t stream);

// front.cu ---------------------------------------------------------------------------------------
// dwconv7 + bias + block LayerNorm in one pass; each of u / stats / v / img is written only when non-null
int dwconv7_ln_fwd(const float* x, const float* wt, const float* bias, const float* lnw, const float* lnb, float* u,
                   float* stats, float* v, unsigned short* img, int N, int H, int W, int C, float eps, cudaStream_t stream);

// moe.cu -----------------------------------------------------------------------------------------
struct RouterArgs {
  const float* v;        // [T,C] LN output
  const float* wp;       // [P,C] cosine_projector.weight
  const float* bp;       // [P]
  const float* sim;      // [P,E] sim_matrix (un-normalised)
  const float* temperature;  // [1]
  const float* w_noise;  // [C,E] or null
  const float* noise;    // [T,E] standard-normal draws or null (null => clean logits)
  int T, C, P, E, k;
  // outputs
  int* top_idx;          // [T,k]  (-1 => dropped pair, gate underflowed to 0)
  float* top_gate;       // [T,k]
  float* logits;         // [T,E] optional (clean logits; needed by backward)
  float* top_vals;       // [T,k+1] optional: selected (noisy) logits incl. the (k+1)-th threshold
  float* p_out;          // [T,P] optional: projection Wp v + bp (saved for backward)
  float* sigma;          // [T,E] optional: noise stddev softplus(v w_noise)+0.01 (noisy gating)
  int* top_idx_m;        // [T,min(k+1,E)] optional: all selected experts incl. the (k+1)-th
  float* partials;       // [nblocks][3E] per-block importance / load / hard-count partial sums (workspace)
  int nblocks;           // filled by router_blocks()
};
int router_blocks(int T);
int moe_router(const RouterArgs& a, cudaStream_t stream);

struct PlanArgs {
  const float* partials; int nblocks;   // from the router
  int T, E, k, max_m_tiles;
  // outputs
  float* importance;     // [E]
  float* load;           // [E]
  float* loss;           // [1]  = 1e-2 * (cv2(importance) + cv2(load))
  int* counts;           // [E] pairs per expert (hard count of gate > 0)
  int* seg_begin;        // [E] first slot of expert e (multiple of 128)
  int* seg_end;          // [E] seg_begin + counts
  int* cursor;           // [E] zeroed (used by moe_assign)
  int* tile_group;       // [max_m_tiles]
  int* num_m_tiles;      // [1]
};
int moe_plan(const PlanArgs& a, cudaStream_t stream);

// pair (t,j) -> slot; writes pair_token[slot] = t (caller pre-fills pair_token with -1)
int moe_assign(const int* top_idx, int T, int k, int E, const int* seg_begin, int* cursor, int* slot_of,
               int* pair_token, cudaStream_t stream);

// out[t,:] = resid[t,:] + rowscale[t] * gamma * sum_j gate[t,j] * o[slot_of[t,j],:]   (fixed j order)
int moe_combine(const float* o, const int* slot_of, const int* top_idx, const float* gate, const float* gamma, const float* resid,
                const float* row_scale, float* out, float* y_opt, int T, int C, int k, cudaStream_t stream);

int moe_combine_bwd(const float* dout, const float* o, const int* slot_of, const int* top_idx, const float* gate,
                    const float* gamma, const float* row_scale, float* d_o, float* dgate, float* dgamma, int T, int C,
                    int k, cudaStream_t stream);

struct RouterBwdArgs {
  const float* p;            // [T,P] saved projection (pre-normalisation, incl. bias)
  const float* sim;          // [P,E]
  const float* temperature;  // [1]
  const int* top_idx; const float* top_gate;   // [T,k]
  const float* dgate;        // [T,k] from moe_combine_bwd
  const float* logits;       // [T,E] clean logits saved by the router
  const float* importance;   // [E]
  const float* loss_scale;   // [1] device scalar: upstream grad of this layer's loss (or null)
  // noisy gating only (null for clean gating):
  const float* noise; const float* sigma; const float* top_vals; const int* top_idx_m; const float* load;
  float* dr;                 // [T,32] out: gradient w.r.t. v @ w_noise, zero padded to 32 columns
  int T, P, E, k;
  float* dp;                 // [T,P] out
  float* dsim_hat;           // [P,E] accumulated (pre-zeroed)
  float* dtemperature;       // [1]  accumulated
};
int moe_router_bwd(const RouterBwdArgs& a, cudaStream_t stream);
int moe_router_bwd_finalize(const float* dsim_hat, const float* sim, float* dsim, int P, int E, cudaStream_t stream);

// act.cu -----------------------------------------------------------------------------------------
struct ActPackArgs {
  const float* h;            // [R, W] FFN hidden pre-activation
  const float* da;           // [R, W] upstream gradient (mode 1) or null
  long long R; int W;
  int mode;                  // 0: gelu(h)   1: da * gelu'(h)   2: h   3: mode 1 + gelu(h) into pack_mn2 (one pass)
  const int* live_tiles;     // optional device scalar: only rows < live_tiles*128 hold data (MoE pair space)
  const int* tile_group;     // optional: group (expert) of each 128-row tile, for per-group column sums
  float* out_f32;            // optional [R, W]
  unsigned short* pack_k;    // optional K-major image (128-row tiles)
  unsigned short* pack_mn;   // optional MN-major image (reduction index = row)
  int mn_tile;               // tile width of pack_mn (128 for an A operand, the GEMM tile width for B)
  float* colsum;             // optional [groups][W], accumulated
  unsigned short* pack_mn2;  // mode 3: MN-major image of gelu(h) with tile width mn_tile2
  int mn_tile2;
};
int act_pack(const ActPackArgs& a, cudaStream_t stream);

// reduce.cu --------------------------------------------------------------------------------------
int colsum(const float* a, const float* b, const float* rs, const int* seg_begin, const int* seg_end, int G,
           float* out, long long rows, int C, cudaStream_t stream);
int gather_sum(const float* src, const int* slot_of, const float* add, float* out, int T, int C, int k,
               cudaStream_t stream);
int scale_rows(const float* x, const float* rs, const float* cs, float* out, long long rows, int C,
               cudaStream_t stream);

int gather_rows_peer(const float* const* bases, const int* const* token_lists, const int* src_rank, const int* src_row,
                     const float* scale, float* out, long long rows, int C, cudaStream_t stream);

struct EpPlanArgs {
  const int* allm;            // [W][2][E] all-gathered (pair counts, segment starts) of every rank
  const int* tile_group_s;    // local plan: expert of each 128-slot tile
  const int* num_tiles_s;     // local plan: live tile count (device scalar)
  const int* pair_token;      // [R_s] local slot -> token (-1 = padding)
  int W, me, E, R_s, cap;
  int* src_rank; int* src_slot;     // [cap]   expert side: where each of my rows comes from
  int* tile_group; int* num_tiles;  // [cap/128], [1]  grouped-GEMM schedule of my experts
  int* seg_begin; int* seg_end;     // [E/W]
  int* comb_rank; int* comb_row;    // [R_s]   source side: where each of my slots' outputs lives
  int* overflow;                    // [1]     max rows needed if it ever exceeded cap (else untouched)
};
int ep_plan(const EpPlanArgs& a, cudaStream_t stream);

// lsk.cu (LSKNet-MoE, BASELINE config 5) --------------------------------------------------------------
// wt: depthwise taps transposed to [ks*ks][C]; "same" padding dil*(ks-1)/2.  Instantiated: (3,1) (5,1) (7,3).
int dwconv_fwd(const float* x, const float* wt, const float* bias, const float* resid, float* y, int N, int H, int W, int C,
               int ks, int dil, cudaStream_t stream);
int dwconv_wgrad(const float* x, const float* dy, float* dwt, float* dbias, int N, int H, int W, int C, int ks, int dil,
                 cudaStream_t stream);
int colstat(const float* x, const float* sh1, const float* y, const float* sh2, const float* sc2, float* s1, float* s2,
            long long rows, int C, cudaStream_t stream);
int affine(const float* x1, const float* a1, const float* x2, const float* a2, const float* b, const float* add, float* out,
           long long rows, int C, cudaStream_t stream);
int mul(const float* a, const float* b, const float* add, float* out, long long n, cudaStream_t stream);
int dropout(const float* x, float* out, long long n, float p, unsigned long long seed, cudaStream_t stream);
int dropout_dev(const float* x, float* out, long long n, float p, const unsigned long long* seed_dev, cudaStream_t stream);
int mlp_mid_fwd(const float* h, const float* wt, const float* bias, const float* mask, float* a, int N, int H, int W, int C,
                float p, unsigned long long seed, const unsigned long long* seed_dev, cudaStream_t stream);
int mlp_mid_bwd(const float* h, const float* wt, const float* bias, const float* da, const float* mask, float* dh, float* dwt,
                float* dbias, int N, int H, int W, int C, float p, unsigned long long seed,
                const unsigned long long* seed_dev, cudaStream_t stream);
int lsk_agg(const float* a1, const float* a2, float* agg, int* amax, long long T, int Ch, cudaStream_t stream);
int conv7_c2(const float* x, const float* w, const float* b, float* y, int N, int H, int W, int act, cudaStream_t stream);
int conv7_c2_wgrad(const float* x, const float* dpre, float* dw, float* db, int N, int H, int W, cudaStream_t stream);
int lsk_mix(const float* a1, const float* a2, const float* sig, float* out, long long T, int Ch, cudaStream_t stream);
int lsk_mix_bwd_sig(const float* dout, const float* a1, const float* a2, const float* sig, float* dpre, long long T, int Ch,
                    cudaStream_t stream);
int lsk_mix_bwd_in(const float* dout, const float* sig, const float* dagg, const int* amax, float* da1, float* da2,
                   long long T, int Ch, cudaStream_t stream);
int im2col(const float* x, float* col, int N, int H, int W, int Cin, int ks, int stride, int pad, int Kp, int nchw,
           cudaStream_t stream);
int col2im(const float* dcol, float* dx, int N, int H, int W, int Cin, int ks, int stride, int pad, int Kp, int nchw,
           cudaStream_t stream);

// neck.cu (MultitaskFPN, SURVEY 8f rank 1) ---------------------------------------------------------------------
int upsample_add(const float* a, const float* b, float* out, int N, int H, int W, int h, int w, int C, cudaStream_t stream);
int upsample_add_bwd(const float* d, float* db, int N, int H, int W, int h, int w, int C, cudaStream_t stream);
int transpose_batched(const float* in, float* out, int B, int R, int Cc, cudaStream_t stream);
int fpn_export_pool(const float* in, float* const* outs, int N, int H, int W, int C, int L, cudaStream_t stream);
int fpn_export_pool_bwd(const float* const* douts, float* din, int N, int H, int W, int C, int L, cudaStream_t stream);


// rpn_head.cu ------------------------------------------------------------------------------------
namespace rpn {
long long rows(const int* shapes, int L);
int conv_fwd(const float* const* x, float* const* cls, float* const* reg, const int* shapes, int L, int Cin,
             const uint16_t* wimg, const float* bconv, const uint16_t* himg, const float* bhead, int ncls, int nreg,
             float* h_out, int passes, cudaStream_t stream);
int mid_bwd(const float* h, const float* const* dcls, const float* const* dreg, const int* shapes, int L, const float* whead,
            int ncls, int nreg, float* dpre, float* dwhead, float* dbhead, float* dbconv, cudaStream_t stream);
int conv_dx(const float* dpre, float* const* dx, const int* shapes, int L, int Cin, const uint16_t* wimg, int passes,
            cudaStream_t stream);
int tap_index(const int* shapes, int L, int* idx, cudaStream_t stream);
}  // namespace rpn

}  // namespace sm3
