// extern "C" boundary: thin forwarding layer from include/sm3det_b200.h to the C++ launchers.
#include "../../include/sm3det_b200.h"
#include "common.cuh"
#include "gemm_tc.cuh"
#include "kernels.h"
#include "ffn_fused.cuh"

using namespace sm3;

static inline cudaStream_t S(void* s) { return reinterpret_cast<cudaStream_t>(s); }

extern "C" {

int sm3_abi_version(void) { return SM3_ABI_VERSION; }
const char* sm3_last_error(void) { return sm3::last_error(); }

int sm3_device_supported(void) {
  int dev = 0, major = 0, minor = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) return 0;
  if (cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev) != cudaSuccess) return 0;
  return (major == 9 && minor == 0) ? 1 : 0;
}

int sm3_gemm(const sm3_gemm_args* a, void* stream) {
  if (!a) { set_last_error("sm3_gemm: null args"); return SM3_ERR_INVALID_ARG; }
  gemm::Params p{};
  p.A = a->A; p.a_smn = a->a_stride_mn; p.a_sk = a->a_stride_k;
  p.B = a->B; p.b_smn = a->b_stride_mn; p.b_sk = a->b_stride_k; p.b_group_stride = a->b_group_stride;
  p.a_row_index = a->a_row_index; p.b_k_index = a->b_k_index;
  p.b_packed = a->b_packed; p.b_packed_group_stride = a->b_packed_group_stride; p.a_packed = a->a_packed;
  p.M = a->M; p.N = a->N; p.K = a->K; p.BN = a->tile_n;
  p.sched = a->sched; p.k_splits = a->k_splits; p.num_groups = a->num_groups;
  p.tile_group = a->tile_group; p.num_m_tiles_dev = a->num_m_tiles;
  p.seg_begin = a->seg_begin; p.seg_end = a->seg_end;
  p.D = a->D; p.ldd = a->ldd; p.d_group_stride = a->d_group_stride;
  p.bias = a->bias; p.bias_group_stride = a->bias_group_stride;
  p.epi = a->epilogue;
  p.aux_out = a->aux_out; p.aux_in = a->aux_in; p.ld_aux = a->ld_aux;
  p.col_scale = a->col_scale; p.row_scale = a->row_scale;
  p.resid = a->resid; p.ld_resid = a->ld_resid;
  p.colsum = a->colsum; p.colsum_group_stride = a->colsum_group_stride;
  p.passes = (a->mma_passes == 1) ? 1 : 3;
  return gemm::launch(p, S(stream));
}

int64_t sm3_gemm_packed_elems(int32_t N, int32_t K) { return gemm::packed_elems(N, K); }
int sm3_gemm_pack_b(const float* B, int64_t s_mn, int64_t s_k, int64_t group_stride, int32_t groups, int32_t N, int32_t K,
                    uint16_t* out, void* stream) {
  return gemm::pack_b(B, s_mn, s_k, group_stride, groups, N, K, out, S(stream));
}

int64_t sm3_gemm_packed_act_elems(int64_t rows, int32_t cols, int32_t mn_major, int32_t tile) {
  return gemm::packed_act_elems(rows, cols, mn_major, tile);
}
int sm3_gemm_pack_act(const float* X, int64_t ld, const int32_t* row_index, int64_t rows, int32_t cols, int32_t mn_major,
                      int32_t tile, uint16_t* out, void* stream) {
  return gemm::pack_act(X, ld, row_index, rows, cols, mn_major, tile, out, S(stream));
}
int32_t sm3_gemm_tile_n(int32_t N) { return gemm::pick_bn(N); }
int sm3_gemm_pack_b_tile(const float* B, int64_t s_mn, int64_t s_k, int64_t group_stride, int32_t groups, int32_t N, int32_t K,
                         int32_t tile, uint16_t* out, void* stream) {
  return gemm::pack_b(B, s_mn, s_k, group_stride, groups, N, K, out, S(stream), tile);
}
size_t sm3_gemm_workspace_bytes(const sm3_gemm_args*) { return 0; }

int32_t sm3_ffn_fused_chunk(int32_t mode, int32_t C) { return (mode >= 0 && mode <= 3) ? ffn::chain_chunk(mode, C) : 0; }
size_t sm3_ffn_fused_workspace_bytes(const sm3_ffn_args*) { return 0; }
int sm3_ffn_fused(const sm3_ffn_args* a, void* stream) {
  if (!a) { set_last_error("sm3_ffn_fused: null args"); return SM3_ERR_INVALID_ARG; }
  ffn::ChainParams p{};
  p.a1 = a->a1; p.a2 = a->a2; p.wa1 = a->wa1; p.wa2 = a->wa2; p.wb = a->wb;
  p.bias1 = a->bias1; p.bias2 = a->bias2; p.col_scale = a->col_scale; p.row_scale = a->row_scale; p.resid = a->resid;
  p.out = a->out; p.aux_out = a->aux_out; p.h_out = a->h_out;
  p.dh_mn = a->dh_mn; p.act_mn = a->act_mn; p.db1 = a->db1; p.h_in = a->h_in;
  p.M = a->M; p.C = a->C; p.H4 = a->H4; p.HC = a->chunk; p.passes = a->mma_passes; p.mode = a->mode;
  return ffn::chain(p, S(stream));
}

int sm3_layernorm_fwd(const float* x, const float* w, const float* b, float* y, float* stats, int64_t T, int32_t C,
                      float eps, int32_t out_mode, int32_t H, int32_t W, void* stream) {
  return layernorm_fwd(x, w, b, y, stats, T, C, eps, out_mode, H, W, S(stream));
}
int sm3_layernorm_fwd_img(const float* x, const float* w, const float* b, uint16_t* img, float* y, float* stats, int64_t T,
                          int32_t C, float eps, void* stream) {
  return layernorm_fwd_img(x, w, b, img, y, stats, T, C, eps, S(stream));
}
int sm3_layernorm_bwd(const float* dy, const float* x, const float* stats, const float* w, float* dx, float* dw,
                      float* db, int64_t T, int32_t C, int32_t in_mode, int32_t H, int32_t W, int32_t dx_accum,
                      void* stream) {
  return layernorm_bwd(dy, x, stats, w, dx, dw, db, T, C, in_mode, H, W, dx_accum, S(stream));
}
int sm3_stem_fwd(const float* x, const float* wt, const float* bias, const float* lnw, const float* lnb, float* y,
                 float* conv_out, float* stats, int32_t N, int32_t Cin, int32_t H, int32_t W, int32_t ps, int32_t C0,
                 float eps, void* stream) {
  return stem_fwd(x, wt, bias, lnw, lnb, y, conv_out, stats, N, Cin, H, W, ps, C0, eps, S(stream));
}
int sm3_stem_wgrad(const float* x, const float* du, float* dwt, float* dbias, int32_t N, int32_t Cin, int32_t H,
                   int32_t W, int32_t ps, int32_t C0, void* stream) {
  return stem_wgrad(x, du, dwt, dbias, N, Cin, H, W, ps, C0, S(stream));
}
int sm3_dwconv7_fwd(const float* x, const float* wt, const float* bias, const float* resid, float* y, int32_t N,
                    int32_t H, int32_t W, int32_t C, void* stream) {
  return dwconv7_fwd(x, wt, bias, resid, y, N, H, W, C, S(stream));
}
int sm3_dwconv7_wgrad(const float* x, const float* dy, float* dwt, float* dbias, int32_t N, int32_t H, int32_t W,
                      int32_t C, void* stream) {
  return dwconv7_wgrad(x, dy, dwt, dbias, N, H, W, C, S(stream));
}
int sm3_dwconv7_ln_fwd(const float* x, const float* wt, const float* bias, const float* lnw, const float* lnb, float* u,
                       float* stats, float* v, uint16_t* img, int32_t N, int32_t H, int32_t W, int32_t C, float eps,
                       void* stream) {
  return dwconv7_ln_fwd(x, wt, bias, lnw, lnb, u, stats, v, img, N, H, W, C, eps, S(stream));
}

int sm3_moe_router_blocks(int32_t T) { return router_blocks(T); }
int sm3_moe_router(const sm3_router_args* a, void* stream) {
  if (!a) { set_last_error("sm3_moe_router: null args"); return SM3_ERR_INVALID_ARG; }
  RouterArgs r{};
  r.v = a->v; r.wp = a->proj_weight; r.bp = a->proj_bias; r.sim = a->sim_matrix; r.temperature = a->temperature;
  r.w_noise = a->w_noise; r.noise = a->noise;
  r.T = a->T; r.C = a->C; r.P = a->P; r.E = a->E; r.k = a->k;
  r.top_idx = a->top_idx; r.top_gate = a->top_gate; r.logits = a->logits; r.top_vals = a->top_vals; r.p_out = a->p_out; r.sigma = a->sigma; r.top_idx_m = a->top_idx_m;
  r.partials = a->partials; r.nblocks = router_blocks(a->T);
  return moe_router(r, S(stream));
}
size_t sm3_moe_router_workspace_bytes(const sm3_router_args* a) {
  return a ? (size_t)router_blocks(a->T) * 3u * (size_t)a->E * sizeof(float) : 0;
}
size_t sm3_moe_plan_workspace_bytes(const sm3_plan_args* a) {
  // importance[E] load[E] loss[1] floats + counts / seg_begin / seg_end / cursor [E] each + tile_group[max_m_tiles] + num_m_tiles[1] ints
  return a ? (size_t)(2 * a->E + 1) * sizeof(float) + (size_t)(4 * a->E + a->max_m_tiles + 1) * sizeof(int32_t) : 0;
}
int sm3_moe_plan(const sm3_plan_args* a, void* stream) {
  if (!a) { set_last_error("sm3_moe_plan: null args"); return SM3_ERR_INVALID_ARG; }
  PlanArgs p{};
  p.partials = a->partials; p.nblocks = router_blocks(a->T);
  p.T = a->T; p.E = a->E; p.k = a->k; p.max_m_tiles = a->max_m_tiles;
  p.importance = a->importance; p.load = a->load; p.loss = a->loss;
  p.counts = a->counts; p.seg_begin = a->seg_begin; p.seg_end = a->seg_end; p.cursor = a->cursor;
  p.tile_group = a->tile_group; p.num_m_tiles = a->num_m_tiles;
  return moe_plan(p, S(stream));
}
int sm3_moe_assign(const int32_t* top_idx, int32_t T, int32_t k, int32_t E, const int32_t* seg_begin, int32_t* cursor,
                   int32_t* slot_of, int32_t* pair_token, void* stream) {
  return moe_assign(top_idx, T, k, E, seg_begin, cursor, slot_of, pair_token, S(stream));
}
int sm3_moe_combine(const float* o, const int32_t* slot_of, const int32_t* top_idx, const float* gate,
                    const float* gamma, const float* resid, const float* row_scale, float* out, float* y_opt,
                    int32_t T, int32_t C, int32_t k, void* stream) {
  return moe_combine(o, slot_of, top_idx, gate, gamma, resid, row_scale, out, y_opt, T, C, k, S(stream));
}

int sm3_act_pack(const sm3_act_pack_args* a, void* stream) {
  if (!a) { set_last_error("sm3_act_pack: null args"); return SM3_ERR_INVALID_ARG; }
  ActPackArgs r{};
  r.h = a->h; r.da = a->da; r.R = a->R; r.W = a->W; r.mode = a->mode; r.live_tiles = a->live_tiles; r.tile_group = a->tile_group;
  r.out_f32 = a->out_f32; r.pack_k = a->pack_k; r.pack_mn = a->pack_mn; r.mn_tile = a->mn_tile; r.colsum = a->colsum;
  r.pack_mn2 = a->pack_mn2; r.mn_tile2 = a->mn_tile2;
  return act_pack(r, S(stream));
}
int sm3_moe_combine_bwd(const float* dout, const float* o, const int32_t* slot_of, const int32_t* top_idx,
                        const float* gate, const float* gamma, const float* row_scale, float* d_o, float* dgate,
                        float* dgamma, int32_t T, int32_t C, int32_t k, void* stream) {
  return moe_combine_bwd(dout, o, slot_of, top_idx, gate, gamma, row_scale, d_o, dgate, dgamma, T, C, k, S(stream));
}
int sm3_moe_router_bwd(const sm3_router_bwd_args* a, void* stream) {
  if (!a) { set_last_error("sm3_moe_router_bwd: null args"); return SM3_ERR_INVALID_ARG; }
  RouterBwdArgs r{};
  r.p = a->p; r.sim = a->sim_matrix; r.temperature = a->temperature; r.top_idx = a->top_idx; r.top_gate = a->top_gate;
  r.dgate = a->dgate; r.logits = a->logits; r.importance = a->importance; r.loss_scale = a->loss_scale;
  r.T = a->T; r.P = a->P; r.E = a->E; r.k = a->k; r.dp = a->dp; r.dsim_hat = a->dsim_hat; r.dtemperature = a->dtemperature;
  r.noise = a->noise; r.sigma = a->sigma; r.top_vals = a->top_vals; r.top_idx_m = a->top_idx_m; r.load = a->load; r.dr = a->dr;
  return moe_router_bwd(r, S(stream));
}
int sm3_moe_router_bwd_finalize(const float* dsim_hat, const float* sim, float* dsim, int32_t P, int32_t E, void* stream) {
  return moe_router_bwd_finalize(dsim_hat, sim, dsim, P, E, S(stream));
}
int sm3_colsum(const float* a, const float* b, const float* rs, const int32_t* seg_begin, const int32_t* seg_end,
               int32_t G, float* out, int64_t rows, int32_t C, void* stream) {
  return colsum(a, b, rs, seg_begin, seg_end, G, out, rows, C, S(stream));
}
int sm3_gather_sum(const float* src, const int32_t* slot_of, const float* add, float* out, int32_t T, int32_t C,
                   int32_t k, void* stream) {
  return gather_sum(src, slot_of, add, out, T, C, k, S(stream));
}
int sm3_scale_rows(const float* x, const float* rs, const float* cs, float* out, int64_t rows, int32_t C, void* stream) {
  return scale_rows(x, rs, cs, out, rows, C, S(stream));
}

int sm3_gather_rows_peer(const float* const* bases, const int32_t* const* token_lists, const int32_t* src_rank,
                         const int32_t* src_row, const float* scale, float* out, int64_t rows, int32_t C, void* stream) {
  return gather_rows_peer(bases, reinterpret_cast<const int* const*>(token_lists), src_rank, src_row, scale, out, rows, C, S(stream));
}
int sm3_dwconv_fwd(const float* x, const float* wt, const float* bias, const float* resid, float* y, int32_t N, int32_t H,
                   int32_t W, int32_t C, int32_t ks, int32_t dil, void* stream) {
  return dwconv_fwd(x, wt, bias, resid, y, N, H, W, C, ks, dil, S(stream));
}
int sm3_dwconv_wgrad(const float* x, const float* dy, float* dwt, float* dbias, int32_t N, int32_t H, int32_t W, int32_t C,
                     int32_t ks, int32_t dil, void* stream) {
  return dwconv_wgrad(x, dy, dwt, dbias, N, H, W, C, ks, dil, S(stream));
}
int sm3_colstat(const float* x, const float* sh1, const float* y, const float* sh2, const float* sc2, float* s1, float* s2,
                int64_t rows, int32_t C, void* stream) {
  return colstat(x, sh1, y, sh2, sc2, s1, s2, rows, C, S(stream));
}
int sm3_affine(const float* x1, const float* a1, const float* x2, const float* a2, const float* b, const float* add,
               float* out, int64_t rows, int32_t C, void* stream) {
  return affine(x1, a1, x2, a2, b, add, out, rows, C, S(stream));
}
int sm3_mul(const float* a, const float* b, const float* add, float* out, int64_t n, void* stream) {
  return mul(a, b, add, out, n, S(stream));
}
int sm3_dropout(const float* x, float* out, int64_t n, float p, uint64_t seed, void* stream) {
  return dropout(x, out, n, p, seed, S(stream));
}
int sm3_dropout_dev(const float* x, float* out, int64_t n, float p, const uint64_t* seed_dev, void* stream) {
  return dropout_dev(x, out, n, p, reinterpret_cast<const unsigned long long*>(seed_dev), S(stream));
}
int sm3_mlp_mid_fwd(const float* h, const float* weight_t, const float* bias, const float* mask, float* a, int32_t N,
                    int32_t H, int32_t W, int32_t C, float p, uint64_t seed, const uint64_t* seed_dev, void* stream) {
  return mlp_mid_fwd(h, weight_t, bias, mask, a, N, H, W, C, p, seed, reinterpret_cast<const unsigned long long*>(seed_dev),
                     S(stream));
}
int sm3_mlp_mid_bwd(const float* h, const float* weight_t, const float* bias, const float* da, const float* mask, float* dh,
                    float* dweight_t, float* dbias, int32_t N, int32_t H, int32_t W, int32_t C, float p, uint64_t seed,
                    const uint64_t* seed_dev, void* stream) {
  return mlp_mid_bwd(h, weight_t, bias, da, mask, dh, dweight_t, dbias, N, H, W, C, p, seed,
                     reinterpret_cast<const unsigned long long*>(seed_dev), S(stream));
}
int sm3_lsk_agg(const float* a1, const float* a2, float* agg, int32_t* amax, int64_t T, int32_t Ch, void* stream) {
  return lsk_agg(a1, a2, agg, amax, T, Ch, S(stream));
}
int sm3_conv7_c2(const float* x, const float* w, const float* b, float* y, int32_t N, int32_t H, int32_t W, int32_t act,
                 void* stream) {
  return conv7_c2(x, w, b, y, N, H, W, act, S(stream));
}
int sm3_conv7_c2_wgrad(const float* x, const float* dpre, float* dw, float* db, int32_t N, int32_t H, int32_t W, void* stream) {
  return conv7_c2_wgrad(x, dpre, dw, db, N, H, W, S(stream));
}
int sm3_lsk_mix(const float* a1, const float* a2, const float* sig, float* out, int64_t T, int32_t Ch, void* stream) {
  return lsk_mix(a1, a2, sig, out, T, Ch, S(stream));
}
int sm3_lsk_mix_bwd_sig(const float* dout, const float* a1, const float* a2, const float* sig, float* dpre, int64_t T,
                        int32_t Ch, void* stream) {
  return lsk_mix_bwd_sig(dout, a1, a2, sig, dpre, T, Ch, S(stream));
}
int sm3_lsk_mix_bwd_in(const float* dout, const float* sig, const float* dagg, const int32_t* amax, float* da1, float* da2,
                       int64_t T, int32_t Ch, void* stream) {
  return lsk_mix_bwd_in(dout, sig, dagg, amax, da1, da2, T, Ch, S(stream));
}
int sm3_im2col(const float* x, float* col, int32_t N, int32_t H, int32_t W, int32_t Cin, int32_t ks, int32_t stride,
               int32_t pad, int32_t Kp, int32_t nchw, void* stream) {
  return im2col(x, col, N, H, W, Cin, ks, stride, pad, Kp, nchw, S(stream));
}
int sm3_col2im(const float* dcol, float* dx, int32_t N, int32_t H, int32_t W, int32_t Cin, int32_t ks, int32_t stride,
               int32_t pad, int32_t Kp, int32_t nchw, void* stream) {
  return col2im(dcol, dx, N, H, W, Cin, ks, stride, pad, Kp, nchw, S(stream));
}

int sm3_ep_plan(const sm3_ep_plan_args* a, void* stream) {
  if (!a) { set_last_error("sm3_ep_plan: null args"); return SM3_ERR_INVALID_ARG; }
  EpPlanArgs p{};
  p.allm = a->allm; p.tile_group_s = a->tile_group_s; p.num_tiles_s = a->num_tiles_s; p.pair_token = a->pair_token;
  p.W = a->W; p.me = a->me; p.E = a->E; p.R_s = a->R_s; p.cap = a->cap;
  p.src_rank = a->src_rank; p.src_slot = a->src_slot; p.tile_group = a->tile_group; p.num_tiles = a->num_tiles;
  p.seg_begin = a->seg_begin; p.seg_end = a->seg_end; p.comb_rank = a->comb_rank; p.comb_row = a->comb_row; p.overflow = a->overflow;
  return ep_plan(p, S(stream));
}

int sm3_upsample_add(const float* a, const float* b, float* out, int32_t N, int32_t H, int32_t W, int32_t h, int32_t w,
                     int32_t C, void* stream) {
  return upsample_add(a, b, out, N, H, W, h, w, C, S(stream));
}
int sm3_upsample_add_bwd(const float* d, float* db, int32_t N, int32_t H, int32_t W, int32_t h, int32_t w, int32_t C,
                         void* stream) {
  return upsample_add_bwd(d, db, N, H, W, h, w, C, S(stream));
}
int sm3_transpose_batched(const float* in, float* out, int32_t B, int32_t R, int32_t Cc, void* stream) {
  return transpose_batched(in, out, B, R, Cc, S(stream));
}
int sm3_fpn_export_pool(const float* in, float* const* outs, int32_t N, int32_t H, int32_t W, int32_t C, int32_t L,
                        void* stream) {
  return fpn_export_pool(in, outs, N, H, W, C, L, S(stream));
}
int sm3_fpn_export_pool_bwd(const float* const* douts, float* din, int32_t N, int32_t H, int32_t W, int32_t C, int32_t L,
                            void* stream) {
  return fpn_export_pool_bwd(douts, din, N, H, W, C, L, S(stream));
}

int64_t sm3_rpn_head_rows(const int32_t* shapes, int32_t L) { return rpn::rows(shapes, L); }
int sm3_rpn_head_fwd(const float* const* x, float* const* cls, float* const* reg, const int32_t* shapes, int32_t L, int32_t Cin,
                     const uint16_t* wconv_img, const float* bconv, const uint16_t* whead_img, const float* bhead, int32_t ncls,
                     int32_t nreg, float* h_out, int32_t mma_passes, void* stream) {
  return rpn::conv_fwd(x, cls, reg, shapes, L, Cin, wconv_img, bconv, whead_img, bhead, ncls, nreg, h_out, mma_passes, S(stream));
}
int sm3_rpn_head_mid_bwd(const float* h, const float* const* dcls, const float* const* dreg, const int32_t* shapes, int32_t L,
                         const float* whead, int32_t ncls, int32_t nreg, float* dpre, float* dwhead, float* dbhead, float* dbconv,
                         void* stream) {
  return rpn::mid_bwd(h, dcls, dreg, shapes, L, whead, ncls, nreg, dpre, dwhead, dbhead, dbconv, S(stream));
}
int sm3_rpn_head_dx(const float* dpre, float* const* dx, const int32_t* shapes, int32_t L, int32_t Cin, const uint16_t* wdx_img,
                    int32_t mma_passes, void* stream) {
  return rpn::conv_dx(dpre, dx, shapes, L, Cin, wdx_img, mma_passes, S(stream));
}
int sm3_rpn_head_tap_index(const int32_t* shapes, int32_t L, int32_t* idx, void* stream) {
  return rpn::tap_index(shapes, L, idx, S(stream));
}

}  // extern "C"
