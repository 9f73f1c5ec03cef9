// Fused dense-FFN kernels for the narrow ConvNeXt stages (C <= 256): the [T, 4C] hidden tensor never leaves the SM.
//
// Reference math (mmrotate/models/backbones/convnext_moe.py): FFN.forward :397-405 inside
// ConvNeXtBlock._inner_forward :343-372 --   out = x + drop_path(gamma * (W2 gelu(W1 v + b1) + b2))   -- and what autograd
// derives for it (SURVEY.md Appendix F, steps 1-3).  Round 1 ran this as GEMM1 -> act_pack -> GEMM2 with the hidden
// tensor crossing HBM 4x in the forward and ~10x in the backward (805 MB per crossing at stage 0, bs 8); at C = 96 / 192
// those GEMMs are HBM streams (K or N <= 192), not tensor-bound.  Here one persistent CTA per SM walks 128-token tiles:
//
//   ffn_chain_kernel<MODE, HC>      per tile, per hidden chunk j of HC columns:
//        GEMM-a   acc_h[128 x HC]  = A1 . Wa1_j^T                      (wgmma, 3-pass split-bf16, register accumulator)
//        (MODE 1) acc_d[128 x HC]  = A2 . Wa2_j^T
//        middle   MODE 0: y = gelu(acc_h + b1_j)         MODE 1: y = acc_d * gelu'(acc_h + b1_j)
//                 -> split hi/lo -> shared memory, directly in the K-major SWIZZLE_64B operand layout
//        GEMM-b   acc_o[128 x C]  += y . Wb_j^T
//      final epilogue: MODE 0: out = resid + row_scale * gamma * (acc_o + b2), aux = acc_o + b2;   MODE 1: out = acc_o
//      MODE 0 = forward (A1 = v, Wa1 = W1, Wb = W2);  MODE 1 = backward into dv (A1 = v: the hidden pre-activation is
//      RECOMPUTED, A2 = dz, Wa1 = W1, Wa2 = (gamma W2)^T, Wb = W1^T) -- the tensor pipe has >2x slack on these shapes,
//      HBM does not, so nothing hidden-sized is saved by the forward at all.
//      MODE 2 = MODE 1 that also writes, from the middle stage's registers, the two weight-gradient operands as MN-major
//      SWIZZLE_128B images (dh = d * gelu'(h) and gelu(h), 128-column tiles, rows M .. ceil32(M) zero: the layout act_pack
//      writes) and db1 = sum_t dh (per-CTA shared-memory partials, one global atomic per column per CTA).
//      MODE 3 = MODE 2 for C = 192, where v and dz tiles do not both fit: A2 = dz alone, h is read from the forward's
//      saved fp32 h_in straight into the fragment layout instead of being recomputed.
//
// Not fused: the weight gradients (split-K GEMMs).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace sm3 {
namespace ffn {

struct ChainParams {
  // operands (all pre-split bf16 hi|lo tile images, see gemm_tc.cuh pack_act / pack_b)
  const uint16_t* a1;     // K-major image of A1 [M, C], 128-row tiles
  const uint16_t* a2;     // MODE 1: K-major image of A2 [M, C]
  const uint16_t* wa1;    // image of Wa1 [H4, C] packed with tile width HC
  const uint16_t* wa2;    // MODE 1: image of Wa2 [H4, C], tile width HC
  const uint16_t* wb;     // image of Wb [C, H4] packed with tile width C
  const float* bias1;     // [H4]
  const float* bias2;     // [C] or null
  const float* col_scale; // [C] or null (gamma)
  const float* row_scale; // [M] or null (drop-path)
  const float* resid;     // [M, C] or null (shortcut)
  float* out;             // [M, C]
  float* aux_out;         // [M, C] or null: acc_o + bias2 before scaling (y2, needed for dgamma)
  float* h_out;           // MODE 0: [M, H4] or null: hidden pre-activation A1 Wa1^T + b1 (saved for a GEMM-based backward)
  uint16_t* dh_mn;        // MODES 2, 3: MN-major image (128-column tiles) of dh = d * gelu'(h), wgrad1's dy operand
  uint16_t* act_mn;       // MODES 2, 3: MN-major image (128-column tiles) of gelu(h), wgrad2's x operand
  float* db1;             // MODES 2, 3: [H4] += column sums of dh
  const float* h_in;      // MODE 3: [M, H4] the saved pre-activation (b1 included) instead of its recompute
  int M, C, H4, HC, passes, mode;
  int debug;              // perf experiments only: bit0 = middle stage skips the GELU math, bit1 = skip the operand split/stores
};
int chain(const ChainParams& p, cudaStream_t stream);

// largest hidden chunk the shared-memory budget allows for (mode, C); 0 if the shape is unsupported
int chain_chunk(int mode, int C);

}  // namespace ffn
}  // namespace sm3
