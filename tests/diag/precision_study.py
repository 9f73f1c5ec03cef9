"""Measured answer to "would single-pass TF32 (or plain bf16) have been accurate enough?"  (VERDICT r01 item 9/15).

Emulates, on the CPU oracle, what each tensor-core operand format does to the FFN / expert / patchify GEMMs of the cfg2
backbone (ConvNeXt-T, E8 k2, one 1024^2 image, trained-like weights) -- forward AND backward GEMMs -- while everything the
CUDA path keeps in fp32 SIMT (router, LayerNorm, depthwise conv, combine) stays fp32:

  tf32_trunc : operands truncated to 10 mantissa bits (what a tf32 tensor-core MMA does to raw fp32 bits in smem)
  tf32_rn    : operands rounded to nearest-even at 10 bits (needs an extra rounding pass by the producer)
  bf16       : one bf16 pass (round to nearest) -- the AMP recipe
  bf16x3     : hi = truncated bf16, lo = rounded bf16 residual, hi*hi + hi*lo + lo*hi -- what sm3_gemm ships

and reports, against the unmodified fp32 oracle: max-norm relative error of the 4 outputs, gate-loss error, routing flips
and the largest (k)-vs-(k+1) logit gap among the flipped tokens (a flip with a large gap is a real routing change, not a
numerical tie), and the worst parameter-gradient error.  Test infrastructure: imports oracle/, never the product.

    python tests/diag/precision_study.py [--size 1024] [--modes tf32_trunc,tf32_rn,bf16,bf16x3]
"""
import argparse
import os
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from oracle import convnext_moe_oracle as O                      # noqa: E402
from oracle.cases import CFG2_KW, upstream_grads                 # noqa: E402
from sm3det_b200.synth import make_images, make_state_dict       # noqa: E402


def trunc_bits(x, keep):           # keep `keep` explicit mantissa bits, drop the rest (toward zero)
    mask = -(1 << (23 - keep))
    return (x.contiguous().view(torch.int32) & mask).view(torch.float32)


def round_bits(x, keep):           # round to nearest even at `keep` mantissa bits
    i = x.contiguous().view(torch.int32)
    sh = 23 - keep
    bias = ((i >> sh) & 1) + ((1 << (sh - 1)) - 1)
    return ((i + bias) & (-(1 << sh))).view(torch.float32)


def split_bf16(x):
    hi = trunc_bits(x, 7)
    lo = round_bits(x - hi, 7)
    return hi, lo


def emu_matmul(a, b_t, mode):
    """a [M,K] @ b_t[N,K]^T with both operands in the emulated format, fp32 accumulation."""
    if mode == 'fp32':
        return a @ b_t.t()
    if mode == 'tf32_trunc':
        return trunc_bits(a, 10) @ trunc_bits(b_t, 10).t()
    if mode == 'tf32_rn':
        return round_bits(a, 10) @ round_bits(b_t, 10).t()
    if mode == 'bf16':
        return round_bits(a, 7) @ round_bits(b_t, 7).t()
    if mode == 'bf16x3':
        ah, al = split_bf16(a)
        bh, bl = split_bf16(b_t)
        return al @ bh.t() + ah @ bl.t() + ah @ bh.t()
    raise ValueError(mode)


class EmuLinear(torch.autograd.Function):
    MODE = 'fp32'

    @staticmethod
    def forward(ctx, x, w, b):
        ctx.save_for_backward(x, w)
        y = emu_matmul(x.reshape(-1, x.shape[-1]), w, EmuLinear.MODE)
        if b is not None:
            y = y + b
        return y.reshape(*x.shape[:-1], w.shape[0])

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        dy2, x2 = dy.reshape(-1, dy.shape[-1]), x.reshape(-1, x.shape[-1])
        dx = emu_matmul(dy2, w.t().contiguous(), EmuLinear.MODE).reshape(x.shape)
        dw = emu_matmul(dy2.t().contiguous(), x2.t().contiguous(), EmuLinear.MODE)
        return dx, dw, dy2.sum(0)


def emu_ffn(x, sd, p):            # FFN.forward convnext_moe.py:397-405 with emulated GEMMs
    x = EmuLinear.apply(x, sd[p + 'pointwise_conv1.weight'], sd[p + 'pointwise_conv1.bias'])
    x = F.gelu(x)
    return EmuLinear.apply(x, sd[p + 'pointwise_conv2.weight'], sd[p + 'pointwise_conv2.bias'])


class _FProxy:
    """torch.nn.functional with the patchify convolutions (groups == 1: stem 4x4/s4, downsample 2x2/s2) lowered to the
    emulated GEMM; depthwise convs and everything else untouched."""

    def __getattr__(self, name):
        return getattr(F, name)

    @staticmethod
    def conv2d(x, w, b=None, stride=1, padding=0, dilation=1, groups=1):
        if groups != 1 or EmuLinear.MODE == 'fp32':
            return F.conv2d(x, w, b, stride, padding, dilation, groups)
        s = stride if isinstance(stride, int) else stride[0]
        Co, Ci, kh, kw = w.shape
        assert kh == s and kw == s and padding == 0
        N, _, H, W = x.shape
        cols = x.reshape(N, Ci, H // s, s, W // s, s).permute(0, 2, 4, 1, 3, 5).reshape(-1, Ci * s * s)
        y = EmuLinear.apply(cols, w.reshape(Co, -1), b)
        return y.reshape(N, H // s, W // s, Co).permute(0, 3, 1, 2)


def run(mode, cfg, sd, x, train):
    EmuLinear.MODE = mode
    O.ffn, O.F = (O._orig_ffn, F) if mode == 'fp32' else (emu_ffn, _FProxy())
    rec = []
    sdg = {k: (v.clone().requires_grad_(True) if train and 'ffn.mean' not in k and 'ffn.std' not in k else v) for k, v in sd.items()}
    with torch.set_grad_enabled(train):
        outs, loss = O.backbone_forward(sdg, cfg, x, train=train, record=rec)
    grads = None
    if train:
        (sum((o * g).sum() for o, g in zip(outs, upstream_grads(outs))) + loss).backward()
        grads = {k: v.grad for k, v in sdg.items() if getattr(v, 'grad', None) is not None}
    return [o.detach() for o in outs], loss.detach(), rec, grads


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--size', type=int, default=1024)
    ap.add_argument('--modes', default='tf32_trunc,tf32_rn,bf16,bf16x3')
    ap.add_argument('--no-train', action='store_true')
    a = ap.parse_args()
    torch.set_num_threads(os.cpu_count())
    O._orig_ffn = O.ffn
    kw = dict(CFG2_KW, noisy_gating=False)
    cfg = O.OracleConfig(**kw)
    sd = make_state_dict(O.param_shapes(cfg), 0, True)
    x = make_images(1, a.size, a.size, seed=1234)
    print(f'# precision study: ConvNeXt-T E8 k2 last-2 (cfg2 arch), 1x3x{a.size}x{a.size}, trained-like weights, torch {torch.__version__} CPU')
    print('# err = max|a-b| / max|b| vs the fp32 oracle; tolerance of the task: 1e-3, router top-k bit-exact except numerical ties')
    for train in ([False] if a.no_train else [False, True]):
        t0 = time.time()
        ref = run('fp32', cfg, sd, x, train)
        print(f'\n## {"train fwd+bwd (noisy_gating=False)" if train else "eval forward"}   (fp32 oracle: {time.time() - t0:.0f} s)')
        for mode in a.modes.split(','):
            outs, loss, rec, grads = run(mode, cfg, sd, x, train)
            errs = [float((o - r).abs().max() / r.abs().max()) for o, r in zip(outs, ref[0])]
            flips, worst_gap, tokens, scale = 0, 0.0, 0, 1.0
            for g, c in zip(rec, ref[2]):
                m = (g['top_idx'].sort(1).values != c['top_idx'].sort(1).values).any(1)
                tokens += m.numel()
                flips += int(m.sum())
                if m.any():
                    lg = c['logits'][m]
                    k = c['top_idx'].shape[1]
                    top = lg.topk(k + 1, dim=-1).values
                    worst_gap = max(worst_gap, float((top[:, k - 1] - top[:, k]).max()))
                    scale = float(c['logits'].abs().max())
            line = (f'{mode:11s} out errs {" ".join(f"{e:.2e}" for e in errs)} | gate-loss rel err '
                    f'{abs(float(loss) - float(ref[1])) / abs(float(ref[1])):.2e} | routing flips {flips}/{tokens}'
                    f' worst flipped gap {worst_gap:.2e} (max|logit| {scale:.1f})')
            if train:
                ge = {k: float((grads[k] - ref[3][k]).abs().max() / (ref[3][k].abs().max() + 1e-30)) for k in ref[3]}
                top = sorted(ge.items(), key=lambda kv: -kv[1])[:3]
                line += ' | worst grads ' + ', '.join(f'{k.split("stages.")[-1]} {v:.2e}' for k, v in top)
                line += f' | grads over 2e-3: {sum(v > 2e-3 for v in ge.values())}/{len(ge)}'
            print(line, flush=True)
    O.ffn, O.F = O._orig_ffn, F


if __name__ == '__main__':
    main()
