"""Time OrientedRPNHead forward + backward at the SM3Det shape: batch 4 x 1024^2 through the 5-level pyramid (256^2 .. 16^2),
256 channels, 3 anchors (rpn_cls 256 -> 3, rpn_reg 256 -> 18).

    python tools/bench_rpn_head.py [--batch 4] [--size 1024] [--iters 20] [--warmup 3]

Arms, interleaved step by step in the same process:
  kernels  sm3det_b200.OrientedRPNHeadConvs (the fused implicit-GEMM head and its backward)
  library  the library's previous route: PatchEmbedFn (im2col + wgmma GEMM) for the 3x3 conv, torch ReLU, and one
           PatchEmbedFn 1x1 GEMM for the concatenated [rpn_cls; rpn_reg] (21 columns padded to 24: the GEMM needs N % 8 == 0)
  torch    the reference's ops (F.conv2d, F.relu) eagerly, fp32
  tf32     the same with TF32 convolutions
Prints one JSON line: ms per step (median), TFLOP/s from the FLOPs computed from shapes (forward 2 * positions *
(9 Cin 256 + 256 * 21), backward twice that), peak memory per arm, checksums, and the card's name, power limit and SM clock.
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    try:
        out = subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader'], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return dict(zip(q.split(','), [s.strip() for s in out[0].split(',')]))
    except Exception as e:                       # noqa: BLE001  (report what could not be read, do not guess)
        return {'error': str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=4)
    ap.add_argument('--size', type=int, default=1024)
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_rpn_head needs a GPU'
    from sm3det_b200 import OrientedRPNHeadConvs
    from sm3det_b200.lsk_functional import PatchEmbedFn

    dev = torch.device('cuda')
    C, A = 256, 3
    sizes = [a.size // s for s in (4, 8, 16, 32, 64)]
    g = torch.Generator(device=dev).manual_seed(0)
    feats = [torch.randn(a.batch, C, s, s, device=dev, generator=g) for s in sizes]
    dcls = [torch.randn(a.batch, A, s, s, device=dev, generator=g) for s in sizes]
    dreg = [torch.randn(a.batch, 6 * A, s, s, device=dev, generator=g) for s in sizes]
    head = OrientedRPNHeadConvs(C).to(dev)
    with torch.no_grad():
        for p in head.parameters():
            p.normal_(0, 0.02, generator=g)
    wc, bc = head.rpn_conv.weight, head.rpn_conv.bias
    wh = torch.cat([head.rpn_cls.weight, head.rpn_reg.weight, torch.zeros(3, C, 1, 1, device=dev)]).detach().requires_grad_(True)
    bh = torch.cat([head.rpn_cls.bias, head.rpn_reg.bias, torch.zeros(3, device=dev)]).detach().requires_grad_(True)
    xs = [f.clone().requires_grad_(True) for f in feats]

    def zero():
        for t in (*head.parameters(), wh, bh, *xs):
            t.grad = None

    def run_kernels():
        cls, reg = head(xs)
        torch.autograd.backward(cls + reg, dcls + dreg)
        return cls, reg, head.rpn_conv.weight.grad

    def run_library():
        cls, reg = [], []
        for x in xs:
            h = torch.relu(PatchEmbedFn.apply(x, wc, bc, 1, True))               # NHWC
            o = PatchEmbedFn.apply(h, wh, bh, 1, False).permute(0, 3, 1, 2)      # [N, 24, H, W]
            cls.append(o[:, :A])
            reg.append(o[:, A:7 * A])
        torch.autograd.backward(cls + reg, dcls + dreg)
        return cls, reg, wc.grad

    def run_torch():
        cls, reg = [], []
        for x in xs:
            h = F.relu(F.conv2d(x, wc, bc, padding=1))
            cls.append(F.conv2d(h, head.rpn_cls.weight, head.rpn_cls.bias))
            reg.append(F.conv2d(h, head.rpn_reg.weight, head.rpn_reg.bias))
        torch.autograd.backward(cls + reg, dcls + dreg)
        return cls, reg, wc.grad

    def tf32(flag):
        torch.backends.cudnn.allow_tf32 = flag
        torch.backends.cuda.matmul.allow_tf32 = flag

    arms = {'kernels': (run_kernels, False), 'library': (run_library, False), 'torch_fp32': (run_torch, False),
            'torch_tf32': (run_torch, True)}
    times = {k: [] for k in arms}
    peak, check = {}, {}
    for name, (fn, t32) in arms.items():                 # warm-up, peak memory and checksums, one arm at a time
        tf32(t32)
        for _ in range(a.warmup):
            zero()
            fn()
        torch.cuda.synchronize()
        zero()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        cls, reg, dw = fn()
        torch.cuda.synchronize()
        peak[name] = round((torch.cuda.max_memory_allocated() - base) / 2**20, 1)
        check[name] = dict(cls=sum(c.double().sum().item() for c in cls), reg=sum(r.double().sum().item() for r in reg),
                           dw=dw.double().sum().item(), dx0=xs[0].grad.double().abs().sum().item())
        del cls, reg, dw
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(len(arms) * a.iters)]
    i = 0
    for _ in range(a.iters):                             # interleaved timing
        for name, (fn, t32) in arms.items():
            tf32(t32)
            zero()
            ev[i][0].record()
            fn()
            ev[i][1].record()
            i += 1
    torch.cuda.synchronize()
    i = 0
    for _ in range(a.iters):
        for name in arms:
            times[name].append(ev[i][0].elapsed_time(ev[i][1]))
            i += 1
    tf32(False)
    positions = a.batch * sum(s * s for s in sizes)
    flop_fwd = 2 * positions * (9 * C * C + C * 7 * A)
    flop = 3 * flop_fwd
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    res = dict(workload=f'OrientedRPNHead fwd+bwd, batch {a.batch} x {a.size}^2, levels {sizes}, C={C}, {A} anchors',
               gflop_per_step=round(flop / 1e9, 1), ms=dict((k, round(v, 3)) for k, v in med.items()),
               ms_min=dict((k, round(min(v), 3)) for k, v in times.items()),
               tflops=dict((k, round(flop / (v * 1e-3) / 1e12, 1)) for k, v in med.items()),
               peak_mib=peak, checksum=check, iters=a.iters, card=card())
    print(json.dumps(res))


if __name__ == '__main__':
    main()
