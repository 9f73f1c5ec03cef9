#!/usr/bin/env python
"""Side measurement (not the bench.py contract): fwd+bwd images/s of the SM3Det LSKNet-MoE backbones, bs=4 per GPU,
1024x1024, fp32, noisy gating + dropout as configured.
  --arch s: BASELINE config 5, LSKNet-S (configs/SM3Det/SM3Det_lsk_s.py:13-25)
  --arch t: LSKNet-T (configs/SM3Det/SM3Det_lsk_t.py:14-24, without drop path), widths [32, 64, 160, 256]
  --comparator: the same step through the oracle's torch ops on the same GPU, in the same call
  --gemm-tails: instead, event-timed cost of LSK-T's column-tail GEMMs (N = 16 / 80) against N = 32 / 96 at equal M, K
  python tools/bench_lsk.py [--arch s|t] [--batch 4] [--size 1024] [--steps 5] [--comparator] [--gemm-tails]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sm3det_b200 import LSKNet_moe_MultiInput  # noqa: E402
from sm3det_b200.synth import make_images  # noqa: E402

KW = dict(MoE_Block_inds_fc1=[[], [0], [0, 2], [0]], MoE_Block_inds_fc2=[[], [0], [0, 2], [0]], num_experts=4, top_k=2,
          embed_dims=[64, 128, 320, 512], depths=[2, 2, 4, 2], drop_rate=0.1, drop_path_rate=0.,
          norm_cfg=dict(type='SyncBN', requires_grad=True))
KW_T = dict(MoE_Block_inds_fc1=[[], [0, 2], [0, 2, 4, 6, 8], [0]], MoE_Block_inds_fc2=[[], [0, 2], [0, 2, 4, 6, 8], [0]],
            num_experts=4, top_k=2, embed_dims=[32, 64, 160, 256], depths=[3, 3, 5, 2], drop_rate=0.1, drop_path_rate=0.,
            norm_cfg=dict(type='SyncBN', requires_grad=True))
ARCH = {'s': ('LSKNet-S', KW), 't': ('LSKNet-T', KW_T)}


def device_info():
    """Card name and power limit, read in the same process as the measurement."""
    info = {'gpu': torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        info['power_limit'], info['max_sm_clock'] = [s.strip() for s in q.split(',')]
    except Exception as e:                     # noqa: BLE001  (reported, not hidden)
        info['power_limit'] = f'not read ({type(e).__name__})'
    return info


def timed(step, steps, warmup):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def bench_step(a, name, kw):
    torch.manual_seed(0)
    net = LSKNet_moe_MultiInput(**kw).cuda().train()
    x = make_images(a.batch, a.size, a.size, seed=3).cuda()

    def step():
        outs, loss = net(x)
        (sum(o.mean() for o in outs) + loss).backward()
        net.zero_grad(set_to_none=True)

    torch.cuda.reset_peak_memory_stats()
    ms = timed(step, a.steps, a.warmup)
    res = {'metric': f'{name} MoE backbone images/s (fwd+bwd)', 'value': a.batch / ms * 1e3, 'ms_per_step': ms,
           'batch': a.batch, 'size': a.size, 'peak_mem_gb': torch.cuda.max_memory_allocated() / 2 ** 30}
    if a.comparator:
        sd = {k: v.detach().clone() for k, v in net.state_dict().items()}
        del net
        torch.cuda.empty_cache()
        res['comparator'] = comparator(a, kw, sd, x)
    return res


def comparator(a, kw, sd, x):
    """The same training step through the oracle's torch ops (fp32, eager) on the same GPU."""
    from oracle.cases import lsk_plan, make_drop_masks
    from oracle.lsk_moe_oracle import LskConfig, lsk_backbone_forward
    cfg = LskConfig(**{k: v for k, v in kw.items() if k not in ('norm_cfg', 'drop_path_rate')})
    tokens, dshapes = lsk_plan(cfg, a.batch, a.size, a.size)
    noise = [torch.randn(t, cfg.num_experts, device='cuda') for t in tokens]
    drops = [m.cuda() for m in make_drop_masks(dshapes, cfg.drop_rate)] if cfg.drop_rate > 0 else None
    no_grad = ('running_', 'num_batches', '.mean', '.std')
    sdg = {k: (v.requires_grad_(True) if v.is_floating_point() and not any(t in k for t in no_grad) else v) for k, v in sd.items()}

    def step():
        outs, loss = lsk_backbone_forward(sdg, cfg, x, train=True, noise=noise, drop_masks=drops)
        (sum(o.mean() for o in outs) + loss).backward()
        for v in sdg.values():
            v.grad = None

    torch.cuda.reset_peak_memory_stats()
    ms = timed(step, max(2, a.steps // 2), 1)
    return {'what': 'oracle torch ops (eager fp32) on the same GPU', 'value': a.batch / ms * 1e3, 'ms_per_step': ms,
            'peak_mem_gb': torch.cuda.max_memory_allocated() / 2 ** 30}


def gemm_tails(a):
    """LSK-T's LSKblock 1x1 convs at batch a.batch, size a.size: conv1/conv2 forward (N = dim/2), conv dgrad (N = dim/2)
    and conv wgrad (dw[dim, dim/2]: N = dim/2), each against the same launch with N rounded up to its padded tile width."""
    from sm3det_b200 import ops
    out = []
    for dim, level in ((32, 4), (160, 16)):
        T = a.batch * (a.size // level) ** 2
        for half in (dim // 2, ops._pick_bn(dim // 2) * -(-(dim // 2) // ops._pick_bn(dim // 2))):
            g = torch.Generator(device='cuda').manual_seed(dim + half)
            x = torch.randn(T, dim, device='cuda', generator=g)
            w1 = torch.randn(half, dim, device='cuda', generator=g) * 0.1        # conv1: dim -> half
            w = torch.randn(dim, half, device='cuda', generator=g) * 0.1         # conv: half -> dim
            dy = torch.randn(T, dim, device='cuda', generator=g)
            h = torch.randn(T, half, device='cuda', generator=g)
            p1 = ops.pack_weight(w1, transposed=False)
            pt = ops.pack_weight(w, transposed=True)
            dw = torch.zeros(dim, half, device='cuda')
            cases = {'fwd conv1 (N=half, K=dim)': lambda: ops.linear_fwd(x, w1, packed=p1),
                     'dgrad conv (N=half, K=dim)': lambda: ops.linear_dgrad(dy, w, packed=pt),
                     'wgrad conv (M=dim, N=half, K=T)': lambda: ops.linear_wgrad(dy, h, dw)}
            for name, fn in cases.items():
                ms = timed(fn, 50, 5)
                out.append({'dim': dim, 'tokens': T, 'N': half, 'tile': ops._pick_bn(half), 'launch': name, 'us': ms * 1e3})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--arch', choices=sorted(ARCH), default='s')
    ap.add_argument('--batch', type=int, default=4)
    ap.add_argument('--size', type=int, default=1024)
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--comparator', action='store_true')
    ap.add_argument('--gemm-tails', action='store_true')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_lsk.py measures on the GPU; no CUDA device found')
    if a.gemm_tails:
        res = {'metric': 'LSK-T column-tail GEMMs, event-timed (50 launches each)', 'launches': gemm_tails(a)}
    else:
        res = bench_step(a, *ARCH[a.arch])
    res.update(device_info())
    print(json.dumps(res))


if __name__ == '__main__':
    main()
