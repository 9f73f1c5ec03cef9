#!/usr/bin/env python
"""Side measurement (not the bench.py contract): backbone + mmdet FPN neck, forward and backward, batch 4 x 1024^2, fp32.

Two shipped single-dataset configs, with their backbone and neck dicts:
  dota_lsk_s_orcnn       LSKNet-S (local_configs/dota_lsk_s_orcnn.py), FPN [64, 128, 320, 512] -> 256, num_outs=5
  dota_convnext_t_orcnn  ConvNeXt-T without experts (local_configs/dota_convnext_t_orcnn.py), FPN [96, 192, 384, 768] -> 256
Both necks use the max-pool P6 (add_extra_convs=False).  Each config is timed with sm3det_b200.FPN and, as the comparator,
with the same CUDA backbone followed by the oracle's eager torch FPN (tests/fpn_mmdet_ref.py: F.conv2d, F.interpolate,
F.max_pool2d) on the same GPU, in fp32 and with TF32 allowed, as bench.py's comparator runs.  The neck alone is timed the
same way on the backbone's outputs.  The variants alternate --repeats times; the median is reported with the spread.  Card
name and power limit are read in the same process.

  python tools/bench_fpn.py [--batch 4] [--size 1024] [--steps 10] [--warmup 3] [--repeats 3] [--config NAME ...]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from sm3det_b200 import FPN, ConvNeXt_moe_MultiInput, LSKNet  # noqa: E402
from sm3det_b200.synth import make_images  # noqa: E402

SYNC_BN = dict(type='SyncBN', requires_grad=True)
CONFIGS = {
    'dota_lsk_s_orcnn': (LSKNet, dict(embed_dims=[64, 128, 320, 512], drop_rate=0.1, drop_path_rate=0.1, depths=[2, 2, 4, 2],
                                      norm_cfg=SYNC_BN),
                         dict(in_channels=[64, 128, 320, 512], out_channels=256, num_outs=5)),
    'dota_convnext_t_orcnn': (ConvNeXt_moe_MultiInput, dict(MoE_Block_inds=[[], [], [], []], datasets=None, arch='tiny',
                                                            drop_path_rate=0.1),
                              dict(in_channels=[96, 192, 384, 768], out_channels=256, num_outs=5)),
}


def device_info():
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


def _outs(res):
    """A backbone's feature tuple (the ConvNeXt MoE classes return (outs, gate_loss) when they have experts)."""
    return res[0] if isinstance(res[0], (tuple, list)) else res


def eager_neck(neck_kw, sd):
    """The oracle's torch FPN with the parameters of the CUDA neck (copied, on the GPU, requiring grad)."""
    import fpn_mmdet_ref as M
    sdg = {k: v.detach().clone().requires_grad_(True) for k, v in sd.items()}
    return (lambda feats: M.fpn_forward_mmdet(sdg, list(feats), neck_kw['num_outs'])), list(sdg.values())


def bench_config(a, name):
    cls, bb_kw, neck_kw = CONFIGS[name]
    torch.manual_seed(0)
    bb = cls(**bb_kw).cuda().train()
    neck = FPN(**neck_kw).cuda()
    x = make_images(a.batch, a.size, a.size, seed=3).cuda()
    ref_neck, ref_params = eager_neck(neck_kw, neck.state_dict())
    # the eager comparator runs as bench.py's does: fp32, and with TF32 allowed in cuDNN / cuBLAS
    necks = {'sm3det_b200.FPN': (neck, list(neck.parameters()), False), 'eager FPN fp32': (ref_neck, ref_params, False),
             'eager FPN tf32': (ref_neck, ref_params, True)}

    def clear(params):
        bb.zero_grad(set_to_none=True)
        for p in params:
            p.grad = None

    def full_step(which):
        fn, params, _ = necks[which]

        def step():
            outs = fn(_outs(bb(x)))
            sum(o.mean() for o in outs).backward()
            clear(params)
        return step

    with torch.no_grad():
        feats = [f.detach().clone() for f in _outs(bb(x))]
    feats = [f.requires_grad_(True) for f in feats]

    def neck_step(which):
        fn, params, _ = necks[which]

        def step():
            outs = fn(feats)
            sum(o.mean() for o in outs).backward()
            for f in feats:
                f.grad = None
            clear(params)
        return step

    tf32_default = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    with torch.no_grad():                         # the two necks compute the same pyramid
        got, want = neck(feats), ref_neck(feats)
    rel = max(float((g - w).abs().max() / w.abs().max()) for g, w in zip(got, want))
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32_default
    del got, want
    res = {'config': name, 'batch': a.batch, 'size': a.size, 'neck_max_rel_diff_vs_eager': rel,
           'levels': [list(f.shape[2:]) for f in feats]}
    for label, mk in (('backbone+neck', full_step), ('neck only', neck_step)):
        ts = {k: [] for k in necks}
        for _ in range(a.repeats):
            for k, (_, _, tf32) in necks.items():
                torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = tf32
                ts[k].append(timed(mk(k), a.steps, a.warmup))
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32_default
        row = {}
        for k, v in ts.items():
            ms = sorted(v)[len(v) // 2]
            row[k] = {'ms_per_step': ms, 'spread_ms': max(v) - min(v), 'images_per_s': a.batch / ms * 1e3}
        for k in ('eager FPN fp32', 'eager FPN tf32'):
            row[f'speedup_vs_{k.replace(" ", "_")}'] = row[k]['ms_per_step'] / row['sm3det_b200.FPN']['ms_per_step']
        res[label] = row
    del bb, neck, feats
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=4)
    ap.add_argument('--size', type=int, default=1024)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--config', nargs='*', choices=sorted(CONFIGS), default=list(CONFIGS))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_fpn.py measures on the GPU; no CUDA device found')
    res = {'metric': 'backbone + mmdet FPN, fwd+bwd, fp32 (median of alternating repeats)',
           'runs': [bench_config(a, n) for n in a.config]}
    res.update(device_info())
    print(json.dumps(res))


if __name__ == '__main__':
    main()
