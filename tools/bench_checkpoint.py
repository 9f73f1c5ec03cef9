"""Cost and saving of activation checkpointing (`with_cp=True`) on the bench.py cfg2 workload (ConvNeXt-T, E=8, k=2, noisy
gating, 1024^2 images, fp32-accurate GEMMs), whole 32-image step captured in a CUDA graph.

    python tools/bench_checkpoint.py [--steps 5] [--warmup 2] [--out results.json]

Prints one JSON object:
  steps:   for with_cp off/on and 16- or 32-image passes: img/s over the 32-image step and max_memory_allocated, or the error
           when the step (with its graph) does not fit;
  kernels: the fused dwconv7 + LayerNorm kernel vs dwconv7 -> layernorm_fwd[_img] at each cfg2 stage shape of a 16-image
           pass, event-timed (median of the repetitions), for the outputs the checkpointed forward and its recompute ask for;
  gpu:     the card name and power limit of this run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import CONFIGS  # noqa: E402  (the workload definition bench.py times; read only)


def gpu_info():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i',
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in q.split(',')]
    except Exception:            # noqa: BLE001 -- nvidia-smi missing: report the name torch knows
        name, power = torch.cuda.get_device_name(), 'unknown'
    return dict(name=name, power_limit=power)


def build_net():
    from sm3det_b200 import ConvNeXt_moe_MultiInput
    from sm3det_b200.synth import make_state_dict
    net = ConvNeXt_moe_MultiInput(**CONFIGS['t_e8']['kw'])
    net.load_state_dict(make_state_dict({k: tuple(v.shape) for k, v in net.state_dict().items()}, 0, True), strict=True)
    return net.cuda().train()


def time_step(net, x, micro, with_cp, steps, warmup):
    from sm3det_b200.graphed import GraphedStep
    net.with_cp = with_cp
    n_micro = x.shape[0] // micro

    def step(xx):
        tot = None
        for i in range(n_micro):
            outs, loss = net(xx[i * micro:(i + 1) * micro])
            t = (sum(o.float().mean() for o in outs) + loss) / n_micro
            t.backward()
            tot = t.detach() if tot is None else tot + t.detach()
        return tot

    net.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    g = None
    try:
        g = GraphedStep(step, [x], net.parameters(), warmup=warmup,
                        invalidate=[m._packs for m in net.modules() if hasattr(m, '_packs')])
        g(x)
        torch.cuda.synchronize()
        times = []
        for _ in range(steps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            g(x)
            b.record()
            b.synchronize()
            times.append(a.elapsed_time(b) / 1e3)
        dt = statistics.median(times)
        return dict(with_cp=with_cp, micro_batch=micro, fits=True, img_per_s=round(x.shape[0] / dt, 2),
                    step_s=round(dt, 4), max_memory_allocated_gib=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2))
    except Exception as e:       # noqa: BLE001 -- out of memory in the eager warm-up or in the capture: report it
        return dict(with_cp=with_cp, micro_batch=micro, fits=False, error=f'{type(e).__name__}: {str(e)[:160]}',
                    max_memory_allocated_gib=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2))
    finally:
        del g
        net.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


def event_ms(fn, reps=20):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return round(statistics.median(ts), 4)


def time_kernels(images=16, size=1024):
    from sm3det_b200 import ops
    rows = []
    for i, C in enumerate((96, 192, 384, 768)):
        s = size // (4 * 2 ** i)
        x = torch.randn((images, s, s, C), device='cuda')
        wt, b = torch.randn((49, C), device='cuda') * 0.1, torch.randn((C,), device='cuda')
        lnw, lnb = torch.ones((C,), device='cuda'), torch.zeros((C,), device='cuda')
        T = images * s * s
        img = C <= 192 and ops.ffn_chunk(0, C) > 0      # the fused-FFN stages take the operand image
        if img:
            two = lambda: ops.layernorm_fwd_img(ops.dwconv7(x, wt, b), lnw, lnb, 1e-6, tokens=T, C=C)
            two_all = lambda: ops.layernorm_fwd_img(ops.dwconv7(x, wt, b), lnw, lnb, 1e-6, tokens=T, C=C, save_stats=True,
                                                    want_f32=True)
        else:
            two = lambda: ops.layernorm_fwd(ops.dwconv7(x, wt, b), lnw, lnb, 1e-6, tokens=T, C=C)
            two_all = lambda: ops.layernorm_fwd(ops.dwconv7(x, wt, b), lnw, lnb, 1e-6, tokens=T, C=C, save_stats=True)
        fwd = lambda: ops.dwconv7_ln(x, wt, b, lnw, lnb, 1e-6, want_v=not img, want_img=img)
        rec = lambda: ops.dwconv7_ln(x, wt, b, lnw, lnb, 1e-6, want_u=True, want_stats=True, want_v=True, want_img=img)
        rows.append(dict(shape=[images, s, s, C], output='img' if img else 'v',
                         forward_ms=dict(fused=event_ms(fwd), two_kernels=event_ms(two)),
                         recompute_ms=dict(fused=event_ms(rec), two_kernels=event_ms(two_all))))
        del x
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--out', default=None, help='also write the JSON here')
    args = ap.parse_args()
    from sm3det_b200 import _lib
    from sm3det_b200.synth import make_images
    assert _lib.load().sm3_device_supported() == 1, 'needs an sm_90 (H100) device'
    torch.manual_seed(1234)
    res = dict(gpu=gpu_info(), workload=CONFIGS['t_e8']['name'], images_per_step=32, size=1024, kernels=time_kernels())
    net = build_net()
    x = make_images(32, 1024, 1024, seed=1234).cuda()
    res['steps'] = [time_step(net, x, micro, cp, args.steps, args.warmup) for cp, micro in ((False, 16), (True, 16), (True, 32), (False, 32))]
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
