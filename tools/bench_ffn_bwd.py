"""The dense-FFN backward of the bench.py stage shapes (16-image pass at 1024^2: stage 0 [1,048,576 x 96], stage 1
[262,144 x 192]) in its two forms, event-timed over many launches:

  gemm:  linear_dgrad(dz, gamma W2) -> act_pack(ACT_BWD) -> linear_dgrad(dh_k, W1)      (SM3_FUSED_FFN_BWD=0)
  chain: pack_act(dzs) -> ffn_fused_bwd(want_wgrad_images=True), mode 2 (recomputes h) at C = 96, mode 3 (reads h) at 192

Both produce dv, db1 and the MN-major images of dh and gelu(h) the two weight-gradient GEMMs read.  Bytes are the HBM
traffic each sequence needs (fp32 tensors 4 B / element, hi|lo images 4 B / element); achieved GB/s = bytes / time.

    python tools/bench_ffn_bwd.py [--iters 50] [--out results.json]
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_checkpoint import gpu_info  # noqa: E402


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters // 5):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) / (iters // 5))
    return statistics.median(ts), min(ts), max(ts)


def shape_case(T, C, iters):
    from sm3det_b200 import ops
    g = torch.Generator(device='cuda').manual_seed(C)
    H4 = 4 * C
    v = torch.randn((T, C), device='cuda', generator=g)
    dz = torch.randn((T, C), device='cuda', generator=g)
    w1 = torch.randn((H4, C), device='cuda', generator=g) / C ** 0.5
    b1 = 0.2 * torch.randn((H4,), device='cuda', generator=g)
    w2 = torch.randn((C, H4), device='cuda', generator=g) / H4 ** 0.5
    gamma = 0.5 + torch.rand((C,), device='cuda', generator=g)
    v_img, _, _ = ops.layernorm_fwd_img(v, torch.ones(C, device='cuda'), torch.zeros(C, device='cuda'), 1e-6, tokens=T, C=C)
    cf = ops.ffn_chunk(0, C)
    w1c, _ = ops.pack_weight(w1, transposed=False, tile=cf)
    w2n, _ = ops.pack_weight(w2, transposed=False, tile=C)
    _, _, h = ops.ffn_fused_fwd(v_img, w1c, w2n, b1, torch.zeros(C, device='cuda'), T=T, C=C, chunk=cf, want_h=True)
    w2g = ops.scale_rows(w2, row_scale=gamma)
    w2g_t = ops.pack_weight(w2g, transposed=True)
    w1_t = ops.pack_weight(w1, transposed=True)
    mode = 2 if ops.ffn_chunk(2, C) > 0 else 3
    cb = ops.ffn_chunk(mode, C)
    w1cb, _ = ops.pack_weight(w1, transposed=False, tile=cb)
    w2gt, _ = ops.pack_weight(w2g, transposed=True, tile=cb)
    w1tn, _ = ops.pack_weight(w1, transposed=True, tile=C)
    db1 = torch.zeros((H4,), device='cuda')

    def gemm_seq():
        da = ops.linear_dgrad(dz, w2g, packed=w2g_t)
        dh_k, _, _ = ops.act_pack(h, rows=T, width=H4, mode=ops.ACT_BWD, da=da, want_k=True, mn_tile=128,
                                  mn_tile2=ops._pick_bn(H4), colsum=db1)
        del da
        return ops.linear_dgrad(None, w1, rows=T, a_packed=dh_k, packed=w1_t)

    def chain():
        dz_img = ops.pack_act(dz, rows=T, cols=C, mn_major=False)
        return ops.ffn_fused_bwd(v_img, dz_img, w1cb, w2gt, w1tn, b1, T=T, C=C, chunk=cb, want_wgrad_images=True, db1=db1,
                                 h=h if mode == 3 else None)

    n = float(T * C)
    # gemm: dz 4 + da 16 (dgrad2); h 16 + da 16 + dh_k 16 + two MN images 32 (act_pack); dh_k 16 + dv 4 (dgrad1)
    gemm_bytes = (4 + 16 + 16 + 16 + 16 + 32 + 16 + 4) * n
    # chain: dz 4 + dz image 4 (pack); dz image 4 + v image 4 or h 16 + dv 4 + two MN images 32 (kernel)
    chain_bytes = (4 + 4 + 4 + (4 if mode == 2 else 16) + 4 + 32) * n
    out = dict(T=T, C=C, mode=mode, chunk=cb)
    for name, fn, byts in (('gemm', gemm_seq, gemm_bytes), ('chain', chain, chain_bytes)):
        med, lo, hi = timed(fn, iters)
        out[name] = dict(ms=round(med, 4), ms_min=round(lo, 4), ms_max=round(hi, 4), GB=round(byts / 1e9, 3),
                         GBps=round(byts / (med * 1e-3) / 1e9, 1))
    # the chain kernel alone (without the dz pack), for its share of HBM bandwidth
    dz_img = ops.pack_act(dz, rows=T, cols=C, mn_major=False)
    kbytes = (4 + (4 if mode == 2 else 16) + 4 + 32) * n
    med, lo, hi = timed(lambda: ops.ffn_fused_bwd(v_img, dz_img, w1cb, w2gt, w1tn, b1, T=T, C=C, chunk=cb,
                                                  want_wgrad_images=True, db1=db1, h=h if mode == 3 else None), iters)
    out['chain_kernel'] = dict(ms=round(med, 4), GB=round(kbytes / 1e9, 3), GBps=round(kbytes / (med * 1e-3) / 1e9, 1))
    out['speedup'] = round(out['gemm']['ms'] / out['chain']['ms'], 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'needs an H100'
    res = dict(gpu=gpu_info(), shapes=[])
    for T, C in ((1048576, 96), (262144, 192)):
        res['shapes'].append(shape_case(T, C, args.iters))
        torch.cuda.empty_cache()
    print(json.dumps(res))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
