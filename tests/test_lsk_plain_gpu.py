"""LSKNet / VAN (dense single-dataset backbones) and the fused Mlp middle stage on the GPU.

* sm3_mlp_mid_fwd / _bwd against the three-Function sequence they replace (DWConvFn(3, 1) -> GeluFn -> DropoutFn, or MulFn
  with an injected mask) on the same seed: the output and dh bit for bit, dw / db against float64 under the n u sum|terms|
  rule of tests/simt_ref.py.  Outputs lie in sentinel-filled buffers, inputs in NaN-filled ones (tests/test_simt_gpu.py),
  and the profiler confirms which kernel ran.
* A CUDA-graph-captured step draws a new mask per replay and matches eager launches on the replay's seed.
* The whole backbones against the tests/golden/lsk_plain fixtures (tools/gen_golden_lsk_plain.py), with the LSK
  channel-argmax teacher forcing of tests/test_lsk_gpu.py: forward <= 1e-3, gradients <= 3e-3, BatchNorm statistics.
"""
import os

import numpy as np
import pytest
import torch

import simt_ref as R
from oracle.cases import load_golden, lsk_injections, upstream_grads
from oracle.lsk_moe_oracle import lsk_backbone_forward, lsk_param_shapes
from parity_util import GAP_TOL, MAX_FLIP_FRACTION
from sm3det_b200 import lsk_functional as LF
from sm3det_b200.synth import make_images, make_state_dict
from test_lsk_plain_contract import FIXTURES, SYNC_BN, _config
from test_simt_gpu import Out, call, cu, kernels_run, ran, sms

pytestmark = pytest.mark.gpu
TOL, GRAD_TOL = 1e-3, 3e-3
# LSKNet() at its defaults (depths 3/4/6/3) in eval mode is ill-conditioned at stage 3: the oracle in fp32 and in fp64
# differ by 2.3e-5 there (~380x the fp32 unit roundoff), so the split-bf16 GEMMs' ~1e-5 relative error per product shows
# as 1.7e-3 (measured on an H100), as for LSK-T at 1024^2 in tests/test_lsk_t_gpu.py.  That fixture is held to 2e-3.
FORWARD_TOL = {'lsk_default_256_eval': 2e-3}


@pytest.fixture(scope='module')
def L():
    from sm3det_b200 import _lib
    return _lib.load()


def bits(a):
    return np.ascontiguousarray(R.f32(a)).view(np.uint32)


def rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).abs().max() / (b.abs().max() + 1e-30)).item()


# every Mlp hidden width of the shipped LSK / VAN configs; H, W not multiples of 16, N = 1..3
MID_CASES = [(128, 1, 19, 33), (256, 2, 23, 17), (512, 3, 13, 29), (640, 1, 37, 21), (1024, 2, 18, 35),
             (1280, 3, 9, 50), (2048, 2, 21, 14)]


def old_sequence(h, w, b, da, p, seed, mask):
    """(a, dh, du) of DWConvFn(3, 1) -> GeluFn -> DropoutFn / MulFn, du = the gradient at the conv output."""
    hg, wg, bg = (t.cuda().requires_grad_(True) for t in (h, w, b))
    u = LF.DWConvFn.apply(hg, wg, bg, 3, 1)
    u.retain_grad()
    a = LF.GeluFn.apply(u)
    if mask is not None:
        a = LF.MulFn.apply(a, mask.cuda())
    elif p > 0:
        a = LF.DropoutFn.apply(a, p, seed)
    a.backward(da.cuda())
    return a.detach(), hg.grad, u.grad


@pytest.mark.parametrize('drop', ['none', 'hashed', 'mask'])
@pytest.mark.parametrize('C,N,H,W', MID_CASES)
def test_mlp_mid_matches_three_function_sequence(L, C, N, H, W, drop):
    g = torch.Generator().manual_seed(C + N + H)
    h = torch.randn(N, H, W, C, generator=g) * 2.0
    w = torch.randn(C, 1, 3, 3, generator=g) * 0.3
    b = torch.randn(C, generator=g) * 0.2
    da = torch.randn(N, H, W, C, generator=g)
    p = 0.0 if drop == 'none' else 0.1
    seed = 987654321 + C
    mask = (torch.rand(N, H, W, C, generator=g) >= p).float() / (1.0 - p) if drop == 'mask' else None
    a_old, dh_old, du = old_sequence(h, w, b, da, p, seed, mask)
    wt = w.reshape(C, 9).t().contiguous()

    def fwd():
        a = Out((N, H, W, C))
        call(L, 'sm3_mlp_mid_fwd', cu(h), cu(wt), cu(b), cu(mask), a, N, H, W, C, p, seed, None)
        return a
    # the profiler confirms the kernels once (one session per direction), not per case: every profiler session of a long
    # single-process GPU run is another chance for torch.profiler to return no CUDA activity at all
    profile = C == 512 and drop == 'hashed'
    if profile:
        names, a = kernels_run(fwd)
        assert ran(names, 'mlp_mid_fwd_kernel'), names
    else:
        a = fwd()
    a = a.get('a')
    assert np.array_equal(bits(a), bits(a_old)), 'forward differs from the three-Function sequence'
    if drop != 'none':
        assert 0.05 < float((a == 0).mean()) < 0.15

    dwt0, db0 = torch.randn(9, C, generator=g), torch.randn(C, generator=g)

    def bwd():
        dh, dwt, db = Out((N, H, W, C)), Out((9, C), init=dwt0), Out((C,), init=db0)
        call(L, 'sm3_mlp_mid_bwd', cu(h), cu(wt), cu(b), cu(da), cu(mask), dh, dwt, db, N, H, W, C, p, seed, None)
        return dh, dwt, db
    if profile:
        names, (dh, dwt, db) = kernels_run(bwd)
        assert ran(names, 'mlp_mid_bwd_kernel'), names
    else:
        dh, dwt, db = bwd()
    assert np.array_equal(bits(dh.get('dh')), bits(dh_old)), 'dh differs from the three-Function sequence'
    # chain per (tap, channel): <= 41 pixels per warp and tile, tiles per block, the 8-warp sum, one atomic per block
    tiles = N * -(-H // 16) * -(-W // 16)
    bpc = max(1, min(tiles, -(-(sms() * 2) // (C // 32))))
    n = 41 * -(-tiles // bpc) + 8 + bpc + 1
    ref_w, ref_b = R.dwconv_wgrad(h, du, ks=3, dil=1)
    bw, bb = R.dwconv_wgrad_bound(h, du, n, ks=3, dil=1, dwt0=dwt0, db0=db0)
    assert R.ratio(dwt.get('dwt'), ref_w + R.f64(dwt0), bw) <= 1.0
    assert R.ratio(db.get('db'), ref_b + R.f64(db0), bb) <= 1.0


def test_mlp_mid_function_and_grid_limit(L):
    """MlpMidFn (the autograd wrapper) returns the kernel's values; eval / p = 0 applies no mask; N*C/32 >= 65536 is refused."""
    from sm3det_b200 import ops
    g = torch.Generator().manual_seed(5)
    h = torch.randn(2, 20, 24, 256, generator=g)
    w, b = torch.randn(256, 1, 3, 3, generator=g) * 0.3, torch.randn(256, generator=g) * 0.1
    hg, wg, bg = (t.cuda().requires_grad_(True) for t in (h, w, b))
    a = LF.MlpMidFn.apply(hg, wg, bg, 0.1, 77, None)
    da = torch.randn(a.shape, generator=g).cuda()
    a.backward(da)
    a_old, dh_old, _ = old_sequence(h, w, b, da.cpu(), 0.1, 77, None)
    assert torch.equal(a.detach(), a_old) and torch.equal(hg.grad, dh_old)
    assert torch.equal(LF.MlpMidFn.apply(hg.detach(), wg.detach(), bg.detach(), 0.0, 77, None),
                       LF.GeluFn.apply(LF.DWConvFn.apply(hg.detach(), wg.detach(), bg.detach(), 3, 1)))
    big = torch.empty(1, 1, 1, 32 * 65536, device='cuda')
    with pytest.raises(RuntimeError, match='N\\*C/32'):
        ops.mlp_mid_fwd(big, torch.zeros(9, big.shape[-1], device='cuda'), torch.zeros(big.shape[-1], device='cuda'))


def test_graphed_mlp_mid_draws_fresh_mask_per_replay():
    """Captured: the seed is drawn on the device inside the graph (as Mlp does under capture); every replay draws a new
    mask, and each replay equals eager launches given that replay's seed (a and dh bit for bit)."""
    from sm3det_b200 import ops
    g = torch.Generator().manual_seed(11)
    C = 512
    h = (torch.randn(2, 33, 40, C, generator=g)).cuda()
    wt = (torch.randn(9, C, generator=g) * 0.3).cuda()
    b = (torch.randn(C, generator=g) * 0.1).cuda()
    da = torch.randn(h.shape, generator=g).cuda()
    dwt, db, seed_out = torch.zeros(9, C, device='cuda'), torch.zeros(C, device='cuda'), torch.zeros(1, dtype=torch.int64, device='cuda')

    def step():
        seed = torch.randint(0, 2 ** 62, (1,), device='cuda')
        seed_out.copy_(seed)
        dwt.zero_()
        db.zero_()
        return ops.mlp_mid_fwd(h, wt, b, p=0.1, seed=seed), ops.mlp_mid_bwd(h, wt, b, da, dwt, db, p=0.1, seed=seed)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        a_s, dh_s = step()
    seen = []
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        sd = int(seed_out.item())
        a, dh, w1, b1 = a_s.clone(), dh_s.clone(), dwt.clone(), db.clone()
        ea = ops.mlp_mid_fwd(h, wt, b, p=0.1, seed=sd)
        ew, eb = torch.zeros_like(dwt), torch.zeros_like(db)
        edh = ops.mlp_mid_bwd(h, wt, b, da, ew, eb, p=0.1, seed=sd)
        assert torch.equal(a, ea) and torch.equal(dh, edh)
        assert torch.allclose(w1, ew, rtol=1e-5, atol=1e-5) and torch.allclose(b1, eb, rtol=1e-5, atol=1e-5)
        seen.append((sd, a == 0))
    assert seen[0][0] != seen[1][0]
    assert not torch.equal(seen[0][1], seen[1][1]), 'two replays drew the same dropout mask'


# ------------------------------------------------------------------------------------------------
def build(gold):
    import sm3det_b200
    cfg = _config(dict(type=gold['cls'], **gold['kw']))
    sd = make_state_dict(lsk_param_shapes(cfg), 0, True)
    net = getattr(sm3det_b200, gold['cls'])(norm_cfg=dict(SYNC_BN), **gold['kw'])
    net.load_state_dict(sd, strict=True)
    return cfg, sd, net.cuda()


def zero_grad_bias(name):
    """A conv bias in front of a training-mode BatchNorm: the true gradient is exactly 0, both sides hold fp32 noise."""
    return name.startswith('patch_embed') and name.endswith('proj.bias')


@pytest.mark.parametrize('path', FIXTURES, ids=lambda p: os.path.basename(p)[:-3])
def test_plain_backbone_matches_reference_golden(path):
    gold = load_golden(path)
    tol = FORWARD_TOL.get(gold['name'], TOL)
    cfg, sd, net = build(gold)
    n, h, w = gold['img']
    x = make_images(n, h, w, seed=1234)
    train = gold['mode'] != 'eval'
    net.train(train)
    _, drops = lsk_injections(cfg, gold)
    dps = gold.get('dp_masks')
    if train:
        blocks = [blk for i in range(cfg.num_stages) for blk in getattr(net, f'block{i + 1}')]
        it = iter(drops)
        for blk, m in zip(blocks, dps):
            m1, m2 = next(it), next(it)
            blk.mlp._injected_drop_masks = [m1.permute(0, 2, 3, 1).contiguous(), m2.permute(0, 2, 3, 1).contiguous()]
            blk._injected_drop_mask = m
    amax = []
    LF.AMAX_RECORD = amax
    try:
        with torch.set_grad_enabled(train):
            outs = net(x.cuda())
    finally:
        LF.AMAX_RECORD = None
    assert isinstance(outs, list) and len(outs) == 4 and all(o.is_contiguous() for o in outs)
    ups = upstream_grads([o.detach().cpu() for o in outs])
    if train:
        sum((o * u.cuda()).sum() for o, u in zip(outs, ups)).backward()
    # the oracle teacher-forced to the CUDA path's LSK channel argmax (tests/test_lsk_gpu.py); flips must be near-ties
    is_lsk = gold['unit'] == 'lsk'
    no_grad = ('running_', 'num_batches')
    sdo = {k: (v.clone().requires_grad_(True) if train and v.is_floating_point() and not any(t in k for t in no_grad) else v)
           for k, v in sd.items()}
    bn_state, arec = {}, []
    with torch.set_grad_enabled(train):
        oc = lsk_backbone_forward(sdo, cfg, x, train=train, drop_masks=drops,
                                  dp_masks=[m.view(n, 1, 1, 1) for m in dps] if train else None, bn_state=bn_state,
                                  forced_amax=[a.cpu() for a in amax] if is_lsk else None, amax_record=arec)
    amax_flips = 0
    for a in arec:
        flip = a['own'] != a['forced']
        amax_flips += int(flip.sum())
        if flip.any():
            assert float((a['gap'][flip] / a['scale'][flip]).max()) < GAP_TOL, (a['prefix'], 'channel-argmax flip is not a near-tie')
        assert int(flip.sum()) <= max(2, MAX_FLIP_FRACTION * flip.numel()), (a['prefix'], int(flip.sum()), flip.numel())
    errs = [rel(a, b) for a, b in zip(outs, oc)]
    print(os.path.basename(path), 'channel-argmax flips', amax_flips, 'rel errs vs forced oracle', errs)
    assert max(errs) < tol
    new_sd = net.state_dict()
    if train:
        sum((o * u).sum() for o, u in zip(oc, ups)).backward()
        bad = []
        for name, p in net.named_parameters():
            want, got = sdo[name].grad, p.grad.detach().float().cpu()
            if zero_grad_bias(name):
                assert (got - want).abs().max().item() < 1e-5, name
                continue
            bad.append((((got - want).abs().max() / max(want.abs().max().item(), 1e-5)).item(), name))
        bad.sort(reverse=True)
        print('worst grads vs forced oracle', bad[:5])
        assert bad[0][0] < GRAD_TOL, bad[:8]
        for k, v in bn_state.items():
            assert rel(new_sd[k], v) < 1e-4, k
    # the reference-generated fixture itself
    st = gold['stride']
    errs = [rel(o[:, :, ::st, ::st], g) for o, g in zip(outs, gold['outs'])]
    print(os.path.basename(path), 'rel errs vs fixture', errs)
    assert max(errs) < tol
    if train and amax_flips == 0:
        bad = []
        for name, p in net.named_parameters():
            gg = gold['grads'][name]
            got = p.grad.detach().float().cpu().reshape(-1)
            want, got = (gg['full'], got) if 'full' in gg else (gg['sample'], got[gg['idx']])
            scale = (gg['l2'] / (p.numel() ** 0.5)) if 'l2' in gg else want.abs().max().item()
            if zero_grad_bias(name):
                continue
            bad.append((((got - want).abs().max() / max(want.abs().max().item(), scale, 1e-5)).item(), name))
        bad.sort(reverse=True)
        print('worst grads vs fixture', bad[:5])
        assert bad[0][0] < GRAD_TOL, bad[:8]
        for k, v in gold['bn'].items():
            assert rel(new_sd[k], v) < 1e-4, k


def test_return_convention_and_fused_mlp_kernels(monkeypatch):
    """LSKNet returns a list of 4 NCHW maps; VAN concatenates a list input along N; every Mlp of a training step runs the
    fused middle stage (one sm3_mlp_mid_fwd and one sm3_mlp_mid_bwd per block)."""
    from sm3det_b200 import LSKNet, VAN, ops
    kw = dict(embed_dims=[32, 64, 160, 256], depths=[1, 1, 1, 1], drop_rate=0.1)
    x = make_images(2, 96, 64, seed=3).cuda()
    van = VAN(**kw).cuda().eval()
    with torch.no_grad():
        o1 = van(x)
        o2 = van([x[:1], x[1:]], datasets=['a', 'b'])
    assert isinstance(o1, list) and all(torch.equal(a, b) for a, b in zip(o1, o2))
    assert [tuple(o.shape) for o in o1] == [(2, 32, 24, 16), (2, 64, 12, 8), (2, 160, 6, 4), (2, 256, 3, 2)]
    calls = []
    for name in ('mlp_mid_fwd', 'mlp_mid_bwd', 'dwconv'):
        fn = getattr(ops, name)
        monkeypatch.setattr(ops, name, lambda *a, _f=fn, _n=name, **k: (calls.append(_n), _f(*a, **k))[1])
    net = LSKNet(**kw).cuda().train()
    outs = net(x)
    sum(o.square().mean() for o in outs).backward()
    torch.cuda.synchronize()
    assert isinstance(outs, list) and len(outs) == 4
    assert calls.count('mlp_mid_fwd') == 4 and calls.count('mlp_mid_bwd') == 4, calls
    assert all(torch.isfinite(p.grad).all() for p in net.parameters() if p.grad is not None)
