"""Activation checkpointing (`with_cp=True`) of the ConvNeXt backbones and its fused dwconv7 + LayerNorm kernel.

The checkpointed blocks recompute their activations in backward with the forward's own kernels, so the forward is
bit-identical to the plain one and gradients differ only by the order of split-K / atomic sums."""
import itertools

import pytest
import torch

GRAD_REL = 1e-5            # cp vs plain gradients, relative to max|g| of each tensor


def _ops():
    from sm3det_b200 import ops
    return ops


def _front_inputs(N, H, W, C, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((N, H, W, C), generator=g)
    wt = torch.randn((49, C), generator=g) * 0.2
    b = torch.randn((C,), generator=g)
    lnw = 1.0 + 0.5 * torch.randn((C,), generator=g)
    lnb = 0.3 * torch.randn((C,), generator=g)
    return [t.cuda() for t in (x, wt, b, lnw, lnb)]


SHAPES = [(1, 1, 1), (1, 7, 9), (3, 33, 17), (3, 64, 64)]


@pytest.mark.parametrize('mode,C', [('ln', c) for c in (32, 96, 384, 768, 1024)] + [('img', c) for c in (32, 96, 160, 192, 256)])
@pytest.mark.gpu
def test_dwconv7_ln_matches_the_two_kernels(mode, C):
    """sm3_dwconv7_ln_fwd == dwconv7 -> layernorm_fwd (or -> layernorm_fwd_img), bit for bit, for every output subset."""
    ops = _ops()
    eps = 1e-6
    names = ('u', 'stats', 'v', 'img') if mode == 'img' else ('u', 'stats', 'v')
    for N, H, W in SHAPES:
        x, wt, b, lnw, lnb = _front_inputs(N, H, W, C, seed=N * 1000 + H * 10 + W + C)
        T = N * H * W
        u_ref = ops.dwconv7(x, wt, b)
        v_ref, st_ref = ops.layernorm_fwd(u_ref, lnw, lnb, eps, tokens=T, C=C, save_stats=True)
        ln_ref = dict(u=u_ref, stats=st_ref, v=v_ref.view(T, C))
        if mode == 'img':
            img_ref, v_ref, st_ref = ops.layernorm_fwd_img(u_ref, lnw, lnb, eps, tokens=T, C=C, save_stats=True, want_f32=True)
            img_ref = dict(u=u_ref, stats=st_ref, v=v_ref, img=img_ref)
        for r in range(1, len(names) + 1):
            for subset in itertools.combinations(names, r):
                ref = img_ref if 'img' in subset else ln_ref        # v and stats follow the image kernel's order with img
                got = ops.dwconv7_ln(x, wt, b, lnw, lnb, eps, **{f'want_{n}': True for n in subset})
                got = dict(zip(('u', 'stats', 'v', 'img'), got))
                for n in ('u', 'stats', 'v', 'img'):
                    if n in subset:
                        assert torch.equal(got[n].view(ref[n].shape), ref[n]), (N, H, W, C, subset, n)
                    else:
                        assert got[n] is None


@pytest.mark.gpu
def test_dwconv7_ln_zeroes_the_image_padding_rows():
    """Rows of the last 128-row tile beyond T are written as zeros (the buffer starts as garbage)."""
    ops = _ops()
    from sm3det_b200 import _lib
    lib = _lib.load()
    N, H, W, C = 1, 7, 9, 96                                        # T = 63: 65 padding rows
    x, wt, b, lnw, lnb = _front_inputs(N, H, W, C, seed=3)
    T = N * H * W
    img = torch.full((lib.sm3_gemm_packed_act_elems(T, C, 0, 128),), 0x5555, device='cuda', dtype=torch.int16)
    _lib.check(lib.sm3_dwconv7_ln_fwd(x.data_ptr(), wt.data_ptr(), b.data_ptr(), lnw.data_ptr(), lnb.data_ptr(), None, None,
                                      None, img.data_ptr(), N, H, W, C, 1e-6, torch.cuda.current_stream().cuda_stream), 'x')
    img_ref, _, _ = ops.layernorm_fwd_img(ops.dwconv7(x, wt, b), lnw, lnb, 1e-6, tokens=T, C=C)
    assert torch.equal(img, img_ref)
    # a zero row splits into zero hi and lo halves: the image holds exactly 2 * T * C non-padding 16-bit words
    assert int((img != 0).sum()) <= 2 * T * C


# ---- block level ------------------------------------------------------------------------------------------------------

def _block(C, moe=None, drop=0.0, seed=0):
    from sm3det_b200.backbone import ConvNeXtBlock
    torch.manual_seed(seed)
    blk = ConvNeXtBlock(C, dict(type='LN2d', eps=1e-6), MoE_cfg=moe, drop_path_rate=drop)
    with torch.no_grad():
        for n, p in blk.named_parameters():
            if n.endswith('gamma'):
                p.copy_(0.5 + torch.rand_like(p))
            elif 'norm' in n:
                p.copy_((1.0 if n.endswith('weight') else 0.0) + 0.3 * torch.randn_like(p))
            elif n.endswith('depthwise_conv.bias'):
                p.copy_(0.2 * torch.randn_like(p))
            elif 'w_noise' in n:
                p.copy_(0.1 * torch.randn_like(p))
    return blk.cuda().train()


def _run_block(blk, x, up, shortcut, with_cp):
    blk.with_cp = with_cp
    blk.zero_grad(set_to_none=True)
    xg = x.clone().requires_grad_(True)
    out, loss = blk._run(xg, blk._row_scale(xg), None, shortcut)
    tot = (out * up).sum() + (loss if loss is not None else 0.0)
    tot.backward()
    grads = {n: p.grad.clone() for n, p in blk.named_parameters() if p.grad is not None}
    grads['x'] = xg.grad.clone()
    return out.detach(), (loss.detach() if loss is not None else None), grads


def _compare_cp(blk, x, shortcut=True):
    up = torch.randn_like(x)
    o0, l0, g0 = _run_block(blk, x, up, shortcut, False)
    o1, l1, g1 = _run_block(blk, x, up, shortcut, True)
    assert torch.equal(o0, o1)
    if l0 is not None:
        assert torch.equal(l0, l1)
    assert set(g0) == set(g1)
    for n in g0:
        scale = float(g0[n].abs().max())
        err = float((g0[n] - g1[n]).abs().max())
        assert err <= GRAD_REL * scale, (n, err, scale)


def _inject(blk, x, noise_E=None, drop=False, seed=5):
    g = torch.Generator(device='cuda').manual_seed(seed)
    N, H, W, _ = x.shape
    if drop:
        blk._injected_drop_mask = torch.tensor([1.0 / 0.9, 0.0, 1.0 / 0.9][:N], device='cuda')
    if noise_E is not None:
        blk.ffn._injected_noise = torch.randn((N * H * W, noise_E), device='cuda', generator=g)


@pytest.mark.parametrize('C,fused_env', [(96, '1'), (192, '1'), (384, '1'), (96, '0')])
@pytest.mark.parametrize('shortcut', [True, False])
@pytest.mark.gpu
def test_dense_block_checkpoint_is_exact(monkeypatch, C, fused_env, shortcut):
    monkeypatch.setenv('SM3_FUSED_FFN', fused_env)
    blk = _block(C, drop=0.1, seed=C)
    x = torch.randn((3, 20, 28, C), device='cuda')                  # T = 1680, not a multiple of 128
    _inject(blk, x, drop=True)
    _compare_cp(blk, x, shortcut)


@pytest.mark.parametrize('k', [1, 2, 3])
@pytest.mark.parametrize('noisy', [False, True])
@pytest.mark.gpu
def test_moe_block_checkpoint_is_exact(k, noisy):
    E = 4
    blk = _block(96, moe=dict(noisy_gating=noisy, num_experts=E, top_k=k, gating='cosine'), drop=0.1, seed=k)
    x = torch.randn((3, 20, 28, 96), device='cuda')
    _inject(blk, x, noise_E=E if noisy else None, drop=True)
    _compare_cp(blk, x)
    _compare_cp(blk, x, shortcut=False)


# ---- backbone --------------------------------------------------------------------------------------------------------

@pytest.fixture
def cp_build(monkeypatch):
    """parity_util.run_case, building every backbone with with_cp=True (the oracle config takes no with_cp)."""
    import parity_util
    orig = parity_util.build

    def build(kw, *a, **k):
        cfg, sd, net = orig(kw, *a, **k)
        net.with_cp = True
        return cfg, sd, net
    monkeypatch.setattr(parity_util, 'build', build)
    return parity_util


@pytest.mark.parametrize('name', ['cfg2_t_e8k2_1024_eval', 'cfg2_t_e8k2_1024_train_clean', 'cfg2_t_e8k2_1024_train_noisy',
                                  'da_mini_moe_e4k2_train_noisy_3mod'])
@pytest.mark.gpu
def test_checkpointed_backbone_matches_reference_golden(cp_build, name):
    import os
    from oracle.cases import load_golden
    gold = load_golden(os.path.join(os.path.dirname(__file__), 'golden', name + '.pt'))
    errs = cp_build.run_case(gold['kw'], gold['img'], gold['mode'], gold['weights'], gold=gold, datasets=gold.get('datasets'))
    print(name, errs)


def _backbone_step(net, x, ups, with_cp):
    net.with_cp = with_cp
    net.zero_grad(set_to_none=True)
    outs, loss = net(x)
    (sum((o * u).sum() for o, u in zip(outs, ups)) + loss).backward()
    return [o.detach().clone() for o in outs], loss.detach().clone(), \
        {n: p.grad.clone() for n, p in net.named_parameters() if p.grad is not None}


def _inject_backbone(net, N, H, W, seed=9):
    from sm3det_b200.backbone import ConvNeXtBlock
    g = torch.Generator(device='cuda').manual_seed(seed)
    for si, stage in enumerate(net.stages):
        s = 4 * 2 ** si
        for blk in stage:
            assert isinstance(blk, ConvNeXtBlock)
            if blk.drop_path_rate > 0:
                blk._injected_drop_mask = (torch.rand((N,), device='cuda', generator=g) > 0.3).float() / (1 - blk.drop_path_rate)
            if blk.MoE_cfg is not None and blk.ffn.noisy_gating:
                blk.ffn._injected_noise = torch.randn(((N * (H // s) * (W // s)), blk.ffn.num_experts), device='cuda', generator=g)


@pytest.mark.parametrize('amp', [False, True])
@pytest.mark.gpu
def test_checkpointed_backbone_is_exact(amp):
    """cfg2 (ConvNeXt-T, E=8, k=2, noisy gating, drop path): outputs and gate loss bit-identical, gradients within 1e-5."""
    from oracle.cases import CFG2_KW
    from sm3det_b200 import ConvNeXt_moe_MultiInput
    from sm3det_b200.synth import make_images
    torch.manual_seed(0)
    net = ConvNeXt_moe_MultiInput(**CFG2_KW, drop_path_rate=0.2).cuda().train()
    net.amp = amp
    N, H, W = 2, 256, 320
    x = make_images(N, H, W, seed=4).cuda()
    _inject_backbone(net, N, H, W)
    ups = [torch.randn((N, c, H // (4 * 2 ** i), W // (4 * 2 ** i)), device='cuda') for i, c in enumerate(net.channels)]
    o0, l0, g0 = _backbone_step(net, x, ups, False)
    o1, l1, g1 = _backbone_step(net, x, ups, True)
    assert all(torch.equal(a, b) for a, b in zip(o0, o1))
    assert torch.equal(l0, l1)
    assert set(g0) == set(g1)
    worst = max((float((g0[n] - g1[n]).abs().max()) / (float(g0[n].abs().max()) + 1e-30), n) for n in g0)
    print('amp', amp, 'worst grad rel', worst)
    assert worst[0] <= GRAD_REL, worst


@pytest.mark.gpu
def test_graphed_checkpointed_step():
    """A captured cp step replays to the eager loss and gradients, and draws fresh gating noise on every replay."""
    from oracle.cases import CASES
    from parity_util import build
    from sm3det_b200.graphed import GraphedStep
    from sm3det_b200.synth import make_images

    def fwd_bwd(net):
        def step(x):
            outs, loss = net(x)
            tot = sum(o.square().mean() for o in outs) + loss
            tot.backward()
            return tot.detach()
        return step

    spec = CASES['mini2_moe_e8k2_train_clean']
    _, _, net = build(spec['kw'])
    net.with_cp = True
    net.train()
    x = make_images(*spec['img'], seed=1).cuda()
    step = fwd_bwd(net)
    net.zero_grad(set_to_none=True)
    ref = step(x).clone()
    want = {n: p.grad.clone() for n, p in net.named_parameters() if p.grad is not None}
    net.zero_grad(set_to_none=True)
    g = GraphedStep(step, [x], net.parameters(), invalidate=[m._packs for m in net.modules() if hasattr(m, '_packs')])
    got = g(x)
    torch.cuda.synchronize()
    assert abs(got.item() - ref.item()) <= 1e-4 * abs(ref.item())
    now = {n: p.grad for n, p in net.named_parameters() if p.grad is not None}
    assert set(now) == set(want)
    worst = max((float((now[k] - want[k]).abs().max() / want[k].abs().max()) / (5.0 if k.endswith('temperature') else 1.0), k)
                for k in want if float(want[k].abs().max()) > 1e-8)
    assert worst[0] <= 1e-4, worst
    # noisy gating: the noise is drawn inside the graph, fresh on every replay
    kw = dict(spec['kw'], noisy_gating=True)
    _, _, net = build(kw)
    net.with_cp = True
    net.train()
    g = GraphedStep(fwd_bwd(net), [x], net.parameters())
    losses = []
    for _ in range(3):
        losses.append(g(x).item())
        assert all(torch.isfinite(p.grad).all() for p in net.parameters() if p.grad is not None)
    assert len({round(v, 10) for v in losses}) == 3, losses


@pytest.mark.gpu
def test_checkpoint_memory():
    """ConvNeXt-T cfg2, 2 x 1024^2, train: what the forward leaves allocated for backward, and the backward peak."""
    from oracle.cases import CFG2_KW
    from sm3det_b200 import ConvNeXt_moe_MultiInput
    from sm3det_b200.synth import make_images
    torch.manual_seed(0)
    net = ConvNeXt_moe_MultiInput(**CFG2_KW).cuda().train()
    x = make_images(2, 1024, 1024, seed=3).cuda()
    res = {}
    for cp in (False, True, False):                                 # the first pass also warms up packs and the allocator
        net.with_cp = cp
        net.zero_grad(set_to_none=False)
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated()
        outs, loss = net(x)
        torch.cuda.synchronize()
        kept = torch.cuda.memory_allocated() - before
        torch.cuda.reset_peak_memory_stats()
        (sum(o.square().mean() for o in outs) + loss).backward()
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - before
        del outs, loss
        res[cp] = (kept, peak)
    ratio = res[True][0] / res[False][0]
    print(f'saved for backward: {res[False][0] / 2**30:.3f} GiB plain, {res[True][0] / 2**30:.3f} GiB with cp (ratio {ratio:.3f}); '
          f'backward peak {res[False][1] / 2**30:.3f} vs {res[True][1] / 2**30:.3f} GiB')
    assert ratio <= 0.25                                            # measured 0.19 on an H100 (3.47 -> 0.68 GiB)
    assert res[True][1] < res[False][1]


def test_with_cp_is_a_pure_memory_option():
    """CPU: with_cp=True builds from the registry and has exactly the state_dict layout of with_cp=False."""
    from sm3det_b200.registry import build_backbone
    kw = dict(arch='tiny', MoE_Block_inds=[[], [], [0, 2, 4, 6, 8], [0, 2]], num_experts=8, top_k=2)
    for typ in ('ConvNeXt_moe', 'ConvNeXt_moe_MultiInput', 'ConvNeXt_DA_MultiInput'):
        a = build_backbone(dict(type=typ, with_cp=True, **kw))
        b = build_backbone(dict(type=typ, with_cp=False, **kw))
        assert a.with_cp and not b.with_cp
        assert all(blk.with_cp for st in a.stages for blk in st)
        sa, sb = a.state_dict(), b.state_dict()
        assert list(sa) == list(sb)
        assert all(sa[k].shape == sb[k].shape for k in sa)

