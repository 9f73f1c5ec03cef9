"""OrientedRPNHead convolutions on the CUDA library (sm3det_b200.head).

CPU: tests/rpn_head_ref.py reproduces the fixtures tools/gen_golden_rpn_head.py wrote and, when the reference tree is present,
matches the unmodified RotatedRPNHead.forward_single / OrientedRPNHead._init_layers bit for bit; the config inventory; the
options the kernels do not cover raise; CPU inputs raise; the head is not force-registered.  GPU: forward and every
gradient against the oracle, the kernels against float64 at odd shapes with sentinel-guarded outputs, eval / no_grad,
autocast, CUDA-graph replay, bitwise-repeatable launches, and MultitaskFPN followed by the head."""
import glob
import inspect
import os
import re

import pytest
import torch
import torch.nn.functional as F

import rpn_head_ref as M
from oracle.cases import load_golden
from sm3det_b200 import OrientedRPNHeadConvs

GOLD = os.path.join(os.path.dirname(__file__), 'golden', 'rpn_head')
FIXTURES = sorted(glob.glob(os.path.join(GOLD, '*.pt')))
ODD = [(20, 24), (10, 12), (5, 6), (3, 3), (1, 2), (1, 1)]      # H != W, not tile multiples, 1x1 and 1x2 levels


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


def head_from(sd):
    cin = sd['rpn_conv.weight'].shape[1]
    m = OrientedRPNHeadConvs(in_channels=cin)
    m.load_state_dict({k: v.float() for k, v in sd.items()}, strict=True)
    return m


# ---- CPU -------------------------------------------------------------------------------------------------------------
def _reference_heads():
    mod = M.load_reference_heads()
    if mod is None:
        pytest.skip('reference tree not present')
    return mod


def test_oracle_matches_reference_forward_single():
    ref = _reference_heads()
    head = ref.OrientedRPNHead(in_channels=256)
    shapes = {k: tuple(v.shape) for k, v in head.state_dict().items()}
    assert shapes == M.rpn_head_param_shapes(256)
    sd = M.make_params(256, seed=7)
    head.load_state_dict(sd, strict=True)
    feats = M.make_feats(2, [(9, 14), (5, 7), (1, 1)], 256, seed=7)
    with torch.no_grad():
        for x in feats:
            rc, rr = head.forward_single(x.clone())
            oc, orr = M.forward_single(sd, x)
            assert torch.equal(rc, oc) and torch.equal(rr, orr)


def test_mixin_composes_over_reference_class():
    ref = _reference_heads()
    from sm3det_b200 import SM3RPNHeadMixin
    cls = type('SM3OrientedRPNHead', (SM3RPNHeadMixin, ref.OrientedRPNHead), {})
    a, b = cls(in_channels=256), ref.OrientedRPNHead(in_channels=256)
    assert list(a.state_dict()) == list(b.state_dict()) == list(OrientedRPNHeadConvs(256).state_dict())
    assert cls.forward is SM3RPNHeadMixin.forward
    with pytest.raises(RuntimeError, match='CUDA'):
        a([torch.zeros(1, 256, 4, 4)])


def test_config_inventory():
    """76 reference configs build an OrientedRPNHead; every one is 256 -> 256 with one scale and three ratios."""
    from oracle import ref_shim
    if not ref_shim.reference_available():
        pytest.skip('reference tree not present')
    root = ref_shim.REFERENCE_ROOT
    files = [f for f in glob.glob(os.path.join(root, '**', '*.py'), recursive=True)
             if ('/configs/' in f or '/local_configs/' in f) and "type='OrientedRPNHead'" in open(f, errors='ignore').read()]
    assert len(files) == 76
    for f in files:
        src = open(f, errors='ignore').read()
        for blk in re.findall(r"type='OrientedRPNHead'(.*?)bbox_coder", src, re.S):
            assert re.search(r'in_channels=256', blk) and re.search(r'feat_channels=256', blk), f
            assert re.search(r'scales=\[8\]', blk) and re.search(r'ratios=\[0\.5, 1\.0, 2\.0\]', blk), f


@pytest.mark.parametrize('path', FIXTURES, ids=[os.path.basename(p)[:-3] for p in FIXTURES])
def test_oracle_reproduces_fixture(path):
    gold = load_golden(path)
    cls, reg = M.rpn_head_forward(gold['params'], gold['feats'])
    assert all(torch.equal(a, b) for a, b in zip(cls, gold['cls']))
    assert all(torch.equal(a, b) for a, b in zip(reg, gold['reg']))


def test_fixtures_present():
    assert {os.path.basename(p)[:-3] for p in FIXTURES} == set(M.GOLDEN_CASES)


@pytest.mark.parametrize('kw', [dict(in_channels=48), dict(in_channels=512), dict(feat_channels=128), dict(num_anchors=9)])
def test_unsupported_shapes_raise(kw):
    with pytest.raises(NotImplementedError):
        OrientedRPNHeadConvs(**kw)


def test_unsupported_layers_raise_in_mixin():
    from sm3det_b200.head import rpn_head_forward
    m = OrientedRPNHeadConvs()
    m.rpn_conv = torch.nn.Conv2d(256, 256, 3, padding=2, dilation=2)
    with pytest.raises(NotImplementedError):
        rpn_head_forward(m.rpn_conv, m.rpn_cls, m.rpn_reg, [torch.zeros(1, 256, 4, 4)])
    m = OrientedRPNHeadConvs()
    with pytest.raises(NotImplementedError):
        m([torch.zeros(1, 256, 2, 2)] * 9)


def test_cpu_inputs_raise():
    with pytest.raises(RuntimeError, match='CUDA'):
        OrientedRPNHeadConvs()([torch.zeros(1, 256, 4, 4)])


def test_not_force_registered():
    from sm3det_b200 import registry
    src = inspect.getsource(registry.register_into_mmrotate)
    assert 'RPN' not in src and 'HEADS' not in src


# ---- GPU -------------------------------------------------------------------------------------------------------------
def _run(sd, feats, dcls=None, dreg=None, **fwd):
    head = head_from(sd).cuda()
    xs = [x.float().cuda().requires_grad_(True) for x in feats]
    cls, reg = head(xs, **fwd)
    if dcls is None:
        return head, xs, cls, reg
    torch.autograd.backward(cls + reg, [d.float().cuda() for d in dcls + dreg])
    return head, xs, cls, reg


def _kernel_masks(sd, feats):
    """The ReLU mask the kernels used (h > 0 of their saved hidden map), per level as [N, 256, H, W] on the CPU."""
    from sm3det_b200 import ops
    head = head_from(sd).cuda()
    xs = [x.detach().float().cuda() for x in feats]
    cin = xs[0].shape[1]
    wc = head.rpn_conv.weight.detach()
    wc_img, _ = ops.pack_weight(wc.permute(0, 2, 3, 1).reshape(256, 9 * cin).contiguous(), transposed=False, tile=256)
    wh = torch.zeros(32, 256, device='cuda')
    wh[:3] = head.rpn_cls.weight.detach().view(3, 256)
    wh[3:21] = head.rpn_reg.weight.detach().view(18, 256)
    wh_img, _ = ops.pack_weight(wh, transposed=False, tile=32)
    bh = torch.cat([head.rpn_cls.bias, head.rpn_reg.bias]).detach()
    _, _, h = ops.rpn_head_fwd(xs, wc_img, head.rpn_conv.bias.detach(), wh_img, bh, ncls=3, nreg=18, want_h=True)
    masks, r0 = [], 0
    for x in xs:
        n, _, hh, ww = x.shape
        masks.append((h[r0:r0 + n * hh * ww] > 0).view(n, hh, ww, 256).permute(0, 3, 1, 2).cpu())
        r0 += -(-n * hh * ww // 128) * 128
    return masks


def _oracle(sd, feats, dcls, dreg, masks=None):
    """float64 oracle forward + backward.  With `masks` the ReLU is teacher-forced to the kernels' mask: a pre-activation
    within rounding of zero may land on the other side in fp32, which moves that position's whole gradient; every such
    disagreement must be a near tie."""
    sd64 = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    xs64 = [x.double().requires_grad_(True) for x in feats]
    if masks is None:
        cls, reg = M.rpn_head_forward(sd64, xs64)
    else:
        cls, reg = _masked_forward(sd64, xs64, masks)
    torch.autograd.backward(cls + reg, [d.double() for d in dcls + dreg])
    return sd64, xs64, cls, reg


def _masked_forward(sd64, xs64, masks):
    cls, reg = [], []
    for x, m in zip(xs64, masks):
        pre = F.conv2d(x, sd64['rpn_conv.weight'], sd64['rpn_conv.bias'], padding=1)
        flips = m != (pre.detach() > 0)
        tie = 1e-4 * pre.detach().abs().max()
        assert flips.sum().item() <= max(2, pre.numel() // 20000)
        assert (pre.detach()[flips].abs() < tie).all()
        h = pre * m.double()
        cls.append(F.conv2d(h, sd64['rpn_cls.weight'], sd64['rpn_cls.bias']))
        reg.append(F.conv2d(h, sd64['rpn_reg.weight'], sd64['rpn_reg.bias']))
    return cls, reg


def _grads_out(feats, cin, seed):
    g = torch.Generator().manual_seed(seed)
    return ([torch.randn(x.shape[0], 3, x.shape[2], x.shape[3], generator=g) for x in feats],
            [torch.randn(x.shape[0], 18, x.shape[2], x.shape[3], generator=g) for x in feats])


@pytest.mark.gpu
@pytest.mark.parametrize('cin,batch', [(256, 1), (256, 3), (64, 1), (64, 3)])
def test_parity_with_oracle(cin, batch):
    sd = M.make_params(cin, seed=cin + batch)
    feats = M.make_feats(batch, ODD, cin, seed=batch)
    dcls, dreg = _grads_out(feats, cin, batch)
    head, xs, cls, reg = _run(sd, feats, dcls, dreg)
    sd64, xs64, c64, r64 = _oracle(sd, feats, dcls, dreg, _kernel_masks(sd, feats))
    for a, b in zip(cls + reg, c64 + r64):
        assert a.dtype == torch.float32 and rel(a, b) < 1e-4
    for n, p in head.named_parameters():
        assert rel(p.grad, sd64[n].grad) < 5e-4, n
    for a, b in zip(xs, xs64):
        assert rel(a.grad, b.grad) < 5e-4


@pytest.mark.gpu
@pytest.mark.parametrize('path', FIXTURES, ids=[os.path.basename(p)[:-3] for p in FIXTURES])
def test_fixture_forward(path):
    gold = load_golden(path)
    head = head_from(gold['params']).cuda()
    with torch.no_grad():
        cls, reg = head([x.cuda() for x in gold['feats']])
    for a, b in zip(cls + reg, gold['cls'] + gold['reg']):
        assert rel(a, b) < 1e-4


def _guarded(shapes, pad=64):
    """Output tensors inside NaN-filled buffers with `pad` guard elements on each side."""
    bufs, views = [], []
    for s in shapes:
        n = 1
        for v in s:
            n *= v
        b = torch.full((n + 2 * pad,), float('nan'), device='cuda')
        bufs.append(b)
        views.append(b[pad:pad + n].view(s))
    return bufs, views


def _guards_intact(bufs, pad=64):
    return all(torch.isnan(b[:pad]).all() and torch.isnan(b[-pad:]).all() for b in bufs)


@pytest.mark.gpu
@pytest.mark.parametrize('cin', [256, 96])
def test_kernels_vs_float64(cin):
    """The forward kernel and the dx kernel alone, at odd shapes (positions not a multiple of 128, H != W, 1x1 levels),
    writing into NaN-guarded buffers: every output element is written, nothing outside."""
    from sm3det_b200 import _lib, ops
    lib = _lib.load()
    sd = M.make_params(cin, seed=11)
    feats = [x.cuda() for x in M.make_feats(2, ODD, cin, seed=11)]
    shapes = [(x.shape[0], x.shape[2], x.shape[3]) for x in feats]
    wc, bc = sd['rpn_conv.weight'].cuda(), sd['rpn_conv.bias'].cuda()
    wh = torch.zeros(32, 256, device='cuda')
    wh[:3] = sd['rpn_cls.weight'].view(3, 256).cuda()
    wh[3:21] = sd['rpn_reg.weight'].view(18, 256).cuda()
    bh = torch.cat([sd['rpn_cls.bias'], sd['rpn_reg.bias']]).cuda()
    wc_img, _ = ops.pack_weight(wc.permute(0, 2, 3, 1).reshape(256, 9 * cin).contiguous(), transposed=False, tile=256)
    wh_img, _ = ops.pack_weight(wh, transposed=False, tile=32)
    cb, cls = _guarded([(n, 3, h, w) for n, h, w in shapes])
    rb, reg = _guarded([(n, 18, h, w) for n, h, w in shapes])
    R = ops.rpn_head_rows(shapes)
    hbuf = torch.full((R, 256), float('nan'), device='cuda')
    rc = lib.sm3_rpn_head_fwd(ops._ptr_array(feats), ops._ptr_array(cls), ops._ptr_array(reg), ops._shape_array(shapes), len(shapes),
                              cin, wc_img.data_ptr(), bc.data_ptr(), wh_img.data_ptr(), bh.data_ptr(), 3, 18, hbuf.data_ptr(), 3,
                              ops._stream())
    assert rc == 0, lib.sm3_last_error()
    torch.cuda.synchronize()
    assert _guards_intact(cb) and _guards_intact(rb)
    sd64 = {k: v.double() for k, v in sd.items()}
    c64, r64 = M.rpn_head_forward(sd64, [x.double().cpu() for x in feats])
    for a, b in zip(cls + reg, c64 + r64):
        assert not torch.isnan(a).any() and rel(a, b) < 1e-4
    # the saved ReLU output: every position row written, equal to the float64 hidden map
    r0 = 0
    for x in feats:
        n, _, h, w = x.shape
        hid = F.relu(F.conv2d(x.double().cpu(), sd64['rpn_conv.weight'], sd64['rpn_conv.bias'], padding=1))
        got = hbuf[r0:r0 + n * h * w].view(n, h, w, 256).permute(0, 3, 1, 2)
        assert not torch.isnan(got).any() and rel(got, hid) < 1e-4
        r0 += -(-n * h * w // 128) * 128

    # dx: the 3x3 conv of a row-major gradient with the flipped, transposed weight
    g = torch.Generator().manual_seed(5)
    dpre = torch.randn(R, 256, generator=g).cuda()
    wd = torch.zeros(256, 9 * 256, device='cuda')
    wd[:cin] = wc.flip(2, 3).permute(1, 2, 3, 0).reshape(cin, 9 * 256)
    wd_img, _ = ops.pack_weight(wd, transposed=False, tile=256)
    db, dx = _guarded([(n, cin, h, w) for n, h, w in shapes])
    rc = lib.sm3_rpn_head_dx(dpre.data_ptr(), ops._ptr_array(dx), ops._shape_array(shapes), len(shapes), cin, wd_img.data_ptr(), 3,
                             ops._stream())
    assert rc == 0, lib.sm3_last_error()
    torch.cuda.synchronize()
    assert _guards_intact(db)
    r0 = 0
    for d, (n, h, w) in zip(dx, shapes):
        dp = dpre[r0:r0 + n * h * w].double().cpu().view(n, h, w, 256).permute(0, 3, 1, 2)
        ref = F.conv_transpose2d(dp, sd64['rpn_conv.weight'], padding=1)
        assert not torch.isnan(d).any() and rel(d, ref) < 1e-4
        r0 += -(-n * h * w // 128) * 128


@pytest.mark.gpu
def test_eval_and_no_grad_save_nothing():
    sd = M.make_params(256, seed=2)
    feats = [x.cuda() for x in M.make_feats(2, [(64, 64), (32, 32)], 256, seed=2)]
    head = head_from(sd).cuda()
    cls_t, reg_t = head(feats)
    assert cls_t[0].grad_fn is not None
    h_bytes = (2 * 64 * 64 + 2 * 32 * 32) * 256 * 4
    for ctx in (torch.no_grad, torch.inference_mode):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        with ctx():
            head.eval()
            cls, reg = head(feats)
            head.train()
        torch.cuda.synchronize()
        assert cls[0].grad_fn is None
        assert torch.cuda.max_memory_allocated() - base < h_bytes
        assert all(torch.equal(a, b) for a, b in zip(cls + reg, cls_t + reg_t))


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
def test_autocast(dtype):
    sd = M.make_params(256, seed=9)
    feats = M.make_feats(2, ODD[:4], 256, seed=9)
    head = head_from(sd).cuda()
    xs = [x.cuda() for x in feats]
    c64, r64 = M.rpn_head_forward({k: v.double() for k, v in sd.items()}, [x.double() for x in feats])
    scaler = torch.amp.GradScaler('cuda') if dtype == torch.float16 else None
    with torch.autocast('cuda', dtype=dtype):
        cls, reg = head([x.to(dtype) for x in xs] if dtype == torch.float16 else xs)
    assert all(o.dtype == torch.float32 for o in cls + reg)
    l2 = lambda a, b: ((a.detach().double().cpu() - b).norm() / b.norm()).item()
    e = max(l2(a, b) for a, b in zip(cls + reg, c64 + r64))
    assert 1e-4 < e < 5e-2
    loss = sum(o.square().mean() for o in cls + reg)
    (scaler.scale(loss) if scaler else loss).backward()
    assert all(torch.isfinite(p.grad).all() for p in head.parameters())
    from sm3det_b200 import ops
    assert ops.current_passes() == 3


@pytest.mark.gpu
def test_graph_replay_matches_eager():
    sd = M.make_params(256, seed=4)
    feats = [x.cuda() for x in M.make_feats(2, ODD[:5], 256, seed=4)]
    dcls, dreg = _grads_out(feats, 256, 4)
    dcls, dreg = [d.cuda() for d in dcls], [d.cuda() for d in dreg]
    head = head_from(sd).cuda()
    xs = [x.clone().requires_grad_(True) for x in feats]

    def step():
        for p in head.parameters():
            p.grad = None
        for x in xs:
            x.grad = None
        cls, reg = head(xs)
        torch.autograd.backward(cls + reg, dcls + dreg)
        return [o.detach() for o in cls + reg]

    eager = [o.clone() for o in step()]
    eager_g = [p.grad.clone() for p in head.parameters()] + [x.grad.clone() for x in xs]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    for p in head.parameters():
        p.grad = None
    with torch.cuda.graph(graph):
        outs = step()
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(outs, eager))
    got_g = [p.grad for p in head.parameters()] + [x.grad for x in xs]
    for a, b in zip(got_g, eager_g):
        assert rel(a, b) < 1e-5       # split-K weight gradients add their partials with atomics in any order


@pytest.mark.gpu
def test_repeated_launches_bitwise_identical():
    sd = M.make_params(256, seed=6)
    feats = M.make_feats(3, ODD, 256, seed=6)
    dcls, dreg = _grads_out(feats, 256, 6)
    runs = []
    for _ in range(2):
        head, xs, cls, reg = _run(sd, feats, dcls, dreg)
        runs.append(([o.detach() for o in cls + reg], [x.grad for x in xs], head.rpn_conv.bias.grad, head.rpn_cls.bias.grad))
    (o1, dx1, _, _), (o2, dx2, _, _) = runs
    assert all(torch.equal(a, b) for a, b in zip(o1, o2))
    assert all(torch.equal(a, b) for a, b in zip(dx1, dx2))


@pytest.mark.gpu
def test_fpn_then_head_matches_oracle():
    """MultitaskFPN (start_level 0, 'on_output', 5 outs) followed by the head, against the oracle FPN + oracle head."""
    from oracle.fpn_oracle import fpn_forward, fpn_param_shapes
    from sm3det_b200.neck import MultitaskFPN
    widths, sizes = [32, 64, 96, 128], [(32, 40), (16, 20), (8, 10), (4, 5)]
    kw = dict(in_channels=widths, out_channels=256, num_outs=5, start_level=0, add_extra_convs='on_output')
    g = torch.Generator().manual_seed(8)
    fsd = {k: torch.randn(s, generator=g) * ((s[1] * s[2] * s[3]) ** -0.5 if len(s) == 4 else 0.1)
           for k, s in fpn_param_shapes(widths, 256, 5, 0, 'on_output').items()}
    neck = MultitaskFPN(**kw)
    neck.load_state_dict(fsd, strict=True)
    neck = neck.cuda()
    hsd = M.make_params(256, seed=8)
    head = head_from(hsd).cuda()
    inputs = [torch.randn(2, c, h, w, generator=g) for c, (h, w) in zip(widths, sizes)]
    xs = [x.cuda().requires_grad_(True) for x in inputs]
    cls, reg = head(list(neck(xs)))
    loss = sum(o.square().mean() for o in cls + reg)
    loss.backward()
    fsd64 = {k: v.double().requires_grad_(True) for k, v in fsd.items()}
    hsd64 = {k: v.double().requires_grad_(True) for k, v in hsd.items()}
    xs64 = [x.double().requires_grad_(True) for x in inputs]
    masks = _kernel_masks(hsd, [p.detach() for p in neck(xs)])
    c64, r64 = _masked_forward(hsd64, list(fpn_forward(fsd64, xs64, 4, 5, 0, 'on_output')), masks)
    sum(o.square().mean() for o in c64 + r64).backward()
    for a, b in zip(cls + reg, c64 + r64):
        assert rel(a, b) < 1e-4
    for n, p in head.named_parameters():
        assert rel(p.grad, hsd64[n].grad) < 5e-4, n
    for n, p in neck.named_parameters():
        assert rel(p.grad, fsd64[n].grad) < 5e-4, n
    for a, b in zip(xs, xs64):
        assert rel(a.grad, b.grad) < 5e-4
