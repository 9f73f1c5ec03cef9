"""mmdet FPN (sm3det_b200.neck.FPN), the neck of the single-dataset LSKNet, VAN and ConvNeXt configs.

CPU: tests/fpn_mmdet_ref.py reproduces the fixtures tools/gen_golden_fpn.py made from the unmodified reference (and the live
reference when its tree is present); every neck dict of the shipped configs builds with mmdet's state_dict layout; the
options no config uses raise.  GPU: forward and every gradient against the oracle in the three modes, the max-pool export
kernels against a float64 reference, which kernels ran, and a CUDA-graph replay."""
import glob
import os
import re

import numpy as np
import pytest
import torch

import fpn_mmdet_ref as M
from oracle.cases import load_golden
from sm3det_b200.synth import make_state_dict

GOLD = os.path.join(os.path.dirname(__file__), 'golden', 'fpn_mmdet')
T, S, CT, CB = [32, 64, 160, 256], [64, 128, 320, 512], [96, 192, 384, 768], [128, 256, 512, 1024]
ON_OUTPUT = dict(start_level=1, add_extra_convs='on_output')
ON_INPUT = dict(start_level=1, add_extra_convs='on_input')
# The distinct neck dicts of the 39 shipped configs that pair mmdet's FPN with a backbone of this project
# (configs/lsknet/*, local_configs/{dota,dronevehicle,sardet50k}_*; StripLSKNet has no backbone source), and their configs.
CONFIG_NECKS = {
    'maxpool_t': ({}, T, ['lsk_t_fpn_1x_dota_le90', 'dota_lsk_t_orcnn', 'dronevehicle_lsk_t_orcnn', 'dota_van_t_orcnn',
                          'dronevehicle_van_t_orcnn']),
    'maxpool_s': ({}, S, ['lsk_s_ema_fpn_1x_dota_le90', 'lsk_s_fpn_1x_dota_le90', 'lsk_s_fpn_1x_fair_le90',
                          'lsk_s_fpn_3x_hrsc_le90', 'dota_lsk_s_orcnn', 'dronevehicle_lsk_s_orcnn', 'dota_lsk_b_orcnn',
                          'dronevehicle_lsk_b_orcnn', 'dota_van_s_orcnn', 'dronevehicle_van_s_orcnn', 'dota_van_b_orcnn',
                          'dronevehicle_van_b_orcnn']),
    'maxpool_convnext_t': ({}, CT, ['dota_convnext_t_orcnn', 'dota_convnext_t_roitrans', 'dota_convnext_s_orcnn',
                                    'dronevehicle_convnext_t_orcnn', 'dronevehicle_convnext_t_roitrans',
                                    'dronevehicle_convnext_s_orcnn', 'sardet50k_convnext_t_cascade',
                                    'sardet50k_convnext_t_frcnn']),
    'maxpool_convnext_b': ({}, CB, ['dota_convnext_b_orcnn', 'dronevehicle_convnext_b_orcnn']),
    'on_output_t': (ON_OUTPUT, T, ['sardet50k_lsk_t_gfl', 'sardet50k_van_t_gfl']),
    'on_output_s': (ON_OUTPUT, S, ['sardet50k_lsk_s_gfl', 'sardet50k_lsk_b_gfl', 'sardet50k_van_s_gfl',
                                   'sardet50k_van_b_gfl']),
    'on_output_convnext_t': (ON_OUTPUT, CT, ['sardet50k_convnext_t_gfl', 'sardet50k_convnext_t_retina',
                                             'sardet50k_convnext_s_gfl']),
    'on_output_convnext_b': (ON_OUTPUT, CB, ['sardet50k_convnext_b_gfl']),
    'on_input_convnext_t': (ON_INPUT, CT, ['dota_convnext_t_s2anet', 'dronevehicle_convnext_t_s2anet']),
}


def neck_dict(name):
    extra, widths, _ = CONFIG_NECKS[name]
    return dict(type='FPN', in_channels=list(widths), out_channels=256, num_outs=5, **extra)


def _shapes(kw):
    return M.fpn_mmdet_param_shapes(kw['in_channels'], kw['out_channels'], kw['num_outs'], kw.get('start_level', 0),
                                    kw.get('add_extra_convs', False))


def _reference_module():
    from oracle import ref_shim
    if not ref_shim.reference_available():
        pytest.skip('reference tree not present')
    return ref_shim.load_reference_module('Multitask_FPN', 'necks')


def _reference_fpn(mod, kw):
    """The reference MultitaskFPN that computes FPN(**kw): start_level=0, extra_level=s (called with start_level=s)."""
    s = kw.get('start_level', 0)
    return mod.MultitaskFPN(start_level=0, extra_level=s, **{k: v for k, v in kw.items() if k not in ('type', 'start_level')})


# ---- CPU -------------------------------------------------------------------------------------------------------------
def test_config_inventory():
    names = [c for _, _, cfgs in CONFIG_NECKS.values() for c in cfgs]
    assert len(names) == len(set(names)) == 39
    assert sum(len(c) for e, _, c in CONFIG_NECKS.values() if not e) == 27
    assert sum(len(c) for e, _, c in CONFIG_NECKS.values() if e == ON_OUTPUT) == 10


FIXTURES = sorted(glob.glob(os.path.join(GOLD, '*.pt')))


def test_fixtures_present():
    assert {os.path.basename(p)[:-3] for p in FIXTURES} == set(M.GOLDEN_CASES)


@pytest.mark.parametrize('path', FIXTURES, ids=lambda p: os.path.basename(p)[:-3])
def test_oracle_reproduces_fixture(path):
    gold = load_golden(path)
    kw = gold['kw']
    assert kw == M.GOLDEN_CASES[gold['name']]
    sd = make_state_dict(_shapes(kw), gold['sd_seed'], True)
    assert sorted(sd) == gold['keys']
    xs = M.fpn_inputs(kw['in_channels'], gold['batch'], gold['sizes'], gold['seed'])
    with torch.no_grad():
        outs = M.fpn_forward_mmdet(sd, xs, kw['num_outs'], kw.get('start_level', 0), kw.get('add_extra_convs', False))
    assert len(outs) == len(gold['outs']) == kw['num_outs']
    for o, g in zip(outs, gold['outs']):       # generated bit-exact; 2e-6 tolerates another CPU's kernel selection
        torch.testing.assert_close(o, g, rtol=2e-6, atol=2e-6)


@pytest.mark.parametrize('name', ['maxpool_t', 'on_output_t', 'on_input_convnext_t'])
def test_oracle_matches_live_reference(name):
    """Odd map sizes (17/9/5/3: P6 = 2x2, and a 17 -> 9 top-down step) on the reference under the re-indexing."""
    mod = _reference_module()
    kw = dict(neck_dict(name), out_channels=32)
    s = kw.get('start_level', 0)
    sd = make_state_dict(_shapes(kw), 8, True)
    torch.manual_seed(0)
    ref = _reference_fpn(mod, kw)
    rsd = ref.state_dict()
    rsd.update({M.to_multitask_key(k, s): v for k, v in sd.items()})
    ref.load_state_dict(rsd, strict=True)
    xs = M.fpn_inputs(kw['in_channels'], 2, (17, 9, 5, 3), 4)
    with torch.no_grad():
        want = ref(xs, start_level=s)
        got = M.fpn_forward_mmdet(sd, xs, 5, s, kw.get('add_extra_convs', False))
    assert len(want) == len(got) == 5
    for a, b in zip(want, got):
        torch.testing.assert_close(b, a, rtol=2e-6, atol=2e-6)


@pytest.mark.parametrize('name', list(CONFIG_NECKS))
def test_config_neck_builds_with_mmdet_layout(name):
    from sm3det_b200.neck import FPN, ROTATED_NECKS
    d = neck_dict(name)
    net = ROTATED_NECKS.build(dict(d))
    assert type(net) is FPN
    sd = {k: tuple(v.shape) for k, v in net.state_dict().items()}
    assert sd == {k: tuple(v) for k, v in _shapes(d).items()}
    net.load_state_dict(make_state_dict(_shapes(d), 0, True), strict=True)
    from oracle import ref_shim
    if not ref_shim.reference_available():
        return
    rsd = M.from_multitask_state_dict(_reference_fpn(_reference_module(), d).state_dict(), d.get('start_level', 0))
    assert {k: tuple(v.shape) for k, v in rsd.items()} == sd


@pytest.mark.parametrize('bad', [dict(norm_cfg=dict(type='GN', num_groups=32)), dict(act_cfg=dict(type='ReLU')),
                                 dict(conv_cfg=dict(type='Conv2d')), dict(relu_before_extra_convs=True),
                                 dict(upsample_cfg=dict(scale_factor=2, mode='nearest')),
                                 dict(upsample_cfg=dict(mode='bilinear')),
                                 dict(in_channels=[32, 64, 160, 250]), dict(out_channels=200)],
                         ids=['norm_cfg', 'act_cfg', 'conv_cfg', 'relu_before_extra_convs', 'scale_factor', 'bilinear',
                              'in_channels', 'out_channels'])
def test_unsupported_options_raise(bad):
    from sm3det_b200.neck import FPN
    kw = dict(neck_dict('maxpool_t'), add_extra_convs='on_output', **bad)
    kw.pop('type')
    with pytest.raises(NotImplementedError, match='sm3det_b200 FPN'):
        FPN(**kw)


def test_cpu_inputs_raise():
    from sm3det_b200 import FPN
    kw = neck_dict('maxpool_t')
    kw.pop('type')
    net = FPN(**kw)
    with pytest.raises(RuntimeError, match='CUDA'):
        net(M.fpn_inputs(T, 1, (16, 8, 4, 2), 0))          # no fallback path


def test_fpn_is_not_force_registered_as_a_backbone():
    """FPN is opt-in: register_into_mmrotate() exposes the backbones only, so mmdet's own FPN stays the default."""
    import sm3det_b200
    from sm3det_b200.neck import FPN, ROTATED_NECKS
    assert sm3det_b200.FPN is FPN and ROTATED_NECKS.get('FPN') is FPN
    assert 'FPN' not in sm3det_b200.ROTATED_BACKBONES.module_dict


# ---- GPU: the neck against the oracle --------------------------------------------------------------------------------
def _rel(a, b):
    return ((a.detach().cpu() - b.detach()).abs().max() / (b.detach().abs().max() + 1e-30)).item()


@pytest.mark.gpu
@pytest.mark.parametrize('widths', ['t', 'convnext_b'])
@pytest.mark.parametrize('mode', ['maxpool', 'on_output', 'on_input'])
def test_fpn_gpu_matches_oracle(mode, widths):
    """40/20/10/5 maps at batch 2: P5 is 5x5 and the max-pool P6 3x3 (ceil)."""
    from sm3det_b200.neck import ROTATED_NECKS
    extra = {'maxpool': {}, 'on_output': ON_OUTPUT, 'on_input': ON_INPUT}[mode]
    kw = dict(type='FPN', in_channels={'t': T, 'convnext_b': CB}[widths], out_channels=256, num_outs=5, **extra)
    s, src = kw.get('start_level', 0), kw.get('add_extra_convs', False)
    sd = make_state_dict(_shapes(kw), 3, True)
    net = ROTATED_NECKS.build(dict(kw))
    net.load_state_dict(sd, strict=True)
    net = net.cuda()
    xs = M.fpn_inputs(kw['in_channels'], 2, (40, 20, 10, 5), 6)
    xc = [x.clone().requires_grad_(True) for x in xs]
    sdg = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    want = M.fpn_forward_mmdet(sdg, xc, 5, s, src)
    xg = [x.cuda().requires_grad_(True) for x in xs]
    got = net(xg)
    assert len(got) == len(want) == 5
    assert all(g.is_contiguous() and g.shape == w.shape for g, w in zip(got, want))
    assert max(_rel(g, w) for g, w in zip(got, want)) < 1e-4
    ups = [torch.randn(w.shape, generator=torch.Generator().manual_seed(50 + i)) / w.numel() ** 0.5 for i, w in enumerate(want)]
    sum((w * u).sum() for w, u in zip(want, ups)).backward()
    sum((g * u.cuda()).sum() for g, u in zip(got, ups)).backward()
    for name, p in net.named_parameters():
        assert sdg[name].grad is not None and p.grad is not None, name
        assert _rel(p.grad, sdg[name].grad) < 5e-4, name
    for i in range(4):
        if i < s:
            assert xg[i].grad is None and xc[i].grad is None, i
        else:
            assert _rel(xg[i].grad, xc[i].grad) < 5e-4, i


# ---- GPU: the export kernels against float64 ------------------------------------------------------------------------
SENT = 0x7FA11A11        # a NaN payload no kernel produces
FRONT, PAD_IN = 64, 256


class _Out:
    """An output window inside a sentinel-filled buffer as long as the window on each side."""

    def __init__(self, shape):
        self.shape, self.n = tuple(shape), int(np.prod(shape))
        self.big = torch.full((FRONT + 2 * self.n + FRONT,), SENT, dtype=torch.int32).cuda()
        self.t = self.big[FRONT:FRONT + self.n].view(torch.float32).view(self.shape)

    def get(self, what):
        b = self.big.cpu().numpy()
        assert np.all(b[:FRONT] == SENT) and np.all(b[FRONT + self.n:] == SENT), f'{what}: written outside its window'
        return b[FRONT:FRONT + self.n].view(np.float32).reshape(self.shape)


def _cu(t):
    """t on the GPU inside a NaN-filled buffer: a read past either end turns an output into NaN."""
    flat = t.contiguous().reshape(-1)
    big = torch.full((FRONT + flat.numel() + PAD_IN,), float('nan'))
    big[FRONT:FRONT + flat.numel()] = flat
    return big.cuda()[FRONT:FRONT + flat.numel()].view(t.shape)


def _scaled(g, *shape):
    """randn with a per-channel (last axis) scale 2^k, k in [-8, 8], mixed signs."""
    k = torch.randint(-8, 9, (shape[-1],), generator=g).double()
    return (torch.randn(*shape, generator=g, dtype=torch.float64) * torch.exp2(k)).float()


def _ptrs(ts):
    import ctypes
    return (ctypes.c_void_p * len(ts))(*[None if t is None else t.data_ptr() for t in ts])


@pytest.mark.gpu
@pytest.mark.parametrize('N,H,W,C,L', [(2, 5, 5, 36, 1), (2, 7, 6, 64, 2), (3, 8, 8, 256, 1), (2, 33, 17, 96, 2),
                                       (1, 1, 1, 32, 2), (4, 256, 256, 64, 2)])
def test_export_pool_kernels_vs_float64(N, H, W, C, L):
    from sm3det_b200 import _lib, ops
    lib = _lib.load()
    g = torch.Generator().manual_seed(H * 1000 + W * 10 + L)
    shapes = ops.fpn_pool_shapes(N, C, H, W, L)
    x = _scaled(g, N, H, W, C)
    outs = [_Out(s) for s in shapes]
    _lib.check(lib.sm3_fpn_export_pool(_cu(x).data_ptr(), _ptrs([o.t for o in outs]), N, H, W, C, L,
                                       torch.cuda.current_stream().cuda_stream), 'sm3_fpn_export_pool')
    levels = [x.permute(0, 3, 1, 2).double()]
    for _ in range(L):
        levels.append(torch.nn.functional.max_pool2d(levels[-1], 1, stride=2))
    for k, (o, want) in enumerate(zip(outs, levels)):
        assert want.shape == torch.Size(shapes[k])
        assert torch.equal(want, levels[0][:, :, ::2 ** k, ::2 ** k])
        got = o.get(f'level {k}')
        assert np.array_equal(got.view(np.uint32), want.float().numpy().view(np.uint32)), k     # a copy: bit for bit
    ds = [_scaled(g, s[0], s[2], s[3], s[1]).permute(0, 3, 1, 2).contiguous() for s in shapes]
    din = _Out((N, H, W, C))
    dcu = [_cu(d) for d in ds]
    _lib.check(lib.sm3_fpn_export_pool_bwd(_ptrs(dcu), din.t.data_ptr(), N, H, W, C, L,
                                           torch.cuda.current_stream().cuda_stream), 'sm3_fpn_export_pool_bwd')
    got = din.get('din')
    # float64 autograd of the same outputs
    xr = levels[0].clone().requires_grad_(True)
    lv = [xr]
    for _ in range(L):
        lv.append(torch.nn.functional.max_pool2d(lv[-1], 1, stride=2))
    sum((a * d.double()).sum() for a, d in zip(lv, ds)).backward()
    want = xr.grad.permute(0, 2, 3, 1).numpy()
    terms = torch.zeros_like(xr)
    for k, d in enumerate(ds):
        terms[:, :, ::2 ** k, ::2 ** k] += d.double().abs()
    u = 2.0 ** -24
    bound = L * u / (1 - L * u) * terms.permute(0, 2, 3, 1).numpy()      # an (L+1)-term fp32 sum: L roundings
    err = np.abs(got.astype(np.float64) - want)
    assert np.all(np.isfinite(got))
    assert np.all(err <= bound), float((err - bound).max())
    # and the summation order the kernel documents: P_top, then levels 1..L
    emu = ds[0].permute(0, 2, 3, 1).numpy().copy()
    for k in range(1, L + 1):
        emu[:, ::2 ** k, ::2 ** k] += ds[k].permute(0, 2, 3, 1).numpy()
    assert np.array_equal(got.view(np.uint32), emu.view(np.uint32))


@pytest.mark.gpu
def test_export_pool_rejects_bad_arguments():
    from sm3det_b200 import _lib
    lib = _lib.load()
    x = torch.zeros(1, 4, 4, 32, device='cuda')
    o = [torch.zeros(1, 32, 4, 4, device='cuda'), torch.zeros(1, 32, 2, 2, device='cuda')]
    stream = torch.cuda.current_stream().cuda_stream
    assert lib.sm3_fpn_export_pool(x.data_ptr(), _ptrs(o), 1, 4, 4, 32, 0, stream) != 0       # L = 0
    assert lib.sm3_fpn_export_pool(x.data_ptr(), _ptrs(o), 1, 4, 4, 32, 9, stream) != 0       # L > SM3_FPN_MAX_POOL_LEVELS
    assert lib.sm3_fpn_export_pool(x.data_ptr(), _ptrs([o[0], None]), 1, 4, 4, 32, 1, stream) != 0
    assert lib.sm3_fpn_export_pool_bwd(_ptrs(o), None, 1, 4, 4, 32, 1, stream) != 0
    assert b'fpn_export_pool' in lib.sm3_last_error()


# ---- GPU: which kernels ran, and a captured step ---------------------------------------------------------------------
def _cuda_kernels(fn, tries=5):
    """Names of the CUDA kernels fn launches (retried: the profiler occasionally records no CUDA activity)."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(tries):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
        if any(not n.startswith(('Memcpy', 'Memset')) for n in names):
            return names
    return names


def _maxpool_net_and_inputs():
    from sm3det_b200 import FPN
    kw = neck_dict('maxpool_t')
    kw.pop('type')
    net = FPN(**kw)
    net.load_state_dict(make_state_dict(_shapes(neck_dict('maxpool_t')), 2, True), strict=True)
    xs = [x.cuda().requires_grad_(True) for x in M.fpn_inputs(T, 2, (32, 16, 8, 4), 9)]
    return net.cuda(), xs


@pytest.mark.gpu
def test_export_pool_kernels_run():
    net, xs = _maxpool_net_and_inputs()
    held = {}
    fwd = _cuda_kernels(lambda: held.__setitem__('outs', net(xs)))
    assert any(re.search(r'fpn_export_pool_kernel', n) for n in fwd), sorted(fwd)
    assert not any('max_pool' in n for n in fwd)
    outs = held['outs']
    bwd = _cuda_kernels(lambda: sum(o.sum() for o in outs).backward())
    assert any(re.search(r'fpn_export_pool_bwd_kernel', n) for n in bwd), sorted(bwd)
    assert not any('max_pool' in n for n in bwd)


@pytest.mark.gpu
def test_graph_replay_matches_eager():
    from sm3det_b200.graphed import GraphedStep
    net, xs = _maxpool_net_and_inputs()
    xs = [x.detach() for x in xs]
    ups = None

    def step(*inp):
        nonlocal ups
        outs = net(list(inp))
        if ups is None:
            ups = [torch.randn(o.shape, generator=torch.Generator().manual_seed(70 + i)).cuda() / o.numel() ** 0.5
                   for i, o in enumerate(outs)]
        loss = sum((o * u).sum() for o, u in zip(outs, ups))
        loss.backward()
        return tuple(o.detach() for o in outs)

    g = GraphedStep(step, xs, net.parameters())
    got = [o.clone() for o in g(*xs)]
    got_grads = {n: p.grad.clone() for n, p in net.named_parameters()}
    for p in net.parameters():
        p.grad = None
    eager = step(*xs)
    torch.cuda.synchronize()
    assert len(got) == len(eager) == 5
    for a, b in zip(got, eager):
        assert float((a - b).abs().max()) <= 1e-6 * float(b.abs().max()), 'replayed outputs differ from eager'
    for n, p in net.named_parameters():
        assert float((got_grads[n] - p.grad).abs().max()) <= 1e-5 * float(p.grad.abs().max()) + 1e-30, n
