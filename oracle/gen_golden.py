"""Generate tests/golden/*.pt by running the UNMODIFIED reference (via oracle/ref_shim.py).

Needs the reference tree (SM3DET_REFERENCE_ROOT):  python -m oracle.gen_golden [case ...]   or   python -m oracle.gen_golden live
Every case also asserts that the restated oracle reproduces the reference bit-for-bit on CPU
(forward outputs, gate loss, routing decisions, parameter gradients) -- this is what pins the
oracle.  Fixtures hold no weights: those are regenerated from seeds by sm3det_b200.synth.
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_shim                                   # noqa: E402
from oracle.cases import CASES, make_noise, save_golden, summarize_grad, upstream_grads   # noqa: E402
from oracle.convnext_moe_oracle import OracleConfig, backbone_forward, param_shapes, tie_da_weights  # noqa: E402
from sm3det_b200.synth import make_images, make_state_dict, state_dict_checksum    # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden')


def moe_token_counts(cfg, n, h, w):
    counts = []
    for i in range(4):
        t = n * (h // (4 * 2 ** i)) * (w // (4 * 2 ** i))
        counts += [t] * len(cfg.moe_blocks(i))
    return counts


def moe_digest(r, full):
    """What a fixture keeps of one MoE layer.  Full-size cases: int8 indices + the (k)-vs-(k+1) logit gap per token (the
    margin a routing flip is judged against) instead of the gate values."""
    d = dict(prefix=r['prefix'], importance=r['importance'], load=r['load'], loss=r['loss'])
    if not full:
        d.update(top_idx=r['top_idx'].to(torch.int16), top_gates=r['top_gates'])
        return d
    k = r['top_idx'].shape[1]
    lg = r['logits']
    top = lg.topk(min(k + 1, lg.shape[1]), dim=-1).values
    d.update(top_idx=r['top_idx'].to(torch.int8), logit_scale=float(lg.abs().max()),
             gap=(top[:, k - 1] - top[:, k]).float() if top.shape[1] > k else torch.full((lg.shape[0],), float('inf')))
    return d


def run_case(name, spec):
    kw = dict(spec['kw'])
    da = bool(spec.get('da', False))
    datasets = spec.get('datasets')
    cfg = OracleConfig(da=da, **kw)
    if da:
        net = ref_shim.build_reference_backbone('ConvNeXt_DA_MultiInput', seed=0, module='convnext_moe_DA', **kw)
    else:
        net = ref_shim.build_reference_backbone('ConvNeXt_moe_MultiInput', seed=0, **kw)
    call = (lambda inp: net(inp, datasets)) if da else net
    okw = dict(datasets=datasets) if da else {}
    shapes = param_shapes(cfg)
    rsd = net.state_dict()
    assert set(shapes) == set(rsd), set(shapes) ^ set(rsd)
    for k, s in shapes.items():
        assert tuple(rsd[k].shape) == tuple(s), k
    sd = make_state_dict(shapes, seed=0, trained_like=(spec['weights'] == 'trained'))
    if da:
        tie_da_weights(sd)                      # the reference registers ONE Sequential three times (fc.2's values survive a load)
    net.load_state_dict(sd, strict=True)
    n, h, w = spec['img']
    x = make_images(n, h, w, seed=1234)
    mode = spec['mode']
    gold = dict(name=name, kw=kw, img=spec['img'], mode=mode, weights=spec['weights'],
                sd_checksum=state_dict_checksum(sd), x_checksum=float(x.double().abs().sum()))
    if da:
        gold.update(da=True, datasets=list(datasets))
        if len(datasets) > 1:
            x = [x[i:i + 1] for i in range(n)]      # the detector passes one tensor per modality (trisource detector :141-153)
    record = []
    st = spec['stride']
    if mode == 'eval':
        net.eval()
        with torch.no_grad():
            ref = call(x)
            orc = backbone_forward(sd, cfg, x, train=False, record=record, **okw)
    else:
        net.train()
        noise = None
        if mode == 'train_noisy':
            noise = make_noise(cfg, moe_token_counts(cfg, n, h, w))
            it = iter(noise)
            orig = torch.randn_like
            torch.randn_like = lambda t, *a, **k: next(it).to(t.dtype)   # inject the noise stream
        try:
            ref = call(x)
        finally:
            if mode == 'train_noisy':
                torch.randn_like = orig
        sdg = {k: (v.clone().requires_grad_(True) if v.is_floating_point() and 'ffn.mean' not in k and 'ffn.std' not in k else v)
               for k, v in sd.items()}
        if da:
            tie_da_weights(sdg)
        orc = backbone_forward(sdg, cfg, x, train=True, noise=noise, record=record, **okw)
    has_loss = isinstance(ref, tuple) and len(ref) == 2 and isinstance(ref[0], tuple)
    r_outs, r_loss = (ref if has_loss else (ref, None))
    o_outs, o_loss = (orc if has_loss else (orc, None))
    for a, b in zip(r_outs, o_outs):
        assert torch.equal(a, b), f'{name}: oracle output differs from reference by {(a - b).abs().max()}'
    if has_loss:
        assert torch.equal(r_loss, o_loss), (r_loss, o_loss)
        gold['gate_loss'] = r_loss.detach().clone()
    gold['outs'] = [o.detach()[:, :, ::st, ::st].clone() for o in r_outs]
    gold['out_l2'] = [o.detach().double().norm().item() for o in r_outs]
    gold['stride'] = st
    gold['moe'] = [moe_digest(r, spec.get('full', False)) for r in record]
    if mode != 'eval':
        ups = upstream_grads(r_outs)
        (sum((o * g).sum() for o, g in zip(r_outs, ups)) + (r_loss if has_loss else 0.0)).backward()
        (sum((o * g).sum() for o, g in zip(o_outs, ups)) + (o_loss if has_loss else 0.0)).backward()
        grads = {}
        for pname, p in net.named_parameters():
            og = sdg[pname].grad
            if p.grad is None:
                assert og is None or float(og.abs().max()) == 0.0, pname
                continue
            assert og is not None, pname
            if spec.get('full', False):
                # multi-threaded CPU reductions over >= 10^5 tokens are not run-to-run bit-stable (the reference differs
                # from ITSELF in the last bit between runs); forward outputs, loss and routing above stay bit-exact
                assert float((p.grad - og).abs().max()) <= 1e-5 * float(og.abs().max()) + 1e-12, \
                    f'{name}: grad {pname} differs by {(p.grad - og).abs().max()}'
            else:
                assert torch.equal(p.grad, og), f'{name}: grad {pname} differs by {(p.grad - og).abs().max()}'
            # thousands of expert parameters (config 4): keep the digests small -- the GPU test compares full gradients
            # against the live oracle anyway, the digests only pin oracle == reference
            grads[pname] = summarize_grad(p.grad, 256, 24) if len(shapes) > 1500 else summarize_grad(p.grad)
        gold['grads'] = grads
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, name + '.pt')
    save_golden(gold, path)
    print(f'{name}: ok, moe layers {len(record)}')


def run_lsk_case(name, spec):
    """LSKNet-MoE: run the unmodified reference lsk_moe.py, assert the restated oracle reproduces it bit-for-bit
    (outputs, gate loss, routing, parameter gradients, BatchNorm running statistics), save the fixture."""
    import torch.nn.functional as F
    from oracle.cases import lsk_plan, make_drop_masks
    from oracle.lsk_moe_oracle import LskConfig, lsk_backbone_forward, lsk_param_shapes
    kw = dict(spec['kw'])
    unit = spec.get('unit', 'lsk')
    cfg = LskConfig(spatial_unit=unit, **kw)
    mod = ref_shim.load_reference_module('lsk_moe' if unit == 'lsk' else 'van_moe')
    torch.manual_seed(0)
    cls = mod.LSKNet_moe_MultiInput if unit == 'lsk' else mod.VAN_moe_MultiInput
    net = cls(norm_cfg=dict(type='SyncBN', requires_grad=True), **kw)
    shapes = lsk_param_shapes(cfg)
    rsd = net.state_dict()
    assert set(shapes) == set(rsd), set(shapes) ^ set(rsd)
    for k, sh in shapes.items():
        assert tuple(rsd[k].shape) == tuple(sh), k
    sd = make_state_dict(shapes, seed=0, trained_like=True)
    net.load_state_dict(sd, strict=True)
    n, h, w = spec['img']
    x = make_images(n, h, w, seed=1234)
    mode = spec['mode']
    gold = dict(name=name, kw=kw, img=spec['img'], mode=mode, weights='trained', family='lsk', unit=unit,
                sd_checksum=state_dict_checksum({k: v.float() for k, v in sd.items()}), x_checksum=float(x.double().abs().sum()))
    record, bn_state = [], {}
    no_grad_keys = ('running_', 'num_batches', '.mean', '.std')
    if mode == 'eval':
        net.eval()
        with torch.no_grad():
            ref = net(x)
            orc = lsk_backbone_forward(sd, cfg, x, train=False, record=record)
    else:
        net.train()
        noise = drops = None
        tokens, dshapes = lsk_plan(cfg, n, h, w)
        orig_randn, orig_drop = torch.randn_like, F.dropout
        if mode == 'train_noisy':
            noise = [torch.randn(t, cfg.num_experts, generator=torch.Generator().manual_seed(7 + i)) for i, t in enumerate(tokens)]
            it = iter(noise)
            torch.randn_like = lambda t, *a, **k: next(it).to(t.dtype)
        if cfg.drop_rate > 0:
            drops = make_drop_masks(dshapes, cfg.drop_rate)
            dit = iter(drops)
            F.dropout = lambda t, p=0.5, training=True, inplace=False: t * next(dit) if training else t
        try:
            ref = net(x)
        finally:
            torch.randn_like, F.dropout = orig_randn, orig_drop
        sdg = {k: (v.clone().requires_grad_(True) if v.is_floating_point() and not any(t in k for t in no_grad_keys) else v)
               for k, v in sd.items()}
        orc = lsk_backbone_forward(sdg, cfg, x, train=True, noise=noise, drop_masks=drops, record=record, bn_state=bn_state)
    has_loss = isinstance(ref, tuple) and len(ref) == 2 and isinstance(ref[0], tuple)
    r_outs, r_loss = (ref if has_loss else (ref, None))
    o_outs, o_loss = (orc if has_loss else (orc, None))
    for a, b in zip(r_outs, o_outs):
        assert torch.equal(a, b), f'{name}: oracle output differs from reference by {(a - b).abs().max()}'
    if has_loss:
        assert torch.equal(r_loss, o_loss), (r_loss, o_loss)
        gold['gate_loss'] = r_loss.detach().clone()
    st = spec.get('stride', 1)
    gold['outs'] = [o.detach()[:, :, ::st, ::st].clone() for o in r_outs]
    gold['out_l2'] = [o.detach().double().norm().item() for o in r_outs]
    gold['stride'] = st
    gold['moe'] = [moe_digest(r, spec.get('full', False)) for r in record]
    if mode != 'eval':
        ups = upstream_grads(r_outs)
        (sum((o * g).sum() for o, g in zip(r_outs, ups)) + (r_loss if has_loss else 0.0)).backward()
        (sum((o * g).sum() for o, g in zip(o_outs, ups)) + (o_loss if has_loss else 0.0)).backward()
        grads = {}
        for pname, p in net.named_parameters():
            og = sdg[pname].grad
            if p.grad is None:
                assert og is None or float(og.abs().max()) == 0.0, pname
                continue
            assert og is not None, pname
            if spec.get('full', False):
                # multi-threaded CPU reductions over >= 10^5 tokens are not run-to-run bit-stable (the reference differs
                # from ITSELF in the last bit between runs); forward outputs, loss and routing above stay bit-exact
                assert float((p.grad - og).abs().max()) <= 1e-5 * float(og.abs().max()) + 1e-12, \
                    f'{name}: grad {pname} differs by {(p.grad - og).abs().max()}'
            else:
                assert torch.equal(p.grad, og), f'{name}: grad {pname} differs by {(p.grad - og).abs().max()}'
            grads[pname] = summarize_grad(p.grad)
        gold['grads'] = grads
        new_sd = net.state_dict()
        for k, v in bn_state.items():
            assert torch.equal(v, new_sd[k]), k
        gold['bn'] = {k: v.clone() for k, v in bn_state.items()}
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, name + '.pt')
    save_golden(gold, path)
    print(f'{name}: ok, moe layers {len(record)}')


# kwargs of the state_dict-layout checks in tests/test_contract.py (tiny arch: the reference cannot be built on 'meta')
LAYOUT_CASES = {
    'tiny_dense_multi': ('ConvNeXt_moe_MultiInput', dict(arch='tiny')),
    'tiny_e8k2_multi': ('ConvNeXt_moe_MultiInput', dict(arch='tiny', MoE_Block_inds=[[], [], [0, 2, 4, 6, 8], [0, 2]], num_experts=8, top_k=2)),
    'tiny_e8k3_plain': ('ConvNeXt_moe', dict(arch='tiny', MoE_Block_inds=[[], [], [0, 2, 4, 6, 8], [0, 2]], num_experts=8, top_k=3)),
}
LSK_S_KW = dict(MoE_Block_inds_fc1=[[], [0], [0, 2], [0]], MoE_Block_inds_fc2=[[], [0], [0, 2], [0]], num_experts=4, top_k=2,
                embed_dims=[64, 128, 320, 512], depths=[2, 2, 4, 2], drop_rate=0.1, drop_path_rate=0.,
                norm_cfg=dict(type='SyncBN', requires_grad=True))          # configs/SM3Det/SM3Det_lsk_s.py:13-25
VAN_KW = dict(MoE_Block_inds_fc1=[[], [0], [0], []], MoE_Block_inds_fc2=[[], [0], [0], []], num_experts=2, top_k=1,
              embed_dims=[32, 64, 160, 256], depths=[1, 1, 2, 1])
FPN_KW = dict(in_channels=[96, 192, 384, 768], out_channels=256, extra_level=1, add_extra_convs='on_output', num_outs=5)


def fpn_inputs(n=2, s=64, seed=3):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(n, c, s // (4 * 2 ** i), s // (4 * 2 ** i), generator=g) for i, c in enumerate(FPN_KW['in_channels'])]


def run_live_reference():
    """tests/golden/live/reference.pt: what the unmodified reference modules return for the small live-comparison cases
    (forward outputs, state_dict layouts, parameter names), so the tests compare against it without the reference tree."""
    from oracle.cases import LSK_CASES
    from oracle.fpn_oracle import fpn_param_shapes
    from oracle.lsk_moe_oracle import LskConfig, lsk_param_shapes
    gold = {'convnext': {}, 'layout': {}}
    for name in ('mini_moe_e4k2_eval', 'mini_moe_e8k3_eval'):
        kw = dict(CASES[name]['kw'])
        net = ref_shim.build_reference_backbone('ConvNeXt_moe_MultiInput', seed=0, **kw)
        net.load_state_dict(make_state_dict(param_shapes(OracleConfig(**kw)), 3, True), strict=True)
        net.eval()
        with torch.no_grad():
            outs, loss = net(make_images(2, 64, 64, seed=5))
        gold['convnext'][name] = dict(outs=[o.clone() for o in outs], loss=loss.clone())
    kw = dict(arch=dict(depths=[1, 1, 2, 1], channels=[32, 64, 96, 128]), MoE_Block_inds=[[], [], [1], []], num_experts=4, top_k=2)
    net = ref_shim.build_reference_backbone('ConvNeXt_moe', seed=0, **kw)
    keys = sorted(net.state_dict())
    net.load_state_dict(make_state_dict(param_shapes(OracleConfig(multi_input=False, **kw)), 1, True), strict=True)
    net.eval()
    with torch.no_grad():
        outs = net(make_images(1, 64, 64, seed=2))[0]
    gold['convnext_plain'] = dict(keys=keys, outs=[o.clone() for o in outs])
    spec = LSK_CASES['lsk_mini_moe_e4k2_eval']
    mod = ref_shim.load_reference_module('lsk_moe')
    torch.manual_seed(0)
    net = mod.LSKNet_moe_MultiInput(norm_cfg=dict(type='SyncBN', requires_grad=True), **spec['kw'])
    net.load_state_dict(make_state_dict(lsk_param_shapes(LskConfig(**spec['kw'])), 0, True), strict=True)
    net.eval()
    with torch.no_grad():
        outs, loss = net(make_images(*spec['img'], seed=5))
    gold['lsk'] = dict(outs=[o.clone() for o in outs], loss=loss.clone())
    fpn = ref_shim.load_reference_module('Multitask_FPN', 'necks').MultitaskFPN(**FPN_KW)
    sd = make_state_dict(fpn_param_shapes(FPN_KW['in_channels'], 256, 5, 1, 'on_output'), 5, True)
    gold['fpn_keys'] = sorted(fpn.state_dict())
    fpn.load_state_dict(sd, strict=True)
    with torch.no_grad():
        gold['fpn'] = {0: [o.clone() for o in fpn(fpn_inputs())],
                       1: [o.clone() for o in fpn(fpn_inputs(), start_level=1, add_extra_convs='on_output')]}
    for case, (cls, kw) in LAYOUT_CASES.items():
        net = ref_shim.build_reference_backbone(cls, **kw)
        gold['layout'][case] = dict(shapes={k: tuple(v.shape) for k, v in net.state_dict().items()},
                                    params=sorted(n for n, _ in net.named_parameters()))
    net = ref_shim.build_reference_backbone('ConvNeXt_DA_MultiInput', module='convnext_moe_DA', arch='tiny', drop_path_rate=0.1, datasets=None)
    gold['layout']['da_tiny'] = dict(keys=list(net.state_dict()), params=[n for n, _ in net.named_parameters()])
    for case, net in (('lsk_s', mod.LSKNet_moe_MultiInput(**LSK_S_KW)),
                      ('van', ref_shim.load_reference_module('van_moe').VAN_moe_MultiInput(**VAN_KW))):
        sd = net.state_dict()
        gold['layout'][case] = dict(keys=sorted(sd), shapes={k: tuple(v.shape) for k, v in sd.items()})
    path = os.path.join(OUT, 'live', 'reference.pt')
    save_golden(gold, path)
    print('live reference: ok')


if __name__ == '__main__':
    from oracle.cases import LSK_CASES
    torch.set_num_threads(8)
    if sys.argv[1:] == ['live']:
        run_live_reference()
        sys.exit(0)
    names = sys.argv[1:] or (list(CASES) + list(LSK_CASES))
    for nm in names:
        if nm in LSK_CASES:
            run_lsk_case(nm, LSK_CASES[nm])
        else:
            run_case(nm, CASES[nm])
