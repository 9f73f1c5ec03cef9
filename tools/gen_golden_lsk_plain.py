"""Generate tests/golden/lsk_plain/: fixtures of the dense single-dataset LSKNet and VAN backbones (lsknet.py, van.py).

    python tools/gen_golden_lsk_plain.py [case ...]      (needs the reference tree, SM3DET_REFERENCE_ROOT)

Every case runs the UNMODIFIED reference lsknet.py / van.py through oracle/ref_shim.py and asserts that the oracle
(oracle/lsk_moe_oracle.py with no expert layer, multi_input=False) reproduces it bit for bit: forward outputs, every
parameter gradient and the BatchNorm running statistics, in eval and in training with dropout and drop path.  The
dropout masks are the ones oracle/cases.py:lsk_injections regenerates; the drop-path masks (one per block, shared by the
block's two residual branches, [N]) are stored in the fixture.  The fixtures live in their own subdirectory so the tests
that glob tests/golden/lsk_*.pt do not pick them up.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, 'tests', 'golden', 'lsk_plain')

SYNC_BN = dict(type='SyncBN', requires_grad=True)
# configs/lsknet/lsk_s_fpn_1x_dota_le90.py (= local_configs/dota_lsk_s_orcnn.py)
LSK_S_KW = dict(embed_dims=[64, 128, 320, 512], drop_rate=0.1, drop_path_rate=0.1, depths=[2, 2, 4, 2])
# local_configs/dota_van_t_orcnn.py
VAN_T_KW = dict(embed_dims=[32, 64, 160, 256], drop_rate=0.1, drop_path_rate=0.1, depths=[3, 3, 5, 2])

# name -> (class, constructor kwargs without norm_cfg, image (n, h, w), mode, output stride).  Training cases use batch 2
# (oracle/cases.py: torch 2.11's CPU autograd disagrees with finite differences on this op sequence at batch 1).
CASES = {
    'lsk_s_1024_eval': dict(cls='LSKNet', kw=LSK_S_KW, img=(1, 1024, 1024), mode='eval', stride=8),
    'lsk_s_b2_512_train_drop': dict(cls='LSKNet', kw=LSK_S_KW, img=(2, 512, 512), mode='train', stride=8),
    'van_t_b2_512_train_drop': dict(cls='VAN', kw=VAN_T_KW, img=(2, 512, 512), mode='train', stride=8),
    'lsk_default_256_eval': dict(cls='LSKNet', kw={}, img=(1, 256, 256), mode='eval', stride=2),
    # short depth at the S widths: small enough that every gradient is compared bit for bit
    'lsk_s_short_b2_128_train_drop': dict(cls='LSKNet', kw=dict(LSK_S_KW, depths=[1, 1, 2, 1], drop_path_rate=0.3),
                                          img=(2, 128, 128), mode='train', stride=1),
}

_CFG_FIELDS = ('embed_dims', 'depths', 'mlp_ratios', 'drop_rate', 'drop_path_rate', 'num_stages')


def oracle_config(cls, kw):
    """LskConfig of an LSKNet / VAN constructor call (defaults of lsknet.py:130-132)."""
    from oracle.lsk_moe_oracle import LskConfig
    full = dict(embed_dims=[64, 128, 256, 512], depths=[3, 4, 6, 3], mlp_ratios=[8, 8, 4, 4], drop_rate=0.0,
                drop_path_rate=0.0, num_stages=4)
    full.update({k: v for k, v in kw.items() if k in _CFG_FIELDS})
    n = full['num_stages']
    return LskConfig(multi_input=False, spatial_unit='lka' if cls == 'VAN' else 'lsk', MoE_Block_inds_fc1=[[]] * n,
                     MoE_Block_inds_fc2=[[]] * n, **full)


def drop_path_masks(cfg, n):
    """One [n] keep mask per block, pre-scaled by 1/(1 - rate) of that block; every third block drops one sample."""
    dpr = [v.item() for v in torch.linspace(0, cfg.drop_path_rate, sum(cfg.depths))]
    out = []
    for b, rate in enumerate(dpr):
        keep = torch.ones(n)
        if b % 3 == 1:
            keep[b % n] = 0.0
        out.append(keep / (1.0 - rate))
    return out


def run_case(name, spec):
    import torch.nn.functional as F
    from oracle import ref_shim
    from oracle.cases import lsk_injections, save_golden, summarize_grad, upstream_grads
    from oracle.lsk_moe_oracle import lsk_backbone_forward, lsk_param_shapes
    from sm3det_b200.synth import make_images, make_state_dict, state_dict_checksum
    cls, kw = spec['cls'], dict(spec['kw'])
    cfg = oracle_config(cls, kw)
    mod = ref_shim.load_reference_module('lsknet' if cls == 'LSKNet' else 'van')
    torch.manual_seed(0)
    net = getattr(mod, cls)(norm_cfg=dict(SYNC_BN), **kw)
    shapes = lsk_param_shapes(cfg)
    rsd = net.state_dict()
    assert list(shapes) == list(rsd), set(shapes) ^ set(rsd)
    for k, sh in shapes.items():
        assert tuple(rsd[k].shape) == tuple(sh), k
    sd = make_state_dict(shapes, seed=0, trained_like=True)
    net.load_state_dict(sd, strict=True)
    n, h, w = spec['img']
    x = make_images(n, h, w, seed=1234)
    mode = spec['mode']
    gold = dict(name=name, cls=cls, kw=kw, img=spec['img'], mode=mode, weights='trained', unit=cfg.spatial_unit,
                sd_checksum=state_dict_checksum({k: v.float() for k, v in sd.items()}), x_checksum=float(x.double().abs().sum()))
    bn_state = {}
    if mode == 'eval':
        net.eval()
        with torch.no_grad():
            ref = net(x)
            orc = lsk_backbone_forward(sd, cfg, x, train=False)
    else:
        net.train()
        _, drops = lsk_injections(cfg, gold)
        dps = drop_path_masks(cfg, n)
        gold['dp_masks'] = dps
        blocks = [blk for i in range(cfg.num_stages) for blk in getattr(net, f'block{i + 1}')]
        for blk, m in zip(blocks, dps):
            blk.drop_path._mask = m.view(n, 1, 1, 1)
        dit = iter(drops)
        orig_dp, orig_drop = ref_shim._DropPath.forward, F.dropout
        ref_shim._DropPath.forward = lambda self, t: t * self._mask if (self.training and self.drop_prob > 0.0) else t
        F.dropout = lambda t, p=0.5, training=True, inplace=False: t * next(dit) if training else t
        try:
            ref = net(x)
        finally:
            ref_shim._DropPath.forward, F.dropout = orig_dp, orig_drop
        assert next(dit, None) is None, 'every injected dropout mask is consumed'
        sdg = {k: (v.clone().requires_grad_(True) if v.is_floating_point() and 'running_' not in k and 'num_batches' not in k
                   else v) for k, v in sd.items()}
        orc = lsk_backbone_forward(sdg, cfg, x, train=True, drop_masks=drops, dp_masks=[m.view(n, 1, 1, 1) for m in dps],
                                   bn_state=bn_state)
    assert isinstance(ref, list) and len(ref) == cfg.num_stages
    for a, b in zip(ref, orc):
        assert torch.equal(a, b), f'{name}: oracle output differs from reference by {(a - b).abs().max()}'
    st = spec['stride']
    gold['outs'] = [o.detach()[:, :, ::st, ::st].clone() for o in ref]
    gold['out_l2'] = [o.detach().double().norm().item() for o in ref]
    gold['stride'] = st
    if mode != 'eval':
        ups = upstream_grads(ref)
        sum((o * g).sum() for o, g in zip(ref, ups)).backward()
        sum((o * g).sum() for o, g in zip(orc, ups)).backward()
        big = h * w * n >= 2 * 512 * 512
        grads = {}
        for pname, p in net.named_parameters():
            og = sdg[pname].grad
            assert p.grad is not None and og is not None, pname
            if big:
                # multi-threaded CPU reductions over >= 10^5 tokens are not run-to-run bit-stable (the reference differs
                # from ITSELF in the last bit between runs); forward outputs and BN statistics stay bit-exact
                assert float((p.grad - og).abs().max()) <= 1e-5 * float(og.abs().max()) + 1e-12, \
                    f'{name}: grad {pname} differs by {(p.grad - og).abs().max()}'
            else:
                assert torch.equal(p.grad, og), f'{name}: grad {pname} differs by {(p.grad - og).abs().max()}'
            grads[pname] = summarize_grad(p.grad)
        gold['grads'] = grads
        new_sd = net.state_dict()
        assert set(bn_state) == {k for k in new_sd if 'running_' in k}
        for k, v in bn_state.items():
            assert torch.equal(v, new_sd[k]), k
        gold['bn'] = {k: v.clone() for k, v in bn_state.items()}
    save_golden(gold, os.path.join(OUT, name + '.pt'))
    print(f'{name}: ok')


if __name__ == '__main__':
    torch.set_num_threads(8)
    for nm in sys.argv[1:] or list(CASES):
        run_case(nm, CASES[nm])
