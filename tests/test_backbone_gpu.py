"""End-to-end parity of the CUDA backbone against the CPU oracle (and the reference-generated goldens)."""
import glob
import os

import pytest
import torch

from oracle.cases import CASES, load_golden, make_noise
from oracle.convnext_moe_oracle import OracleConfig, backbone_forward, param_shapes
from oracle.gen_golden import moe_token_counts
from sm3det_b200.synth import make_images, make_state_dict
from parity_util import TOL, build, rel, run_case

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), 'golden')
CONV_GOLDENS = sorted(p for p in glob.glob(os.path.join(GOLD, '*.pt')) if not os.path.basename(p).startswith(('lsk_', 'van_')))


@pytest.mark.parametrize('path', CONV_GOLDENS, ids=lambda p: os.path.basename(p)[:-3])
def test_matches_reference_golden(path):
    """Every ConvNeXt fixture (small ones, the ConvNeXt_DA ones and the full-size cfg2 / shipped-k3 / cfg4 shapes): routing vs the reference's
    (flips must be numerical ties), then outputs / loss / pre-gamma MoE outputs / every gradient vs the teacher-forced
    oracle on all elements, plus the fixture values themselves when no token flipped.  No assertion is conditional on
    the number of flips (see parity_util)."""
    gold = load_golden(path)
    errs = run_case(gold['kw'], gold['img'], gold['mode'], gold['weights'], gold=gold, datasets=gold.get('datasets'))
    print(os.path.basename(path), errs)


@pytest.mark.parametrize('name', ['mini_moe_e4k2_eval', 'mini_moe_e8k3_eval', 'mini_moe_e6k1_eval', 'mini_moe_e2k2_eval'])
def test_moe_layers_match_oracle(name):
    """A second input (seed 77) the fixtures do not hold, against the live oracle."""
    spec = CASES[name]
    print(name, run_case(spec['kw'], spec['img'], 'eval', img_seed=77))


def test_list_input_and_plain_class():
    from sm3det_b200 import ConvNeXt_moe
    kw = dict(arch=dict(depths=[1, 1, 2, 1], channels=[32, 64, 96, 128]), MoE_Block_inds=[[], [], [1], []], num_experts=4, top_k=2)
    cfg, sd, net = build(kw)
    xs = [make_images(1, 64, 64, seed=s) for s in (1, 2, 3)]
    net.eval()
    with torch.no_grad():
        a = net([t.cuda() for t in xs], ['sar', 'rgb', 'ifr'])
        b = net(torch.cat(xs).cuda())
    assert isinstance(a, tuple) and len(a) == 2 and len(a[0]) == 4
    for p, q in zip(a[0], b[0]):
        assert torch.equal(p, q) and p.is_contiguous()
    assert a[0][0].shape == (3, 32, 16, 16) and a[0][3].shape == (3, 128, 2, 2)
    # plain class: tuple only when dense, (tuple, loss) with MoE
    cfgp = OracleConfig(multi_input=False, **kw)
    sdp = make_state_dict(param_shapes(cfgp), 1, True)
    netp = ConvNeXt_moe(**kw)
    netp.load_state_dict(sdp, strict=True)
    netp = netp.cuda().eval()
    x = make_images(2, 64, 64, seed=5)
    with torch.no_grad():
        og, lg = netp(x.cuda())
        oc, lc = backbone_forward(sdp, cfgp, x)
    for p, q in zip(og, oc):
        assert rel(p, q) < TOL
    dense = ConvNeXt_moe(arch=kw['arch']).cuda().eval()
    with torch.no_grad():
        r = dense(x.cuda())
    assert isinstance(r, tuple) and len(r) == 4 and torch.is_tensor(r[0])


@pytest.mark.parametrize('name', ['mini_moe_e8k3_noisy', 'mini_moe_e2k2_noisy'])
def test_backward_matches_oracle(name):
    """Training-mode cases without a fixture: k = 3 with noise, and k == E with noise (w_noise still gets its gradient
    through the gates even though the load falls back to the hard count, convnext_moe.py:219-222)."""
    spec = CASES[name.replace('_noisy', '_eval')]
    print(name, run_case(spec['kw'], spec['img'], 'train_noisy'))


def test_mixed_precision_mode():
    """AMP recipe (SURVEY 8f rank 2): under torch.autocast the GEMMs run single-pass bf16; the result stays within bf16
    accuracy of the fp32 oracle, differs from the fp32-accurate mode, and the next plain forward is fp32-accurate again."""
    spec = CASES['mini_moe_e4k2_train_clean']
    cfg, sd, net = build(spec['kw'])
    net.train()
    n, h, w = spec['img']
    x = make_images(n, h, w, seed=1234).cuda()
    with torch.no_grad():
        ref, _ = backbone_forward(sd, cfg, x.cpu(), train=True)
    from sm3det_b200 import ops
    o32, l32 = net(x)
    with torch.autocast('cuda', dtype=torch.bfloat16):
        o16, l16 = net(x)
    # an interleaved fp32-mode forward (EMA / validation hook) must not change the precision of the pending bf16 backward
    # (round-1 advisor finding): the Functions captured their own mode
    with torch.no_grad():
        net(x)
    assert ops.current_passes() == 3
    (sum(o.float().square().mean() for o in o16) + l16).backward()
    assert all(p.grad is None or torch.isfinite(p.grad).all() for p in net.parameters())
    e32 = max(rel(a, b) for a, b in zip(o32, ref))
    l2 = lambda a, b: ((a.detach().float().cpu() - b).norm() / b.norm()).item()     # a routing flip moves single tokens a lot
    e16 = max(l2(a, b) for a, b in zip(o16, ref))
    print('fp32-mode err', e32, 'bf16-mode rel-L2 err', e16)
    assert e32 < TOL
    assert 1e-4 < e16 < 5e-2
    o32b, _ = net(x)
    assert max(rel(a, b) for a, b in zip(o32b, ref)) < TOL


def test_fp16_autocast_with_grad_scaler():
    """The reference's recipe (configs/SM3Det/SM3Det_convnext_t.py:8 fp16=dict(loss_scale='dynamic'); mmcv Fp16OptimizerHook
    = fp16 autocast + dynamic loss scaling): the backbone takes the fp32 image, returns fp32 maps (the fp16-sensitive combine is
    fp32 like convnext_moe.py:283 forces it), gradients arrive multiplied by the loss scale and come out finite; after
    unscaling they match the unscaled run to the single-pass tolerance, and the optimizer step is not skipped."""
    spec = CASES['mini_moe_e4k2_train_clean']
    cfg, sd, net = build(spec['kw'])
    net.train()
    n, h, w = spec['img']
    x = make_images(n, h, w, seed=1234).cuda()

    def loss_of(outs, gl):
        return sum(o.float().square().mean() for o in outs) + gl
    with torch.autocast('cuda', dtype=torch.float16):
        outs, gl = net(x)
        assert all(o.dtype == torch.float32 for o in outs) and gl.dtype == torch.float32
        loss_of(outs, gl).backward()
    plain = {k: p.grad.detach().clone() for k, p in net.named_parameters() if p.grad is not None}
    net.zero_grad(set_to_none=True)
    opt = torch.optim.SGD(net.parameters(), lr=1e-6)
    scaler = torch.amp.GradScaler('cuda', init_scale=2.0 ** 16)
    before = {k: p.detach().clone() for k, p in net.named_parameters()}
    with torch.autocast('cuda', dtype=torch.float16):
        outs, gl = net(x)
        loss = loss_of(outs, gl)
    scaler.scale(loss).backward()
    big = max(float(p.grad.abs().max()) for p in net.parameters() if p.grad is not None)
    assert big > 1.0                                                  # the scale really went through the hand-written backward
    scaler.unscale_(opt)
    worst = max((rel(p.grad, plain[k]), k) for k, p in net.named_parameters() if p.grad is not None and float(plain[k].abs().max()) > 1e-8)
    assert worst[0] < 5e-3, worst                                     # same single-pass arithmetic, scaled by a power of two
    scaler.step(opt)
    scaler.update()
    assert scaler.get_scale() == 2.0 ** 16                            # no inf/nan found -> step taken, scale kept
    assert any(not torch.equal(p.detach(), before[k]) for k, p in net.named_parameters())
