"""Pins tests/moe_ref.py (the float64-capable MoE reference of tests/test_moe_gpu.py) to the CPU oracle.

Evaluated in float32 on the oracle's own routing, the reference must reproduce the oracle's outputs, gate loss,
importance / load and the autograd gradients with respect to every input, in eval, train-clean and train-noisy mode
(soft load for k < E, hard counts for k == E).  CPU only."""
import math

import pytest
import torch

import moe_ref
from oracle.convnext_moe_oracle import OracleConfig, convnext_block
from oracle.lsk_moe_oracle import LskConfig, moe_conv_layer

TOL = 1e-6
TOL_ROUTER = 3e-6


def rel(a, b):
    return ((a.detach().double() - b.detach().double()).abs().max() / (b.detach().double().abs().max() + 1e-30)).item()


def routing(rec, k, E):
    """The oracle's top-k (descending) and its (k+1)-th expert, from its recorded selection logits."""
    idx_k1 = rec['logits'].topk(k + 1, dim=1).indices[:, k] if k < E else None
    return rec['top_idx'], idx_k1


MODES = [  # (name, train, noisy, k)
    ('eval', False, False, 2), ('train_clean', True, False, 2), ('train_noisy', True, True, 2),
    ('train_noisy_k_eq_E', True, True, 4)]


def leaves(shapes, g):
    sd = {}
    for n, s in shapes.items():
        t = torch.randn(s, generator=g)
        if n.endswith('temperature'):
            t = torch.tensor([math.log(10.0)])
        elif 'w_noise' in n:
            t = t * 0.1
        elif n.endswith('.weight') and len(s) >= 2:
            t = t / math.sqrt(s[1])
        sd[n] = t.requires_grad_(True)
    return sd


def compare_grads(sd_o, sd_r, gi):
    for n in sd_o:
        go, gr = sd_o[n].grad, sd_r[n].grad
        if go is None or not go.abs().max() > 0:
            assert gr is None or not gr.abs().max() > 0, n
        elif n.endswith('temperature'):
            # one fp32 sum over all tokens of terms of both signs, summed in a different order by the two sides: the
            # rounding is bounded by the sum of the magnitudes of the per-token terms, not by the (cancelled) result
            bound = TOL * (gi['clean'].grad * gi['clean']).sum(1).abs().sum().item()
            assert abs(gr.item() - go.item()) <= bound, (n, abs(gr.item() - go.item()), bound)
        elif '.w_gate.' in '.' + n:
            # the projector / sim gradients are sums over all tokens of terms that pass through both normalisations,
            # the softmax and (noisy) 1 / sigma; in fp32 the oracle and this reference each land ~1e-6 from the float64
            # value (measured 0.7-1.1e-6 each, train_noisy), so they may be twice that apart
            assert rel(gr, go) <= TOL_ROUTER, (n, rel(gr, go))
        else:
            assert rel(gr, go) <= TOL, (n, rel(gr, go))


@pytest.mark.parametrize('mode,train,noisy,k', MODES, ids=[m[0] for m in MODES])
def test_convnext_block_matches_oracle(mode, train, noisy, k):
    g = torch.Generator().manual_seed(7 + k)
    N, H, W, C, E = 2, 6, 6, 32, 4
    P = C // 2
    T = N * H * W
    shapes = {'depthwise_conv.weight': (C, 1, 7, 7), 'depthwise_conv.bias': (C,), 'norm.weight': (C,), 'norm.bias': (C,),
              'gamma': (C,), 'ffn.w_noise': (C, E), 'ffn.w_gate.temperature': (1,), 'ffn.w_gate.sim_matrix': (P, E),
              'ffn.w_gate.cosine_projector.weight': (P, C), 'ffn.w_gate.cosine_projector.bias': (P,)}
    for e in range(E):
        q = f'ffn.experts.{e}.'
        shapes.update({q + 'pointwise_conv1.weight': (4 * C, C), q + 'pointwise_conv1.bias': (4 * C,),
                       q + 'pointwise_conv2.weight': (C, 4 * C), q + 'pointwise_conv2.bias': (C,)})
    x = torch.randn(N, C, H, W, generator=g)
    noise = torch.randn(T, E, generator=g) if noisy else None
    mask = torch.tensor([0.0, 1.25]).view(N, 1, 1, 1) if train else None
    dout = torch.randn(N, C, H, W, generator=g)
    cfg = OracleConfig(num_experts=E, top_k=k, noisy_gating=noisy)

    sd_o = leaves(shapes, torch.Generator().manual_seed(1))
    xo = x.clone().requires_grad_(True)
    rec = []
    out_o, loss_o = convnext_block(xo, {'b.' + n: t for n, t in sd_o.items()}, 'b.', cfg, True, 0.2 if train else 0.0,
                                   train, noise, mask, rec)
    ((out_o * dout).sum() + loss_o).backward()

    sd_r = leaves(shapes, torch.Generator().manual_seed(1))
    xr = x.permute(0, 2, 3, 1).contiguous().requires_grad_(True)
    top_idx, idx_k1 = routing(rec[0], k, E)
    rs = mask.view(N).repeat_interleave(H * W) if train else None
    out_r, gr = moe_ref.convnext_moe_block(xr, sd_r, E=E, top_idx=top_idx, idx_k1=idx_k1, noise=noise, row_scale=rs)
    ((out_r * dout.permute(0, 2, 3, 1)).sum() + gr['loss']).backward()

    assert bool(gr['live'].all())
    assert rel(out_r, out_o.permute(0, 2, 3, 1)) <= TOL
    assert rel(gr['y'], rec[0]['y']) <= TOL
    assert rel(gr['loss'], loss_o) <= TOL
    assert rel(gr['importance'], rec[0]['importance']) <= TOL and rel(gr['load'], rec[0]['load']) <= TOL
    assert rel(xr.grad, xo.grad.permute(0, 2, 3, 1)) <= TOL
    compare_grads(sd_o, sd_r, gr)


@pytest.mark.parametrize('mode,train,noisy,k', MODES, ids=[m[0] for m in MODES])
def test_lsk_moe_layer_matches_oracle(mode, train, noisy, k):
    g = torch.Generator().manual_seed(11 + k)
    N, H, W, Cin, Cout, E = 2, 5, 7, 64, 96, 4
    P = Cin // 2
    T = N * H * W
    shapes = {'w_noise': (Cin, E), 'w_gate.temperature': (1,), 'w_gate.sim_matrix': (P, E),
              'w_gate.cosine_projector.weight': (P, Cin), 'w_gate.cosine_projector.bias': (P,)}
    for e in range(E):
        shapes.update({f'experts.{e}.weight': (Cout, Cin, 1, 1), f'experts.{e}.bias': (Cout,)})
    x = torch.randn(N, Cin, H, W, generator=g)
    noise = torch.randn(T, E, generator=g) if noisy else None
    dout = torch.randn(N, Cout, H, W, generator=g)
    cfg = LskConfig(num_experts=E, top_k=k, noisy_gating=noisy)

    sd_o = leaves(shapes, torch.Generator().manual_seed(2))
    xo = x.clone().requires_grad_(True)
    rec = []
    out_o, loss_o = moe_conv_layer(xo, {'m.' + n: t for n, t in sd_o.items()}, 'm.', cfg, train, noise, record=rec)
    ((out_o * dout).sum() + loss_o).backward()

    sd_r = leaves(shapes, torch.Generator().manual_seed(2))
    xr = x.permute(0, 2, 3, 1).contiguous().requires_grad_(True)
    top_idx, idx_k1 = routing(rec[0], k, E)
    out_r, gr = moe_ref.lsk_moe_layer(xr, sd_r, E=E, top_idx=top_idx, idx_k1=idx_k1, noise=noise)
    ((out_r * dout.permute(0, 2, 3, 1)).sum() + gr['loss']).backward()

    assert rel(out_r, out_o.permute(0, 2, 3, 1)) <= TOL
    assert rel(gr['loss'], loss_o) <= TOL
    assert rel(gr['importance'], rec[0]['importance']) <= TOL and rel(gr['load'], rec[0]['load']) <= TOL
    assert rel(xr.grad, xo.grad.permute(0, 2, 3, 1)) <= TOL
    compare_grads(sd_o, sd_r, gr)


def test_fp32_live_drops_underflowed_gates():
    """A second gate exp(-110) is ~1e-48 in float64 but exactly 0 in fp32: the pair is not dispatched, not counted in the
    load, and its gate is 0 in the float64 reference too."""
    clean = torch.tensor([[55.0, -60.0, -55.0], [1.0, 0.5, 0.0]], dtype=torch.float64)
    top_idx = torch.tensor([[0, 2], [0, 1]])
    gi = moe_ref.gating_from_logits(clean, top_idx)
    assert gi['live'].tolist() == [[True, False], [True, True]]
    assert gi['top_gates'][0, 1].item() == 0.0 and gi['top_gates'][0, 0].item() == 1.0
    assert gi['load'].tolist() == [2.0, 1.0, 0.0]
