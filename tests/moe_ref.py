"""Float64-capable functional reference of one sparse-MoE layer, for the kernel and layer tests.

Restates oracle.convnext_moe_oracle.noisy_top_k_gating + moe_layer + the ConvNeXt block tail (layer scale, drop path,
shortcut) and the LSKNet MoE_layer.  Unlike the oracle it works at any dtype (the oracle casts to fp32 in cv_squared and
in the combine), and it takes the routing as an input instead of computing a top-k, so a test never depends on how a tie
is broken:

* ``top_idx`` [T, k]: the chosen experts of each token, in descending order of the selection logit;
* ``idx_k1`` [T]: the (k+1)-th expert (only read by the soft load, noisy gating with k < E);
* ``live`` [T, k] bool: which pairs are dispatched.  The CUDA router and the reference evaluate the gates in fp32, and a
  gate that underflows to 0 there is not dispatched (the kernel writes top_idx = -1).  In float64 the same gate would be
  ~1e-46 and would count as a token of that expert, so the dispatch decision is made in fp32 (``fp32_live``) and passed in.

Parameters are looked up by their module names (``w_gate.sim_matrix``, ``experts.0.pointwise_conv1.weight`` ...), so a
test can hand over ``dict(module.named_parameters())`` converted to float64.
"""
import math

import torch
import torch.nn.functional as F

LN100 = math.log(100.0)       # CosineTopKGate clamp_max = log(1 / 0.01)


def cv_squared(z):
    if z.shape[0] == 1:
        return z.new_zeros(())
    return z.var() / (z.mean() ** 2 + 1e-10)


def fp32_live(sel, top_idx):
    """Dispatch mask of the chosen pairs: the fp32 softmax over the chosen selection logits is nonzero."""
    vals = sel.detach().float().gather(1, top_idx)
    g = torch.exp(vals - vals[:, :1])
    return (g / g.sum(1, keepdim=True)) > 0


def gating(v, prm, top_idx, *, idx_k1=None, noise=None, live=None, pre='w_gate.', noise_key='w_noise'):
    """Cosine top-k gating of tokens v [T, C] with the routing given.  Returns a dict with clean / sel logits, sigma,
    raw noise logits r, top_gates [T, k] (0 on undispatched pairs), live, importance, load and the gate loss.
    ``clean`` keeps its gradient (``retain_grad``) so a test can form the per-token terms of d loss / d temperature."""
    proj = F.linear(v, prm[pre + 'cosine_projector.weight'], prm[pre + 'cosine_projector.bias'])
    clean = (F.normalize(proj, dim=1) @ F.normalize(prm[pre + 'sim_matrix'], dim=0)) * \
        torch.clamp(prm[pre + 'temperature'], max=LN100).exp()
    if clean.requires_grad:
        clean.retain_grad()
    return gating_from_logits(clean, top_idx, idx_k1=idx_k1, noise=noise, live=live,
                              r=None if noise is None else v @ prm[noise_key])


def gating_from_logits(clean, top_idx, *, idx_k1=None, noise=None, r=None, live=None):
    T, E = clean.shape
    k = top_idx.shape[1]
    sigma, sel = None, clean
    if noise is not None:
        sigma = F.softplus(r) + 1e-2
        sel = clean + noise * sigma
    if live is None:
        live = fp32_live(sel, top_idx)
    top_gates = torch.softmax(sel.gather(1, top_idx), -1) * live
    gates = clean.new_zeros(T, E).scatter(1, top_idx, top_gates)
    importance = gates.sum(0)
    if noise is not None and k < E:
        # _prob_in_top_k: an expert inside the top k is compared with the (k+1)-th noisy value, the others with the k-th
        thr_in = sel.gather(1, idx_k1.view(T, 1))
        thr_out = sel.gather(1, top_idx[:, k - 1:k])
        is_in = torch.zeros(T, E, dtype=torch.bool).scatter(1, top_idx, True)
        z = (clean - torch.where(is_in, thr_in, thr_out)) / sigma
        load = (0.5 * (1 + torch.erf(z / math.sqrt(2)))).sum(0)
    else:
        load = torch.zeros(T, E, dtype=clean.dtype).scatter(1, top_idx, live.to(clean.dtype)).sum(0)
    loss = (cv_squared(importance) + cv_squared(load)) * 1e-2
    return dict(clean=clean, sel=sel, sigma=sigma, r=r, top_gates=top_gates, live=live, importance=importance,
                load=load, loss=loss)


def combine(v, top_idx, top_gates, live, experts, Cout):
    """y[t] = sum over the dispatched pairs (t, j) of top_gates[t, j] * experts[top_idx[t, j]](v[t])."""
    y = v.new_zeros(v.shape[0], Cout)
    for e, f in enumerate(experts):
        t, j = ((top_idx == e) & live).nonzero(as_tuple=True)
        if t.numel():
            y = y.index_add(0, t, top_gates[t, j].unsqueeze(1) * f(v[t]))
    return y


def ffn_expert(prm, pre):
    return lambda u: F.linear(F.gelu(F.linear(u, prm[pre + 'pointwise_conv1.weight'], prm[pre + 'pointwise_conv1.bias'])),
                              prm[pre + 'pointwise_conv2.weight'], prm[pre + 'pointwise_conv2.bias'])


def conv1x1_expert(prm, pre):
    return lambda u: F.linear(u, prm[pre + 'weight'].flatten(1), prm[pre + 'bias'])


def tail(y, gamma=None, resid=None, row_scale=None):
    """resid + (y * gamma) * row_scale: layer scale, drop path as a per-token scale, shortcut."""
    if gamma is not None:
        y = y * gamma
    if row_scale is not None:
        y = y * row_scale.view(-1, 1)
    return y if resid is None else resid + y


def convnext_moe_block(x, prm, *, E, top_idx, idx_k1=None, noise=None, row_scale=None, live=None, eps=1e-6):
    """ConvNeXtBlock with a MoE_layer FFN on x [N, H, W, C] (NHWC).  prm: the block's parameters by module name.
    Returns (out [N, H, W, C], gating dict)."""
    N, H, W, C = x.shape
    u = F.conv2d(x.permute(0, 3, 1, 2), prm['depthwise_conv.weight'], prm['depthwise_conv.bias'], padding=3, groups=C)
    v = F.layer_norm(u.permute(0, 2, 3, 1).reshape(-1, C), (C,), prm['norm.weight'], prm['norm.bias'], eps)
    g = gating(v, prm, top_idx, idx_k1=idx_k1, noise=noise, live=live, pre='ffn.w_gate.', noise_key='ffn.w_noise')
    y = combine(v, top_idx, g['top_gates'], g['live'], [ffn_expert(prm, f'ffn.experts.{e}.') for e in range(E)], C)
    g['y'] = y
    out = tail(y, prm['gamma'], x.reshape(-1, C), row_scale)
    return out.view(N, H, W, C), g


def lsk_moe_layer(x, prm, *, E, top_idx, idx_k1=None, noise=None, gamma=None, resid=None, row_scale=None, live=None):
    """LSKNet MoE_layer (single 1x1-conv experts) on x [..., Cin]; gamma / resid / row_scale as the fused fc2 tail.
    Returns (out [..., Cout], gating dict)."""
    lead, Cin = x.shape[:-1], x.shape[-1]
    Cout = prm['experts.0.weight'].shape[0]
    v = x.reshape(-1, Cin)
    g = gating(v, prm, top_idx, idx_k1=idx_k1, noise=noise, live=live)
    y = combine(v, top_idx, g['top_gates'], g['live'], [conv1x1_expert(prm, f'experts.{e}.') for e in range(E)], Cout)
    g['y'] = y
    out = tail(y, gamma, None if resid is None else resid.reshape(-1, Cout), row_scale)
    return out.view(*lead, Cout), g
