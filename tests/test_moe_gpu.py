"""MoE combine, router-backward and expert-dispatch kernels against a float64 reference, and the two MoE layers at
designed expert loads.

Kernel tests call the ops.* wrappers on fp32 inputs.  Where a kernel's summation order is fixed (moe_combine, the d_o
of moe_combine_bwd, gather_sum) it is compared bit-exactly with the same fp32 formula on the CPU; everything else is
compared with tests/moe_ref.py (or plain float64 sums) evaluated in float64 on the same values.  "rel" is the max-norm
relative error.  The layer tests set the routing by construction (one-hot sim matrix, projector = [I_E | 0], tokens
built from the wanted experts), so the reference is handed the designed routing and the test asserts the kernel chose
exactly it.
"""
import math

import pytest
import torch
import torch.nn.functional as F

import moe_ref

pytestmark = pytest.mark.gpu

FAST_V = (1, 2, 3, 4, 5, 6, 8, 10, 12, 16, 20, 24, 32)     # moe_combine_bwd's templated widths C / 32 (moe.cu)
SENTINEL = 12345.0


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).abs().max() / (b.abs().max() + 1e-30)).item()


WORST = {}


def within(quantity, err, tol):
    """err <= tol, remembering the worst err per quantity (printed at the end of the module, run with -s to see it)."""
    WORST[quantity] = max(WORST.get(quantity, 0.0), err)
    return err <= tol


@pytest.fixture(scope='module', autouse=True)
def report_worst():
    yield
    print('\nworst errors:', ', '.join(f'{q} {e:.2e}' for q, e in sorted(WORST.items())))


@pytest.fixture(scope='module')
def ops():
    from sm3det_b200 import ops as o
    return o


def kernels_run(fn):
    """Names of the CUDA kernels fn launches (torch.profiler), and fn's result."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        res = fn()
        torch.cuda.synchronize()
    return {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}, res


# ---- synthetic dispatch: random distinct experts per token, some pairs dead (-1), padded 128-row expert segments ----
def synth_dispatch(T, E, k, g, dead=0.15):
    top_idx = torch.rand(T, E, generator=g).argsort(1)[:, :k].int()
    kill = torch.rand(T, k, generator=g) < dead
    kill[:, 0] = False
    top_idx[kill] = -1
    flat = top_idx.flatten()
    slot = torch.full_like(flat, -1)
    pos = 0
    for e in range(E):
        where = (flat == e).nonzero().flatten()
        slot[where] = (pos + torch.arange(where.numel())).int()
        pos += (where.numel() + 127) // 128 * 128
    gate = torch.rand(T, k, generator=g) * 0.9 + 0.05
    gate[kill] = 0.0
    return top_idx, slot.view(T, k), gate, pos + 128          # one extra 128-row tile that no slot points at


def combine_fp32(o, slot_of, top_idx, gate, gamma, resid, rs):
    """moe_combine's formula in fp32 with separate multiply and add: the live pairs in ascending expert id, then
    r + (y * gamma) * rs."""
    T, k = top_idx.shape
    order = torch.where(top_idx < 0, 1 << 20, top_idx).argsort(1)
    y = torch.zeros(T, o.shape[1])
    for r in range(k):
        j = order[:, r:r + 1]
        s = slot_of.gather(1, j)[:, 0].long()
        live = (top_idx.gather(1, j)[:, 0] >= 0) & (s >= 0)
        y = torch.where(live[:, None], y + gate.gather(1, j) * o[s.clamp_min(0)], y)
    out = y
    if gamma is not None:
        out = out * gamma
    if rs is not None:
        out = out * rs[:, None]
    if resid is not None:
        out = resid + out
    return out, y


def drop_path_scale(T, g):
    rs = torch.rand(T, generator=g) * 1.5 + 0.5
    rs[torch.rand(T, generator=g) < 0.2] = 0.0
    return rs


@pytest.mark.parametrize('C', [32, 96, 384, 2048])
@pytest.mark.parametrize('k', [1, 2, 3])
def test_combine_bit_exact(ops, k, C):
    g = torch.Generator().manual_seed(100 * k + C)
    T, E = 333, 8
    top_idx, slot_of, gate, R = synth_dispatch(T, E, k, g)
    assert k == 1 or bool((top_idx < 0).any())
    o = torch.randn(R, C, generator=g)
    gamma = torch.rand(C, generator=g) + 0.3
    resid = torch.randn(T, C, generator=g)
    rs = drop_path_scale(T, g)
    assert bool((rs == 0).any())
    dv = lambda t: None if t is None else t.cuda()
    for use in range(8):
        gm, rd, r = (gamma if use & 1 else None), (resid if use & 2 else None), (rs if use & 4 else None)
        out, y = ops.moe_combine(o.cuda(), slot_of.cuda(), top_idx.cuda(), gate.cuda(), dv(gm), dv(rd), dv(r), T=T, Cc=C,
                                 k=k, want_y=True)
        want, want_y = combine_fp32(o, slot_of, top_idx, gate, gm, rd, r)
        assert torch.equal(y.cpu(), want_y), use
        assert torch.equal(out.cpu(), want), use


def fast_kernel_expected(C, has_gamma):
    return has_gamma and C % 32 == 0 and C // 32 in FAST_V


BWD_CASES = [  # (id, C, gamma, k, T or 'tpw' = enough tokens that tokens_per_warp > 8, row_scale)
    ('fast_c96_tpw', 96, True, 2, 'tpw', True), ('fast_c32_k1', 32, True, 1, 1000, False),
    ('fast_c384_k3', 384, True, 3, 3000, True), ('fast_c1024', 1024, True, 2, 500, True),
    ('generic_c224_gamma', 224, True, 2, 2000, True), ('generic_c352_gamma', 352, True, 3, 1500, False),
    ('lsk_c64', 64, False, 2, 2000, True), ('lsk_c2048', 2048, False, 2, 700, False)]


@pytest.mark.parametrize('name,C,has_gamma,k,T,has_rs', BWD_CASES, ids=[c[0] for c in BWD_CASES])
def test_combine_bwd(ops, name, C, has_gamma, k, T, has_rs):
    g = torch.Generator().manual_seed(C + k)
    if T == 'tpw':
        T = ops.num_sms() * 32 * 8 + 4321
        warps = ops.num_sms() * 32
        assert -(-T // warps) > 8                             # the fast kernel's tokens_per_warp leaves its minimum
    E = 8
    top_idx, slot_of, gate, R = synth_dispatch(T, E, k, g)
    o = torch.randn(R, C, generator=g)
    dout = torch.randn(T, C, generator=g)
    gamma = torch.rand(C, generator=g) + 0.3 if has_gamma else None
    rs = drop_path_scale(T, g) if has_rs else None
    d_o = torch.full((R, C), SENTINEL, device='cuda')
    dgamma = torch.zeros(C, device='cuda') if has_gamma else None
    dv = lambda t: None if t is None else t.cuda()
    names, dgate = kernels_run(lambda: ops.moe_combine_bwd(dout.cuda(), o.cuda(), slot_of.cuda(), top_idx.cuda(), gate.cuda(),
                                                           dv(gamma), dv(rs), d_o, dgamma, T=T, Cc=C, k=k))
    generic = any('moe_combine_bwd_generic_kernel' in n for n in names)
    fast = any('moe_combine_bwd_kernel' in n for n in names)
    assert (fast, generic) == ((True, False) if fast_kernel_expected(C, has_gamma) else (False, True)), names
    assert name.startswith('fast') == fast_kernel_expected(C, has_gamma)

    # d_o: live slots exactly g * ((dout * rs) * gamma); padding rows and the slots of -1 pairs never written
    d_o = d_o.cpu()
    live = slot_of >= 0
    s = slot_of[live].long()
    dy = dout if rs is None else dout * rs[:, None]
    if gamma is not None:
        dy = dy * gamma
    tok = torch.arange(T).view(T, 1).expand(T, k)[live]
    assert torch.equal(d_o[s], gate[live].view(-1, 1) * dy[tok])
    untouched = torch.ones(R, dtype=torch.bool)
    untouched[s] = False
    assert bool(untouched.any()) and bool((d_o[untouched] == SENTINEL).all())

    # dgate = <o[slot], dout * rs * gamma>, exactly 0 on -1 pairs; dgamma = sum_t rs * dout * y   (float64)
    dgate = dgate.cpu()
    o64, dy64 = o.double(), dout.double() * (1.0 if rs is None else rs.double()[:, None]) * \
        (1.0 if gamma is None else gamma.double())
    want = torch.zeros(T, k, dtype=torch.float64)
    want[live] = (o64[s] * dy64[tok]).sum(1)
    assert bool((dgate[~live] == 0).all())
    assert within('combine_bwd.dgate', rel(dgate, want), 1e-5)
    if gamma is not None:
        y = torch.zeros(T, C, dtype=torch.float64).index_add(0, tok, gate[live].double().view(-1, 1) * o64[s])
        dz = dout.double() * (1.0 if rs is None else rs.double()[:, None])
        assert within('combine_bwd.dgamma', rel(dgamma, (dz * y).sum(0)), 1e-5)


def test_gather_sum_bit_exact(ops):
    g = torch.Generator().manual_seed(9)
    for C, k in ((32, 1), (384, 3), (2048, 2)):
        T = 517
        top_idx, slot_of, _, R = synth_dispatch(T, 8, k, g)
        src = torch.randn(R, C, generator=g)
        add = torch.randn(T, C, generator=g)
        for a in (None, add):
            out = ops.gather_sum(src.cuda(), slot_of.cuda(), None if a is None else a.cuda(), T=T, Cc=C, k=k).cpu()
            want = torch.zeros(T, C) if a is None else a.clone()
            for j in range(k):
                s = slot_of[:, j].long()
                want = torch.where((s >= 0)[:, None], want + src[s.clamp_min(0)], want)
            assert torch.equal(out, want), (C, k, a is None)


@pytest.mark.parametrize('C', [96, 200])
def test_colsum_segments(ops, C):
    """Per-expert column sums over padded segments: an empty segment, one shorter than the number of row chunks the
    launch splits a segment into, ragged lengths; with and without b / row_scale; accumulates into out."""
    g = torch.Generator().manual_seed(C)
    R = 5000
    segs = [(0, 0), (128, 138), (256, 1301), (1408, 1409), (1536, 4999)]
    G = len(segs)
    gy = (C + 63) // 64
    chunks = min(max(ops.num_sms() * 8 // (gy * G), 1), (R + 63) // 64)
    assert chunks > 10                                          # segment 1 (10 rows) is shorter than the chunk count
    sb = torch.tensor([s[0] for s in segs], dtype=torch.int32)
    se = torch.tensor([s[1] for s in segs], dtype=torch.int32)
    a = torch.randn(R, C, generator=g)
    b = torch.randn(R, C, generator=g)
    rs = drop_path_scale(R, g)
    init = torch.randn(G, C, generator=g)
    for use in range(4):
        bb, rr = (b if use & 1 else None), (rs if use & 2 else None)
        out = init.clone().cuda()
        ops.colsum(a.cuda(), out, rows=R, Cc=C, b=None if bb is None else bb.cuda(), row_scale=None if rr is None else rr.cuda(),
                   segs=(sb.cuda(), se.cuda()), groups=G)
        out = out.cpu()
        v = a.double() * (1.0 if bb is None else bb.double()) * (1.0 if rr is None else rr.double()[:, None])
        want = init.double() + torch.stack([v[s0:s1].sum(0) for s0, s1 in segs])
        assert torch.equal(out[0], init[0])                     # empty segment: nothing added
        for gi in range(1, G):
            assert within('colsum', rel(out[gi] - init[gi], want[gi] - init[gi].double()), 1e-5), (use, gi)


# ---- router backward ------------------------------------------------------------------------------------------------
def hub_sim(P, E, g):
    """Sim columns: s_0 = h, s_e = -h + 0.6 u_e (+ 1 % noise), with h, u_e orthonormal.  A token along h has cosine ~1 with
    expert 0 and ~ -0.86 with every other, so at the clamped scale of 100 its second gate underflows to 0 in fp32."""
    sim = torch.zeros(P, E)
    sim[P - 1, 0] = 1.0
    for e in range(1, E):
        sim[P - 1, e] = -1.0
        sim[e - 1, e] = 0.6
    return sim + 0.01 * torch.randn(P, E, generator=g)


def live_fp32(vals):
    ex = torch.exp(vals - vals[:, :1])
    return (ex / ex.sum(1, keepdim=True)) > 0


ROUTER_CASES = []
for _i, (_E, _k) in enumerate([(2, 1), (8, 2), (8, 3), (16, 2), (16, 8)]):
    for _mode in ('clean', 'noisy'):
        ROUTER_CASES.append((_E, _k, _mode))
ROUTER_CASES += [(2, 2, 'noisy'), (8, 8, 'noisy')]             # noisy with k == E: hard load, sigma still in the gates


@pytest.mark.parametrize('tau', [math.log(10.0), 5.0], ids=['tau_ln10', 'tau_clamped'])
@pytest.mark.parametrize('E,k,mode', ROUTER_CASES, ids=[f'E{c[0]}_k{c[1]}_{c[2]}' for c in ROUTER_CASES])
def test_router_bwd(ops, E, k, mode, tau):
    P = (48, 192, 256)[(E + k) % 3]
    C = max(64, (P + 31) // 32 * 32)
    g = torch.Generator().manual_seed(E * 10 + k + (P if mode == 'noisy' else 0))
    T, U = 3000, 64                                             # U designed tokens along h (second gate underflows at scale 100)
    sim = hub_sim(P, E, g)
    p = torch.randn(T, P, generator=g)
    p[:, P - 1] *= 0.3                                          # random tokens stay far from the underflow regime
    p[:U] = sim[:, 0] * 5.0 + 1e-3 * torch.randn(U, P, generator=g)
    v = torch.cat([p, torch.randn(T, C - P, generator=g)], 1)
    wp = torch.zeros(P, C)
    wp[:, :P] = torch.eye(P)                                    # projector = [I | 0], bias 0: p = v[:, :P] exactly
    bp = torch.zeros(P)
    tau_t = torch.tensor([tau])
    noisy = mode == 'noisy'
    w_noise = torch.randn(C, E, generator=g) * (0.3 / math.sqrt(C)) if noisy else None
    noise = torch.randn(T, E, generator=g) if noisy else None
    dv = lambda t: None if t is None else t.cuda()
    r = ops.moe_router(v.cuda(), wp.cuda(), bp.cuda(), sim.cuda(), tau_t.cuda(), T=T, Cc=C, E=E, k=k, w_noise=dv(w_noise),
                       noise=dv(noise), save=True)
    plan = ops.moe_plan(r['partials'], T=T, E=E, k=k)
    logits = r['logits'].cpu()
    assert torch.equal(r['p'].cpu(), p)

    # the kernel's routing: its own (k+1) ranking when noisy, else its fp32 clean logits sorted (ties -> lower id)
    if noisy:
        idx_m = r['top_idx_m'].cpu().long()
        vals = r['top_vals'].cpu()[:, :k]
    else:
        idx_m = logits.sort(dim=1, descending=True, stable=True).indices[:, :min(k + 1, E)]
        vals = logits.gather(1, idx_m[:, :k])
    top_idx, idx_k1 = idx_m[:, :k], (idx_m[:, k] if k < E else None)
    live = live_fp32(vals)
    assert torch.equal(r['top_idx'].cpu().long(), torch.where(live, top_idx, -1))
    underflow = tau > moe_ref.LN100 and k > 1
    assert bool(live[U:].all())
    if k > 1:
        assert bool((~live[:U, 1:]).all()) == underflow

    for upstream in ('gate', 'load'):
        leaves = dict(p=p.double(), sim=sim.double(), tau=tau_t.double())
        if noisy:
            leaves['r'] = v.double() @ w_noise.double()
        for t in leaves.values():
            t.requires_grad_(True)
        shat = F.normalize(leaves['sim'], dim=0)
        clean = (F.normalize(leaves['p'], dim=1) @ shat) * torch.clamp(leaves['tau'], max=moe_ref.LN100).exp()
        clean.retain_grad()
        gi = moe_ref.gating_from_logits(clean, top_idx, idx_k1=idx_k1, noise=None if noise is None else noise.double(),
                                        r=leaves.get('r'), live=live)
        dgate = torch.randn(T, k, generator=g) if upstream == 'gate' else torch.zeros(T, k)
        ls = 0.0 if upstream == 'gate' else 1.0
        ((gi['top_gates'] * dgate.double()).sum() + ls * gi['loss']).backward()

        dsim = torch.zeros(P, E, device='cuda')
        dtau = torch.zeros(1, device='cuda')
        nz = dict(noise=noise.cuda(), sigma=r['sigma'], top_vals=r['top_vals'], top_idx_m=r['top_idx_m'],
                  load=plan['load']) if noisy else None
        dp, dr = ops.moe_router_bwd(r['p'], sim.cuda(), tau_t.cuda(), r['top_idx'], r['top_gate'], dgate.cuda(), r['logits'],
                                    plan['importance'], torch.tensor([ls], device='cuda'), dsim, dtau, T=T, E=E, k=k,
                                    noisy=nz)
        assert within(f'router_bwd.dp.{upstream}', rel(dp, leaves['p'].grad), 1e-5)
        assert within(f'router_bwd.dsim.{upstream}', rel(dsim, leaves['sim'].grad), 1e-5)
        if noisy:
            dr = dr.cpu()
            assert bool((dr[:, E:] == 0).all())                  # padding columns of the 32-wide dw_noise / dv GEMMs
            assert within(f'router_bwd.dr.{upstream}', rel(dr[:, :E], leaves['r'].grad), 1e-5)
        if tau > moe_ref.LN100:
            assert dtau.item() == 0.0
        else:
            # one sum over T tokens with cancellation: bound by the sum of the per-token magnitudes
            bound = 1e-5 * (clean.grad * clean).sum(1).abs().sum().item()
            err = abs(dtau.item() - leaves['tau'].grad.item())
            assert err == 0.0 if bound == 0.0 else within(f'router_bwd.dtau/bound.{upstream}', err / bound, 1.0)


# ---- layers at designed expert loads --------------------------------------------------------------------------------
def design_tokens(counts, k, E, g, *, w=(1.0, 0.8, 0.62), w_next=0.35):
    """Routing from per-expert pair counts (sum = k*T, each <= T): token t takes the t-th and (t+T)-th ... entries of the
    expert list sorted by id (distinct because no count exceeds T), in random rank order; tokens shuffled.  Returns the
    top-k in rank order, the (k+1)-th expert (a random other one) and the expert-space coordinates x[:, :E]."""
    T = sum(counts) // k
    assert sum(counts) == k * T and max(counts) <= T and len(counts) == E
    L = torch.repeat_interleave(torch.arange(E), torch.tensor(counts))
    sets = L.view(k, T).t()
    top = sets.gather(1, torch.rand(T, k, generator=g).argsort(1))[torch.randperm(T, generator=g)]
    xe = torch.zeros(T, E)
    xe.scatter_(1, top, torch.tensor(w[:k]).expand(T, k).contiguous())
    idx_k1 = None
    if k < E:
        sc = torch.rand(T, E, generator=g).scatter(1, top, -1.0)
        idx_k1 = sc.argmax(1)
        xe.scatter_(1, idx_k1.view(T, 1), w_next)
    return top, idx_k1, xe


def expert_counts(top, live, E):
    return torch.zeros(E, dtype=torch.long).scatter_add(0, top[live], torch.ones(int(live.sum()), dtype=torch.long))


def check_design(gi, k):
    """Designed gates: top gate in 0.6-0.9 and the (k)-vs-(k+1) gap >= 5 % of max|logit| (float64 reference values)."""
    sel = gi['sel'].detach()
    s = sel.sort(1, descending=True).values
    ok = gi['live'].all(1)
    if k > 1:
        g0 = gi['top_gates'][ok, 0].detach()
        assert 0.6 <= g0.min().item() and g0.max().item() <= 0.9, (g0.min().item(), g0.max().item())
    if k < sel.shape[1]:
        assert ((s[ok, k - 1] - s[ok, k]) >= 0.05 * sel.abs().max()).all()


def compare_params(named, ref, gi, fwd_tol=5e-5, grad_tol=1e-4):
    """Every parameter gradient of the CUDA module vs the float64 reference leaves; temperature by the per-token rule."""
    for n, prm in named:
        want = ref[n].grad
        got = prm.grad
        if want is None:
            assert got is None or not bool(got.abs().max() > 0), n
        elif n.endswith('temperature'):
            bound = grad_tol * (gi['clean'].grad * gi['clean']).sum(1).abs().sum().item()
            err = abs(got.item() - want.item())
            assert err == 0.0 if bound == 0.0 else within('layer.dtau/bound', err / bound, 1.0), (n, err, bound)
        else:
            assert within('layer.param_grads', rel(got, want), grad_tol), n


CNX_CASES = [  # (id, E, k, counts, (N, H, W), noisy, drop_path)
    ('loads_e8_k2', 8, 2, [0, 1, 127, 128, 129, 256, 255, 128], (2, 16, 16), False, False),
    ('tiles_exceed_sms', 8, 2, [129, 4000, 12000, 0, 9000, 6000, 8000, 871], (1, 100, 200), False, False),
    ('k1', 8, 1, [1, 127, 128, 129, 0, 100, 27, 0], (2, 16, 16), False, False),
    ('k3', 8, 3, [128, 129, 127, 256, 1, 383, 512, 0], (2, 16, 16), False, False),
    ('e16', 16, 2, [0, 1, 127, 128, 129] + [49] * 10 + [149], (2, 16, 16), False, False),
    ('noisy_droppath', 8, 2, [0, 1, 127, 128, 129, 256, 255, 128], (2, 16, 16), True, True)]


@pytest.mark.parametrize('name,E,k,counts,nhw,noisy,drop', CNX_CASES, ids=[c[0] for c in CNX_CASES])
def test_convnext_moe_block_designed_loads(ops, name, E, k, counts, nhw, noisy, drop):
    from sm3det_b200.backbone import ConvNeXtBlock
    g = torch.Generator().manual_seed(len(name) * 7 + E + k)
    N, H, W = nhw
    C = 96
    T = N * H * W
    top, idx_k1, xe = design_tokens(counts, k, E, g)
    assert top.shape[0] == T
    x = torch.cat([xe, torch.zeros(T, C - E)], 1) + 0.01 * torch.randn(T, C, generator=g)
    blk = ConvNeXtBlock(C, dict(type='LN2d', eps=1e-6), MoE_cfg=dict(num_experts=E, top_k=k, noisy_gating=noisy,
                                                                     gating='cosine'),
                        drop_path_rate=0.25 if drop else 0.0)
    P = blk.ffn.w_gate.sim_matrix.shape[0]
    with torch.no_grad():
        blk.depthwise_conv.weight.zero_()
        blk.depthwise_conv.weight[:, 0, 3, 3] = 1.0                # centre tap: u = x
        blk.depthwise_conv.bias.zero_()
        blk.norm.weight.fill_(1.0)
        blk.norm.bias.zero_()
        blk.gamma.copy_(torch.rand(C, generator=g) * 0.5 + 0.5)
        gw = blk.ffn.w_gate
        gw.temperature.fill_(math.log(10.0))
        gw.sim_matrix.copy_(torch.eye(P, E))
        gw.cosine_projector.weight.copy_(torch.eye(P, C) * (torch.arange(P) < E).view(P, 1) +
                                         1e-3 * torch.randn(P, C, generator=g))     # [I_E | 0]
        gw.cosine_projector.bias.zero_()
        blk.ffn.w_noise.copy_(torch.randn(C, E, generator=g) * 0.05 / math.sqrt(C))
        for ex in blk.ffn.experts:
            ex.pointwise_conv1.weight.copy_(torch.randn(4 * C, C, generator=g) / math.sqrt(C))
            ex.pointwise_conv1.bias.copy_(torch.randn(4 * C, generator=g) * 0.1)
            ex.pointwise_conv2.weight.copy_(torch.randn(C, 4 * C, generator=g) / math.sqrt(4 * C))
            ex.pointwise_conv2.bias.copy_(torch.randn(C, generator=g) * 0.1)
    noise = 0.1 * torch.randn(T, E, generator=g) if noisy else None
    mask = torch.tensor([0.0, 1.0 / 0.75])[:N] if drop else None
    ref = {n: p.detach().double().clone().requires_grad_(True) for n, p in blk.named_parameters()}
    blk = blk.cuda().train()
    if noisy:
        blk.ffn._injected_noise = noise.cuda()
    if drop:
        blk._injected_drop_mask = mask.cuda()
    xd = x.view(N, H, W, C).cuda().requires_grad_(True)
    dout = torch.randn(N, H, W, C, generator=g)
    rec = []
    out, loss = blk(xd, record=rec)
    ((out * dout.cuda()).sum() + loss).backward()
    torch.cuda.synchronize()

    x64 = x.double().view(N, H, W, C).requires_grad_(True)
    rs = None if mask is None else mask.double().repeat_interleave(H * W)
    out_r, gi = moe_ref.convnext_moe_block(x64, ref, E=E, top_idx=top, idx_k1=idx_k1,
                                           noise=None if noise is None else noise.double(), row_scale=rs)
    ((out_r * dout.double()).sum() + gi['loss']).backward()

    check_design(gi, k)
    assert torch.equal(rec[0]['top_idx'].cpu().long(), top)
    assert torch.equal(rec[0]['counts'].cpu().long(), torch.tensor(counts))
    if name == 'tiles_exceed_sms':
        assert sum((c + 127) // 128 for c in counts) > ops.num_sms()
    assert within('layer.out', rel(out, out_r), 5e-5)
    assert within('layer.y', rel(rec[0]['y'], gi['y']), 5e-5)
    assert within('layer.gate_loss', rel(loss, gi['loss']), 5e-5)
    assert within('layer.importance', rel(rec[0]['importance'], gi['importance']), 5e-5)
    assert within('layer.load', rel(rec[0]['load'], gi['load']), 5e-5)
    assert within('layer.dx', rel(xd.grad, x64.grad), 1e-4)
    compare_params(blk.named_parameters(), ref, gi)


LSK_CASES = [  # (id, E, k, Cin, Cout, counts, (N, H, W), noisy, tail, tau, underflow tokens)
    ('fc1_c2048', 8, 2, 256, 2048, [0, 1, 127, 128, 129, 256, 255, 128], (2, 16, 16), False, False, math.log(10.0), 0),
    ('fc2_tail_noisy', 8, 2, 512, 64, [0, 1, 127, 128, 129, 256, 255, 128], (2, 16, 16), True, True, math.log(10.0), 0),
    ('underflow', 4, 2, 64, 64, [385, 1, 127, 511], (2, 16, 16), False, False, 5.0, 96)]


@pytest.mark.parametrize('name,E,k,Cin,Cout,counts,nhw,noisy,tail,tau,U', LSK_CASES, ids=[c[0] for c in LSK_CASES])
def test_lsk_moe_layer_designed_loads(ops, name, E, k, Cin, Cout, counts, nhw, noisy, tail, tau, U):
    from sm3det_b200.lsk_backbone import MoE_layer
    g = torch.Generator().manual_seed(len(name) + E + Cin)
    N, H, W = nhw
    T = N * H * W
    clamped = tau > moe_ref.LN100
    # at the clamped scale of 100 the designed gaps must be 10x narrower in cosine for gates of 0.6-0.9
    top, idx_k1, xe = design_tokens(counts, k, E, g, **(dict(w=(1.0, 0.99), w_next=0.85) if clamped else {}))
    if U:
        # first U tokens: x = e_a - 0.3 e_c - 0.36 (the other two): cos_a - cos_c = 1.12 -> the second gate is
        # exp(-112) = 0 in fp32; cos_c - cos_other = 0.05 keeps the second choice unambiguous
        assert E == 4 and k == 2
        xe[:U] = -0.36
        xe[:U].scatter_(1, top[:U, 1:2], -0.30)
        xe[:U].scatter_(1, top[:U, 0:1], 1.0)
    amp = 1e-4 if clamped else 0.01
    x = torch.cat([xe, torch.zeros(T, Cin - E)], 1) + amp * torch.randn(T, Cin, generator=g)
    m = MoE_layer(dict(noisy_gating=noisy, num_experts=E, in_channels=Cin, out_channels=Cout, top_k=k, gating='cosine'))
    P = m.w_gate.sim_matrix.shape[0]
    with torch.no_grad():
        m.w_gate.temperature.fill_(tau)
        m.w_gate.sim_matrix.copy_(torch.eye(P, E))
        m.w_gate.cosine_projector.weight.copy_(torch.eye(P, Cin) * (torch.arange(P) < E).view(P, 1) +
                                               (1e-5 if clamped else 1e-3) * torch.randn(P, Cin, generator=g))
        m.w_gate.cosine_projector.bias.zero_()
        m.w_noise.copy_(torch.randn(Cin, E, generator=g) * 0.05 / math.sqrt(Cin))
        for ex in m.experts:
            ex.weight.copy_(torch.randn(Cout, Cin, 1, 1, generator=g) / math.sqrt(Cin))
            ex.bias.copy_(torch.randn(Cout, generator=g) * 0.1)
    noise = 0.1 * torch.randn(T, E, generator=g) if noisy else None
    gamma = torch.rand(Cout, generator=g) * 0.5 + 0.5 if tail else None
    resid = torch.randn(N, H, W, Cout, generator=g) if tail else None
    rs = drop_path_scale(T, g) if tail else None
    ref = {n: p.detach().double().clone().requires_grad_(True) for n, p in m.named_parameters()}
    m = m.cuda().train()
    if noisy:
        m._injected_noise = noise.cuda()
    leaf = lambda t: None if t is None else t.cuda().requires_grad_(True)
    xd, gd, rd = leaf(x.view(N, H, W, Cin)), leaf(gamma), leaf(resid)
    dout = torch.randn(N, H, W, Cout, generator=g)
    rec = []
    out, loss = m(xd, gamma=gd, resid=rd, row_scale=None if rs is None else rs.cuda(), record=rec)
    ((out * dout.cuda()).sum() + loss).backward()
    torch.cuda.synchronize()

    leaf64 = lambda t: None if t is None else t.double().requires_grad_(True)
    x64, g64, r64 = leaf64(x.view(N, H, W, Cin)), leaf64(gamma), leaf64(resid)
    out_r, gi = moe_ref.lsk_moe_layer(x64, ref, E=E, top_idx=top, idx_k1=idx_k1,
                                      noise=None if noise is None else noise.double(), gamma=g64, resid=r64,
                                      row_scale=None if rs is None else rs.double())
    ((out_r * dout.double()).sum() + gi['loss']).backward()

    check_design(gi, k)
    live = gi['live']
    assert bool((~live[:U, 1]).all()) and bool(live[U:].all())   # exactly the designed tokens lose their second pair
    assert torch.equal(rec[0]['top_idx'].cpu().long(), torch.where(live, top, -1))
    assert torch.equal(rec[0]['counts'].cpu().long(), expert_counts(top, live, E))
    assert within('layer.out', rel(out, out_r), 5e-5)
    assert within('layer.gate_loss', rel(loss, gi['loss']), 5e-5)
    assert within('layer.importance', rel(rec[0]['importance'], gi['importance']), 5e-5)
    assert within('layer.load', rel(rec[0]['load'], gi['load']), 5e-5)
    assert within('layer.dx', rel(xd.grad, x64.grad), 1e-4)
    if tail:
        assert within('layer.dgamma', rel(gd.grad, g64.grad), 1e-4)
        assert within('layer.dresid', rel(rd.grad, r64.grad), 1e-4)
    if clamped:
        assert m.w_gate.temperature.grad.item() == 0.0
    compare_params(m.named_parameters(), ref, gi)
