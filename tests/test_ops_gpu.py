"""GPU parity of each C-ABI kernel against plain torch fp32 on the CPU (oracle arithmetic)."""
import math
import os

import pytest
import torch
import torch.nn.functional as F

from gemm_ref import decode_k_image

pytestmark = pytest.mark.gpu


def rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).abs().max() / (b.abs().max() + 1e-30)).item()


@pytest.fixture(scope='module')
def ops():
    from sm3det_b200 import ops as o
    return o


@pytest.mark.parametrize('C', [32, 96, 192, 384, 768, 1024])
def test_layernorm_modes(ops, C):
    g = torch.Generator().manual_seed(C)
    N, H, W = 2, 6, 8
    x = torch.randn(N, H, W, C, generator=g) * 2 + 0.5
    w, b = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.1
    ref = F.layer_norm(x, (C,), w, b, 1e-6)
    xd, wd, bd = x.cuda(), w.cuda(), b.cuda()
    T = N * H * W
    y, stats = ops.layernorm_fwd(xd, wd, bd, 1e-6, tokens=T, C=C, save_stats=True)
    assert rel(y, ref) < 1e-5
    # NCHW output
    y2 = torch.empty(N, C, H, W, device='cuda')
    ops.layernorm_fwd(xd, wd, bd, 1e-6, tokens=T, C=C, out=y2, out_mode=ops.LN_NCHW, H=H, W=W)
    assert rel(y2, ref.permute(0, 3, 1, 2)) < 1e-5
    # 2x2 patch output
    y3 = torch.empty(T // 4, 4 * C, device='cuda')
    ops.layernorm_fwd(xd, wd, bd, 1e-6, tokens=T, C=C, out=y3, out_mode=ops.LN_PATCH2, H=H, W=W)
    refp = ref.view(N, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(T // 4, 4 * C)
    assert rel(y3, refp) < 1e-5
    # backward (all three gradient layouts)
    xr = x.clone().requires_grad_(True); wr = w.clone().requires_grad_(True); br = b.clone().requires_grad_(True)
    out = F.layer_norm(xr, (C,), wr, br, 1e-6)
    dy = torch.randn(N, H, W, C, generator=g)
    out.backward(dy)
    for mode, dyl in ((ops.LN_NHWC, dy), (ops.LN_NCHW, dy.permute(0, 3, 1, 2).contiguous()),
                      (ops.LN_PATCH2, dy.view(N, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(T // 4, 4 * C).contiguous())):
        dw = torch.zeros(C, device='cuda'); db = torch.zeros(C, device='cuda')
        dx = ops.layernorm_bwd(dyl.cuda(), xd, stats, wd, dw, db, tokens=T, C=C, in_mode=mode, H=H, W=W)
        assert rel(dx.view(N, H, W, C), xr.grad) < 2e-5, mode
        assert rel(dw, wr.grad) < 2e-5 and rel(db, br.grad) < 2e-5, mode


@pytest.mark.parametrize('C,H,W', [(32, 8, 8), (96, 25, 13), (192, 7, 50), (384, 16, 16), (768, 1, 3)])
def test_dwconv7(ops, C, H, W):
    g = torch.Generator().manual_seed(C + H)
    N = 2
    x = torch.randn(N, C, H, W, generator=g, requires_grad=True)
    w = (torch.randn(C, 1, 7, 7, generator=g) * 0.2).requires_grad_(True)
    b = (torch.randn(C, generator=g) * 0.1).requires_grad_(True)
    ref = F.conv2d(x, w, b, padding=3, groups=C)
    dy = torch.randn(N, C, H, W, generator=g)
    ref.backward(dy)
    xh = x.detach().permute(0, 2, 3, 1).contiguous().cuda()
    wt = w.detach().reshape(C, 49).t().contiguous().cuda()
    y = ops.dwconv7(xh, wt, b.detach().cuda())
    assert rel(y.permute(0, 3, 1, 2), ref) < 1e-5
    dyh = dy.permute(0, 2, 3, 1).contiguous().cuda()
    wtf = w.detach().flip(2, 3).reshape(C, 49).t().contiguous().cuda()
    res = torch.randn(N, H, W, C, generator=g)
    dx = ops.dwconv7(dyh, wtf, None, resid=res.cuda())
    assert rel(dx.cpu() - res, x.grad.permute(0, 2, 3, 1)) < 1e-5
    dwt = torch.zeros(49, C, device='cuda'); dbb = torch.zeros(C, device='cuda')
    ops.dwconv7_wgrad(xh, dyh, dwt, dbb)
    assert rel(dwt.t().reshape(C, 1, 7, 7), w.grad) < 2e-5
    assert rel(dbb, b.grad) < 2e-5


@pytest.mark.parametrize('C0', [32, 96, 128])
def test_stem(ops, C0):
    g = torch.Generator().manual_seed(C0)
    N, H, W = 2, 64, 96
    x = torch.randn(N, 3, H, W, generator=g)
    w = (torch.randn(C0, 3, 4, 4, generator=g) * 0.2).requires_grad_(True)
    b = (torch.randn(C0, generator=g) * 0.1).requires_grad_(True)
    lw = (torch.rand(C0, generator=g) + 0.5).requires_grad_(True); lb = (torch.randn(C0, generator=g) * 0.1).requires_grad_(True)
    u = F.conv2d(x, w, b, stride=4)
    ref = F.layer_norm(u.permute(0, 2, 3, 1), (C0,), lw, lb, 1e-6)
    dy = torch.randn(ref.shape, generator=g)
    ref.backward(dy)
    wt = w.detach().reshape(C0, -1).t().contiguous().cuda()
    y, conv, stats = ops.stem_fwd(x.cuda(), wt, b.detach().cuda(), lw.detach().cuda(), lb.detach().cuda(), 1e-6, 4, save=True)
    assert rel(y, ref) < 1e-5
    assert rel(conv, u.permute(0, 2, 3, 1)) < 1e-5
    T = N * (H // 4) * (W // 4)
    dlw = torch.zeros(C0, device='cuda'); dlb = torch.zeros(C0, device='cuda')
    du = ops.layernorm_bwd(dy.cuda(), conv, stats, lw.detach().cuda(), dlw, dlb, tokens=T, C=C0)
    dwt = torch.zeros(48, C0, device='cuda'); dbb = torch.zeros(C0, device='cuda')
    ops.stem_wgrad(x.cuda(), du, dwt, dbb, 4)
    assert rel(dwt.t().reshape(C0, 3, 4, 4), w.grad) < 2e-5
    assert rel(dbb, b.grad) < 2e-5 and rel(dlw, lw.grad) < 2e-5 and rel(dlb, lb.grad) < 2e-5


@pytest.mark.parametrize('M,N,K', [(300, 384, 96), (1000, 96, 384), (130, 768, 3072), (64, 256, 128)])
def test_linear_fwd_dgrad_wgrad(ops, M, N, K):
    g = torch.Generator().manual_seed(M + N)
    x = torch.randn(M, K, generator=g, requires_grad=True)
    w = (torch.randn(N, K, generator=g) / math.sqrt(K)).requires_grad_(True)
    b = (torch.randn(N, generator=g) * 0.1).requires_grad_(True)
    h = F.linear(x, w, b)
    ref = F.gelu(h)
    dy = torch.randn(M, N, generator=g)
    ref.backward(dy)
    xd, wd, bd = x.detach().cuda(), w.detach().cuda(), b.detach().cuda()
    hbuf = torch.empty(M, N, device='cuda')
    y = ops.linear_fwd(xd, wd, bd, epilogue=ops.EPI_GELU, aux_out=hbuf)
    assert rel(y, ref) < 5e-5 and rel(hbuf, h) < 5e-5
    # dgrad with fused GELU'
    dh_ref = torch.autograd.grad(F.gelu(h.detach().requires_grad_(True)), [], allow_unused=True) if False else None
    hd = h.detach().clone().requires_grad_(True)
    F.gelu(hd).backward(dy)
    dh = hd.grad
    dx = ops.linear_dgrad(dh.cuda(), wd)
    assert rel(dx, x.grad) < 5e-5
    ident = torch.eye(N)
    dh_gpu = ops.linear_dgrad(dy.cuda(), ident.cuda().contiguous(), epilogue=ops.EPI_DGELU, aux_in=hbuf)
    assert rel(dh_gpu, dh) < 5e-5
    dw = torch.zeros(N, K, device='cuda')
    ops.linear_wgrad(dh.cuda(), xd, dw)
    assert rel(dw, w.grad) < 5e-5
    db = torch.zeros(N, device='cuda')
    ops.colsum(dh.cuda(), db, rows=M, Cc=N)
    assert rel(db, b.grad) < 2e-5


@pytest.mark.parametrize('C,E,k,T', [(96, 4, 2, 500), (384, 8, 2, 4096), (768, 8, 3, 1000), (128, 6, 1, 777), (64, 2, 2, 256),
                                      (512, 16, 2, 2048)])
@pytest.mark.parametrize('tau', [math.log(2.0), math.log(10.0), 5.0])
def test_router_matches_oracle_bit_exact(ops, C, E, k, T, tau):
    from oracle.convnext_moe_oracle import OracleConfig, noisy_top_k_gating, cv_squared
    g = torch.Generator().manual_seed(C * E + k)
    P = min(C // 2, 256)
    v = torch.randn(T, C, generator=g)
    sd = {'w_gate.cosine_projector.weight': torch.randn(P, C, generator=g) / math.sqrt(C),
          'w_gate.cosine_projector.bias': torch.randn(P, generator=g) * 0.05,
          'w_gate.sim_matrix': torch.randn(P, E, generator=g), 'w_gate.temperature': torch.tensor([tau]),
          'w_noise': torch.zeros(C, E)}
    cfg = OracleConfig(num_experts=E, top_k=k)
    gates, load, info = noisy_top_k_gating(v, sd, '', cfg, train=False)
    r = ops.moe_router(v.cuda(), sd['w_gate.cosine_projector.weight'].cuda(), sd['w_gate.cosine_projector.bias'].cuda(),
                       sd['w_gate.sim_matrix'].cuda(), sd['w_gate.temperature'].cuda(), T=T, Cc=C, E=E, k=k, save=True)
    idx = r['top_idx'].cpu().long()
    ref_idx = info['top_idx']
    mism = (idx != ref_idx).any(dim=1)
    # fp32 summation order differs from MKL's: only (k)-vs-(k+1) near-ties (margin < 1e-5 * scale) may flip
    if mism.any():
        top = info['logits'].topk(min(k + 1, E), dim=-1).values
        gaps = (top[:, :-1] - top[:, 1:]).min(dim=1).values
        assert (gaps[mism] < 1e-5 * math.exp(min(tau, math.log(100)))).all(), f'{int(mism.sum())} real routing mismatches'
        assert mism.sum() <= 2
    ok = ~mism
    scale = math.exp(min(tau, math.log(100)))
    # gates = softmax of logits that reach +-scale: fp32 rounding of the logits (1e-7 * scale) carries through exp
    assert (r['top_gate'].cpu()[ok] - info['top_gates'][ok]).abs().max() < 2e-6 + 3e-7 * scale
    assert rel(r['logits'], info['logits']) < 2e-6
    plan = ops.moe_plan(r['partials'], T=T, E=E, k=k)
    imp = gates.sum(0)
    loss = (cv_squared(imp) + cv_squared(load)) * 1e-2
    if not mism.any():
        assert rel(plan['importance'], imp) < 1e-5
        assert torch.equal(plan['counts'].cpu().long(), load)
        assert abs(plan['loss'].item() - loss.item()) <= 1e-5 * abs(loss.item()) + 1e-9
    # dispatch plan invariants
    slot_of, pair_token = ops.moe_assign(r['top_idx'], plan, T=T, E=E, k=k)
    sb, se, cnt = plan['seg_begin'].cpu(), plan['seg_end'].cpu(), plan['counts'].cpu()
    assert (sb % 128 == 0).all() and torch.equal(se - sb, cnt)
    so, pt = slot_of.cpu().long(), pair_token.cpu().long()
    assert (pt[so.flatten()] == torch.arange(T).repeat_interleave(k)).all()
    for e in range(E):
        assert ((so >= sb[e]) & (so < se[e])).sum() == cnt[e]
        assert (idx[(so >= sb[e]) & (so < se[e])] == e).all()
    assert (pt >= 0).sum() == T * k
    ntile = plan['num_m_tiles'].item()
    tg = plan['tile_group'].cpu()[:ntile]
    assert ntile == sum((int(c) + 127) // 128 for c in cnt)
    for t in range(ntile):
        assert sb[tg[t]] <= t * 128 < sb[tg[t]] + ((cnt[tg[t]] + 127) // 128) * 128


def test_router_noisy_soft_load(ops):
    from oracle.convnext_moe_oracle import OracleConfig, noisy_top_k_gating, cv_squared
    g = torch.Generator().manual_seed(3)
    C, E, k, T = 96, 4, 2, 1000
    P = C // 2
    v = torch.randn(T, C, generator=g)
    sd = {'w_gate.cosine_projector.weight': torch.randn(P, C, generator=g) / math.sqrt(C),
          'w_gate.cosine_projector.bias': torch.randn(P, generator=g) * 0.05,
          'w_gate.sim_matrix': torch.randn(P, E, generator=g), 'w_gate.temperature': torch.tensor([math.log(10.)]),
          'w_noise': torch.randn(C, E, generator=g) * 0.05}
    noise = torch.randn(T, E, generator=g)
    cfg = OracleConfig(num_experts=E, top_k=k)
    gates, load, info = noisy_top_k_gating(v, sd, '', cfg, train=True, noise=noise)
    r = ops.moe_router(v.cuda(), sd['w_gate.cosine_projector.weight'].cuda(), sd['w_gate.cosine_projector.bias'].cuda(),
                       sd['w_gate.sim_matrix'].cuda(), sd['w_gate.temperature'].cuda(), T=T, Cc=C, E=E, k=k,
                       w_noise=sd['w_noise'].cuda(), noise=noise.cuda(), save=True)
    assert torch.equal(r['top_idx'].cpu().long(), info['top_idx'])
    plan = ops.moe_plan(r['partials'], T=T, E=E, k=k)
    assert rel(plan['load'], load) < 1e-5
    loss = (cv_squared(gates.sum(0)) + cv_squared(load)) * 1e-2
    assert abs(plan['loss'].item() - loss.item()) <= 1e-5 * abs(loss.item())


@pytest.mark.parametrize('R,W', [(256, 384), (1000, 128), (300, 1536)])
def test_act_pack_images_feed_gemms(ops, R, W):
    """act_pack's bf16 hi/lo tile images (modes 0 and 3) are consumed by the packed GEMMs exactly like torch's
    gelu / gelu-backward followed by matmuls (forward GEMM2, dgrad1, wgrad1, wgrad2) -- incl. 16-lane column groups (W=384)."""
    g = torch.Generator().manual_seed(R + W)
    C = 64
    h = torch.randn(R, W, generator=g)
    da = torch.randn(R, W, generator=g)
    w2 = torch.randn(C, W, generator=g) / W ** 0.5          # GEMM2 weight [C, 4C]
    w1 = torch.randn(W, C, generator=g) / C ** 0.5          # GEMM1 weight [4C, C]
    v = torch.randn(R, C, generator=g)
    dz = torch.randn(R, C, generator=g)
    hd, dad = h.cuda(), da.cuda()
    a_ref = F.gelu(h)
    hr = h.clone().requires_grad_(True)
    F.gelu(hr).backward(da)
    dh_ref = hr.grad
    # mode 0: K-major image -> forward GEMM2
    a_k, _, a_f32 = ops.act_pack(hd, rows=R, width=W, mode=ops.ACT_GELU, want_k=True, want_f32=True)
    assert rel(a_f32, a_ref) < 2e-6
    y = ops.linear_fwd(None, w2.cuda(), None, rows=R, a_packed=a_k, packed=ops.pack_weight(w2.cuda(), transposed=False))
    assert rel(y, a_ref @ w2.t()) < 5e-5
    # mode 3: one pass -> dgrad1 (K-major dh), wgrad1 (MN-major dh), wgrad2 (MN-major gelu(h)), db1
    db1 = torch.zeros(W, device='cuda')
    dh_k, dh_mn, a_mn = ops.act_pack(hd, rows=R, width=W, mode=ops.ACT_BWD, da=dad, want_k=True, mn_tile=128,
                                     mn_tile2=ops._pick_bn(W), colsum=db1)
    assert rel(db1, dh_ref.sum(0)) < 5e-5
    dv = ops.linear_dgrad(None, w1.cuda(), rows=R, a_packed=dh_k, packed=ops.pack_weight(w1.cuda(), transposed=True))
    assert rel(dv, dh_ref @ w1) < 5e-5
    dw1 = torch.zeros(W, C, device='cuda')
    ops.linear_wgrad(None, v.cuda(), dw1, rows=R, dy_packed=dh_mn)
    assert rel(dw1, dh_ref.t() @ v) < 5e-5
    dw2 = torch.zeros(C, W, device='cuda')
    ops.linear_wgrad(dz.cuda(), None, dw2, rows=R, x_packed=a_mn)
    assert rel(dw2, dz.t() @ a_ref) < 5e-5


def test_gather_rows_peer_single_device(ops):
    """sm3_gather_rows_peer with a one-entry pointer table (the expert-parallel row gather, world size 1): direct rows,
    rows through a token list, per-row scale, and -1 -> zero rows."""
    g = torch.Generator().manual_seed(5)
    T, C, R = 200, 96, 333
    x = torch.randn(T, C, generator=g).cuda()
    toks = torch.randint(0, T, (400,), generator=g, dtype=torch.int32).cuda()
    src_rank = torch.zeros(R, dtype=torch.int32); src_rank[::7] = -1
    src_slot = torch.randint(0, 400, (R,), generator=g, dtype=torch.int32)
    scale = torch.rand(R, generator=g)
    bases = torch.tensor([x.data_ptr()], dtype=torch.int64, device='cuda')
    lists = torch.tensor([toks.data_ptr()], dtype=torch.int64, device='cuda')
    out = ops.gather_rows_peer(bases, src_rank.cuda(), src_slot.cuda(), rows=R, Cc=C, token_lists=lists, scale=scale.cuda())
    want = x.cpu()[toks.cpu().long()[src_slot.long()]] * scale[:, None]
    want[src_rank < 0] = 0
    assert torch.equal(out.cpu(), want)
    direct = ops.gather_rows_peer(bases, src_rank.cuda(), (src_slot % T).cuda(), rows=R, Cc=C)
    want2 = x.cpu()[(src_slot % T).long()]
    want2[src_rank < 0] = 0
    assert torch.equal(direct.cpu(), want2)


@pytest.mark.parametrize('W,E,k', [(2, 4, 2), (4, 8, 2), (8, 16, 2), (8, 8, 3)])
def test_ep_plan_kernel_matches_host_plan(W, E, k):
    """sm3_ep_plan (the device-side expert-parallel exchange plan, no host sync) against the host plan the world-2 gloo test
    validates (expert_parallel._build_plan), for every rank of a simulated W-rank group: ragged counts, an idle expert."""
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(__file__), 'dist'))
    from ep_plan_worker import local_plan
    from sm3det_b200.expert_parallel import EPContext, _build_plan, device_plan
    T = 700
    plans = []
    for r in range(W):
        g = torch.Generator().manual_seed(40 + r)
        logits = torch.randn(T, E, generator=g)
        if r == 1:
            logits[:, E - 1] = -1e9               # an expert that receives nothing from this rank
        plans.append(local_plan(logits.topk(k, dim=1).indices, E))
    allm = torch.stack([torch.stack([p[0], p[1]]) for p in plans]).to(torch.int32)          # [W, 2, E]
    for me in range(W):
        counts, seg_begin, tile_group, num_tiles, pair_token, slot_of = plans[me]
        R_s = pair_token.numel()
        ctx = EPContext.__new__(EPContext)
        ctx.world, ctx.rank = W, me
        ctx.overflow = torch.zeros(1, device='cuda', dtype=torch.int32)
        ref = _build_plan(ctx, allm[:, 0], allm[:, 1], tile_group, num_tiles, pair_token, E, R_s, torch.device('cpu'))
        cap = (ref['R_d'] // 128 + 3) * 128
        tg = tile_group.clone()
        tg[tg == 12345] = 0                        # the device plan clamps garbage tile ids itself; keep the input in range too
        P = device_plan(ctx, allm.cuda(), tile_group.cuda(), num_tiles.cuda(), pair_token.cuda(), E, R_s, cap)
        torch.cuda.synchronize()
        R_d = ref['R_d']
        assert int(P['num_tiles']) * 128 == R_d and int(ctx.overflow) == 0
        assert torch.equal(P['src_rank'][:R_d].cpu(), ref['src_rank'][:R_d]) and bool((P['src_rank'][R_d:] == -1).all())
        live = ref['src_rank'][:R_d] >= 0
        assert torch.equal(P['src_slot'][:R_d].cpu()[live], ref['src_slot'][:R_d][live])
        assert torch.equal(P['tile_group'][:R_d // 128].cpu(), ref['tile_group'][:R_d // 128])
        assert torch.equal(P['seg_begin'].cpu(), ref['seg_begin']) and torch.equal(P['seg_end'].cpu(), ref['seg_end'])
        assert torch.equal(P['comb_rank'].cpu(), ref['comb_rank'])
        lv = ref['comb_rank'] >= 0
        assert torch.equal(P['comb_row'].cpu()[lv], ref['comb_row'][lv])
        # capacity overflow is reported, not silently truncated
        ctx.overflow.zero_()
        device_plan(ctx, allm.cuda(), tile_group.cuda(), num_tiles.cuda(), pair_token.cuda(), E, R_s, 128)
        assert int(ctx.overflow) == R_d or R_d <= 128


@pytest.mark.parametrize('T,C', [(300, 96), (1024, 64), (129, 192), (5, 128), (256, 32)])
def test_layernorm_to_operand_image(T, C):
    """sm3_layernorm_fwd_img: LN output written directly as the fused FFN's A-operand image (hi + lo = fp32 value to 2^-17),
    statistics as the plain kernel's, rows of the last 128-row tile beyond T zero."""
    from sm3det_b200 import ops
    g = torch.Generator().manual_seed(T + C)
    x = torch.randn(T, C, generator=g) * 2 + 0.5
    w, b = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.1
    ref = F.layer_norm(x, (C,), w, b, 1e-6)
    img, v, stats = ops.layernorm_fwd_img(x.cuda(), w.cuda(), b.cuda(), 1e-6, tokens=T, C=C, save_stats=True, want_f32=True)
    T_pad = (T + 127) // 128 * 128
    dec = decode_k_image(img, T_pad, C)
    assert (dec[:T] - ref).abs().max() < 2e-5 * ref.abs().max()
    assert (v.cpu() - ref).abs().max() < 1e-5 * ref.abs().max()
    assert (dec[:T] - v.cpu()).abs().max() <= 2.0 ** -16 * ref.abs().max()
    assert float(dec[T:].abs().max() if T_pad > T else 0.0) == 0.0
    assert torch.allclose(stats[:, 0].cpu(), x.mean(1), atol=1e-5) and torch.allclose(stats[:, 1].cpu(), (x.var(1, unbiased=False) + 1e-6).rsqrt(), rtol=1e-5)
    # and the same image as the separate pack of the fp32 output, up to LN rounding
    dec2 = decode_k_image(ops.pack_act(v, rows=T, cols=C, mn_major=False), T_pad, C)
    assert (dec2[:T] - dec[:T]).abs().max() <= 2.0 ** -16 * ref.abs().max()


@pytest.mark.parametrize('T,C', [(640, 96), (200, 64), (384, 32), (300, 128)])
def test_fused_ffn_matches_torch(T, C):
    """sm3_ffn_fused (forward incl. the stored pre-activation, backward into dv) vs plain torch fp32 on the CPU."""
    from sm3det_b200 import ops
    g = torch.Generator().manual_seed(C)
    v = torch.randn(T, C, generator=g, requires_grad=True)
    x = torch.randn(T, C, generator=g)
    w1 = (torch.randn(4 * C, C, generator=g) / C ** 0.5).requires_grad_(True)
    b1 = (torch.randn(4 * C, generator=g) * 0.2).requires_grad_(True)
    w2 = (torch.randn(C, 4 * C, generator=g) / (4 * C) ** 0.5).requires_grad_(True)
    b2 = torch.randn(C, generator=g) * 0.2
    gamma = torch.rand(C, generator=g) * 0.9 + 0.1
    y2 = F.linear(F.gelu(F.linear(v, w1, b1)), w2, b2)
    out = x + gamma * y2
    dz = torch.randn(T, C, generator=g) * 0.1
    out.backward(dz)
    cf, cb = ops.ffn_chunk(0, C), ops.ffn_chunk(1, C)
    assert cf and cb
    dev = lambda t: t.detach().cuda().contiguous()
    v_img = ops.pack_act(dev(v), rows=T, cols=C, mn_major=False)
    w1c, _ = ops.pack_weight(dev(w1), transposed=False, tile=cf)
    w2n, _ = ops.pack_weight(dev(w2), transposed=False, tile=C)
    o, aux, h = ops.ffn_fused_fwd(v_img, w1c, w2n, dev(b1), dev(b2), T=T, C=C, chunk=cf, gamma=dev(gamma), resid=dev(x), want_aux=True,
                                  want_h=True)
    assert rel(o, out) < 5e-5 and rel(aux, y2) < 5e-5
    assert rel(h, F.linear(v, w1, b1)) < 5e-5                       # the pre-activation stored for the GEMM backward
    assert bool(torch.isfinite(o).all()) and bool(torch.isfinite(h).all())
    dz_img = ops.pack_act(dev(dz), rows=T, cols=C, mn_major=False)
    w1cb, _ = ops.pack_weight(dev(w1), transposed=False, tile=cb)
    w2gt, _ = ops.pack_weight(dev(w2) * dev(gamma)[:, None], transposed=True, tile=cb)
    w1tn, _ = ops.pack_weight(dev(w1), transposed=True, tile=C)
    dv = ops.ffn_fused_bwd(v_img, dz_img, w1cb, w2gt, w1tn, dev(b1), T=T, C=C, chunk=cb)
    assert bool(torch.isfinite(dv).all()) and rel(dv, v.grad) < 1e-4
