"""tests/simt_ref.py on the CPU: each float64 reference against the independent torch float64 op, the dropout
re-implementation's statistics, and every bound against torch's own fp32 CPU op on the same inputs (no bound may be
tighter than an fp32 computation of the same kind meets)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import simt_ref as R

TOL = 1e-12


def close(a, b, tol=TOL):
    a, b = R.f64(a), R.f64(b)
    return float(np.abs(a - b).max()) <= tol * max(1.0, float(np.abs(b).max()))


def scaled(g, *shape, lo=-8, hi=8):
    """randn with a per-channel (last axis) scale 2^k, k in [lo, hi], and mixed signs."""
    k = torch.randint(lo, hi + 1, (shape[-1],), generator=g).double()
    return (torch.randn(*shape, generator=g, dtype=torch.float64) * torch.exp2(k)).float()


def t64(a):
    return torch.from_numpy(np.ascontiguousarray(R.f64(a)))


@pytest.mark.parametrize('C', [32, 160, 640])
def test_layernorm_ref(C):
    g = torch.Generator().manual_seed(C)
    x = scaled(g, 50, C) + 1e3 * torch.randn(50, 1, generator=g)
    x[3] = 7.0                                                     # constant row
    w, b = torch.randn(C, generator=g), torch.randn(C, generator=g)
    y, mu, rstd = R.ln_fwd(x, w, b, 1e-6)
    assert close(y, F.layer_norm(x.double(), (C,), w.double(), b.double(), 1e-6))
    by, bm, br = R.ln_fwd_bound(x, w, b, 1e-6, C // 32 + 5)
    y32 = F.layer_norm(x, (C,), w, b, 1e-6)
    assert R.ratio(y32, y, by) <= 1
    # backward against autograd
    xr = x.double().requires_grad_(True)
    wr, br_ = w.double().requires_grad_(True), b.double().requires_grad_(True)
    dy = scaled(g, 50, C)
    F.layer_norm(xr, (C,), wr, br_, 1e-6).backward(dy.double())
    dx, dw, db = R.ln_bwd(dy, x, mu, rstd, w)
    assert close(dx, xr.grad, 1e-9) and close(dw, wr.grad) and close(db, br_.grad)   # 1e-9: constant row, rstd = 1e3
    # torch's fp32 layer_norm backward recomputes its own statistics, which differ from any given fp32 (mean, rstd) by
    # roundings that rstd = 1e3 amplifies, so it is not comparable; the same formula in torch fp32 ops on the given
    # statistics is
    m32 = x.mean(1)
    r32 = torch.rsqrt(((x - m32[:, None]) ** 2).mean(1) + 1e-6)
    xh = (x - m32[:, None]) * r32[:, None]
    gg = dy * w
    dx32 = r32[:, None] * (gg - gg.mean(1, keepdim=True) - xh * (gg * xh).mean(1, keepdim=True))
    dx64, dw64, db64 = R.ln_bwd(dy, x, m32, r32, w)
    bdx, bdw, bdb = R.ln_bwd_bound(dy, x, m32, r32, w, C // 32 + 5, 50 + 8 + 1)
    assert R.ratio(dx32, dx64, bdx) <= 1
    assert R.ratio((dy * xh).sum(0), dw64, bdw) <= 1 and R.ratio(dy.sum(0), db64, bdb) <= 1


def test_stem_ref():
    g = torch.Generator().manual_seed(1)
    x = scaled(g, 2, 3, 12, 20)
    w = torch.randn(64, 3, 4, 4, generator=g)
    b = torch.randn(64, generator=g)
    wt = w.reshape(64, -1).t()
    u = R.stem_conv(x, wt, b, 4)
    ref = F.conv2d(x.double(), w.double(), b.double(), stride=4).permute(0, 2, 3, 1).reshape(-1, 64)
    assert close(u, ref)
    u32 = F.conv2d(x, w, b, stride=4).permute(0, 2, 3, 1).reshape(-1, 64)
    assert R.ratio(u32, u, R.stem_conv_bound(x, wt, b, 4)) <= 1
    du = torch.randn(u.shape[0], 64, generator=g, dtype=torch.float64)
    xr, wr, br = x.double().requires_grad_(True), w.double().requires_grad_(True), b.double().requires_grad_(True)
    F.conv2d(xr, wr, br, stride=4).permute(0, 2, 3, 1).reshape(-1, 64).backward(du)
    dwt, db = R.stem_wgrad(x, du, 4)
    assert close(dwt, wr.grad.reshape(64, -1).t()) and close(db, br.grad)


@pytest.mark.parametrize('ks,dil', [(7, 1), (3, 1), (5, 1), (7, 3)])
def test_dwconv_ref(ks, dil):
    g = torch.Generator().manual_seed(ks + dil)
    N, H, W, C = 2, 9, 4, 8
    x = scaled(g, N, H, W, C)
    w = torch.randn(C, 1, ks, ks, generator=g)
    b = torch.randn(C, generator=g)
    res = torch.randn(N, H, W, C, generator=g)
    wt = w.reshape(C, ks * ks).t()
    pad = dil * (ks // 2)
    xr = x.permute(0, 3, 1, 2).double().requires_grad_(True)
    wr, br = w.double().requires_grad_(True), b.double().requires_grad_(True)
    ref = F.conv2d(xr, wr, br, padding=pad, dilation=dil, groups=C)
    assert close(R.dwconv(x, wt, b, res, ks, dil), ref.permute(0, 2, 3, 1) + res.double())
    y32 = F.conv2d(x.permute(0, 3, 1, 2), w, b, padding=pad, dilation=dil, groups=C).permute(0, 2, 3, 1) + res
    assert R.ratio(y32, R.dwconv(x, wt, b, res, ks, dil), R.dwconv_bound(x, wt, b, res, ks, dil)) <= 1
    dy = scaled(g, N, H, W, C)
    ref.backward(dy.permute(0, 3, 1, 2).double())
    assert close(R.dwconv(dy, R.flip_taps(wt, ks), None, None, ks, dil), xr.grad.permute(0, 2, 3, 1))
    dwt, db = R.dwconv_wgrad(x, dy, ks, dil)
    assert close(dwt, wr.grad.reshape(C, -1).t()) and close(db, br.grad)


@pytest.mark.parametrize('d_over_sigma', [0, 1, 4, 16])
def test_batchnorm_ref(d_over_sigma):
    g = torch.Generator().manual_seed(d_over_sigma)
    rows, C = 3000, 12
    sig = torch.exp2(torch.randint(-8, 9, (C,), generator=g).double())
    mu = 256 * sig * torch.where(torch.rand(C, generator=g) < 0.5, -1.0, 1.0)
    x = (mu + sig * torch.randn(rows, C, generator=g, dtype=torch.float64)).float()
    w, b = torch.randn(C, generator=g), torch.randn(C, generator=g)
    xb = x.double()
    rm = (xb.mean(0) - d_over_sigma * xb.std(0, unbiased=False)).float()
    y, m, v = R.bn_fwd(x, w, b, 1e-5)
    assert close(y, F.batch_norm(xb, None, None, w.double(), b.double(), training=True, eps=1e-5), 1e-10)
    assert close(m, xb.mean(0)) and close(v, xb.var(0, unbiased=False), 1e-10)
    n_c = R.colstat_n(rows, C, 132)[0]
    by, em, rel_r = R.bn_fwd_bound(x, w, b, 1e-5, rm, n_c)
    y32 = F.batch_norm(x, None, None, w, b, training=True, eps=1e-5)
    assert R.ratio(y32, y, by) <= 1
    xr, wr, br = xb.clone().requires_grad_(True), w.double().requires_grad_(True), b.double().requires_grad_(True)
    dy = torch.randn(rows, C, generator=g)
    F.batch_norm(xr, None, None, wr, br, training=True, eps=1e-5).backward(dy.double())
    dx, xh, rstd = R.bn_bwd(dy, x, w, 1e-5, True)
    assert close(dx, xr.grad, 1e-10)
    assert close((R.f64(dy) * xh).sum(0), wr.grad, 1e-10) and close(R.f64(dy).sum(0), br.grad)
    x32, w32, b32 = x.clone().requires_grad_(True), w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    F.batch_norm(x32, None, None, w32, b32, training=True, eps=1e-5).backward(dy)
    assert R.ratio(x32.grad, dx, R.bn_bwd_bound(dy, x, w, 1e-5, em, rel_r, n_c, True, xh, rstd)) <= 1


def test_colstat_affine_ref():
    g = torch.Generator().manual_seed(3)
    x, y = scaled(g, 100, 12), scaled(g, 100, 12)
    sh1, sh2, sc2 = torch.randn(12, generator=g), torch.randn(12, generator=g), torch.rand(12, generator=g)
    s1, s2 = R.colstat(x, sh1, y, sh2, sc2)
    xd, yd = x.double() - sh1.double(), (y.double() - sh2.double()) * sc2.double()
    assert close(s1, xd.sum(0)) and close(s2, (xd * yd).sum(0))
    out, _ = R.affine(x, sh1, y, sc2, sh2, x)
    assert close(out, x.double() * sh1.double() + y.double() * sc2.double() + sh2.double() + x.double())


def test_lsk_ref():
    g = torch.Generator().manual_seed(4)
    T, Ch = 40, 36
    a1 = torch.randint(-3, 4, (T, Ch), generator=g).float()      # small integers: many exact ties
    a2 = torch.randint(-3, 4, (T, Ch), generator=g).float()
    agg, am = R.lsk_agg(a1, a2)
    cat = torch.cat([a1, a2], 1).double()
    mx, idx = cat.max(1)
    assert close(agg[:, 0], cat.mean(1)) and close(agg[:, 1], mx)
    assert np.array_equal(am, idx.numpy())                       # torch's max(dim): the first maximal index
    # conv_squeeze (2 -> 2, 7x7, pad 3) and sigmoid against F.conv2d / torch.sigmoid
    N, H, W = 2, 5, 9
    x = scaled(g, N, H, W, 2)
    w = torch.randn(2, 2, 7, 7, generator=g) * 4
    b = torch.randn(2, generator=g)
    s, z, za = R.conv7_c2(x, w, b, N, H, W, 1)
    zr = F.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), b.double(), padding=3).permute(0, 2, 3, 1).reshape(-1, 2)
    assert close(z, zr) and close(s, torch.sigmoid(zr))
    s32 = torch.sigmoid(F.conv2d(x.permute(0, 3, 1, 2), w, b, padding=3).permute(0, 2, 3, 1).reshape(-1, 2))
    assert R.ratio(s32, s, R.conv7_c2_bound(z, za, 1)) <= 1
    dpre = torch.randn(N * H * W, 2, generator=g, dtype=torch.float64)
    xr, wr, br = x.double().requires_grad_(True), w.double().requires_grad_(True), b.double().requires_grad_(True)
    F.conv2d(xr.permute(0, 3, 1, 2), wr, br, padding=3).permute(0, 2, 3, 1).reshape(-1, 2).backward(dpre)
    dw, db = R.conv7_c2_wgrad(x, dpre, N, H, W)
    assert close(dw, wr.grad.reshape(-1)) and close(db, br.grad)


@pytest.mark.parametrize('nchw', [True, False])
@pytest.mark.parametrize('ks,stride,pad', [(7, 4, 3), (3, 2, 1)])
def test_im2col_col2im_ref(nchw, ks, stride, pad):
    g = torch.Generator().manual_seed(ks)
    N, H, W, Cin = 2, 13, 11, 4
    x = torch.randn(N, Cin, H, W, generator=g) if nchw else torch.randn(N, H, W, Cin, generator=g)
    Kp = ks * ks * Cin + 4
    col, Ho, Wo = R.im2col(x, N, H, W, Cin, ks, stride, pad, Kp, nchw)
    xn = x if nchw else x.permute(0, 3, 1, 2)
    un = F.unfold(xn.double(), ks, padding=pad, stride=stride)       # [N, Cin*ks*ks (ci, kh, kw), L]
    un = un.view(N, Cin, ks * ks, -1).permute(0, 3, 2, 1).reshape(N * Ho * Wo, ks * ks * Cin)
    assert np.array_equal(col[:, :ks * ks * Cin], un.numpy()) and not col[:, ks * ks * Cin:].any()
    dcol = torch.randn(N * Ho * Wo, Kp, generator=g)
    dc = dcol[:, :ks * ks * Cin].double().view(N, Ho * Wo, ks * ks, Cin).permute(0, 3, 2, 1).reshape(N, -1, Ho * Wo)
    folded = F.fold(dc, (H, W), ks, padding=pad, stride=stride)
    ref = R.col2im(dcol, N, H, W, Cin, ks, stride, pad, Kp, nchw)
    assert close(ref, folded if nchw else folded.permute(0, 2, 3, 1))
    fp = R.col2im_fp32(dcol, N, H, W, Cin, ks, stride, pad, Kp, nchw)
    assert np.abs(fp - ref).max() <= 8 * R.U * np.abs(ref).max() + 1e-30


def test_upsample_ref():
    g = torch.Generator().manual_seed(5)
    for H, h in ((25, 13), (13, 7), (7, 4), (16, 8)):
        b = torch.randn(2, h, h + 1, 3, generator=g, dtype=torch.float64)
        W = 2 * h + 3
        ref = F.interpolate(b.permute(0, 3, 1, 2), size=(H, W), mode='nearest').permute(0, 2, 3, 1)
        assert np.array_equal(R.upsample(b.numpy(), H, W), ref.numpy()), (H, h)
        d = torch.randn(2, H, W, 3, generator=g, dtype=torch.float64).requires_grad_(True)
        br = b.clone().requires_grad_(True)
        F.interpolate(br.permute(0, 3, 1, 2), size=(H, W), mode='nearest').permute(0, 2, 3, 1).backward(d)
        assert close(R.upsample_add_bwd(d.detach(), h, h + 1), br.grad)


def test_dropout_reimplementation():
    n = 4 * 50000 + 4 * 3
    for p in (0.1, 0.5):
        keep = R.dropout_mask(n, p, 1234)
        sd = np.sqrt(n * p * (1 - p))
        assert abs(keep.sum() - n * (1 - p)) < 5 * sd
    a, b = R.dropout_mask(n, 0.5, 1), R.dropout_mask(n, 0.5, 2)
    assert 0.4 < (a != b).mean() < 0.6                              # differs across seeds
    assert 0.4 < (a[:n // 2] != a[n // 2:]).mean() < 0.6             # depends on the element index
    assert R.dropout_mask(n, 0.0, 7).all()
    x = np.ones(8, np.float32)
    _, scale = R.dropout_params(0.1)
    assert set(np.unique(R.dropout_fp32(x, 0.1, 9))) <= {np.float32(0.0), scale}
