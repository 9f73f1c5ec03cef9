"""Float64 references and per-element error bounds for the SIMT (CUDA-core fp32) kernels: LayerNorm and the stem
(csrc/norm.cu), the depthwise convolutions (csrc/stencil.cu, csrc/lsk.cu), BatchNorm statistics and `affine`, the LSK
spatial selection, im2col / col2im and dropout (csrc/lsk.cu), the FPN helpers (csrc/neck.cu) and `scale_rows`
(csrc/reduce.cu).

Needs numpy only, so the CPU suite checks it without a GPU (tests/test_simt_ref.py).

Every reference takes the fp32 values the kernel is given and computes in float64.  Where a kernel only moves data, or
rounds in a fixed order without fused multiply-adds, the `*_fp32` functions reproduce its result bit for bit.

Bound rule (as for the GEMM): |got - ref| <= n * u * sum|terms|, u = 2^-24, where n is the longest chain of roundings
the kernel performs for that output: sequential terms per thread, then the shuffle or shared-memory reduction steps,
then the atomic adds into it (the output's initial value counts as one more term).  Each `n_*` helper reads n from the
launcher's arithmetic; the wgrads use the per-thread chain, never the total pixel count.  Operations built on
divisions, square roots or exponentials have bounds derived from their parts, written out in each docstring.
"""

import numpy as np

U = 2.0 ** -24          # unit roundoff of fp32
TINY = 2.0 ** -126      # smallest normal fp32: absolute slack where expf over/underflows


def f64(t):
    if hasattr(t, 'detach'):
        t = t.detach().cpu().numpy()
    return np.asarray(t, dtype=np.float64)


def f32(t):
    if hasattr(t, 'detach'):
        t = t.detach().cpu().numpy()
    return np.asarray(t, dtype=np.float32)


def ratio(got, ref, bound):
    """max |got - ref| / bound (0 where both error and bound are 0; inf where only the bound is)."""
    err = np.abs(f64(got) - f64(ref))
    b = np.broadcast_to(f64(bound), err.shape)
    with np.errstate(divide='ignore', invalid='ignore'):
        r = np.where(err == 0, 0.0, err / b)
    return float(r.max()) if r.size else 0.0


def chain(n, terms):
    """n * u * terms (terms = sum of |terms| of each output)."""
    return n * U * f64(terms)


# ---- LayerNorm (norm.cu: ln_fwd_kernel, ln_fwd_nchw_kernel, ln_fwd_img_kernel, ln_bwd_kernel, ln_bwd_nchw_kernel) ---
def ln_fwd(x, w, b, eps):
    """(y, mean, rstd) of F.layer_norm over the last axis of x [T, C], biased variance."""
    x = f64(x)
    mu = x.mean(1)
    var = ((x - mu[:, None]) ** 2).mean(1)
    rstd = 1.0 / np.sqrt(var + eps)
    y = (x - mu[:, None]) * rstd[:, None] * f64(w) + f64(b)
    return y, mu, rstd


def ln_fwd_bound(x, w, b, eps, n_red, ex=None):
    """Per-element bounds (y, mean, rstd) of the two-pass fp32 LayerNorm of the kernels.

    The kernels sum the row in a chain of n_red = V + 5 roundings (V = C/32 per lane, then 5 shuffle steps) and divide
    by C: the fp32 mean errs by em <= (n_red + 1) u S, S = sum|x| / C.  The second pass squares d = fl(x - mean_f);
    sum (x - mean_f)^2 / C = var + (mu - mean_f)^2, so the fp32 variance lies within
        ev = (var + em^2) (n_red + 4) u + em^2 + u eps
    of var (3 roundings per term, the chain, the division, + eps).  rstd = rsqrtf(.) (<= 2 ulp, 4u) then errs by
        rel_r <= ev / (2 (var + eps)) + 5u       (1 - (1 + a)^-1/2 <= a / 2 for a >= 0).
    y = ((x - mean_f) rstd_f) w + b:
        |dy| <= |w| rstd (em + ex_mean + ex + u |x - mu|) (1 + rel_r) + |xhat w| (rel_r + 3u) + u |y|.
    For a constant row var = 0, rstd = eps^-1/2, and the bound keeps the amplified |w| eps^-1/2 em term: an fp32 mean one
    rounding away from the row value moves y by about 10^3 of that rounding.
    `ex` is an optional per-element absolute error of x itself (the stem's convolution), which moves the mean by its
    row mean and the variance by 2 mean(|x - mu| ex) + mean(ex)^2.
    """
    x, w, b = f64(x), f64(w), f64(b)
    C = x.shape[1]
    y, mu, rstd = ln_fwd(x, w, b, eps)
    var = 1.0 / rstd ** 2 - eps
    em = (n_red + 1) * U * np.abs(x).sum(1) / C
    ex = np.zeros_like(x) if ex is None else f64(ex)
    exm = ex.mean(1)
    ev = (var + em ** 2) * (n_red + 4) * U + em ** 2 + U * eps
    ev = ev + 2 * (np.abs(x - mu[:, None]) * ex).mean(1) + exm ** 2 + 2 * em * exm
    rel_r = ev / (2 * (var + eps)) + 5 * U
    xh = (x - mu[:, None]) * rstd[:, None]
    by = (np.abs(w) * (rstd * (em + exm) * (1 + rel_r))[:, None]
          + np.abs(w) * rstd[:, None] * (ex + U * np.abs(x - mu[:, None])) * (1 + rel_r)[:, None]
          + np.abs(xh * w) * (rel_r[:, None] + 3 * U) + U * np.abs(y))
    return by * (1 + 16 * U), em + exm, rel_r * rstd


def ln_bwd(dy, x, mean, rstd, w):
    """(dx, dw, db) of LayerNorm given the saved (fp32) statistics: xhat = (x - mean) rstd, g = dy w,
    dx = rstd (g - mean_c g - xhat mean_c(g xhat)), dw = sum_t dy xhat, db = sum_t dy."""
    dy, x, w = f64(dy), f64(x), f64(w)
    mean, rstd = f64(mean)[:, None], f64(rstd)[:, None]
    C = x.shape[1]
    xh = (x - mean) * rstd
    g = dy * w
    dx = rstd * (g - g.mean(1, keepdims=True) - xh * (g * xh).mean(1, keepdims=True))
    return dx, (dy * xh).sum(0), dy.sum(0)


def ln_bwd_bound(dy, x, mean, rstd, w, n_red, n_param, dx0=None, dw0=None, db0=None):
    """Bounds of ln_bwd_token: xhat = fl(fl(x - mean) rstd) errs by 2u|xhat|, g = fl(dy w) by u|g|; s1 = mean(g) and
    s2 = mean(g xhat) are chains of n_red = V + 5 (+1 for / C, +2 for xhat in s2);
        |d dx| <= rstd ((n_red + 4) u (|g| + mean|g| + |xhat| mean|g xhat|)) + u |dx0| (dx_accumulate adds one rounding).
    dw and db are per-warp fmaf chains of tokens_per_warp (4 per warp in the NCHW kernel, times its chunks), the 8-warp
    shared-memory sum and one atomic per block: n_param = that chain length; dw also carries xhat's 2u.
    """
    dy, x, w = f64(dy), f64(x), f64(w)
    mean, rstd = f64(mean)[:, None], f64(rstd)[:, None]
    xh = np.abs((x - mean) * rstd)
    g = np.abs(dy * w)
    bdx = rstd * (n_red + 4) * U * (g + g.mean(1, keepdims=True) + xh * (g * xh).mean(1, keepdims=True))
    dx, dw, db = ln_bwd(dy, x, mean[:, 0], rstd[:, 0], w)
    if dx0 is not None:
        bdx = bdx + U * np.abs(dx + f64(dx0))
    bdw = (n_param + 3) * U * ((np.abs(dy) * xh).sum(0) + (0 if dw0 is None else np.abs(f64(dw0))))
    bdb = (n_param + 1) * U * (np.abs(dy).sum(0) + (0 if db0 is None else np.abs(f64(db0))))
    return bdx, bdw, bdb


def ln_bwd_schedule(T, C, nchw, sms):
    """(tokens_per_warp or chunks_per_block, blocks) that layernorm_bwd launches (norm.cu)."""
    V = C // 32
    target = sms * (64 if V <= 6 else 32 if V <= 12 else 16) * 2
    if nchw:
        chunks = -(-T // 32)
        cpb = max(1, -(-(chunks * 8) // target))
        return cpb, -(-chunks // cpb)
    tpw = max(2, -(-T // target))
    return tpw, -(-(-(-T // tpw)) // 8)


def to_patch2(y, N, H, W):
    """[N*H*W, C] NHWC tokens -> the LN_PATCH2 layout [N*H/2*W/2, 4C] (column block (h%2)*2 + w%2)."""
    C = y.shape[-1]
    return y.reshape(N, H // 2, 2, W // 2, 2, C).transpose(0, 1, 3, 2, 4, 5).reshape(-1, 4 * C)


def to_nchw(y, N, H, W):
    return y.reshape(N, H, W, -1).transpose(0, 3, 1, 2)


# ---- stem: 4x4/s4 conv (NCHW in) + LayerNorm (stem_fwd_kernel), and stem_wgrad_kernel ---------------------------------
def patches(x, ps):
    """x [N, Cin, H, W] -> [N*Ho*Wo, Cin*ps*ps] with k = (c, i, j), the stem's patch order."""
    x = f64(x)
    N, Cin, H, W = x.shape
    Ho, Wo = H // ps, W // ps
    p = x[:, :, :Ho * ps, :Wo * ps].reshape(N, Cin, Ho, ps, Wo, ps).transpose(0, 2, 4, 1, 3, 5)
    return p.reshape(N * Ho * Wo, Cin * ps * ps)


def stem_conv(x, wt, bias, ps):
    """u [P, C0] = patches @ wt + bias (wt = [K, C0])."""
    return patches(x, ps) @ f64(wt) + f64(bias)


def stem_conv_bound(x, wt, bias, ps):
    """The kernel's fmaf chain starts from the bias and adds K = Cin ps^2 products: n = K + 1."""
    P = patches(np.abs(f64(x)), ps)
    return chain(P.shape[1] + 1, P @ np.abs(f64(wt)) + np.abs(f64(bias)))


def stem_wgrad(x, du, ps):
    """(dWt [K, C0], dbias [C0]) = (patches^T du, sum du)."""
    P = patches(x, ps)
    du = f64(du)
    return P.T @ du, du.sum(0)


def stem_wgrad_n(P, sms):
    """Chain of stem_wgrad_kernel: per 32-pixel chunk a 32-term fmaf chain added to the block's accumulator
    (ppb / 32 chunks), then one atomic per block (+ the initial value)."""
    blocks = sms * 2
    ppb = -(-P // blocks)
    ppb = -(-ppb // 32) * 32
    blocks = -(-P // ppb)
    return 32 + ppb // 32 + blocks + 1, ppb, blocks


# ---- depthwise convolutions (dwconv7_*, dwconv_* with KS x KS taps, dilation DIL, "same" padding) ---------------------
def dwconv(x, wt, bias=None, resid=None, ks=7, dil=1):
    """y[n,h,w,c] = bias[c] + sum_{i,j} x[n, h+i*dil-R, w+j*dil-R, c] wt[i*ks+j, c] (+ resid), R = dil (ks // 2)."""
    x, wt = f64(x), f64(wt)
    N, H, W, C = x.shape
    R = dil * (ks // 2)
    xp = np.zeros((N, H + 2 * R, W + 2 * R, C))
    xp[:, R:R + H, R:R + W] = x
    y = np.zeros_like(x)
    for i in range(ks):
        for j in range(ks):
            y += xp[:, i * dil:i * dil + H, j * dil:j * dil + W] * wt[i * ks + j]
    if bias is not None:
        y += f64(bias)
    if resid is not None:
        y += f64(resid)
    return y


def dwconv_bound(x, wt, bias=None, resid=None, ks=7, dil=1):
    """fmaf chain from the bias over ks^2 taps, then the residual add: n = ks^2 + 2."""
    ab = lambda t: None if t is None else np.abs(f64(t))
    return chain(ks * ks + 2, dwconv(ab(x), ab(wt), ab(bias), ab(resid), ks, dil))


def flip_taps(wt, ks):
    """Taps of the dgrad convolution: dx = dwconv(dy, flip_taps(wt))."""
    wt = f64(wt)
    return wt.reshape(ks, ks, -1)[::-1, ::-1].reshape(ks * ks, -1)


def dwconv_wgrad(x, dy, ks=7, dil=1):
    """(dwt [ks^2, C], dbias [C]): dwt[i*ks+j, c] = sum_{n,h,w} x[n, h+i*dil-R, w+j*dil-R, c] dy[n,h,w,c]."""
    x, dy = f64(x), f64(dy)
    N, H, W, C = x.shape
    R = dil * (ks // 2)
    xp = np.zeros((N, H + 2 * R, W + 2 * R, C))
    xp[:, R:R + H, R:R + W] = x
    dwt = np.zeros((ks * ks, C))
    for i in range(ks):
        for j in range(ks):
            dwt[i * ks + j] = (xp[:, i * dil:i * dil + H, j * dil:j * dil + W] * dy).sum((0, 1, 2))
    return dwt, dy.sum((0, 1, 2))


def dwconv_wgrad_bound(x, dy, n, ks=7, dil=1, dwt0=None, db0=None):
    a, b = dwconv_wgrad(np.abs(f64(x)), np.abs(f64(dy)), ks, dil)
    if dwt0 is not None:
        a, b = a + np.abs(f64(dwt0)), b + np.abs(f64(db0))
    return chain(n, a), chain(n, b)


def dw_tile_wgrad_n(N, H, W, C, sms, rows_per_warp, warps):
    """Chain of the tiled wgrads (dwconv7_wgrad_tile_kernel: 16 half-warps of one row each; dwconv_wgrad_tile_kernel:
    8 warps of two rows each): 16 columns x rows_per_warp per tile, tiles_per_block tiles, the `warps`-way shared-memory
    sum, then one atomic per block of the channel chunk (+ the initial value).  Returns (n, bpc, tiles)."""
    tiles = N * -(-H // 16) * -(-W // 16)
    chunks = C // 32
    bpc = max(1, min(tiles, -(-(sms * 2) // chunks)))
    per_block = -(-tiles // bpc)
    return 16 * rows_per_warp * per_block + warps + bpc + 1, bpc, tiles


def dw7_generic_wgrad_n(N, H, W, C, sms):
    """Chain of dwconv7_wgrad_kernel: rows_per_band x W fmafs per thread, one atomic per (image, band) block.
    Returns (n, bands_per_img, rows_per_band)."""
    gy = -(-(C // 4) // 32)
    want = max(1, sms * 4 // gy)
    bands = max(1, min(H, -(-want // N)))
    rpb = -(-H // bands)
    bands = -(-H // rpb)
    return rpb * W + N * bands + 1, bands, rpb


# ---- BatchNorm: colstat (one pass, shifted by the running mean) + affine, and its backward -----------------------------
def colstat(x, sh1=None, y=None, sh2=None, sc2=None):
    """(s1, s2): s1 = sum_r (x - sh1), s2 = sum_r (x - sh1) * (y ? (y - sh2) sc2 : (x - sh1))."""
    v = f64(x) - (0 if sh1 is None else f64(sh1))
    u = v if y is None else (f64(y) - (0 if sh2 is None else f64(sh2))) * (1 if sc2 is None else f64(sc2))
    return v.sum(0), (v * u).sum(0)


def colstat_n(rows, C, sms):
    """Chain of colstat_kernel: ceil(rows_per_block / 8) per thread, the 8-row-lane shared sum, one atomic per row
    chunk (+ the initial value), + 3 for forming x - sh1 and (y - sh2) sc2.  Returns (n, row chunks, rows per block)."""
    gx = -(-(C // 4) // 32)
    gy = max(1, sms * 8 // gx)
    rpb = max(32, -(-rows // gy))
    gy = -(-rows // rpb)
    return -(-rpb // 8) + 8 + gy + 1 + 3, gy, rpb


def colstat_bound(x, n, sh1=None, y=None, sh2=None, sc2=None, s0=(0, 0)):
    ab = lambda t: None if t is None else np.abs(f64(t))
    a1 = np.abs(f64(x) - (0 if sh1 is None else f64(sh1))).sum(0)
    u = None if y is None else np.abs((f64(y) - (0 if sh2 is None else f64(sh2))) * (1 if sc2 is None else f64(sc2)))
    a2 = (np.abs(f64(x) - (0 if sh1 is None else f64(sh1))) * (np.abs(f64(x) - (0 if sh1 is None else f64(sh1)))
                                                                if u is None else u)).sum(0)
    return chain(n, a1 + np.abs(f64(s0[0]))), chain(n, a2 + np.abs(f64(s0[1])))


def affine(x1, a1=None, x2=None, a2=None, b=None, add=None):
    """out = a1 x1 + a2 x2 + b + add (None operands skipped; a1 None = 1); also sum|terms|."""
    t = [f64(x1) * (1 if a1 is None else f64(a1))]
    if x2 is not None:
        t.append(f64(x2) * f64(a2))
    if b is not None:
        t.append(np.broadcast_to(f64(b), t[0].shape))
    if add is not None:
        t.append(f64(add))
    return sum(t), sum(np.abs(v) for v in t)


AFFINE_N = 4      # a1 x1, fmaf(x2, a2, .), + b, + add: one rounding each


def bn_fwd(x, w, b, eps):
    """Training-mode BatchNorm over the rows of x [rows, C]: (y, mean, biased var)."""
    x = f64(x)
    mu = x.mean(0)
    var = ((x - mu) ** 2).mean(0)
    return (x - mu) / np.sqrt(var + eps) * f64(w) + f64(b), mu, var


def bn_fwd_bound(x, w, b, eps, running_mean, n_c):
    """Bound of BatchNormFn.forward in training mode (per element), and the (mean, rstd) errors it implies.

    colstat sums v = fl(x - rm) (rm = running mean) in chains of n_c:  d = s1 / n errs by ed <= (n_c + 2) u mean|v|,
    s2 / n = sigma^2 + d^2 by (n_c + 4) u (sigma^2 + d^2).  var = s2 / n - d^2 (torch fp32) therefore errs by
        |dvar| <= (n_c + 6) u sigma^2 (1 + (d / sigma)^2) + 2 |d| ed + ed^2,
    the (d / sigma)^2 factor being the cancellation of the one-pass formula (d = batch mean - running mean).
    mean = rm + d errs by ed + u |mean|; rstd = rsqrt(var + eps) by rel_r <= |dvar| / (2 (var + eps)) + 5u.
    scale = w rstd, shift = b - mean scale, y = fl(fl(x scale) + shift) (affine_kernel):
        |dy| <= |x w rstd| (rel_r + 3u) + |mean w rstd| (rel_r + 4u) + |w| rstd (ed + u |mean|) + u (|b| + |y|).
    The |x w rstd| and |mean w rstd| terms are the cancellation of x scale + shift when |mean| >> sigma; torch's CPU
    BatchNorm uses the same scale / shift form.
    """
    x, w, b, rm = f64(x), f64(w), f64(b), f64(running_mean)
    y, mu, var = bn_fwd(x, w, b, eps)
    d = mu - rm
    v = x - rm
    ed = (n_c + 2) * U * np.abs(v).mean(0)
    dvar = (n_c + 6) * U * (var + d * d) + 2 * np.abs(d) * ed + ed * ed
    rstd = 1.0 / np.sqrt(var + eps)
    rel_r = dvar / (2 * (var + eps)) + 5 * U
    em = ed + U * np.abs(mu)
    by = (np.abs(x * w * rstd) * (rel_r + 3 * U) + np.abs(mu * w * rstd) * (rel_r + 4 * U)
          + np.abs(w) * rstd * em + U * (np.abs(b) + np.abs(y)))
    return by * (1 + 16 * U), em, rel_r


def bn_bwd(dy, x, w, eps, train, running_var=None):
    """(dx, dw, db) of BatchNorm.  train: batch statistics of x; eval: rstd from the running variance and the
    running mean is irrelevant to dx."""
    dy, x, w = f64(dy), f64(x), f64(w)
    n = x.shape[0]
    if train:
        mu = x.mean(0)
        rstd = 1.0 / np.sqrt(((x - mu) ** 2).mean(0) + eps)
        xh = (x - mu) * rstd
        dx = w * rstd * (dy - dy.mean(0) - xh * (dy * xh).mean(0))
    else:
        rstd = 1.0 / np.sqrt(f64(running_var) + eps)
        dx = dy * w * rstd
        xh = None
    return dx, xh, rstd


def bn_bwd_bound(dy, x, w, eps, mean_err, rstd_rel, n_c, train, xh, rstd):
    """Bound of BatchNormFn.backward.  It uses the forward's fp32 mean and rstd (errors mean_err, rstd_rel from
    bn_fwd_bound), so xhat = (x - mean) rstd carries |d xhat| <= rstd mean_err + |xhat| rstd_rel.
    colstat forms s1 = sum dy, s2 = sum dy xhat (chains n_c); A = w rstd, Bc = -(A rstd) s2 / n,
    D = -(A s1 / n) - Bc mean, dx = fl(fl(fl(A dy) + Bc x) + D):
        |d dx| <= |A| (rstd_rel |dy - mean dy - xhat m2| + |d xhat| |m2| + (mean|dy| + |xhat| mean|dy xhat|)(n_c + 2) u
                  + (mean|dy| |d xhat|)) + (6 + ...)u (|A dy| + |Bc x| + |Bc mean| + |A s1 / n|),
    the last group being the cancellation of Bc x + D when |mean| >> sigma.  Eval: dx = fl(A dy), A = fl(w rstd) with
    rstd = rsqrt(running_var + eps): 7u |dx|.
    """
    dy, x, w = f64(dy), f64(x), f64(w)
    A = np.abs(w * rstd)
    if not train:
        return 7 * U * np.abs(dy) * A
    mu = x.mean(0)
    m1, m2 = dy.mean(0), (dy * xh).mean(0)
    dxh = rstd * mean_err + np.abs(xh) * rstd_rel
    core = np.abs(dy - m1 - xh * m2)
    Bc = A * rstd * np.abs(m2)
    b = A * (rstd_rel * core + dxh * np.abs(m2) + (np.abs(dy).mean(0) + np.abs(xh) * np.abs(dy * xh).mean(0)) * (n_c + 2) * U
             + np.abs(xh) * (np.abs(dy) * dxh).mean(0))
    b = b + 8 * U * (A * np.abs(dy) + Bc * np.abs(x) + Bc * np.abs(mu) + A * np.abs(m1))
    return b * (1 + 16 * U)


# ---- LSK selection -----------------------------------------------------------------------------------------------------
def lsk_agg(a1, a2):
    """(agg [T, 2] = (mean, max) over cat(a1, a2) channels, argmax with the lowest index on ties)."""
    a = np.concatenate([f64(a1), f64(a2)], 1)
    return np.stack([a.mean(1), a.max(1)], 1), a.argmax(1)


def lsk_agg_mean_bound(a1, a2):
    """Mean: per lane 2 ceil(Ch/32) sequential adds, 5 shuffle steps, / 2Ch: n = 2 ceil(Ch/32) + 6."""
    Ch = f64(a1).shape[1]
    return chain(2 * -(-Ch // 32) + 6, (np.abs(f64(a1)).sum(1) + np.abs(f64(a2)).sum(1)) / (2 * Ch))


def conv7_c2(x, w, b, N, H, W, act):
    """y [N*H*W, 2]: act(b[co] + sum_{ci,i,j} x[n, h+i-3, w+j-3, ci] w[co, ci, i, j]), act 1 = sigmoid.
    Also returns the pre-activation and sum|terms|."""
    x = f64(x).reshape(N, H, W, 2)
    w = f64(w).reshape(2, 2, 7, 7)
    xp = np.zeros((N, H + 6, W + 6, 2))
    xp[:, 3:3 + H, 3:3 + W] = x
    z = np.zeros((N, H, W, 2)) + (0 if b is None else f64(b))
    za = np.zeros((N, H, W, 2)) + (0 if b is None else np.abs(f64(b)))
    for i in range(7):
        for j in range(7):
            s = xp[:, i:i + H, j:j + W]                # [N, H, W, ci]
            z += s @ w[:, :, i, j].T
            za += np.abs(s) @ np.abs(w[:, :, i, j]).T
    z, za = z.reshape(-1, 2), za.reshape(-1, 2)
    return (1.0 / (1.0 + np.exp(-z)) if act else z), z, za


def conv7_c2_bound(z, za, act):
    """Pre-activation: bias + 98 fmafs, n = 99.  Sigmoid s = 1 / (1 + E), E = expf(-z) (<= 2 ulp, 4u relative):
        |ds| <= s (1 - s) (|dz| + 4u) + 2u s + TINY
    (dE moves s by s^2 E = s (1 - s) per unit relative error; 1 + E and the IEEE division round once each; TINY covers
    expf overflowing to inf and s flushing to 0 for z < -88)."""
    ez = chain(99, za)
    if not act:
        return ez
    s = 1.0 / (1.0 + np.exp(-z))
    return s * (1 - s) * (ez + 4 * U) + 2 * U * s + TINY


def conv7_c2_wgrad(x, dpre, N, H, W):
    """(dw [196] = [co, ci, i, j], db [2])."""
    x = f64(x).reshape(N, H, W, 2)
    d = f64(dpre).reshape(N, H, W, 2)
    xp = np.zeros((N, H + 6, W + 6, 2))
    xp[:, 3:3 + H, 3:3 + W] = x
    dw = np.zeros((2, 2, 7, 7))
    for i in range(7):
        for j in range(7):
            dw[:, :, i, j] = np.einsum('nhwo,nhwi->oi', d, xp[:, i:i + H, j:j + W])
    return dw.reshape(-1), d.reshape(-1, 2).sum(0)


def conv7_c2_wgrad_n(total, sms):
    """Chain of conv7_c2_wgrad_kernel: px_per_block fmafs per thread, one atomic per block.  Returns (n, blocks)."""
    blocks = sms * 8
    ppb = max(64, -(-total // blocks))
    blocks = -(-total // ppb)
    return ppb + blocks + 1, blocks


def lsk_mix(a1, a2, sig):
    """out = a1 sig[:, 0] + a2 sig[:, 1] (fmaf(a1, s0, fl(a2 s1)): n = 2) and sum|terms|."""
    a1, a2, s = f64(a1), f64(a2), f64(sig)
    t1, t2 = a1 * s[:, :1], a2 * s[:, 1:]
    return t1 + t2, np.abs(t1) + np.abs(t2)


def lsk_mix_bwd_sig(dout, a1, a2, sig):
    """dpre[t, s] = (sum_c dout a_s) sig_s (1 - sig_s), on the fp32 sig the kernel reads, and sum|terms|.  For
    sig >= 1/2 the fp32 1 - sig is exact (Sterbenz), so saturated sigmoids lose nothing here."""
    d, s = f64(dout), f64(sig)
    r = np.stack([(d * f64(a1)).sum(1), (d * f64(a2)).sum(1)], 1) * s * (1 - s)
    ra = np.stack([np.abs(d * f64(a1)).sum(1), np.abs(d * f64(a2)).sum(1)], 1) * s * np.abs(1 - s)
    return r, ra


def lsk_mix_bwd_sig_n(Ch):
    """ceil(Ch/32) fmafs per lane, 5 shuffle steps, 1 - s, two products."""
    return -(-Ch // 32) + 5 + 3


def lsk_mix_bwd_in(dout, sig, dagg, amax):
    """(da1, da2): da_s[t, c] = dout sig_s + dagg[t, 0] / (2 Ch) + (amax[t] == s Ch + c) dagg[t, 1]; and sum|terms|
    (n = 3: the division, the fmaf, the add of d(max))."""
    d, s, g = f64(dout), f64(sig), f64(dagg)
    T, Ch = d.shape
    am = np.asarray(amax).astype(np.int64)
    gm = g[:, :1] / (2 * Ch)
    outs, abss = [], []
    for k in range(2):
        hit = (am[:, None] == k * Ch + np.arange(Ch)[None, :]) * g[:, 1:]
        outs.append(d * s[:, k:k + 1] + gm + hit)
        abss.append(np.abs(d * s[:, k:k + 1]) + np.abs(gm) + np.abs(hit))
    return outs, abss


# ---- im2col / col2im (bit-exact) ---------------------------------------------------------------------------------------
def im2col(x, N, H, W, Cin, ks, stride, pad, Kp, nchw):
    """col [N*Ho*Wo, Kp]: column (kh*ks + kw)*Cin + ci = x at (ho*stride - pad + kh, wo*stride - pad + kw), zero
    outside the image and in the Kp - ks^2 Cin padding columns."""
    x = f32(x)
    xh = x.reshape(N, Cin, H, W).transpose(0, 2, 3, 1) if nchw else x.reshape(N, H, W, Cin)
    Ho, Wo = (H + 2 * pad - ks) // stride + 1, (W + 2 * pad - ks) // stride + 1
    xp = np.zeros((N, H + 2 * pad + stride * 2, W + 2 * pad + stride * 2, Cin), dtype=np.float32)
    xp[:, pad:pad + H, pad:pad + W] = xh
    col = np.zeros((N, Ho, Wo, Kp), dtype=np.float32)
    for kh in range(ks):
        for kw in range(ks):
            t = kh * ks + kw
            col[..., t * Cin:(t + 1) * Cin] = xp[:, kh:kh + (Ho - 1) * stride + 1:stride, kw:kw + (Wo - 1) * stride + 1:stride]
    return col.reshape(N * Ho * Wo, Kp), Ho, Wo


def col2im_fp32(dcol, N, H, W, Cin, ks, stride, pad, Kp, nchw):
    """col2im_kernel bit for bit: per input pixel, fp32 adds over kh, then kw, in ascending order.  Returns NHWC or NCHW."""
    Ho, Wo = (H + 2 * pad - ks) // stride + 1, (W + 2 * pad - ks) // stride + 1
    d = f32(dcol).reshape(N, Ho, Wo, Kp)
    acc = np.zeros((N, H, W, Cin), dtype=np.float32)
    hh, ww = np.arange(H), np.arange(W)
    for kh in range(ks):
        hn = hh + pad - kh
        hok = (hn >= 0) & (hn % stride == 0) & (hn // stride < Ho)
        for kw in range(ks):
            wn = ww + pad - kw
            wok = (wn >= 0) & (wn % stride == 0) & (wn // stride < Wo)
            t = kh * ks + kw
            src = np.zeros((N, H, W, Cin), dtype=np.float32)
            hi, wi = np.nonzero(hok)[0], np.nonzero(wok)[0]
            src[:, hi[:, None], wi[None, :]] = d[:, (hn[hi] // stride)[:, None], (wn[wi] // stride)[None, :], t * Cin:(t + 1) * Cin]
            m = hok[:, None] & wok[None, :]
            acc = np.where(m[None, :, :, None], acc + src, acc)
    return acc.transpose(0, 3, 1, 2) if nchw else acc


def col2im(dcol, N, H, W, Cin, ks, stride, pad, Kp, nchw):
    """float64 col2im: the adjoint of im2col (sum of every column entry that copied the pixel)."""
    Ho, Wo = (H + 2 * pad - ks) // stride + 1, (W + 2 * pad - ks) // stride + 1
    d = f64(dcol).reshape(N, Ho, Wo, Kp)
    acc = np.zeros((N, H + 2 * pad + 2 * stride, W + 2 * pad + 2 * stride, Cin))
    for kh in range(ks):
        for kw in range(ks):
            t = kh * ks + kw
            acc[:, kh:kh + (Ho - 1) * stride + 1:stride, kw:kw + (Wo - 1) * stride + 1:stride] += d[..., t * Cin:(t + 1) * Cin]
    acc = acc[:, pad:pad + H, pad:pad + W]
    return acc.transpose(0, 3, 1, 2) if nchw else acc


# ---- dropout (dropout_kernel), bit-exact in uint64 arithmetic ----------------------------------------------------------
_GOLD = np.uint64(0x9E3779B97F4A7C15)
_M1, _M2 = np.uint64(0xBF58476D1CE4E5B9), np.uint64(0x94D049BB133111EB)
_IDX, _LANE = np.uint64(0xD1342543DE82EF95), np.uint64(0x632BE59BD9B4E019)


def mix32(z):
    """splitmix64 finaliser, upper 32 bits (uint64 arrays, wrap-around arithmetic)."""
    with np.errstate(over='ignore'):
        z = z + _GOLD
        z = (z ^ (z >> np.uint64(30))) * _M1
        z = (z ^ (z >> np.uint64(27))) * _M2
        return ((z ^ (z >> np.uint64(31))) >> np.uint64(32)).astype(np.uint32)


def dropout_params(p):
    """(thresh, scale) as the launcher computes them from the fp32 p: (uint32)((double)p * 2^32), 1.0f / (1.0f - p)."""
    p32 = np.float32(p)
    return np.uint32(int(float(p32) * 4294967296.0)), np.float32(1.0) / (np.float32(1.0) - p32)


def dropout_mask(n, p, seed):
    """keep mask of n elements (n % 4 == 0): element 4i + e keeps iff mix32(seed ^ (4i * IDX) + e * LANE) >= thresh."""
    thresh, _ = dropout_params(p)
    i = np.arange(n // 4, dtype=np.uint64)
    with np.errstate(over='ignore'):
        base = np.uint64(seed) ^ (i * np.uint64(4) * _IDX)
        keep = np.stack([mix32(base + np.uint64(e) * _LANE) >= thresh for e in range(4)], 1)
    return keep.reshape(-1)


def dropout_fp32(x, p, seed):
    x = f32(x).reshape(-1)
    _, scale = dropout_params(p)
    return np.where(dropout_mask(x.size, p, seed), x * scale, np.float32(0.0)).astype(np.float32)


# ---- FPN helpers and scale_rows ----------------------------------------------------------------------------------------
def nearest_index(out_size, in_size):
    """source index of each destination index: floor(y * in / out) in integers."""
    return (np.arange(out_size) * in_size) // out_size


def upsample(b, H, W):
    """nearest upsampling of b [N, h, w, C] to [N, H, W, C]."""
    b = np.asarray(b)
    return b[:, nearest_index(H, b.shape[1])][:, :, nearest_index(W, b.shape[2])]


def upsample_add_fp32(a, b):
    a, b = f32(a), f32(b)
    return a + upsample(b, a.shape[1], a.shape[2])


def upsample_add_bwd_fp32(d, h, w):
    """upsample_add_bwd_kernel bit for bit: fp32 adds over destination rows, then columns, in ascending order."""
    d = f32(d)
    N, H, W, C = d.shape
    ys, xs = nearest_index(H, h), nearest_index(W, w)
    out = np.zeros((N, h, w, C), dtype=np.float32)
    for y in range(H):
        for x in range(W):
            out[:, ys[y], xs[x]] += d[:, y, x]
    return out


def upsample_add_bwd(d, h, w):
    d = f64(d)
    N, H, W, C = d.shape
    out = np.zeros((N, h, w, C))
    np.add.at(out, (slice(None), nearest_index(H, h)[:, None], nearest_index(W, w)[None, :]), d)
    return out


def scale_rows_fp32(x, rs=None, cs=None):
    """out = x * (rs * cs) with the scale product formed first in fp32, as scale_rows_kernel does."""
    x = f32(x)
    s = np.ones((x.shape[0], 1), np.float32) if rs is None else f32(rs)[:, None]
    m = np.ones((1, x.shape[1]), np.float32) if cs is None else f32(cs)[None, :]
    return x * (s * m)
