"""The SIMT kernels (LayerNorm, stem, depthwise convolutions, BatchNorm statistics / affine, LSK selection, im2col /
col2im, dropout, FPN helpers, scale_rows) against tests/simt_ref.py on every launch path.

All calls go straight to the C ABI.  Every output lies inside a sentinel-filled buffer and no word outside its window may
change; outputs the ABI accumulates into start from non-zero values.  Inputs carry per-channel scales 2^k, k in [-8, 8],
and mixed signs, so the per-element bounds of simt_ref bite where a max-norm tolerance would not.  Which kernel ran is
read from the profiler; schedule parameters the profiler cannot show (tokens per warp, chunks per block, persistent
tile loops, row bands) are recomputed from the launcher's formula and the SM count, and the test asserts the shape
crosses the threshold it is meant to.  Run with -s to see the worst err / bound per family.
"""
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import gemm_ref
import simt_ref as R

pytestmark = pytest.mark.gpu

WIDTHS = (1, 2, 3, 4, 5, 6, 8, 10, 12, 16, 20, 24, 32)     # SM3_V_DISPATCH: C / 32
SENT = 0x7FA11A11                                          # sentinel bit pattern (a NaN payload no kernel produces)
FRONT = 64                                                 # words of padding before every buffer (256 B)
PAD_IN = 256                                               # NaN words after every input

WORST = {}


def within(family, r):
    """r = max err / bound <= 1, remembering the worst per family (printed at the end of the module)."""
    WORST[family] = max(WORST.get(family, 0.0), r)
    return r <= 1.0


@pytest.fixture(scope='module', autouse=True)
def report_worst():
    yield
    print('\nworst err / bound:', ', '.join(f'{q} {e:.3f}' for q, e in sorted(WORST.items())))


@pytest.fixture(scope='module')
def L():
    from sm3det_b200 import _lib
    return _lib.load()


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def kernels_run(fn, tries=5):
    """(names of the CUDA kernels fn launches, fn's result).  fn allocates its own outputs, so a retry (the profiler
    occasionally records only the input copies, or no CUDA activity at all) starts from the same state."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(tries):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            res = fn()
            torch.cuda.synchronize()
        names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
        if any(not n.startswith(('Memcpy', 'Memset')) for n in names):
            break
    return names, res


def ran(names, pattern):
    return any(re.search(pattern, n) for n in names)


class Out:
    """A [shape] output window inside a sentinel-filled CUDA buffer (optionally pre-filled with `init`).  The sentinel
    tail is as long as the window, so a kernel that overruns its output by up to its own size is caught, not a fault."""

    def __init__(self, shape, init=None, dtype=torch.float32):
        self.shape = tuple(shape)
        self.n = int(np.prod(self.shape))
        words = self.n if dtype != torch.int16 else (self.n + 1) // 2
        big = torch.full((FRONT + 2 * words + FRONT,), SENT, dtype=torch.int32)
        if init is not None:
            big.view(torch.float32)[FRONT:FRONT + self.n] = torch.as_tensor(np.asarray(init, np.float32)).reshape(-1)
        self.words = words
        self.big = big.cuda()
        self.t = self.big[FRONT:FRONT + words].view(dtype)[:self.n].view(self.shape)

    def get(self, what):
        allb = self.big.cpu().numpy()
        assert np.all(allb[:FRONT] == SENT) and np.all(allb[FRONT + self.words:] == SENT), f'{what}: written outside its window'
        return self.big[FRONT:FRONT + self.words].view(self.t.dtype)[:self.n].cpu().numpy().reshape(self.shape)


def call(L, name, *args):
    from sm3det_b200 import _lib
    conv = []
    for a in args:
        if isinstance(a, Out):
            conv.append(a.t.data_ptr())
        elif torch.is_tensor(a):
            conv.append(a.data_ptr())
        else:
            conv.append(a)
    _lib.check(getattr(L, name)(*conv, torch.cuda.current_stream().cuda_stream), name)


def scaled(g, *shape, lo=-8, hi=8):
    """randn with a per-channel (last axis) scale 2^k, k in [lo, hi], and mixed signs (fp32, CPU)."""
    k = torch.randint(lo, hi + 1, (shape[-1],), generator=g).double()
    return (torch.randn(*shape, generator=g, dtype=torch.float64) * torch.exp2(k)).float()


def cu(t):
    """t on the GPU inside a NaN-filled buffer: a read past either end of an input turns the output into NaN."""
    if t is None:
        return None
    flat = t.contiguous().reshape(-1)
    big = torch.full((FRONT + flat.numel() + PAD_IN,), float('nan'), dtype=t.dtype)
    big[FRONT:FRONT + flat.numel()] = flat
    return big.cuda()[FRONT:FRONT + flat.numel()].view(t.shape)


# ---- LayerNorm forward ----------------------------------------------------------------------------------------------
def ln_input(g, T, C):
    """Per-channel scales, per-token offsets of 10^3 sigma, two constant rows."""
    x = scaled(g, T, C, lo=-4, hi=4)
    x += 1e3 * x.std() * torch.randn(T, 1, generator=g)
    x[1] = 3.0
    x[T - 2] = -1.0 / 3.0
    return x


@pytest.mark.parametrize('eps', [1e-6, 1e-5])
@pytest.mark.parametrize('V', WIDTHS)
def test_layernorm_fwd(L, V, eps):
    C = 32 * V
    g = torch.Generator().manual_seed(V)
    w, b = scaled(g, C), scaled(g, C)
    for N, H, W in ((3, 3, 5), (2, 6, 7), (1, 4, 10)):      # HW = 15 < 32; HW = 42: NCHW blocks straddle images
        T = N * H * W                                       # 45, 84, 40: not multiples of 32; (1, 4, 10) for PATCH2
        x = ln_input(g, T, C)
        y64, mu, rstd = R.ln_fwd(x, w, b, eps)
        by, bm, br = R.ln_fwd_bound(x, w, b, eps, V + 5)
        modes = [(0, y64, by, (T, C)), (2, R.to_nchw(y64, N, H, W), R.to_nchw(by, N, H, W), (N, C, H, W))]
        if H % 2 == 0 and W % 2 == 0:
            modes.append((1, R.to_patch2(y64, N, H, W), R.to_patch2(by, N, H, W), (T // 4, 4 * C)))
        for mode, ref, bnd, shape in modes:
            def run():
                y, st = Out(shape), Out((T, 2))
                call(L, 'sm3_layernorm_fwd', cu(x), cu(w), cu(b), y, st, T, C, eps, mode, H, W)
                return y, st
            names, (y, st) = kernels_run(run)
            kern = 'ln_fwd_nchw_kernel' if mode == 2 else 'ln_fwd_kernel'
            assert ran(names, rf'{kern}<{V}>'), names
            assert within('layernorm_fwd', R.ratio(y.get('y'), ref, bnd)), mode
            s = st.get('stats')
            assert within('layernorm_fwd stats', max(R.ratio(s[:, 0], mu, bm), R.ratio(s[:, 1], rstd, br))), mode


@pytest.mark.parametrize('C,T', [(32, 5), (128, 300), (160, 129), (256, 1000)])
def test_layernorm_fwd_img(L, C, T):
    g = torch.Generator().manual_seed(C + T)
    x = ln_input(g, T, C)
    w, b = scaled(g, C), scaled(g, C)
    T_pad = -(-T // 128) * 128
    elems = L.sm3_gemm_packed_act_elems(T, C, 0, 128)

    def run():
        img, y, st = Out((elems,), dtype=torch.int16), Out((T, C)), Out((T, 2))
        call(L, 'sm3_layernorm_fwd_img', cu(x), cu(w), cu(b), img, y, st, T, C, 1e-6)
        return img, y, st
    names, (img, y, st) = kernels_run(run)
    assert ran(names, rf'ln_fwd_img_kernel<{16 if C <= 128 else 32}>'), names
    y32 = y.get('y')
    by, bm, br = R.ln_fwd_bound(x, w, b, 1e-6, 8 + (4 if C <= 128 else 5))     # 8 per lane, log2(G) shuffles
    assert within('layernorm_fwd_img', R.ratio(y32, R.ln_fwd(x, w, b, 1e-6)[0], by))
    hi, lo = gemm_ref.decode_k(img.get('img'), T_pad, C)
    h_ref, l_ref = gemm_ref.split_bits(y32)
    assert np.array_equal(hi[:T], h_ref) and np.array_equal(lo[:T], l_ref)
    assert not hi[T:].any() and not lo[T:].any()            # padding rows of the last 128-row tile are zero


# ---- LayerNorm backward ---------------------------------------------------------------------------------------------
def ln_bwd_case(L, g, V, N, H, W, mode, accum, fam):
    C, T = 32 * V, N * H * W
    x = ln_input(g, T, C)
    w = scaled(g, C)
    _, mu, rstd = R.ln_fwd(x, w, w, 1e-6)
    stats = torch.from_numpy(np.stack([mu, rstd], 1).astype(np.float32))
    dy = scaled(g, T, C)
    dx0, dw0, db0 = scaled(g, T, C), scaled(g, C), scaled(g, C)
    dyl = (dy if mode == 0 else torch.from_numpy(np.ascontiguousarray(
        R.to_patch2(dy.numpy(), N, H, W) if mode == 1 else R.to_nchw(dy.numpy(), N, H, W))))
    nchw = mode == 2
    per, blocks = R.ln_bwd_schedule(T, C, nchw, sms())

    def run():
        dx = Out((T, C), init=dx0 if accum else None)
        dw, db = Out((C,), init=dw0), Out((C,), init=db0)
        call(L, 'sm3_layernorm_bwd', cu(dyl), cu(x), cu(stats), cu(w), dx, dw, db, T, C, mode, H, W, int(accum))
        return dx, dw, db
    names, (dx, dw, db) = kernels_run(run)
    assert ran(names, rf'{"ln_bwd_nchw_kernel" if nchw else "ln_bwd_kernel"}<{V}>'), names
    s = R.f64(stats)
    dx64, dw64, db64 = R.ln_bwd(dy, x, s[:, 0], s[:, 1], w)
    n_param = (4 * per if nchw else per) + 8 + blocks + 1
    bdx, bdw, bdb = R.ln_bwd_bound(dy, x, s[:, 0], s[:, 1], w, V + 5, n_param, dx0=dx0 if accum else None, dw0=dw0, db0=db0)
    want_dx = dx64 + (R.f64(dx0) if accum else 0)
    assert within(fam, R.ratio(dx.get('dx'), want_dx, bdx))
    assert within(fam + ' dw/db', max(R.ratio(dw.get('dw'), dw64 + R.f64(dw0), bdw),
                                      R.ratio(db.get('db'), db64 + R.f64(db0), bdb)))
    return per


@pytest.mark.parametrize('mode', [0, 1, 2])
@pytest.mark.parametrize('V', WIDTHS)
def test_layernorm_bwd(L, V, mode):
    g = torch.Generator().manual_seed(100 * V + mode)
    ln_bwd_case(L, g, V, 2, 6, 10, mode, accum=(V + mode) % 2 == 1, fam='layernorm_bwd')


@pytest.mark.parametrize('accum', [0, 1])
@pytest.mark.parametrize('V,nchw', [(1, False), (32, False), (1, True), (8, True)])
def test_layernorm_bwd_schedules(L, V, nchw, accum):
    """ln_bwd_kernel at more than 2 tokens per warp and ln_bwd_nchw_kernel at more than one 32-token chunk per block."""
    C = 32 * V
    wps = 64 if V <= 6 else 32 if V <= 12 else 16
    target = sms() * wps * 2
    T_min = 4 * target if nchw else 2 * target            # above this, per > 1 (chunks) / per > 2 (tokens per warp)
    H, W = 7, 17
    N = -(-(T_min + T_min // 2) // (H * W))
    per, _ = R.ln_bwd_schedule(N * H * W, C, nchw, sms())
    assert per > (1 if nchw else 2)
    g = torch.Generator().manual_seed(V + 10 * accum)
    ln_bwd_case(L, g, V, N, H, W, 2 if nchw else 0, accum=bool(accum), fam='layernorm_bwd schedules')


# ---- stem -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('V', [v for v in WIDTHS if v <= 16])
def test_stem_fwd(L, V):
    C0 = 32 * V
    g = torch.Generator().manual_seed(V)
    N, Cin, H, W = 1, 3, 4 * 5, 4 * 7                      # P = 35: one full 32-pixel block and a tail of 3
    x = scaled(g, N, Cin, H, W)
    wt, bias = scaled(g, Cin * 16, C0), scaled(g, C0)
    lnw, lnb = scaled(g, C0), scaled(g, C0)
    P = N * (H // 4) * (W // 4)
    assert P % 32 != 0

    def run():
        y, conv, st = Out((P, C0)), Out((P, C0)), Out((P, 2))
        call(L, 'sm3_stem_fwd', cu(x), cu(wt), cu(bias), cu(lnw), cu(lnb), y, conv, st, N, Cin, H, W, 4, C0, 1e-6)
        return y, conv, st
    names, (y, conv, st) = kernels_run(run)
    assert ran(names, rf'stem_fwd_kernel<{V}>'), names
    u = R.stem_conv(x, wt, bias, 4)
    eu = R.stem_conv_bound(x, wt, bias, 4)
    assert within('stem_fwd conv', R.ratio(conv.get('conv'), u, eu))
    by, bm, br = R.ln_fwd_bound(u, lnw, lnb, 1e-6, V + 5, ex=eu)
    assert within('stem_fwd', R.ratio(y.get('y'), R.ln_fwd(u, lnw, lnb, 1e-6)[0], by))
    s = st.get('stats')
    _, mu, rstd = R.ln_fwd(u, lnw, lnb, 1e-6)
    assert within('stem_fwd stats', max(R.ratio(s[:, 0], mu, bm), R.ratio(s[:, 1], rstd, br)))


@pytest.mark.parametrize('C0', [32, 160])
def test_stem_wgrad(L, C0):
    """(K + 1) C0 up to its 8192 limit (C0 = 160 at K = 48), over several 32-pixel chunks per block and many blocks."""
    g = torch.Generator().manual_seed(C0)
    N, Cin = 1, 3
    target = 2 * sms() * 32 * 2 + 5                          # > 2 chunks per block
    Ho = 61
    Wo = -(-target // Ho)
    H, W = 4 * Ho, 4 * Wo
    P = N * Ho * Wo
    n, ppb, blocks = R.stem_wgrad_n(P, sms())
    assert ppb >= 64 and blocks > 1
    x = scaled(g, N, Cin, H, W)
    du = scaled(g, P, C0)
    dw0, db0 = scaled(g, Cin * 16, C0), scaled(g, C0)

    def run():
        dwt, dbias = Out((Cin * 16, C0), init=dw0), Out((C0,), init=db0)
        call(L, 'sm3_stem_wgrad', cu(x), cu(du), dwt, dbias, N, Cin, H, W, 4, C0)
        return dwt, dbias
    names, (dwt, dbias) = kernels_run(run)
    assert ran(names, r'stem_wgrad_kernel'), names
    rw, rb = R.stem_wgrad(x, du, 4)
    aw, ab = R.stem_wgrad(np.abs(R.f64(x)), np.abs(R.f64(du)), 4)
    assert within('stem_wgrad', R.ratio(dwt.get('dwt'), rw + R.f64(dw0), R.chain(n, aw + np.abs(R.f64(dw0)))))
    assert within('stem_wgrad', R.ratio(dbias.get('db'), rb + R.f64(db0), R.chain(n, ab + np.abs(R.f64(db0)))))


# ---- dwconv7 ----------------------------------------------------------------------------------------------------------
def dw7_fwd_dgrad(L, g, N, H, W, C, kern, fam):
    x, dy = scaled(g, N, H, W, C), scaled(g, N, H, W, C)
    wt, bias, res = scaled(g, 49, C), scaled(g, C), scaled(g, N, H, W, C)
    wtf = torch.from_numpy(R.flip_taps(wt, 7).astype(np.float32))
    for inp, taps, bb, rr, what in ((x, wt, bias, None, 'fwd'), (dy, wtf, None, res, 'dgrad')):
        def run():
            y = Out((N, H, W, C))
            call(L, 'sm3_dwconv7_fwd', cu(inp), cu(taps), cu(bb), cu(rr), y, N, H, W, C)
            return y
        names, y = kernels_run(run)
        assert ran(names, kern), names
        assert within(fam, R.ratio(y.get(what), R.dwconv(inp, taps, bb, rr, 7), R.dwconv_bound(inp, taps, bb, rr, 7))), what


@pytest.mark.parametrize('N,H,W,C', [(3, 1, 1, 64), (2, 2, 17, 32), (2, 15, 33, 64), (1, 16, 16, 96), (2, 17, 2, 32),
                                     (1, 33, 15, 64), (64, 2, 2, 256)])
def test_dwconv7_tile(L, N, H, W, C):
    dw7_fwd_dgrad(L, torch.Generator().manual_seed(N + H + W + C), N, H, W, C, r'dwconv7_tile_kernel', 'dwconv7 tile')


@pytest.mark.parametrize('C', [4, 36, 100])
def test_dwconv7_generic(L, C):
    """C % 32 != 0: dwconv7_fwd_kernel / dwconv7_wgrad_kernel, the latter with several row bands of several rows."""
    g = torch.Generator().manual_seed(C)
    dw7_fwd_dgrad(L, g, 2, 9, 19, C, r'dwconv7_fwd_kernel', 'dwconv7 generic')
    want = sms() * 4 // -(-(C // 4) // 32)
    N, W = 4, 11
    H = 3 * -(-want // N) + 5                                # > want / N rows: every band holds several rows
    n, bands, rpb = R.dw7_generic_wgrad_n(N, H, W, C, sms())
    assert bands >= 2 and rpb >= 2
    wgrad_case(L, g, N, H, W, C, 7, 1, n, r'dwconv7_wgrad_kernel', 'dwconv7_wgrad generic')


def wgrad_case(L, g, N, H, W, C, ks, dil, n, kern, fam):
    x, dy = scaled(g, N, H, W, C), scaled(g, N, H, W, C)
    dw0, db0 = scaled(g, ks * ks, C), scaled(g, C)
    name = 'sm3_dwconv7_wgrad' if ks == 7 and dil == 1 else 'sm3_dwconv_wgrad'
    extra = () if name == 'sm3_dwconv7_wgrad' else (ks, dil)

    def run():
        dwt, db = Out((ks * ks, C), init=dw0), Out((C,), init=db0)
        call(L, name, cu(x), cu(dy), dwt, db, N, H, W, C, *extra)
        return dwt, db
    names, (dwt, db) = kernels_run(run)
    assert ran(names, kern), names
    rw, rb = R.dwconv_wgrad(x, dy, ks, dil)
    bw, bb = R.dwconv_wgrad_bound(x, dy, n, ks, dil, dw0, db0)
    assert within(fam, max(R.ratio(dwt.get('dwt'), rw + R.f64(dw0), bw), R.ratio(db.get('db'), rb + R.f64(db0), bb)))


@pytest.mark.parametrize('N,H,W,C', [(2, 17, 33, 64), (1, 1, 2, 32)])
def test_dwconv7_wgrad_tile(L, N, H, W, C):
    g = torch.Generator().manual_seed(H * W)
    n, bpc, tiles = R.dw_tile_wgrad_n(N, H, W, C, sms(), 1, 16)
    wgrad_case(L, g, N, H, W, C, 7, 1, n, r'dwconv7_wgrad_tile_kernel', 'dwconv7_wgrad tile')


def test_dwconv7_wgrad_tile_persistent(L):
    """More tiles than blocks per channel chunk: each block loops over several tiles."""
    C, H, W = 64, 40, 40
    bpc = -(-(sms() * 2) // (C // 32))
    N = -(-3 * bpc // 9)
    n, bpc2, tiles = R.dw_tile_wgrad_n(N, H, W, C, sms(), 1, 16)
    assert tiles > 2 * bpc2
    wgrad_case(L, torch.Generator().manual_seed(7), N, H, W, C, 7, 1, n, r'dwconv7_wgrad_tile_kernel', 'dwconv7_wgrad tile')


@pytest.mark.parametrize('C', [64, 192, 256])
def test_dwconv7_ln(L, C):
    """The fused front kernel at each strip height (C <= 64: 8 rows, <= 192: 4, > 192: 2) against float64."""
    g = torch.Generator().manual_seed(C)
    N, H, W = 2, 11, 19
    x = scaled(g, N, H, W, C)
    wt, bias, lnw, lnb = scaled(g, 49, C), scaled(g, C), scaled(g, C), scaled(g, C)
    T = N * H * W

    def run():
        u, st, v = Out((N, H, W, C)), Out((T, 2)), Out((T, C))
        call(L, 'sm3_dwconv7_ln_fwd', cu(x), cu(wt), cu(bias), cu(lnw), cu(lnb), u, st, v, None, N, H, W, C, 1e-6)
        return u, st, v
    names, (u, st, v) = kernels_run(run)
    assert ran(names, rf'front_ln_kernel<{C // 32}>'), names
    u64 = R.dwconv(x, wt, bias, None, 7)
    eu = R.dwconv_bound(x, wt, bias, None, 7)
    assert within('dwconv7_ln u', R.ratio(u.get('u'), u64, eu))
    u2, eu2 = u64.reshape(T, C), eu.reshape(T, C)
    by, bm, br = R.ln_fwd_bound(u2, lnw, lnb, 1e-6, C // 32 + 5, ex=eu2)
    y64, mu, rstd = R.ln_fwd(u2, lnw, lnb, 1e-6)
    assert within('dwconv7_ln v', R.ratio(v.get('v'), y64, by))
    s = st.get('stats')
    assert within('dwconv7_ln stats', max(R.ratio(s[:, 0], mu, bm), R.ratio(s[:, 1], rstd, br)))


# ---- generic depthwise convs (LSK) ------------------------------------------------------------------------------------
@pytest.mark.parametrize('ks,dil', [(3, 1), (5, 1), (7, 3)])
@pytest.mark.parametrize('N,H,W,C', [(2, 4, 37, 64), (1, 19, 5, 32)])
def test_dwconv(L, ks, dil, N, H, W, C):
    g = torch.Generator().manual_seed(ks * dil + H)
    kern = rf'dwconv_tile_kernel<{ks},\s*{dil}>'
    x, dy = scaled(g, N, H, W, C), scaled(g, N, H, W, C)
    wt, bias, res = scaled(g, ks * ks, C), scaled(g, C), scaled(g, N, H, W, C)
    wtf = torch.from_numpy(R.flip_taps(wt, ks).astype(np.float32))
    for inp, taps, bb, rr, what in ((x, wt, bias, None, 'fwd'), (dy, wtf, None, res, 'dgrad')):
        def run():
            y = Out((N, H, W, C))
            call(L, 'sm3_dwconv_fwd', cu(inp), cu(taps), cu(bb), cu(rr), y, N, H, W, C, ks, dil)
            return y
        names, y = kernels_run(run)
        assert ran(names, kern), names
        assert within('dwconv', R.ratio(y.get(what), R.dwconv(inp, taps, bb, rr, ks, dil),
                                        R.dwconv_bound(inp, taps, bb, rr, ks, dil))), what
    n, _, _ = R.dw_tile_wgrad_n(N, H, W, C, sms(), 2, 8)
    wgrad_case(L, g, N, H, W, C, ks, dil, n, rf'dwconv_wgrad_tile_kernel<{ks},\s*{dil}>', 'dwconv_wgrad')


@pytest.mark.parametrize('ks,dil', [(3, 1), (7, 3)])
def test_dwconv_wgrad_persistent(L, ks, dil):
    C, H, W = 64, 33, 35
    bpc = -(-(sms() * 2) // (C // 32))
    N = -(-3 * bpc // 9)
    n, bpc2, tiles = R.dw_tile_wgrad_n(N, H, W, C, sms(), 2, 8)
    assert tiles > 2 * bpc2
    wgrad_case(L, torch.Generator().manual_seed(ks), N, H, W, C, ks, dil, n,
               rf'dwconv_wgrad_tile_kernel<{ks},\s*{dil}>', 'dwconv_wgrad')


# ---- colstat / affine / mul / BatchNormFn -----------------------------------------------------------------------------
@pytest.mark.parametrize('C', [12, 260])
@pytest.mark.parametrize('rows', [7, 'many'])
def test_colstat(L, C, rows):
    g = torch.Generator().manual_seed(C)
    if rows == 'many':
        rows = 40 * 8 * sms() + 13
    n, gy, rpb = R.colstat_n(rows, C, sms())
    x, y = scaled(g, rows, C), scaled(g, rows, C)
    sh1, sh2, sc2 = scaled(g, C), scaled(g, C), scaled(g, C)
    s0 = (scaled(g, C), scaled(g, C))
    for args in ((None, None, None, None), (sh1, None, None, None), (None, y, sh2, sc2), (sh1, y, sh2, sc2)):
        def run():
            s1, s2 = Out((C,), init=s0[0]), Out((C,), init=s0[1])
            call(L, 'sm3_colstat', cu(x), cu(args[0]), cu(args[1]), cu(args[2]), cu(args[3]), s1, s2, rows, C)
            return s1, s2
        names, (s1, s2) = kernels_run(run)
        assert ran(names, 'colstat_kernel'), names
        r1, r2 = R.colstat(x, *args)
        b1, b2 = R.colstat_bound(x, n, *args, s0=s0)
        assert within('colstat', max(R.ratio(s1.get('s1'), r1 + R.f64(s0[0]), b1), R.ratio(s2.get('s2'), r2 + R.f64(s0[1]), b2)))


def test_affine_null_combinations(L):
    g = torch.Generator().manual_seed(1)
    rows, C = 37, 44
    x1, x2, add = scaled(g, rows, C), scaled(g, rows, C), scaled(g, rows, C)
    a1, a2, b = scaled(g, C), scaled(g, C), scaled(g, C)
    for m in range(16):
        A1, X2, B, AD = (a1 if m & 1 else None), (x2 if m & 2 else None), (b if m & 4 else None), (add if m & 8 else None)
        out = Out((rows, C))
        call(L, 'sm3_affine', cu(x1), cu(A1), cu(X2), cu(a2 if X2 is not None else None), cu(B), cu(AD), out, rows, C)
        ref, terms = R.affine(x1, A1, X2, a2 if X2 is not None else None, B, AD)
        assert within('affine', R.ratio(out.get('out'), ref, R.chain(R.AFFINE_N, terms))), m
    a, bb = scaled(g, rows, C), scaled(g, rows, C)
    out = Out((rows, C))
    call(L, 'sm3_mul', cu(a), cu(bb), None, out, rows * C)
    assert np.array_equal(out.get('mul'), (a * bb).numpy())                        # one IEEE product: bit-exact
    out = Out((rows, C))
    call(L, 'sm3_mul', cu(a), cu(bb), cu(add), out, rows * C)
    ref = R.f64(a) * R.f64(bb) + R.f64(add)
    assert within('mul', R.ratio(out.get('mul+add'), ref, R.chain(2, np.abs(R.f64(a) * R.f64(bb)) + np.abs(R.f64(add)))))


BN_TABLE = {}


@pytest.mark.parametrize('d_over_sigma', [0, 1, 4, 16])
def test_batchnorm_fn(d_over_sigma):
    """BatchNormFn train (one pass shifted by the running mean) and eval, with batch mean - running mean = d sigma and
    |mean| = 256 sigma; the forward error is also compared with torch's fp32 CPU BatchNorm (DESIGN.md §4)."""
    from sm3det_b200.lsk_functional import BatchNormFn
    g = torch.Generator().manual_seed(d_over_sigma)
    rows, C = 20000, 44
    sig = torch.exp2(torch.randint(-8, 9, (C,), generator=g).double())
    mu = 256 * sig * torch.where(torch.rand(C, generator=g) < 0.5, -1.0, 1.0)
    x = (mu + sig * torch.randn(rows, C, generator=g, dtype=torch.float64)).float()
    xb = x.double()
    rm = (xb.mean(0) - d_over_sigma * xb.std(0, unbiased=False)).float()
    rv = (xb.var(0) * 1.5).float()
    w, b = scaled(g, C), scaled(g, C)
    dy = scaled(g, rows, C)
    n_c, _, _ = R.colstat_n(rows, C, sms())
    for train in (True, False):
        xd = x.cuda().requires_grad_(True)
        wd, bd = w.cuda().requires_grad_(True), b.cuda().requires_grad_(True)
        y = BatchNormFn.apply(xd, wd, bd, rm.cuda(), rv.cuda(), train, 0.1, 1e-5, False)
        y.backward(dy.cuda())
        if train:
            y64, m64, v64 = R.bn_fwd(x, w, b, 1e-5)
            by, em, rel_r = R.bn_fwd_bound(x, w, b, 1e-5, rm, n_c)
            dx64, xh, rstd = R.bn_bwd(dy, x, w, 1e-5, True)
            bdx = R.bn_bwd_bound(dy, x, w, 1e-5, em, rel_r, n_c, True, xh, rstd)
            y32 = F.batch_norm(x, None, None, w, b, training=True, eps=1e-5)
            scale = np.abs(y64).max()
            BN_TABLE[d_over_sigma] = (np.abs(R.f64(y.detach()) - y64).max() / scale, np.abs(R.f64(y32) - y64).max() / scale)
            dw64, db64 = (R.f64(dy) * xh).sum(0), R.f64(dy).sum(0)
        else:
            rstd = 1.0 / np.sqrt(R.f64(rv) + 1e-5)
            xh = (R.f64(x) - R.f64(rm)) * rstd
            y64 = xh * R.f64(w) + R.f64(b)
            by = (8 * R.U * (np.abs(R.f64(x) * R.f64(w) * rstd) + np.abs(R.f64(rm) * R.f64(w) * rstd) + np.abs(R.f64(b)))
                  + 4 * R.U * np.abs(xh * R.f64(w)))
            dx64 = R.bn_bwd(dy, x, w, 1e-5, False, rv)[0]
            bdx = R.bn_bwd_bound(dy, x, w, 1e-5, None, None, n_c, False, None, rstd)
            dw64, db64 = (R.f64(dy) * xh).sum(0), R.f64(dy).sum(0)
        fam = 'BatchNormFn ' + ('train' if train else 'eval')
        assert within(fam, R.ratio(y.detach(), y64, by))
        assert within(fam + ' dx', R.ratio(xd.grad, dx64, bdx))
        # dw = sum dy xhat, db = sum dy: colstat chains on the forward's fp32 statistics
        dxh = np.abs(xh) * (rel_r if train else 4 * R.U) + (rstd * em if train else 0)
        bdw = R.chain(n_c, (np.abs(R.f64(dy)) * np.abs(xh)).sum(0)) + (np.abs(R.f64(dy)) * dxh).sum(0)
        assert within(fam + ' dw/db', max(R.ratio(wd.grad, dw64, bdw * (1 + 1e-6) + R.chain(4, np.abs(dw64))),
                                          R.ratio(bd.grad, db64, R.chain(n_c, np.abs(R.f64(dy)).sum(0)))))
    if d_over_sigma <= 4:
        ours, torchs = BN_TABLE[d_over_sigma]
        assert ours <= 10 * max(torchs, R.U), BN_TABLE


@pytest.fixture(scope='module', autouse=True)
def report_bn():
    yield
    if BN_TABLE:
        print('\nBatchNorm forward max|err| / max|y|, d/sigma: (BatchNormFn, torch fp32 CPU):',
              ', '.join(f'{k}: ({a:.2e}, {b:.2e})' for k, (a, b) in sorted(BN_TABLE.items())))


# ---- LSK selection ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('Ch', [32, 64, 160, 256, 36])
def test_lsk_agg_ties(L, Ch):
    """Designed exact ties: within a lane (c, c + 32), across lanes (c, c + 1), across a1 / a2.  The lowest index must
    win, as torch's max(dim) does, and lsk_mix_bwd_in must put d(max) exactly there."""
    g = torch.Generator().manual_seed(Ch)
    T = 200
    a1, a2 = scaled(g, T, Ch, lo=-2, hi=2) * 0.01, scaled(g, T, Ch, lo=-2, hi=2) * 0.01
    m = 100.0
    rng = np.random.default_rng(Ch)
    for t in range(T):
        kind = t % 4
        c = int(rng.integers(0, Ch))
        if kind == 0 and Ch > 32:                          # same lane
            c = int(rng.integers(0, Ch - 32)); a1[t, c] = a1[t, c + 32] = m
        elif kind == 1:                                    # neighbouring lanes, the higher lane first in a2
            c = int(rng.integers(0, Ch - 1)); a2[t, c] = a2[t, c + 1] = m; a1[t, Ch - 1] = m if t % 8 == 1 else a1[t, Ch - 1]
        elif kind == 2:                                    # across a1 / a2 at the same channel (same lane)
            a1[t, c] = a2[t, c] = m
        else:                                              # across a1 / a2, a2's copy in a lower lane
            c2 = int(rng.integers(0, c + 1)); a1[t, c] = a2[t, c2] = -m if t % 8 == 3 else m
    a1[:7] = -3.0                                          # rows of one constant value: index 0
    a2[:7] = -3.0

    def run():
        agg, am = Out((T, 2)), Out((T,), dtype=torch.int32)
        call(L, 'sm3_lsk_agg', cu(a1), cu(a2), agg, am, T, Ch)
        return agg, am
    names, (agg, am) = kernels_run(run)
    assert ran(names, 'lsk_agg_kernel'), names
    ref, idx = R.lsk_agg(a1, a2)
    cat = torch.cat([a1, a2], 1)
    tmax, tidx = cat.max(1)
    a = agg.get('agg')
    amx = am.get('amax')
    assert np.array_equal(amx, idx) and np.array_equal(amx, tidx.numpy())
    assert np.array_equal(a[:, 1], tmax.numpy())
    assert within('lsk_agg mean', R.ratio(a[:, 0], ref[:, 0], R.lsk_agg_mean_bound(a1, a2)))
    # lsk_mix_bwd_in with this argmax
    dout, sig, dagg = scaled(g, T, Ch), torch.rand(T, 2, generator=g), scaled(g, T, 2)
    da1, da2 = Out((T, Ch)), Out((T, Ch))
    call(L, 'sm3_lsk_mix_bwd_in', cu(dout), cu(sig), cu(dagg), am.t, da1, da2, T, Ch)
    outs, abss = R.lsk_mix_bwd_in(dout, sig, dagg, amx)
    for got, ref_, ab, nm in ((da1.get('da1'), outs[0], abss[0], 'da1'), (da2.get('da2'), outs[1], abss[1], 'da2')):
        assert within('lsk_mix_bwd_in', R.ratio(got, ref_, R.chain(3, ab))), nm


@pytest.mark.parametrize('Ch', [32, 64, 160, 256, 36])
def test_lsk_mix(L, Ch):
    g = torch.Generator().manual_seed(Ch)
    T = 333
    a1, a2, dout = scaled(g, T, Ch), scaled(g, T, Ch), scaled(g, T, Ch)
    z = torch.randn(T, 2, generator=g) * 12                  # saturated sigmoids on both sides
    sig = torch.sigmoid(z)
    out = Out((T, Ch))
    call(L, 'sm3_lsk_mix', cu(a1), cu(a2), cu(sig), out, T, Ch)
    ref, ab = R.lsk_mix(a1, a2, sig)
    assert within('lsk_mix', R.ratio(out.get('out'), ref, R.chain(2, ab)))
    dpre = Out((T, 2))
    call(L, 'sm3_lsk_mix_bwd_sig', cu(dout), cu(a1), cu(a2), cu(sig), dpre, T, Ch)
    ref, ab = R.lsk_mix_bwd_sig(dout, a1, a2, sig)
    assert within('lsk_mix_bwd_sig', R.ratio(dpre.get('dpre'), ref, R.chain(R.lsk_mix_bwd_sig_n(Ch), ab)))


@pytest.mark.parametrize('act', [0, 1])
@pytest.mark.parametrize('N,H,W', [(2, 1, 1), (1, 3, 5), (3, 7, 7), (2, 20, 31)])
def test_conv7_c2(L, N, H, W, act):
    g = torch.Generator().manual_seed(H * W + act)
    x = scaled(g, N, H, W, 2)
    w = torch.randn(196, generator=g) * 8                    # pre-activations far into both saturated tails
    b = torch.randn(2, generator=g)

    def run():
        y = Out((N * H * W, 2))
        call(L, 'sm3_conv7_c2', cu(x), cu(w), cu(b), y, N, H, W, act)
        return y
    names, y = kernels_run(run)
    assert ran(names, 'conv7_c2_kernel'), names
    s, z, za = R.conv7_c2(x, w, b, N, H, W, act)
    assert within(f'conv7_c2 act{act}', R.ratio(y.get('y'), s, R.conv7_c2_bound(z, za, act)))


def test_conv7_c2_wgrad(L):
    g = torch.Generator().manual_seed(3)
    N, H, W = 2, 61, 67
    n, blocks = R.conv7_c2_wgrad_n(N * H * W, sms())
    assert blocks > 1
    x, dpre = scaled(g, N, H, W, 2), scaled(g, N * H * W, 2)
    dw0, db0 = scaled(g, 196), scaled(g, 2)

    def run():
        dw, db = Out((196,), init=dw0), Out((2,), init=db0)
        call(L, 'sm3_conv7_c2_wgrad', cu(x), cu(dpre), dw, db, N, H, W)
        return dw, db
    names, (dw, db) = kernels_run(run)
    assert ran(names, 'conv7_c2_wgrad_kernel'), names
    rw, rb = R.conv7_c2_wgrad(x, dpre, N, H, W)
    aw, ab = R.conv7_c2_wgrad(np.abs(R.f64(x)), np.abs(R.f64(dpre)), N, H, W)
    assert within('conv7_c2_wgrad', max(R.ratio(dw.get('dw'), rw + R.f64(dw0), R.chain(n, aw + np.abs(R.f64(dw0)))),
                                        R.ratio(db.get('db'), rb + R.f64(db0), R.chain(n, ab + np.abs(R.f64(db0))))))


# ---- im2col / col2im --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('nchw,ks,stride,pad,Cin,H,W', [(True, 7, 4, 3, 3, 29, 23), (False, 3, 2, 1, 12, 15, 9),
                                                        (False, 7, 4, 3, 8, 13, 17), (True, 3, 2, 1, 5, 11, 7)])
def test_im2col_col2im(L, nchw, ks, stride, pad, Cin, H, W):
    g = torch.Generator().manual_seed(ks + Cin)
    N = 2
    K = ks * ks * Cin
    Kp = -(-(K + 1) // 4) * 4                               # at least one zero padding column
    x = torch.randn(N, Cin, H, W, generator=g) if nchw else scaled(g, N, H, W, Cin)
    Ho, Wo = (H + 2 * pad - ks) // stride + 1, (W + 2 * pad - ks) // stride + 1
    col = Out((N * Ho * Wo, Kp))
    call(L, 'sm3_im2col', cu(x), col, N, H, W, Cin, ks, stride, pad, Kp, int(nchw))
    ref, _, _ = R.im2col(x, N, H, W, Cin, ks, stride, pad, Kp, nchw)
    assert np.array_equal(col.get('col'), ref)
    dcol = scaled(g, N * Ho * Wo, Kp)
    dx = Out((N, Cin, H, W) if nchw else (N, H, W, Cin))
    call(L, 'sm3_col2im', cu(dcol), dx, N, H, W, Cin, ks, stride, pad, Kp, int(nchw))
    got = dx.get('dx')
    assert np.array_equal(got, R.col2im_fp32(dcol, N, H, W, Cin, ks, stride, pad, Kp, nchw))
    r64 = R.col2im(dcol, N, H, W, Cin, ks, stride, pad, Kp, nchw)
    a64 = R.col2im(np.abs(R.f64(dcol)), N, H, W, Cin, ks, stride, pad, Kp, nchw)
    assert within('col2im', R.ratio(got, r64, R.chain(-(-ks // stride) ** 2, a64)))


# ---- dropout ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('p', [0.0, 0.1, 0.5])
def test_dropout_bit_exact(L, p):
    g = torch.Generator().manual_seed(int(p * 10))
    n = 4 * 25013                                            # a multiple of 4, not of 1024
    x = scaled(g, n)
    seed = 0x1234567890ABCDEF + int(p * 100)
    out = Out((n,))
    call(L, 'sm3_dropout', cu(x), out, n, p, seed)
    ref = R.dropout_fp32(x, p, seed)
    got = out.get('dropout')
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32))
    seed_dev = torch.tensor([seed - (1 << 64) if seed >= (1 << 63) else seed], dtype=torch.int64).cuda()
    out2 = Out((n,))
    call(L, 'sm3_dropout_dev', cu(x), out2, n, p, seed_dev)
    assert np.array_equal(out2.get('dropout_dev').view(np.uint32), got.view(np.uint32))


# ---- FPN helpers and scale_rows ---------------------------------------------------------------------------------------
@pytest.mark.parametrize('H,h', [(25, 13), (13, 7), (7, 4), (32, 16)])
def test_upsample_add(L, H, h):
    g = torch.Generator().manual_seed(H)
    N, C = 2, 36
    W, w = H + 2, -(-(H + 2) // 2)
    a, b, d = scaled(g, N, H, W, C), scaled(g, N, h, w, C), scaled(g, N, H, W, C)
    out = Out((N, H, W, C))
    call(L, 'sm3_upsample_add', cu(a), cu(b), out, N, H, W, h, w, C)
    got = out.get('out')
    assert np.array_equal(got, R.upsample_add_fp32(a, b))
    ref = R.f64(a) + F.interpolate(b.double().permute(0, 3, 1, 2), size=(H, W), mode='nearest').permute(0, 2, 3, 1).numpy()
    terms = np.abs(R.f64(a)) + np.abs(R.f64(R.upsample(b.numpy(), H, W)))
    assert within('upsample_add', R.ratio(got, ref, R.chain(1, terms)))
    db = Out((N, h, w, C))
    call(L, 'sm3_upsample_add_bwd', cu(d), db, N, H, W, h, w, C)
    got = db.get('db')
    assert np.array_equal(got, R.upsample_add_bwd_fp32(d, h, w))
    br = b.double().requires_grad_(True)
    F.interpolate(br.permute(0, 3, 1, 2), size=(H, W), mode='nearest').permute(0, 2, 3, 1).backward(d.double())
    k = -(-H // h) * -(-W // w)
    assert within('upsample_add_bwd', R.ratio(got, br.grad, R.chain(k, R.upsample_add_bwd(np.abs(R.f64(d)), h, w))))


@pytest.mark.parametrize('B,Rr,Cc', [(3, 45, 70), (2, 1, 33), (1, 100, 31)])
def test_transpose_batched(L, B, Rr, Cc):
    x = scaled(torch.Generator().manual_seed(Rr), B, Rr, Cc)
    out = Out((B, Cc, Rr))
    call(L, 'sm3_transpose_batched', cu(x), out, B, Rr, Cc)
    assert np.array_equal(out.get('out'), x.transpose(1, 2).numpy())


def test_scale_rows(L):
    g = torch.Generator().manual_seed(9)
    rows, C = 77, 52
    x, rs, cs = scaled(g, rows, C), scaled(g, rows), scaled(g, C)
    for r_, c_ in ((rs, None), (None, cs), (rs, cs)):
        out = Out((rows, C))
        call(L, 'sm3_scale_rows', cu(x), cu(r_), cu(c_), out, rows, C)
        assert np.array_equal(out.get('out'), R.scale_rows_fp32(x, r_, c_))
