"""The split-bf16 GEMM (`gemm_bf16x3_kernel`, csrc/gemm_tc.cuh), its pack kernels and the fused FFN (`ffn_chain_kernel`,
csrc/ffn_fused.cu) against tests/gemm_ref.py, on every launch path, in both precision modes (3 passes: hi*hi + hi*lo +
lo*hi; 1 pass: hi*hi).  All calls go through the C ABI (sm3det_b200.ops).

1. Operand images are bit-exact splits of their fp32 source.
2. A launch matrix on integer operands in [-3, 3] (lo = 0, every sum exact) must equal the integer result exactly, for
   every instantiation launch() can choose, dense / grouped / split-K schedules, tile widths 32-128, M and K tails,
   more tiles than SMs and exact epilogues.  Which instantiation ran is read from the profiler.  Every operand lies
   inside a NaN-filled buffer (gaps of lda > K, rows past M, columns past N, bias / resid / aux past their extents),
   and D / aux_out / colsum inside sentinel-filled buffers: sentinels must stay bit-identical and D free of NaN.
3. Float accuracy against the float64 emulation of the split products, with bounds derived below.
4. The packed split-K segment precondition, and that the MoE, LSK and expert-parallel callers meet it.
5. The fused FFN forward (and backward-into-dv) at every C it supports and every chunk width it accepts.
6. A census: every GEMM / fused-FFN launch of short ConvNeXt and LSK training steps has a signature the matrix covers.
"""
import math
import re

import numpy as np
import pytest
import torch

import gemm_ref as R

pytestmark = pytest.mark.gpu

U = 2.0 ** -24          # unit roundoff of fp32
SENT = 0x7FA11A11       # sentinel bit pattern (a NaN payload the kernels never produce)


@pytest.fixture(scope='module')
def ops():
    from sm3det_b200 import ops as o
    return o


def kernels_run(fn, restore=None, tries=5):
    """(names of the CUDA kernels fn launches, fn's result).  The profiler occasionally records no CUDA activity at all;
    fn is then run again, after `restore()` puts back whatever its previous run accumulated into."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(tries):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            res = fn()
            torch.cuda.synchronize()
        names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
        if names:
            break
        if restore is not None:
            restore()
    return names, res


def gemm_instantiations(names):
    """Template arguments (A_MN, B_MN, B_PACKED, A_PACKED, EPI_T) of each gemm_bf16x3_kernel launched."""
    out = set()
    for n in names:
        m = re.search(r'gemm_bf16x3_kernel<([^>]*)>', n)
        if m:
            a = [s.strip() for s in m.group(1).split(',')]
            out.add(tuple(s == 'true' for s in a[:4]) + (int(re.search(r'-?\d+', a[4]).group(0)),))
    return out


# ---- τ(K): fp32 accumulation error of the wgmma main loop --------------------------------------------------------
# Each wgmma k16 step adds 16 exact bf16 x bf16 products to the fp32 accumulator.  The tensor core aligns the addends
# to the largest exponent and truncates, so one step errs by at most a few fp32 ulps of the largest magnitude it sees,
# which is at most S = sum_k |a_k b_k| (the accumulator holds a partial sum of at most that magnitude).  Taking 4 ulps
# (2^-21 relative) per step, a launch of `passes` MMAs per k16 step over ceil(K/16) steps errs by at most
#     τ(K) · S  with  τ(K) = passes · ceil(K / 16) · 2^-21.
# The bound is linear in the number of steps (errors of equal sign add up); rounding errors of random data largely
# cancel, so measured ratios are far below it (see DESIGN.md §4 for the worst measured ratio).
def tau(K, passes):
    return passes * max(1, -(-K // 16)) * 2.0 ** -21


# split error against exact float64 products, relative per product: 3 passes drop lo*lo (|lo| < 2^-7 |x|, so up to
# 2^-14) and keep the residual of each split (2^-16 each, tests/test_gemm_ref.py); 1 pass truncates both operands to
# bf16 (2 · 2^-7 + 2^-14)
def split_err(passes):
    return 2.0 ** -14 + 2 * 2.0 ** -16 + 2.0 ** -31 if passes == 3 else 2 * 2.0 ** -7 + 2.0 ** -14


# ---- buffers ------------------------------------------------------------------------------------------------------
FRONT = 64     # floats of NaN before every operand (256 B: the operand stays 16-byte aligned)


def nan_buffer(x, ld, extra_rows=3, fill=float('nan')):
    """x [rows, cols] stored with row stride ld >= cols inside a `fill`ed CUDA buffer; returns the 1-D view at x[0, 0]."""
    x = np.asarray(x, dtype=np.float32)
    rows, cols = x.shape
    big = torch.full((FRONT + (rows + extra_rows) * ld + FRONT,), fill, dtype=torch.float32)
    big[FRONT:FRONT + rows * ld].view(rows, ld)[:, :cols] = torch.from_numpy(x)
    return big.cuda()[FRONT:]


def sentinel_buffer(rows, cols, ld, init=None):
    big = torch.full((FRONT + (rows + 3) * ld + FRONT,), SENT, dtype=torch.int32)
    if init is not None:
        big.view(torch.float32)[FRONT:FRONT + rows * ld].view(rows, ld)[:, :cols] = torch.from_numpy(
            np.asarray(init, dtype=np.float32))
    return big.cuda().view(torch.float32)[FRONT:]


def window(buf, rows, cols, ld):
    """(values of the [rows, cols] window, bit patterns of everything outside it incl. the front pad)."""
    full = buf._base if buf._base is not None else buf
    allb = full.cpu().view(torch.int32).numpy()
    inside = np.zeros(allb.size, dtype=bool)
    idx = FRONT + (np.arange(rows)[:, None] * ld + np.arange(cols)[None, :])
    inside[idx.ravel()] = True
    vals = allb[idx].view(np.float32)
    return vals, allb[~inside]


def check_sentinels(buf, rows, cols, ld, what):
    vals, outside = window(buf, rows, cols, ld)
    assert np.all(outside == np.int32(SENT)), f'{what}: written outside its [{rows}, {cols}] window'
    return vals


# ---- 1. images ----------------------------------------------------------------------------------------------------
def _special_values(rng, shape):
    x = rng.standard_normal(shape).astype(np.float32) * np.exp2(rng.integers(-30, 30, shape)).astype(np.float32)
    flat = x.reshape(-1)
    sp = np.array([0.0, -0.0, 1e-39, -3e-42, 3.4e38, -3.4e38, 1.0 + 2 ** -8 + 2 ** -16, -(1.0 + 2 ** -9 + 2 ** -17)],
                  dtype=np.float32)
    flat[:sp.size] = sp
    return x


@pytest.mark.parametrize('tile', [32, 64, 96, 128, 160, 256])
@pytest.mark.parametrize('K', [4, 36, 100])
@pytest.mark.parametrize('transposed', [False, True])
def test_pack_b_image_bit_exact(ops, tile, K, transposed):
    rng = np.random.default_rng(tile * K + transposed)
    groups, N = 2, tile * 2
    w = _special_values(rng, (groups, N, K) if not transposed else (groups, K, N))
    wd = torch.from_numpy(w).cuda()
    img, per = ops.pack_weight(wd, transposed=transposed, groups=groups, tile=tile)
    B = w if not transposed else w.transpose(0, 2, 1)          # B(n, k)
    Kp = -(-K // 32) * 32
    for g in range(groups):
        h, l = R.decode_k(img[g * per:(g + 1) * per], N, Kp, tile)
        eh, el = R.split_bits(np.pad(B[g], ((0, 0), (0, Kp - K))))
        assert np.array_equal(h, eh) and np.array_equal(l, el), g
    assert per == N * Kp * 2


@pytest.mark.parametrize('tile', [32, 64, 96, 128])
@pytest.mark.parametrize('mn_major', [False, True])
@pytest.mark.parametrize('rows,cols,gather', [(1, 40, False), (127, 96, True), (129, 256, False), (300, 64, True)])
def test_pack_act_image_bit_exact(ops, tile, mn_major, rows, cols, gather):
    rng = np.random.default_rng(rows + cols + tile)
    src_rows = rows + 7
    x = _special_values(rng, (src_rows, cols))
    ld = cols + 4
    xd = nan_buffer(x, ld)
    idx = None
    logical = x[:rows]
    if gather:
        idx = rng.integers(-1, src_rows, rows).astype(np.int32)
        idx[::5] = -1
        logical = np.where((idx >= 0)[:, None], x[np.maximum(idx, 0)], 0).astype(np.float32)
    img = ops.pack_act(xd, rows=rows, cols=cols, mn_major=mn_major, tile=tile, ld=ld,
                       row_index=None if idx is None else torch.from_numpy(idx).cuda())
    assert img.numel() == R.packed_act_elems(rows, cols, mn_major, tile)
    if mn_major:
        rp, cp = -(-rows // 32) * 32, -(-cols // tile) * tile
        h, l = R.decode_mn(img, rp, cp, tile)
    else:
        rp, cp = -(-rows // tile) * tile, -(-cols // 32) * 32
        h, l = R.decode_k(img, rp, cp, tile)
    eh, el = R.split_bits(np.pad(logical, ((0, rp - rows), (0, cp - cols))))
    assert np.array_equal(h, eh) and np.array_equal(l, el)


# GELU / GELU' of csrc/common.cuh (phi_parts) against float64 erf.  Phi = 1 - q or q with q = poly(t) exp(-z^2) / 2,
# the Abramowitz-Stegun 7.1.26 form of erfc, whose own error is <= 1.5e-7 on erfc, i.e. 7.5e-8 on Phi.  Its fp32
# evaluation adds the rcp.approx of t (1 ulp), five fma of the Horner chain on coefficients up to 1.5 (< 8 ulps of 1.5
# in absolute terms after the final multiply by t <= 1), ex2.approx (2 ulps) and the product 0.5 * poly * e, all
# multiplied by e / 2 <= 1/2: < 16 · 2^-24 = 9.6e-7 absolute on q.  Then 1 - q rounds once (2^-24).  So
#     |ΔPhi| <= 7.5e-8 + 9.6e-7 · 1/2 + 2^-24 < 6.2e-7,
#     |Δgelu|  <= |x| |ΔPhi| + 2^-24 |gelu(x)|,
#     |Δgelu'| <= |ΔPhi| + |x| pdf(x) (4 · 2^-24 + |x|^2 · 2^-24) + 2^-24 |gelu'(x)|,
# the middle term being the rounding of x · 0.3989 and of the exp argument -x^2/2 (relative |x|^2 · 2^-24 on e).
DPHI = 6.2e-7


def gelu_bound(x):
    x = np.abs(np.asarray(x, dtype=np.float64))
    return x * DPHI + U * np.abs(R.gelu64(x)) + 1e-45


def gelu_grad_bound(x):
    x = np.abs(np.asarray(x, dtype=np.float64))
    pdf = np.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)
    return DPHI + x * pdf * (4 + x * x) * U + U * np.abs(R.gelu_grad64(x))


def _act_inputs(rng, R_, W):
    h = (rng.standard_normal((R_, W)) * 3).astype(np.float32)
    flat = h.reshape(-1)
    sweep = np.linspace(-10, 10, min(flat.size // 2, 20001), dtype=np.float32)
    flat[:sweep.size] = sweep
    flat[sweep.size:sweep.size + 8] = [-1e4, 1e4, -40.0, 40.0, -13.5, 13.5, 1e-30, -1e-30]
    return h


@pytest.mark.parametrize('R_,W,mn_tile', [(300, 256, 128), (129, 384, 96), (1000, 96, 32)])
def test_act_pack_modes(ops, R_, W, mn_tile):
    """Modes 0-3: each image is the bit-exact split of the kernel's own fp32 output; the fp32 GELU / GELU' are within
    the bound above of float64 erf; column sums; rows past live_tiles are zero."""
    rng = np.random.default_rng(R_ + W)
    h = _act_inputs(rng, R_, W)
    da = rng.standard_normal((R_, W)).astype(np.float32)
    hd, dad = torch.from_numpy(h).cuda(), torch.from_numpy(da).cuda()
    Rk, Rm = -(-R_ // 128) * 128, -(-R_ // 32) * 32
    Wm = -(-W // mn_tile) * mn_tile
    f32 = {}
    for mode in (0, 1, 2):
        cs = torch.zeros(W, device='cuda')
        pk, pm, of = ops.act_pack(hd, rows=R_, width=W, mode=mode, da=dad if mode == 1 else None, want_k=True,
                                  mn_tile=mn_tile, want_f32=True, colsum=cs)
        y = of.cpu().numpy()
        f32[mode] = y
        # rows up to the next multiple of 32 are zero; the K-major image's rows beyond that (up to its 128-row tile) are
        # not written: a GEMM row depends only on its own A row, and rows >= M are never stored
        eh, el = R.split_bits(np.pad(y, ((0, Rm - R_), (0, 0))))
        h_, l_ = R.decode_k(pk, Rk, W)
        assert np.array_equal(h_[:Rm], eh) and np.array_equal(l_[:Rm], el), mode
        eh, el = R.split_bits(np.pad(y, ((0, Rm - R_), (0, Wm - W))))
        h_, l_ = R.decode_mn(pm, Rm, Wm, mn_tile)
        assert np.array_equal(h_, eh) and np.array_equal(l_, el), mode
        # column sums of fp32 values: at most R_ roundings of partial sums
        ref = y.astype(np.float64).sum(0)
        assert np.all(np.abs(cs.cpu().numpy() - ref) <= R_ * U * np.abs(y).astype(np.float64).sum(0) + 1e-30), mode
    assert np.array_equal(f32[2], h)
    assert np.all(np.abs(f32[0] - R.gelu64(h)) <= gelu_bound(h))
    assert np.all(np.abs(f32[1] - da.astype(np.float64) * R.gelu_grad64(h))
                  <= np.abs(da) * gelu_grad_bound(h) + U * np.abs(f32[1]))
    # mode 3: one pass emits da * gelu'(h) (= mode 1) and gelu(h) (= mode 0) as images
    pk, pm, pm2 = ops.act_pack(hd, rows=R_, width=W, mode=ops.ACT_BWD, da=dad, want_k=True, mn_tile=128, mn_tile2=mn_tile)
    eh, el = R.split_bits(np.pad(f32[1], ((0, Rm - R_), (0, 0))))
    h_, l_ = R.decode_k(pk, Rk, W)
    assert np.array_equal(h_[:Rm], eh) and np.array_equal(l_[:Rm], el)
    eh, el = R.split_bits(np.pad(f32[0], ((0, Rm - R_), (0, Wm - W))))
    h_, l_ = R.decode_mn(pm2, Rm, Wm, mn_tile)
    assert np.array_equal(h_, eh) and np.array_equal(l_, el)


def test_act_pack_live_tiles_and_group_colsum(ops):
    """Expert layout: rows of tiles >= live_tiles are zero in the images (whatever h holds there); the column sums go
    to each tile's group."""
    rng = np.random.default_rng(7)
    R_, W, live = 640, 128, 3
    h = rng.standard_normal((R_, W)).astype(np.float32)
    h[live * 128:] = np.nan
    tg = np.array([2, 0, 2, 99, 99], dtype=np.int32)
    cs = torch.zeros((3, W), device='cuda')
    pk, pm, of = ops.act_pack(torch.from_numpy(h).cuda(), rows=R_, width=W, mode=ops.ACT_COPY, want_k=True, mn_tile=128,
                              colsum=cs, live_tiles=torch.tensor([live], dtype=torch.int32).cuda(),
                              tile_group=torch.from_numpy(tg).cuda())
    hk, lk = R.decode_k(pk, R_, W)
    hm, lm = R.decode_mn(pm, R_, W, 128)
    want_h, want_l = R.split_bits(np.where(np.arange(R_)[:, None] < live * 128, h, 0).astype(np.float32))
    assert np.array_equal(hk, want_h) and np.array_equal(lk, want_l)
    assert np.array_equal(hm, want_h) and np.array_equal(lm, want_l)
    want = np.zeros((3, W))
    for t in range(live):
        want[tg[t]] += h[t * 128:(t + 1) * 128].astype(np.float64).sum(0)
    assert np.all(np.abs(cs.cpu().numpy() - want) <= 256 * U * np.abs(h[:live * 128]).astype(np.float64).sum(0))


# ---- 2. integer-exact launch matrix -------------------------------------------------------------------------------
E_FFN2_TRAIN = R.EPI_BIAS | R.EPI_COLSCALE | R.EPI_RESID | R.EPI_AUXSTORE
E_FFN2_EVAL = R.EPI_BIAS | R.EPI_COLSCALE | R.EPI_RESID

# Layout families: how A and B reach the kernel.
#   kk   A K-major fp32, B K-major fp32        -> <false, false, false, false, -1>
#   kmn  A K-major fp32, B MN-major fp32       -> <false, true,  false, false, -1>   (dgrad without a packed weight)
#   pb   A K-major fp32, B packed (K-major)    -> <false, false, true,  false, -1>
#   pk   A and B packed K-major                -> <false, false, true,  true,  EPI if one of the hot sets else -1>
#   mm   A MN-major fp32, B MN-major fp32      -> <true,  true,  false, false, -1>   (wgrad)
#   pmn  A and B packed MN-major               -> <true,  true,  true,  true,  EPI if one of the hot sets else -1>
HOT_K = (0, R.EPI_BIAS, E_FFN2_TRAIN, E_FFN2_EVAL)
HOT_MN = (R.EPI_ATOMIC, R.EPI_ATOMIC | R.EPI_ROWSCALE)


def instantiation(layout, epi):
    return {'kk': (False, False, False, False, -1), 'kmn': (False, True, False, False, -1),
            'pb': (False, False, True, False, -1),
            'pk': (False, False, True, True, epi if epi in HOT_K else -1),
            'mm': (True, True, False, False, -1),
            'pmn': (True, True, True, True, epi if epi in HOT_MN else -1)}[layout]


# (layout, schedule, epilogue, row gather, k gather, segments).  Every family runs at BN 32 / 64 / 96 / 128 and in
# both precision modes.
FAMILIES = [
    ('kk', 'dense', 0, False, False, False),
    ('kk', 'dense', R.EPI_BIAS | R.EPI_COLSCALE | R.EPI_ROWSCALE | R.EPI_RESID | R.EPI_AUXSTORE, False, False, False),
    ('kk', 'dense', R.EPI_BIAS, True, False, False),
    ('kk', 'grouped', R.EPI_BIAS, True, False, False),
    ('kk', 'dense', R.EPI_COLSUM | R.EPI_ROWSCALE, False, False, False),
    ('kk', 'splitk', R.EPI_ATOMIC, False, False, False),
    ('kmn', 'dense', 0, False, False, False),
    ('kmn', 'dense', R.EPI_ROWSCALE | R.EPI_RESID, False, False, False),
    ('kmn', 'grouped', R.EPI_COLSUM, False, False, False),
    ('kmn', 'grouped', 0, False, False, False),
    ('pb', 'dense', 0, False, False, False),
    ('pb', 'grouped', 0, False, False, False),
    ('pb', 'dense', R.EPI_BIAS | R.EPI_GELU, False, False, False),
    ('pb', 'dense', R.EPI_BIAS, False, False, False),
    ('pb', 'dense', R.EPI_BIAS, True, False, False),
    ('pb', 'grouped', R.EPI_BIAS, True, False, False),
    ('pb', 'dense', R.EPI_COLSCALE | R.EPI_RESID | R.EPI_BIAS | R.EPI_ROWSCALE, False, False, False),
    ('pk', 'dense', 0, False, False, False),
    ('pk', 'dense', R.EPI_BIAS, False, False, False),
    ('pk', 'grouped', R.EPI_BIAS, False, False, False),
    ('pk', 'grouped', 0, False, False, False),
    ('pk', 'dense', E_FFN2_TRAIN, False, False, False),
    ('pk', 'dense', E_FFN2_EVAL, False, False, False),
    ('pk', 'dense', E_FFN2_TRAIN | R.EPI_ROWSCALE, False, False, False),
    ('pk', 'dense', E_FFN2_EVAL | R.EPI_ROWSCALE, False, False, False),
    ('pk', 'dense', R.EPI_ROWSCALE, False, False, False),
    ('pk', 'grouped', R.EPI_COLSUM, False, False, False),
    ('pk', 'dense', R.EPI_COLSUM, False, False, False),
    ('mm', 'splitk', R.EPI_ATOMIC, False, False, False),
    ('mm', 'splitk', R.EPI_ATOMIC | R.EPI_ROWSCALE, False, False, False),
    ('mm', 'splitk', R.EPI_ATOMIC, False, True, True),
    ('mm', 'splitk', 0, False, False, True),
    ('pmn', 'splitk', R.EPI_ATOMIC, False, False, False),
    ('pmn', 'splitk', R.EPI_ATOMIC | R.EPI_ROWSCALE, False, False, False),
    ('pmn', 'splitk', R.EPI_ATOMIC, False, False, True),
    ('pmn', 'splitk', R.EPI_ATOMIC | R.EPI_ROWSCALE, False, False, True),
    ('pmn', 'splitk', 0, False, False, True),
]
BNS = (32, 64, 96, 128)
SCHED = {'dense': 0, 'grouped': 1, 'splitk': 2}


def signature(layout, sched, epi, BN, row_gather, k_gather, segs, passes):
    return (instantiation(layout, epi), sched, epi, BN, row_gather, k_gather, segs, passes)


COVERED = {signature(f[0], f[1], f[2], bn, f[3], f[4], f[5], p) for f in FAMILIES for bn in BNS for p in (1, 3)}


def run_case(ops, layout, sched, epi, BN, row_gather, k_gather, segs, M, K, passes, seed, int_data=True, data=None,
             k_splits=None):
    """Build one launch on NaN-padded operands, run it, check the sentinels, return (D [G, M, N], ref tuple, names)."""
    rng = np.random.default_rng(seed)
    a_mn = layout in ('mm', 'pmn')
    packed_b = layout in ('pb', 'pk', 'pmn')
    packed = layout in ('pk', 'pmn')
    N = BN if packed_b else 2 * BN                       # packed images use the default tile width pick_bn(N) = BN
    G = 3 if sched in ('grouped',) or segs else 1

    def ints(shape):
        return rng.integers(-3, 4, shape).astype(np.float32)

    gen = ints if int_data else (lambda s: rng.standard_normal(s).astype(np.float32))
    kw = dict(M=M, N=N, K=K, sched=SCHED[sched], epilogue=epi, tile_n=0 if packed_b else BN)
    ref_kw = dict(passes=passes, epi=epi)
    # --- A
    src_rows = M + 5 if row_gather else M
    A_src = gen((src_rows, K)) if data is None else data[0]
    if row_gather:
        ri = rng.integers(-1, src_rows, M).astype(np.int32)
        ri[::3] = -1
        ref_kw['a_row_index'] = ri
    A_logical = A_src
    tile_group = num_m_tiles = None
    if sched == 'grouped':
        m_tiles = -(-M // 128)
        nt = max(1, m_tiles - 1) if m_tiles > 1 else 1    # device count below the host upper bound when possible
        tg = rng.integers(0, G, m_tiles + 2).astype(np.int32)
        tg[nt:] = 1000 + np.arange(tg.size - nt)            # out-of-range ids beyond the live tiles
        tile_group, num_m_tiles = tg, nt
        ref_kw.update(tile_group=tg, num_m_tiles=nt)
        kw.update(tile_group=torch.from_numpy(tg).cuda(), num_m_tiles=torch.tensor([nt], dtype=torch.int32).cuda())
    seg_b = seg_e = None
    if segs:
        # ragged segments incl. an empty one; packed: seg_begin % 32 == 0 and A rows up to ceil32(seg_end) zero
        if packed:
            seg_b = np.array([0, 32 * (K // 96), 32 * (K // 64)], dtype=np.int32)
            seg_e = np.array([min(K, 32 * (K // 96) // 2 + 5), 32 * (K // 96), K - 3], dtype=np.int32)
        else:
            seg_b = np.array([3, K // 3, K // 2 + 1], dtype=np.int32)
            seg_e = np.array([K // 3 - 1, K // 3, K], dtype=np.int32)
        seg_e = np.maximum(seg_e, seg_b)
        if packed:
            live = np.zeros(K, dtype=bool)
            for b, e in zip(seg_b, seg_e):
                live[b:e] = True
            A_logical = np.where(live[None, :], A_logical, 0).astype(np.float32)
        ref_kw['segs'] = (seg_b, seg_e)
        kw.update(seg_begin=torch.from_numpy(seg_b).cuda(), seg_end=torch.from_numpy(seg_e).cuda(), num_groups=G)
    if sched == 'splitk':
        if k_splits is None:
            k_splits = 3 if (epi & R.EPI_ATOMIC) else 1
        kw.update(k_splits=k_splits, num_groups=G)
    # --- B: [Gb, N, Kb] logical
    Gb = G if sched == 'grouped' else 1
    Kb = K + 9 if k_gather else K
    B_src = gen((Gb, N, Kb)) if data is None else data[1]
    if k_gather:
        ki = rng.integers(-1, Kb, K).astype(np.int32)
        ki[::4] = -1
        ref_kw['b_k_index'] = ki
        kw['b_k_index'] = torch.from_numpy(ki).cuda()
    if row_gather and not packed:
        kw['a_row_index'] = torch.from_numpy(ref_kw['a_row_index']).cuda()
    keep = []
    if a_mn:
        lda = M + 8
        At = nan_buffer(A_logical.T, lda)                  # [K, lda]: A(m, k) at k * lda + m
        kw.update(a_smn=1, a_sk=lda)
        if packed:
            kw['a_packed'] = ops.pack_act(At, rows=K, cols=M, mn_major=True, tile=128, ld=lda)
            kw['A'] = None
        else:
            kw['A'] = At
    else:
        lda = K + 4
        Ab = nan_buffer(A_src, lda)
        kw.update(a_smn=lda, a_sk=1)
        if packed:
            ridx = None if not row_gather else torch.from_numpy(ref_kw['a_row_index']).cuda()
            kw['a_packed'] = ops.pack_act(Ab, rows=M, cols=K, mn_major=False, tile=128, ld=lda, row_index=ridx)
            kw['A'] = None
        else:
            kw['A'] = Ab
    if layout in ('kk',):
        ldb = Kb + 4
        Bb = nan_buffer(B_src.reshape(Gb * N, Kb), ldb, extra_rows=2)
        kw.update(B=Bb, b_smn=ldb, b_sk=1, b_group_stride=N * ldb if Gb > 1 else 0)
    elif layout in ('kmn', 'mm'):
        ldb = N + 4                                      # [Kb, ldb] per group: B(n, k) at k * ldb + n
        Bt = np.concatenate([np.pad(B_src[g].T, ((0, 1), (0, 0))) for g in range(Gb)])   # one gap row per group
        Bb = nan_buffer(Bt, ldb)
        # split-K groups index D and the segments; B is shared (group stride 0), as in the expert wgrads
        kw.update(B=Bb, b_smn=1, b_sk=ldb, b_group_stride=(Kb + 1) * ldb if Gb > 1 else 0)
    elif layout in ('pb', 'pk'):
        wb = nan_buffer(B_src.reshape(Gb * N, Kb), Kb, extra_rows=2)   # pack_weight reads [groups, N, K] contiguous
        img, per = ops.pack_weight(wb[:Gb * N * Kb].view(Gb, N, Kb), transposed=False, groups=Gb)
        kw.update(B=None, b_packed=img, b_packed_group_stride=per, b_smn=Kb, b_sk=1)
        keep.append(wb)
    else:   # pmn: B(n, k) = x[k, n], x [K, ldb]
        ldb = N + 4
        xb = nan_buffer(B_src[0].T, ldb)
        kw.update(B=None, b_packed=ops.pack_act(xb, rows=K, cols=N, mn_major=True, tile=BN, ld=ldb), b_smn=1, b_sk=ldb)
    # --- epilogue operands (powers of two incl. 0 for the scales, integers for bias / resid / initial D)
    Gd = G if segs or (sched == 'splitk' and G > 1) else 1
    ldd = N + 8
    d_init = ints((Gd * M, N)) if epi & R.EPI_ATOMIC else None
    D = sentinel_buffer(Gd * M, N, ldd, init=d_init)
    kw.update(D=D, ldd=ldd, d_group_stride=M * ldd if Gd > 1 else 0)   # grouped: all groups write the same D rows
    ref_kw['d_init'] = None if d_init is None else d_init.reshape(Gd, M, N)
    if epi & R.EPI_BIAS:
        bs = N + 4
        bias = ints((Gb, N))
        kw.update(bias=nan_buffer(bias, bs), bias_group_stride=bs)
        ref_kw['bias'] = bias
    ld_aux = N + 4
    if epi & (R.EPI_AUXSTORE | R.EPI_GELU):
        aux = sentinel_buffer(M, N, ld_aux)
        kw.update(aux_out=aux, ld_aux=ld_aux)
    if epi & R.EPI_DGELU:
        ai = (rng.standard_normal((M, N)) * 2).astype(np.float32)
        kw.update(aux_in=nan_buffer(ai, ld_aux), ld_aux=ld_aux)
        ref_kw['aux_in'] = ai
    if epi & R.EPI_COLSCALE:
        cs = np.exp2(rng.integers(-2, 3, N)).astype(np.float32)
        cs[::7] = 0
        kw['col_scale'] = nan_buffer(cs[None], N)
        ref_kw['col_scale'] = cs
    if epi & R.EPI_ROWSCALE:
        rs = np.exp2(rng.integers(-2, 3, M)).astype(np.float32)
        rs[::5] = 0
        kw['row_scale'] = nan_buffer(rs[None], M)
        ref_kw['row_scale'] = rs
    if epi & R.EPI_RESID:
        ld_r = N + 4
        res = ints((M, N))
        kw.update(resid=nan_buffer(res, ld_r), ld_resid=ld_r)
        ref_kw['resid'] = res
    ncs = 0
    if epi & R.EPI_COLSUM:
        ncs = Gb
        colsum = sentinel_buffer(ncs, N, N + 4, init=np.zeros((ncs, N)))
        kw.update(colsum=colsum, colsum_group_stride=N + 4)
    A_ref = A_logical if a_mn else A_src
    ref = R.gemm_ref(A_ref, B_src, **ref_kw)
    from sm3det_b200.ops import precision_scope
    outs = [t for t in (D, kw.get('aux_out'), kw.get('colsum')) if t is not None]
    snap = [t._base.clone() for t in outs]

    def restore():
        for t, s_ in zip(outs, snap):
            t._base.copy_(s_)
    with precision_scope(passes):
        names, _ = kernels_run(lambda: ops.gemm(**kw), restore)
    got = check_sentinels(D, Gd * M, N, ldd, 'D').reshape(Gd, M, N)
    aux_got = check_sentinels(kw['aux_out'], M, N, ld_aux, 'aux_out') if 'aux_out' in kw else None
    cs_got = check_sentinels(kw['colsum'], ncs, N, N + 4, 'colsum') if ncs else None
    return got, ref, names, aux_got, cs_got


def _exact_compare(got, ref, gelu=False):
    """D equals the reference exactly where the schedule writes and keeps its sentinel elsewhere.  With EPI_GELU the
    GELU input (the exact accumulator + bias) is exact, so only the fast GELU's own bound applies."""
    D, _, aux, colsum = ref
    unwritten = np.isnan(D)
    assert np.all(got.view(np.int32)[unwritten] == np.int32(SENT)), 'rows the schedule skips were written'
    assert not np.isnan(got[~unwritten]).any(), 'NaN in D'
    g, d = got[~unwritten].astype(np.float64), D[~unwritten]
    if gelu:                                                      # D = gelu(aux)
        assert np.all(np.abs(g - d) <= gelu_bound(aux[~unwritten]))
    else:
        assert np.array_equal(g, d)


def _int_matrix():
    cases = []
    Ms_k = (1, 127, 128, 129)
    Ks = (4, 36, 48, 100)
    i = 0
    for fam in FAMILIES:
        layout, sched, epi, rg, kg, segs = fam
        for bn in BNS:
            for passes in (1, 3):
                if layout in ('mm', 'pmn'):
                    M, K = (128, 136)[i % 2], (100, 200, 300)[i % 3]
                else:
                    M, K = Ms_k[i % 4], Ks[(i // 4) % 4]
                    if sched == 'grouped':
                        M = (300, 257, 384)[i % 3]
                cases.append(pytest.param(fam, bn, passes, M, K, id=f'{layout}-{sched}-e{epi}-rg{int(rg)}-kg{int(kg)}'
                                          f'-s{int(segs)}-bn{bn}-p{passes}-M{M}-K{K}'))
                i += 1
    return cases


@pytest.mark.parametrize('fam,BN,passes,M,K', _int_matrix())
def test_gemm_integer_exact(ops, fam, BN, passes, M, K):
    layout, sched, epi, rg, kg, segs = fam
    got, ref, names, aux_got, cs_got = run_case(ops, layout, sched, epi, BN, rg, kg, segs, M, K, passes, seed=M * K + BN)
    assert gemm_instantiations(names) == {instantiation(layout, epi)}, names
    _exact_compare(got, ref, gelu=bool(epi & R.EPI_GELU))
    D, _, aux, colsum = ref
    if aux_got is not None:
        live = ~np.isnan(aux[0])
        assert np.array_equal(aux_got[live], aux[0][live]) and np.all(aux_got.view(np.int32)[~live] == np.int32(SENT))
    if cs_got is not None:
        assert np.array_equal(cs_got.astype(np.float64), colsum.reshape(cs_got.shape) if colsum.size == cs_got.size
                              else np.pad(colsum, ((0, cs_got.shape[0] - colsum.shape[0]), (0, 0))))


@pytest.mark.parametrize('layout,passes', [('kk', 3), ('pk', 1), ('pk', 3), ('pmn', 3)])
def test_gemm_more_tiles_than_sms(ops, layout, passes):
    """More than 2x SMs output tiles (persistent loop, smem ring wrapping across tiles); exact integer result."""
    sms = ops.num_sms()
    if layout == 'pmn':
        M, K, bn, sched, epi = 128 * 8, 512, 32, 'splitk', R.EPI_ATOMIC     # 8 x 1 tiles x k_splits
        got, ref, names, _, _ = run_case(ops, layout, sched, epi, bn, False, False, False, M, K, passes, seed=5,
                                         k_splits=2 * sms // 8 + 3)
    else:
        bn = 32 if layout == 'kk' else 128
        M = 128 * (2 * sms // (2 if layout == 'kk' else 1) + 7)
        got, ref, names, _, _ = run_case(ops, layout, 'dense', R.EPI_BIAS if layout == 'pk' else 0, bn, False, False,
                                         False, M, 100, passes, seed=6)
    _exact_compare(got, ref)


# ---- 3. float accuracy --------------------------------------------------------------------------------------------
WORST = {}


@pytest.mark.parametrize('layout,sched,epi', [('kk', 'dense', 0), ('kmn', 'dense', 0), ('pb', 'dense', 0),
                                              ('pk', 'dense', 0), ('mm', 'splitk', R.EPI_ATOMIC),
                                              ('pmn', 'splitk', R.EPI_ATOMIC)])
@pytest.mark.parametrize('K', [4, 36, 64, 256, 1024, 8192])
@pytest.mark.parametrize('passes', [1, 3])
def test_gemm_float_accuracy(ops, layout, sched, epi, K, passes):
    """|got - emulated| <= τ(K) · sum_k |a_k b_k| elementwise; against exact float64, the split term is added.  Inputs:
    N(0, 1), rows scaled by 2^20 / 2^-20, and columns of B that cancel (b_2j+1 = -b_2j + tiny)."""
    rng = np.random.default_rng(K + passes)
    M, BN = 136, 64
    N = BN if layout in ('pb', 'pk', 'pmn') else 2 * BN
    A = rng.standard_normal((M, K)).astype(np.float32)
    A[1::4] *= np.float32(2.0 ** 20)
    A[2::4] *= np.float32(2.0 ** -20)
    B = rng.standard_normal((1, N, K)).astype(np.float32)
    B[0, 1::2] = -B[0, 0::2] + (rng.standard_normal((N // 2, K)) * 1e-3).astype(np.float32)
    k_splits = 1 if sched != 'splitk' else 3
    got, ref, names, _, _ = run_case(ops, layout, sched, epi, BN, False, False, False, M, K, passes, seed=K,
                                     int_data=False, data=(A, B), k_splits=k_splits)
    D, mag, _, _ = ref
    err = np.abs(got.astype(np.float64) - D)
    # atomic split-K: the k_splits partial sums and the initial D are added in fp32, one rounding each of <= |D| + mag
    extra = (k_splits + 1) * U * (np.abs(D) + mag) if epi & R.EPI_ATOMIC else 0.0
    t = tau(K, passes)
    ratio = (err - extra) / (t * mag + 1e-300)
    WORST[(layout, K, passes)] = float(ratio.max())
    assert ratio.max() <= 1.0, f'worst {ratio.max():.3g} of τ(K)'
    # against exact float64 products (D minus the emulated product is the integer initial D of the atomic cases)
    exact64 = A.astype(np.float64) @ B[0].T.astype(np.float64) + (D[0] - R.split_product(A, B[0], passes))
    assert np.all(np.abs(got - exact64) <= (t + split_err(passes)) * mag + extra + 1e-300)
    print(f'float accuracy {layout} K={K} passes={passes}: worst err / (τ(K)·Σ|ab|) = {ratio.max():.3g}')


# ---- 4. packed split-K segments -----------------------------------------------------------------------------------
def test_packed_splitk_segment_precondition(ops):
    """The fully packed split-K path bulk-copies whole 32-row k-blocks from k_begin / 32, so it needs seg_begin % 32 == 0
    and reads the rows [seg_end, ceil32(seg_end)) too (the generic path masks them).  With the rows past each segment
    zero in A the two paths agree exactly; with them nonzero in both operands the packed result includes them."""
    rng = np.random.default_rng(11)
    M, N, K = 128, 64, 256
    A = rng.integers(-3, 4, (M, K)).astype(np.float32)
    X = rng.integers(-3, 4, (K, N)).astype(np.float32)
    seg_b = np.array([0, 64, 160], dtype=np.int32)
    seg_e = np.array([45, 64, 237], dtype=np.int32)
    live = np.zeros(K, dtype=bool)
    for b, e in zip(seg_b, seg_e):
        live[b:e] = True

    def run(A_, packed):
        lda, ldb = M + 4, N + 4
        At, Xb = nan_buffer(A_.T, lda), nan_buffer(X, ldb)
        D = torch.zeros((3, M, N), device='cuda')
        kw = dict(a_smn=1, a_sk=lda, b_smn=1, b_sk=ldb, M=M, N=N, K=K, D=D, ldd=N, d_group_stride=M * N,
                  sched=ops.SCHED_SPLITK, k_splits=2, num_groups=3, seg_begin=torch.from_numpy(seg_b).cuda(),
                  seg_end=torch.from_numpy(seg_e).cuda(), epilogue=ops.EPI_ATOMIC)
        if packed:
            kw.update(A=None, B=None, a_packed=ops.pack_act(At, rows=K, cols=M, mn_major=True, tile=128, ld=lda),
                      b_packed=ops.pack_act(Xb, rows=K, cols=N, mn_major=True, tile=64, ld=ldb))
        else:
            kw.update(A=At, B=Xb)
        ops.gemm(**kw)
        return D.cpu().numpy().astype(np.float64)

    want = np.stack([A[:, b:e].astype(np.float64) @ X[b:e].astype(np.float64) for b, e in zip(seg_b, seg_e)])
    A0 = np.where(live[None], A, 0).astype(np.float32)
    assert np.array_equal(run(A0, True), want) and np.array_equal(run(A0, False), want)
    # precondition violated: the generic path still masks, the packed one sums up to the next multiple of 32
    assert np.array_equal(run(A, False), want)
    ceil = [min(K, -(-int(e) // 32) * 32) if e > b else e for b, e in zip(seg_b, seg_e)]
    want_packed = np.stack([A[:, b:e].astype(np.float64) @ X[b:e].astype(np.float64) for b, e in zip(seg_b, ceil)])
    assert np.array_equal(run(A, True), want_packed) and not np.array_equal(want_packed, want)


def _precondition_recorder(monkeypatch, ops, seen):
    """Wrap ops.linear_wgrad: for every segmented call record whether seg_begin % 32 == 0 and whether one operand is
    zero on the rows [seg_end, ceil32(seg_end)) of each group."""
    orig = ops.linear_wgrad

    def rows_zero(t, packed, rows, cols, tile, r0, r1, row_index=None):
        if r1 <= r0:
            return True
        if packed is not None:
            h, l = R.decode_mn(packed, -(-rows // 32) * 32, -(-cols // tile) * tile, tile)
            return not h[r0:r1].any() and not l[r0:r1].any()
        if row_index is not None:
            return bool((row_index[r0:r1].cpu() < 0).all()) or not t[row_index[r0:r1].clamp(min=0).long()].any()
        return not t[r0:r1].any()

    def wrapped(dy, x, dw, *, rows=None, x_row_index=None, row_scale=None, segs=None, num_groups=1, dy_packed=None,
                x_packed=None):
        if segs is not None:
            torch.cuda.synchronize()
            R_ = rows if rows is not None else dy.shape[0]
            N, K = dw.shape[-2], dw.shape[-1]
            sb, se = segs[0].cpu().numpy(), segs[1].cpu().numpy()
            for b, e in zip(sb, se):
                c = min(-(-int(e) // 32) * 32, -(-R_ // 32) * 32)
                ok = rows_zero(dy, dy_packed, R_, N, 128, int(e), c) or \
                    rows_zero(x, x_packed, R_, K, ops._pick_bn(K), int(e), c, x_row_index)
                seen.append((int(b) % 32 == 0, ok))
        return orig(dy, x, dw, rows=rows, x_row_index=x_row_index, row_scale=row_scale, segs=segs,
                    num_groups=num_groups, dy_packed=dy_packed, x_packed=x_packed)

    monkeypatch.setattr(ops, 'linear_wgrad', wrapped)


def test_segmented_wgrad_callers_meet_precondition(ops, monkeypatch):
    """MoE ConvNeXt blocks and the LSK MoE layer, forward + backward: every segmented wgrad starts its segments on a
    multiple of 32 and has one operand zero past each segment end.  The expert-parallel plan gathers -1 (zero rows) for
    every padding slot of its segments."""
    import os
    import sys
    seen = []
    _precondition_recorder(monkeypatch, ops, seen)
    _train_steps(kinds=('moe', 'lsk'), amp=(False,), cp=(False,))
    assert seen and all(a for a, _ in seen) and all(b for _, b in seen), seen
    # expert-parallel plan (device kernel, one device): padding slots of each owned segment gather nothing
    sys.path.insert(0, os.path.join(os.path.dirname(__file__), 'dist'))
    from ep_plan_worker import local_plan
    from sm3det_b200.expert_parallel import EPContext, device_plan
    W, E, k, T = 2, 8, 2, 700
    plans = [local_plan(torch.randn(T, E, generator=torch.Generator().manual_seed(40 + r)).topk(k, dim=1).indices, E)
             for r in range(W)]
    allm = torch.stack([torch.stack([p[0], p[1]]) for p in plans]).to(torch.int32)
    counts, seg_begin, tile_group, num_tiles, pair_token, slot_of = plans[0]
    ctx = EPContext.__new__(EPContext)
    ctx.world, ctx.rank = W, 0
    ctx.overflow = torch.zeros(1, device='cuda', dtype=torch.int32)
    tg = tile_group.clone()
    tg[tg == 12345] = 0
    cap = (T * k * W // 128 + E + 3) * 128
    P = device_plan(ctx, allm.cuda(), tg.cuda(), num_tiles.cuda(), pair_token.cuda(), E, pair_token.numel(), cap)
    sb, se, src = P['seg_begin'].cpu(), P['seg_end'].cpu(), P['src_rank'].cpu()
    assert (sb % 32 == 0).all()
    for b, e in zip(sb.tolist(), se.tolist()):
        assert (src[e:-(-e // 32) * 32] == -1).all()


# ---- 5. fused FFN -------------------------------------------------------------------------------------------------
# smem arithmetic of csrc/ffn_fused.cu (chain_layout / pick_chain), restated to know which layouts exist
SMEM_LIMIT = 232448 - 1024
CAND = ((64, 2, 2), (32, 2, 2), (64, 2, 1), (32, 2, 1), (32, 1, 1))


def chain_fits(mode, C, HC, sa, sb):
    nA = 2 if mode == 1 else 1
    a_tile = C // 32 * 16384
    wa_stage = nA * (C // 32) * HC * 128
    wb_stage = HC // 32 * C * 128
    total = nA * a_tile + sa * wa_stage + sb * wb_stage + HC // 32 * 16384 + 8 * 32 * 20 * 4 + 256 + 1024
    return total <= SMEM_LIMIT + 1024


def chain_layout(mode, C, HC_req=0):
    if C % 32 or C < 32 or C > 256:
        return None
    for c in CAND:
        if (HC_req in (0, c[0])) and chain_fits(mode, C, *c):
            return c
    return None


def test_ffn_chunk_table(ops):
    """ffn_chunk(0, C) is the chunk of the forward layouts below; C = 256 and non-multiples of 32 are unsupported and the
    launcher rejects them without launching; the backward-into-dv mode fits C <= 128."""
    table = {32: (64, 2, 2), 64: (64, 2, 2), 96: (64, 2, 2), 128: (32, 2, 2), 160: (32, 2, 2), 192: (32, 2, 1),
             224: (32, 1, 1)}
    for C in range(16, 300, 16):
        want = table.get(C)
        assert chain_layout(0, C) == want, C
        assert ops.ffn_chunk(0, C) == (want[0] if want else 0), C
        assert (ops.ffn_chunk(1, C) > 0) == (C % 32 == 0 and 32 <= C <= 128), C
    for C in (256, 48, 200):
        T = 130
        z = torch.zeros(1 << 20, dtype=torch.int16, device='cuda')
        b = torch.zeros(4 * C, device='cuda')
        names, exc = kernels_run(lambda: _raises(lambda: ops.ffn_fused_fwd(z, z, z, b, b[:C], T=T, C=C, chunk=32)))
        assert exc is not None and not any('ffn_chain_kernel' in n for n in names), C


def _raises(fn):
    try:
        fn()
    except RuntimeError as e:
        return e
    return None


def ffn_cases():
    cases = []
    for C in (32, 64, 96, 128, 160, 192, 224):
        for HC in (32, 64):
            if chain_layout(0, C, HC) is None:
                continue
            for passes in (1, 3):
                cases.append(pytest.param(C, HC, passes, id=f'C{C}-HC{HC}-p{passes}'))
    return cases


def ffn_bounds(v, W1, b1, W2, b2, passes):
    """float64 reference and elementwise error bounds of h (= v W1^T + b1), y2 (= gelu(h) W2^T + b2)."""
    v64, W164, W264 = v.astype(np.float64), W1.astype(np.float64), W2.astype(np.float64)
    hs = R.split_product(v, W1, passes) + b1                       # GEMM-a on the split operands, exact
    magh = np.abs(v64) @ np.abs(W164).T
    C = v.shape[1]
    # h: fp32 accumulation (τ) + one rounding for + b1
    eh_emul = tau(C, passes) * magh + U * (np.abs(hs) + np.abs(b1))
    h64 = v64 @ W164.T + b1
    eh = eh_emul + split_err(passes) * magh                        # against exact float64
    a64 = R.gelu64(h64)
    # a = gelu_fast(h_fp32): propagated h error (|gelu'| <= 1.13), the fast GELU, then the in-kernel split of a and W2
    ea = 1.13 * eh + gelu_bound(h64 + np.sign(h64) * eh)
    H4 = W2.shape[1]
    mag2 = (np.abs(a64) + ea) @ np.abs(W264).T
    y64 = a64 @ W264.T + b2
    ey = ea @ np.abs(W264).T + (split_err(passes) + tau(H4, passes)) * mag2 + U * (np.abs(y64) + np.abs(b2))
    return hs, eh_emul, y64, ey


@pytest.mark.parametrize('C,HC,passes', ffn_cases())
def test_fused_ffn_forward(ops, C, HC, passes):
    """ffn_chain_kernel forward at every supported C and chunk width, passes 1 and 3, M tails and more tiles than SMs:
    h_out against the emulated GEMM-a (tight bound), aux = y2 and out = resid + row_scale * gamma * y2 against float64
    with the bound of ffn_bounds; NaN past M in v, resid and row_scale is never read."""
    from sm3det_b200.ops import precision_scope
    sms = ops.num_sms()
    rng = np.random.default_rng(C * HC + passes)
    for M in (1, 127, 129, 2 * sms * 128 + 77) if C in (64, 192) and HC == 32 else (129, 300):
        v = rng.standard_normal((M, C)).astype(np.float32)
        W1 = (rng.standard_normal((4 * C, C)) / math.sqrt(C)).astype(np.float32)
        b1 = (rng.standard_normal(4 * C) * 0.2).astype(np.float32)
        W2 = (rng.standard_normal((C, 4 * C)) / math.sqrt(4 * C)).astype(np.float32)
        b2 = (rng.standard_normal(C) * 0.2).astype(np.float32)
        gamma = (rng.random(C) + 0.1).astype(np.float32)
        rs = np.exp2(rng.integers(-1, 2, M)).astype(np.float32)
        rs[::4] = 0
        resid = rng.standard_normal((M, C)).astype(np.float32)
        vd = nan_buffer(v, C)
        v_img = ops.pack_act(vd, rows=M, cols=C, mn_major=False)
        w1c, _ = ops.pack_weight(torch.from_numpy(W1).cuda(), transposed=False, tile=HC)
        w2n, _ = ops.pack_weight(torch.from_numpy(W2).cuda(), transposed=False, tile=C)
        dev = lambda x: torch.from_numpy(x).cuda()
        resid_d = nan_buffer(resid, C)[:M * C].view(M, C)
        rs_d = nan_buffer(rs[None], M)[:M]
        with precision_scope(passes):
            names, (out, aux, h) = kernels_run(lambda: ops.ffn_fused_fwd(
                v_img, w1c, w2n, dev(b1), dev(b2), T=M, C=C, chunk=HC, gamma=dev(gamma), row_scale=rs_d, resid=resid_d,
                want_aux=True, want_h=True))
        assert any(f'ffn_chain_kernel<0, {HC}, {C}>' in n for n in names), names
        hs, eh, y64, ey = ffn_bounds(v, W1, b1, W2, b2, passes)
        h, aux, out = (t.cpu().numpy().astype(np.float64) for t in (h, aux, out))
        assert not np.isnan(out).any() and not np.isnan(aux).any() and not np.isnan(h).any()
        assert np.all(np.abs(h - hs) <= eh), f'h: worst {np.max(np.abs(h - hs) / eh):.3g} of its bound'
        assert np.all(np.abs(aux - y64) <= ey), f'aux: worst {np.max(np.abs(aux - y64) / ey):.3g} of its bound'
        s = np.abs(gamma.astype(np.float64))[None] * rs[:, None]
        o64 = y64 * gamma * rs[:, None] + resid
        eo = s * ey + 3 * U * (s * np.abs(y64) + np.abs(o64))
        assert np.all(np.abs(out - o64) <= eo), f'out: worst {np.max(np.abs(out - o64) / eo):.3g} of its bound'
        print(f'fused ffn C={C} HC={HC} passes={passes} M={M}: h {np.max(np.abs(h - hs) / eh):.3g}, '
              f'aux {np.max(np.abs(aux - y64) / ey):.3g} of bound')


@pytest.mark.parametrize('C', [32, 64, 96, 128])
@pytest.mark.parametrize('passes', [1, 3])
def test_fused_ffn_backward_dv(ops, C, passes):
    """Mode 1 (dv = ((dz gamma W2) * gelu'(v W1^T + b1)) W1) at every C it accepts, against float64."""
    from sm3det_b200.ops import precision_scope
    rng = np.random.default_rng(C + passes)
    M = 300
    cb = ops.ffn_chunk(1, C)
    v = rng.standard_normal((M, C)).astype(np.float32)
    dz = rng.standard_normal((M, C)).astype(np.float32)
    W1 = (rng.standard_normal((4 * C, C)) / math.sqrt(C)).astype(np.float32)
    b1 = (rng.standard_normal(4 * C) * 0.2).astype(np.float32)
    W2g = (rng.standard_normal((C, 4 * C)) / math.sqrt(4 * C)).astype(np.float32)
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()
    v_img = ops.pack_act(dev(v), rows=M, cols=C, mn_major=False)
    dz_img = ops.pack_act(dev(dz), rows=M, cols=C, mn_major=False)
    w1cb, _ = ops.pack_weight(dev(W1), transposed=False, tile=cb)
    w2gt, _ = ops.pack_weight(dev(W2g), transposed=True, tile=cb)
    w1tn, _ = ops.pack_weight(dev(W1), transposed=True, tile=C)
    with precision_scope(passes):
        dv = ops.ffn_fused_bwd(v_img, dz_img, w1cb, w2gt, w1tn, dev(b1), T=M, C=C, chunk=cb).cpu().numpy()
    v64, dz64, W164, W2g64 = (x.astype(np.float64) for x in (v, dz, W1, W2g))
    h = v64 @ W164.T + b1
    d = dz64 @ W2g64
    y = d * R.gelu_grad64(h)
    want = y @ W164
    s = split_err(passes) + tau(C, passes)
    eh = s * (np.abs(v64) @ np.abs(W164).T) + U * np.abs(h)
    ed = s * (np.abs(dz64) @ np.abs(W2g64)) + U * np.abs(d)
    # y error: d's error times |gelu'| <= 1.13, |d| times (|gelu''| <= 0.8 times h's error + the fast GELU' bound)
    ey = 1.13 * ed + (np.abs(d) + ed) * (0.8 * eh + gelu_grad_bound(h)) + U * np.abs(y)
    ev = ey @ np.abs(W164) + (split_err(passes) + tau(4 * C, passes)) * ((np.abs(y) + ey) @ np.abs(W164))
    assert np.all(np.abs(dv - want) <= ev), f'worst {np.max(np.abs(dv - want) / ev):.3g} of the bound'


# ---- 6. census ----------------------------------------------------------------------------------------------------
def _train_steps(kinds, amp, cp):
    """Short forward + backward passes of mini backbones (dense / MoE ConvNeXt, LSK), in fp32 and / or under autocast,
    with and without activation checkpointing."""
    from oracle.convnext_moe_oracle import OracleConfig, param_shapes
    from sm3det_b200 import ConvNeXt_moe_MultiInput
    from sm3det_b200.synth import make_images, make_state_dict
    x = make_images(2, 64, 64, seed=3).cuda()
    for kind in kinds:
        for use_amp in amp:
            for with_cp in cp:
                if kind in ('dense', 'moe'):
                    kw = dict(arch=dict(depths=[1, 1, 2, 1], channels=[32, 64, 96, 128]),
                              MoE_Block_inds=[[], [], [], []] if kind == 'dense' else [[], [0], [0, 1], [0]],
                              num_experts=4, top_k=2, noisy_gating=False)
                    net = ConvNeXt_moe_MultiInput(**kw, with_cp=with_cp)
                    net.load_state_dict(make_state_dict(param_shapes(OracleConfig(**kw)), 0, True), strict=True)
                    net = net.cuda().train()
                elif with_cp:
                    continue                  # the LSK backbone has no activation checkpointing
                else:
                    from oracle.cases import LSK_CASES
                    from test_lsk_gpu import build
                    _, _, net = build(LSK_CASES['lsk_mini_moe_e4k2_train_clean']['kw'])
                    net.train()
                with torch.autocast('cuda', dtype=torch.bfloat16, enabled=use_amp):
                    res = net(x)
                # backbones without MoE blocks return the feature maps alone
                outs, loss = res if isinstance(res, tuple) and len(res) == 2 and torch.is_tensor(res[1]) else (res, 0.0)
                (sum(o.float().square().mean() for o in outs) + loss).backward()
                torch.cuda.synchronize()


def test_launch_census(ops, monkeypatch):
    """Every GEMM and fused-FFN launch the backbones make has a signature the launch matrix and the fused-FFN tests
    cover, so a new kind of launch cannot go untested."""
    seen, ffn_seen = set(), set()
    orig_gemm, orig_ffn = ops.gemm, ops.ffn_fused_fwd

    def gemm(**kw):
        a_mn = kw['a_smn'] == 1 and kw['a_sk'] != 1
        apk, bpk = kw.get('a_packed') is not None, kw.get('b_packed') is not None
        b_mn = a_mn if apk else (False if bpk else (kw['b_smn'] == 1 and kw['b_sk'] != 1))
        layout = {(False, False, False, False): 'kk', (False, True, False, False): 'kmn', (False, False, True, False): 'pb',
                  (False, False, True, True): 'pk', (True, True, False, False): 'mm', (True, True, True, True): 'pmn'}[
            (a_mn, b_mn, bpk, apk)]
        sched = {0: 'dense', 1: 'grouped', 2: 'splitk'}[kw.get('sched', 0)]
        BN = kw.get('tile_n') or ops._pick_bn(kw['N'])
        seen.add(signature(layout, sched, kw.get('epilogue', 0), BN, kw.get('a_row_index') is not None,
                           kw.get('b_k_index') is not None, kw.get('seg_begin') is not None, ops.current_passes()))
        return orig_gemm(**kw)

    def ffn(*a, **kw):
        ffn_seen.add((kw['C'], kw['chunk'], ops.current_passes()))
        return orig_ffn(*a, **kw)

    monkeypatch.setattr(ops, 'gemm', gemm)
    monkeypatch.setattr(ops, 'ffn_fused_fwd', ffn)
    _train_steps(kinds=('dense', 'moe', 'lsk'), amp=(False, True), cp=(False, True))
    missing = sorted(seen - COVERED, key=str)
    assert seen and not missing, f'launch signatures the matrix does not cover: {missing}'
    ffn_covered = {(c.values[0], c.values[1], c.values[2]) for c in ffn_cases()}
    assert ffn_seen and ffn_seen <= ffn_covered, sorted(ffn_seen - ffn_covered)
