"""GEMM column tails: outputs whose width N is a multiple of 8 but not of the tile width (csrc/gemm_tc.cuh, Params).

The last N-tile runs padded to its tile width and masked, so these must hold on every launch path:
1. pick_bn / ops._pick_bn: unchanged for N % 32 == 0, the fewest tiles and then the least padding otherwise (CPU).
2. pack_b images of a tail width are bit-exact and their padding rows are zero, whatever the buffer held before.
3. The launch matrix of tests/test_gemm_gpu.py (every layout, schedule and epilogue flag, both precision modes) on
   integer operands at N in {8, 16, 24, 48, 80, 112, 144, 208, 336}: the exact integer result, and no byte of D past
   column N or past the last row, of aux_out, or of colsum past N changes.  Operands, bias, col_scale and resid lie in
   NaN-padded buffers.
4. Float accuracy under the τ(K) bound of tests/test_gemm_gpu.py.
5. A census: every GEMM launch of an LSKNet-T training step (16- and 80-wide LSK attention convs) has a signature that
   the matrix here or the one of tests/test_gemm_gpu.py runs.
"""
import os

import numpy as np
import pytest
import torch

import gemm_ref as R
import test_gemm_gpu as G

TAIL_N = (8, 16, 24, 48, 80, 112, 144, 208, 336)
GOLD_T = os.path.join(os.path.dirname(__file__), 'golden', 'lsk_t')
gpu = pytest.mark.gpu


@pytest.fixture(scope='module')
def ops():
    from sm3det_b200 import ops as o
    return o


def _old_pick_bn(n):
    return next(bn for bn in (128, 96, 64, 32) if n % bn == 0)


# ---- 1. tile choice (CPU) -----------------------------------------------------------------------------------------
def test_pick_bn_rule_and_c_mirror():
    from sm3det_b200 import _lib, ops
    lib = _lib.load()
    for n in range(32, 4097, 32):                     # every existing launch keeps its tile width and image size
        assert ops._pick_bn(n) == lib.sm3_gemm_tile_n(n) == _old_pick_bn(n), n
        assert lib.sm3_gemm_packed_elems(n, 100) == n * 128 * 2, n
    for n in range(8, 4097, 8):
        bn = ops._pick_bn(n)
        assert lib.sm3_gemm_tile_n(n) == bn, n
        if n % 32:
            best = min((-(-n // b), -(-n // b) * b) for b in (128, 96, 64, 32))
            assert (-(-n // bn), -(-n // bn) * bn) == best, n
            assert lib.sm3_gemm_packed_elems(n, 40) == -(-n // bn) * bn * 64 * 2, n
    assert {n: ops._pick_bn(n) for n in (16, 80, 144, 336)} == {16: 32, 80: 96, 144: 96, 336: 128}
    for n in (4, 12, 100):
        assert lib.sm3_gemm_tile_n(n) == 0
        with pytest.raises(ValueError):
            ops._pick_bn(n)


# ---- 2. pack_b images ---------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize('N', TAIL_N)
@pytest.mark.parametrize('K', [4, 36, 100])
@pytest.mark.parametrize('transposed', [False, True])
def test_pack_b_tail_image_bit_exact(ops, N, K, transposed):
    """Rows [N, ceil(N / BN) BN) of every group's image are zero although the buffer was NaN-filled before packing."""
    rng = np.random.default_rng(N * K + transposed)
    groups = 2
    w = G._special_values(rng, (groups, N, K) if not transposed else (groups, K, N))
    BN = ops._pick_bn(N)
    Np, Kp = -(-N // BN) * BN, -(-K // 32) * 32
    per = Np * Kp * 2
    out = torch.full((groups * per,), -1, dtype=torch.int16, device='cuda')     # 0xFFFF: a bf16 NaN in every plane
    img, per_got = ops.pack_weight(torch.from_numpy(w).cuda(), transposed=transposed, groups=groups, out=out)
    assert per_got == per and img.data_ptr() == out.data_ptr()
    B = w if not transposed else w.transpose(0, 2, 1)
    for g in range(groups):
        h, l = R.decode_k(img[g * per:(g + 1) * per], Np, Kp, BN)
        eh, el = R.split_bits(np.pad(B[g], ((0, Np - N), (0, Kp - K))))
        assert np.array_equal(h, eh) and np.array_equal(l, el), g


# ---- 3. integer-exact launch matrix -------------------------------------------------------------------------------
# the families of tests/test_gemm_gpu.py, plus GELU' (the dgrad through GELU) on the fp32 and the packed path
FAMILIES = G.FAMILIES + [
    ('kk', 'dense', R.EPI_DGELU | R.EPI_BIAS | R.EPI_COLSUM, False, False, False),
    ('pb', 'dense', R.EPI_DGELU | R.EPI_COLSCALE | R.EPI_RESID, False, False, False),
    ('pk', 'dense', R.EPI_DGELU | R.EPI_COLSUM, False, False, False),
    ('pk', 'dense', R.EPI_BIAS | R.EPI_GELU, False, False, False),       # LSK Attention.proj_1 (GELU fused)
    ('kmn', 'dense', R.EPI_RESID, False, False, False),
]
def _bn(n):
    for bn in (128, 96, 64, 32):
        if n % bn == 0:
            return bn
    return min((128, 96, 64, 32), key=lambda b: (-(-n // b), -(-n // b) * b))


COVERED = {G.signature(f[0], f[1], f[2], _bn(n), f[3], f[4], f[5], p) for f in FAMILIES for n in TAIL_N for p in (1, 3)}


def run_tail(ops, layout, sched, epi, N, row_gather, k_gather, segs, M, K, passes, seed, data=None, k_splits=None,
             profile=False):
    """One launch of output width N (tile width pick_bn(N)) on NaN-padded operands and sentinel-filled outputs, as
    tests/test_gemm_gpu.py: run_case.  Returns (D [G, M, N], reference tuple, kernel names, aux_out, colsum); the kernel
    names come from the profiler and only with `profile` (one profiled launch per family keeps the profiler sessions of
    this file few: the suite's later tests read kernel names from the profiler too)."""
    rng = np.random.default_rng(seed)
    a_mn = layout in ('mm', 'pmn')
    packed = layout in ('pk', 'pmn')
    BN = ops._pick_bn(N)
    Gn = 3 if sched == 'grouped' or segs else 1
    ints = lambda shape: rng.integers(-3, 4, shape).astype(np.float32)
    gen = ints if data is None else None
    kw = dict(M=M, N=N, K=K, sched=G.SCHED[sched], epilogue=epi, tile_n=0)
    ref_kw = dict(passes=passes, epi=epi)
    src_rows = M + 5 if row_gather else M
    A_src = gen((src_rows, K)) if data is None else data[0]
    if row_gather:
        ri = rng.integers(-1, src_rows, M).astype(np.int32)
        ri[::3] = -1
        ref_kw['a_row_index'] = ri
    A_logical = A_src
    if sched == 'grouped':
        m_tiles = -(-M // 128)
        nt = max(1, m_tiles - 1)
        tg = rng.integers(0, Gn, m_tiles + 2).astype(np.int32)
        tg[nt:] = 1000 + np.arange(tg.size - nt)
        ref_kw.update(tile_group=tg, num_m_tiles=nt)
        kw.update(tile_group=torch.from_numpy(tg).cuda(), num_m_tiles=torch.tensor([nt], dtype=torch.int32).cuda())
    if segs:
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
        kw.update(seg_begin=torch.from_numpy(seg_b).cuda(), seg_end=torch.from_numpy(seg_e).cuda(), num_groups=Gn)
    if sched == 'splitk':
        if k_splits is None:
            k_splits = 3 if (epi & R.EPI_ATOMIC) else 1
        kw.update(k_splits=k_splits, num_groups=Gn)
    Gb = Gn if sched == 'grouped' else 1
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
        At = G.nan_buffer(A_logical.T, lda)
        kw.update(a_smn=1, a_sk=lda)
        if packed:
            kw.update(A=None, a_packed=ops.pack_act(At, rows=K, cols=M, mn_major=True, tile=128, ld=lda))
        else:
            kw['A'] = At
    else:
        lda = K + 4
        Ab = G.nan_buffer(A_src, lda)
        kw.update(a_smn=lda, a_sk=1)
        if packed:
            ridx = None if not row_gather else torch.from_numpy(ref_kw['a_row_index']).cuda()
            kw.update(A=None, a_packed=ops.pack_act(Ab, rows=M, cols=K, mn_major=False, tile=128, ld=lda, row_index=ridx))
        else:
            kw['A'] = Ab
    if layout == 'kk':
        ldb = Kb + 4
        Bb = G.nan_buffer(B_src.reshape(Gb * N, Kb), ldb, extra_rows=2)
        kw.update(B=Bb, b_smn=ldb, b_sk=1, b_group_stride=N * ldb if Gb > 1 else 0)
    elif layout in ('kmn', 'mm'):
        ldb = N + 4                                          # NaN columns right after column N
        Bt = np.concatenate([np.pad(B_src[g].T, ((0, 1), (0, 0))) for g in range(Gb)])
        Bb = G.nan_buffer(Bt, ldb)
        kw.update(B=Bb, b_smn=1, b_sk=ldb, b_group_stride=(Kb + 1) * ldb if Gb > 1 else 0)
    elif layout in ('pb', 'pk'):
        wb = G.nan_buffer(B_src.reshape(Gb * N, Kb), Kb, extra_rows=2)
        img, per = ops.pack_weight(wb[:Gb * N * Kb].view(Gb, N, Kb), transposed=False, groups=Gb)
        kw.update(B=None, b_packed=img, b_packed_group_stride=per, b_smn=Kb, b_sk=1)
        keep.append(wb)
    else:   # pmn
        ldb = N + 4
        xb = G.nan_buffer(B_src[0].T, ldb)
        kw.update(B=None, b_packed=ops.pack_act(xb, rows=K, cols=N, mn_major=True, tile=BN, ld=ldb), b_smn=1, b_sk=ldb)
    Gd = Gn if segs or (sched == 'splitk' and Gn > 1) else 1
    ldd = N + 40                                             # D columns [N, ldd) and rows past M hold sentinels
    d_init = ints((Gd * M, N)) if epi & R.EPI_ATOMIC else None
    D = G.sentinel_buffer(Gd * M, N, ldd, init=d_init)
    kw.update(D=D, ldd=ldd, d_group_stride=M * ldd if Gd > 1 else 0)
    ref_kw['d_init'] = None if d_init is None else d_init.reshape(Gd, M, N)
    if epi & R.EPI_BIAS:
        bs = N + 4
        bias = ints((Gb, N))
        kw.update(bias=G.nan_buffer(bias, bs), bias_group_stride=bs)
        ref_kw['bias'] = bias
    ld_aux = N + 40
    if epi & (R.EPI_AUXSTORE | R.EPI_GELU):
        kw.update(aux_out=G.sentinel_buffer(M, N, ld_aux), ld_aux=ld_aux)
    if epi & R.EPI_DGELU:
        ai = (rng.standard_normal((M, N)) * 2).astype(np.float32)
        kw.update(aux_in=G.nan_buffer(ai, ld_aux), ld_aux=ld_aux)
        ref_kw['aux_in'] = ai
    if epi & R.EPI_COLSCALE:
        cs = np.exp2(rng.integers(-2, 3, N)).astype(np.float32)
        cs[::7] = 0
        kw['col_scale'] = G.nan_buffer(cs[None], N)
        ref_kw['col_scale'] = cs
    if epi & R.EPI_ROWSCALE:
        rs = np.exp2(rng.integers(-2, 3, M)).astype(np.float32)
        rs[::5] = 0
        kw['row_scale'] = G.nan_buffer(rs[None], M)
        ref_kw['row_scale'] = rs
    if epi & R.EPI_RESID:
        ld_r = N + 4
        res = ints((M, N))
        kw.update(resid=G.nan_buffer(res, ld_r), ld_resid=ld_r)
        ref_kw['resid'] = res
    ncs = 0
    if epi & R.EPI_COLSUM:
        ncs = Gb
        kw.update(colsum=G.sentinel_buffer(ncs, N, N, init=np.zeros((ncs, N))), colsum_group_stride=N)   # N floats, then sentinels
    ref = R.gemm_ref(A_logical if a_mn else A_src, B_src, **ref_kw)
    if epi & R.EPI_DGELU:
        # GELU' is the one inexact step: keep its input (accumulator + bias) and the factors applied after it
        pre_kw = {k: v for k, v in ref_kw.items() if k not in ('aux_in', 'col_scale', 'row_scale', 'resid', 'd_init')}
        pre = R.gemm_ref(A_logical if a_mn else A_src, B_src, **dict(pre_kw, epi=epi & R.EPI_BIAS))[0]
        scale = np.ones((1, 1, N))
        if epi & R.EPI_COLSCALE:
            scale = scale * ref_kw['col_scale'].reshape(1, 1, N)
        if epi & R.EPI_ROWSCALE:
            scale = scale * ref_kw['row_scale'].reshape(1, M, 1)
        ref = ref + (dict(pre=pre, scale=scale, aux_in=ref_kw['aux_in'], resid=ref_kw.get('resid', 0.0)),)
    from sm3det_b200.ops import precision_scope
    outs = [t for t in (D, kw.get('aux_out'), kw.get('colsum')) if t is not None]
    snap = [t._base.clone() for t in outs]

    def restore():
        for t, s_ in zip(outs, snap):
            t._base.copy_(s_)
    with precision_scope(passes):
        if profile:
            names, _ = G.kernels_run(lambda: ops.gemm(**kw), restore)
        else:
            names = None
            ops.gemm(**kw)
            torch.cuda.synchronize()
    got = G.check_sentinels(D, Gd * M, N, ldd, 'D').reshape(Gd, M, N)
    aux_got = G.check_sentinels(kw['aux_out'], M, N, ld_aux, 'aux_out') if 'aux_out' in kw else None
    cs_got = G.check_sentinels(kw['colsum'], ncs, N, N, 'colsum') if ncs else None
    return got, ref, names, aux_got, cs_got


def _tail_matrix():
    cases = []
    i = 0
    for fam in FAMILIES:
        layout, sched, epi, rg, kg, segs = fam
        for N in TAIL_N:
            for passes in (1, 3):
                if layout in ('mm', 'pmn'):
                    M, K = (128, 136, 40)[i % 3], (100, 200, 300)[i % 3]
                else:
                    M, K = (1, 127, 129, 200)[i % 4], (4, 36, 48, 100)[(i // 4) % 4]
                    if sched == 'grouped':
                        M = (300, 257, 384)[i % 3]
                cases.append(pytest.param(fam, N, passes, M, K, id=f'{layout}-{sched}-e{epi}-rg{int(rg)}-kg{int(kg)}'
                                          f'-s{int(segs)}-N{N}-p{passes}-M{M}-K{K}'))
                i += 1
    return cases


def _check_exact(got, ref, aux_got, cs_got, epi):
    G._exact_compare(got, ref, gelu=bool(epi & R.EPI_GELU))
    D, _, aux, colsum = ref
    if aux_got is not None:
        live = ~np.isnan(aux[0])
        assert np.array_equal(aux_got[live], aux[0][live]) and np.all(aux_got.view(np.int32)[~live] == np.int32(G.SENT))
    if cs_got is not None:
        want = colsum if colsum.shape[0] == cs_got.shape[0] else np.pad(colsum, ((0, cs_got.shape[0] - colsum.shape[0]), (0, 0)))
        assert np.array_equal(cs_got.astype(np.float64), want)


def _check_dgelu(got, ref, cs_got):
    """EPI_DGELU multiplies the exact integer accumulator (+ bias) by the fast GELU', so D is exact up to |x| times the
    GELU' bound of tests/test_gemm_gpu.py times the later scales, plus one rounding per later step (resid, store)."""
    D, _, _, colsum, x = ref
    live = ~np.isnan(D)
    assert np.all(got.view(np.int32)[~live] == np.int32(G.SENT)), 'rows the schedule skips were written'
    assert not np.isnan(got[live]).any(), 'NaN in D'
    bound = (np.abs(x['pre']) * np.abs(x['scale']) * G.gelu_grad_bound(x['aux_in'])[None]
             + 3 * G.U * (np.abs(D) + np.abs(x['resid'])))
    assert np.all(np.abs(got[live] - D[live]) <= bound[live])
    if cs_got is not None:
        rows = live[0].all(axis=1)
        cb = bound[0][rows].sum(0) + rows.sum() * G.U * np.abs(D[0][rows]).sum(0) + 1e-30
        assert np.all(np.abs(cs_got[0].astype(np.float64) - colsum[0]) <= cb)


@gpu
@pytest.mark.parametrize('fam,N,passes,M,K', _tail_matrix())
def test_gemm_tail_integer_exact(ops, fam, N, passes, M, K):
    layout, sched, epi, rg, kg, segs = fam
    got, ref, names, aux_got, cs_got = run_tail(ops, layout, sched, epi, N, rg, kg, segs, M, K, passes, seed=M * K + N,
                                                profile=(N == 16))
    if names is not None:
        assert G.gemm_instantiations(names) == {G.instantiation(layout, epi)}, names
    if epi & R.EPI_DGELU:
        _check_dgelu(got, ref, cs_got)
        return
    _check_exact(got, ref, aux_got, cs_got, epi)


@gpu
@pytest.mark.parametrize('layout,epi', [('kk', R.EPI_COLSUM | R.EPI_BIAS), ('pk', R.EPI_COLSUM)])
def test_gemm_tail_global_colsum(ops, layout, epi):
    """N > 3072 takes the global-atomic column-sum variant: padding columns of the last tile must not reach colsum[N:]."""
    N = 3080                                                 # 24 tiles of 128 + a 8-column tail
    got, ref, names, aux_got, cs_got = run_tail(ops, layout, 'dense', epi, N, False, False, False, 130, 36, 3, seed=9)
    _check_exact(got, ref, aux_got, cs_got, epi)


@gpu
def test_gemm_tail_explicit_tile(ops):
    """An explicit tile width that does not divide N (tile_n = 32 at N = 80: three tiles, the last one half padding)."""
    rng = np.random.default_rng(4)
    M, N, K = 200, 80, 68
    A = rng.integers(-3, 4, (M, K)).astype(np.float32)
    B = rng.integers(-3, 4, (N, K)).astype(np.float32)
    ldd = N + 40
    D = G.sentinel_buffer(M, N, ldd)
    ops.gemm(A=torch.from_numpy(A).cuda(), a_smn=K, a_sk=1, B=torch.from_numpy(B).cuda(), b_smn=K, b_sk=1, M=M, N=N, K=K,
             D=D, ldd=ldd, tile_n=32)
    got = G.check_sentinels(D, M, N, ldd, 'D')
    assert np.array_equal(got.astype(np.float64), A.astype(np.float64) @ B.T.astype(np.float64))


# ---- 4. float accuracy --------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize('layout,sched,epi', [('kk', 'dense', 0), ('kmn', 'dense', 0), ('pb', 'dense', 0),
                                              ('pk', 'dense', 0), ('mm', 'splitk', R.EPI_ATOMIC),
                                              ('pmn', 'splitk', R.EPI_ATOMIC)])
@pytest.mark.parametrize('N', [16, 80, 144])
@pytest.mark.parametrize('K', [36, 1024])
@pytest.mark.parametrize('passes', [1, 3])
def test_gemm_tail_float_accuracy(ops, layout, sched, epi, N, K, passes):
    """|got - emulated| <= τ(K) · sum_k |a_k b_k| elementwise (the bound of tests/test_gemm_gpu.py)."""
    rng = np.random.default_rng(K + N + passes)
    M = 136
    A = rng.standard_normal((M, K)).astype(np.float32)
    A[1::4] *= np.float32(2.0 ** 20)
    A[2::4] *= np.float32(2.0 ** -20)
    B = rng.standard_normal((1, N, K)).astype(np.float32)
    B[0, 1::2] = -B[0, 0::2] + (rng.standard_normal((N // 2, K)) * 1e-3).astype(np.float32)
    k_splits = 1 if sched != 'splitk' else 3
    got, ref, names, _, _ = run_tail(ops, layout, sched, epi, N, False, False, False, M, K, passes, seed=K,
                                     data=(A, B), k_splits=k_splits)
    D, mag, _, _ = ref
    err = np.abs(got.astype(np.float64) - D)
    extra = (k_splits + 1) * G.U * (np.abs(D) + mag) if epi & R.EPI_ATOMIC else 0.0
    ratio = (err - extra) / (G.tau(K, passes) * mag + 1e-300)
    print(f'tail float accuracy {layout} N={N} K={K} passes={passes}: worst err / (τ(K)·Σ|ab|) = {ratio.max():.3g}')
    assert ratio.max() <= 1.0


# ---- 5. census ----------------------------------------------------------------------------------------------------
@gpu
def test_lsk_t_launch_census(ops, monkeypatch):
    """Every GEMM launch of an LSKNet-T training step (fp32 and autocast) has a signature that the matrix above or the one
    of tests/test_gemm_gpu.py runs, and the step does launch the 16- and 80-column tails."""
    import test_lsk_gpu as L
    from oracle.cases import load_golden
    from sm3det_b200.synth import make_images
    seen, widths = set(), set()
    orig = ops.gemm

    def gemm(**kw):
        a_mn = kw['a_smn'] == 1 and kw['a_sk'] != 1
        apk, bpk = kw.get('a_packed') is not None, kw.get('b_packed') is not None
        b_mn = a_mn if apk else (False if bpk else (kw['b_smn'] == 1 and kw['b_sk'] != 1))
        layout = {(False, False, False, False): 'kk', (False, True, False, False): 'kmn', (False, False, True, False): 'pb',
                  (False, False, True, True): 'pk', (True, True, False, False): 'mm', (True, True, True, True): 'pmn'}[
            (a_mn, b_mn, bpk, apk)]
        sched = {0: 'dense', 1: 'grouped', 2: 'splitk'}[kw.get('sched', 0)]
        seen.add(G.signature(layout, sched, kw.get('epilogue', 0), kw.get('tile_n') or ops._pick_bn(kw['N']),
                             kw.get('a_row_index') is not None, kw.get('b_k_index') is not None,
                             kw.get('seg_begin') is not None, ops.current_passes()))
        widths.add(kw['N'])
        return orig(**kw)

    monkeypatch.setattr(ops, 'gemm', gemm)
    gold = load_golden(os.path.join(GOLD_T, 'lsk_t_short_e4k2_train_noisy_drop.pt'))
    _, _, net = L.build(gold['kw'])
    net.train()
    x = make_images(2, 96, 96, seed=3).cuda()
    for amp in (False, True):
        with torch.autocast('cuda', dtype=torch.bfloat16, enabled=amp):
            outs, loss = net(x)
        (sum(o.float().square().mean() for o in outs) + loss).backward()
        torch.cuda.synchronize()
    assert {16, 80} <= widths, sorted(widths)
    missing = sorted(seen - COVERED - G.COVERED, key=str)
    assert seen and not missing, f'launch signatures no matrix covers: {missing}'
