"""CPU checks of tests/gemm_ref.py, the reference the GEMM and fused-FFN GPU tests compare against."""
import numpy as np
import pytest

import gemm_ref as R


def _bits(x):
    return np.asarray(x, dtype=np.float32).view(np.uint32)


@pytest.mark.parametrize('tile', [32, 64, 96, 128])
def test_k_image_round_trip(tile):
    rng = np.random.default_rng(tile)
    rows, cols = 3 * tile, 96
    hi = rng.integers(0, 1 << 16, (rows, cols), dtype=np.uint16)
    lo = rng.integers(0, 1 << 16, (rows, cols), dtype=np.uint16)
    img = R.encode_k(hi, lo, tile)
    # every (row, k) of both planes has its own slot and the image holds nothing else
    assert np.count_nonzero(img) == np.count_nonzero(hi) + np.count_nonzero(lo)
    h2, l2 = R.decode_k(img, rows, cols, tile)
    assert np.array_equal(h2, hi) and np.array_equal(l2, lo)


@pytest.mark.parametrize('tile', [32, 64, 96, 128, 160, 256])
def test_mn_image_round_trip(tile):
    rng = np.random.default_rng(tile)
    rows, cols = 64, 2 * tile
    hi = rng.integers(1, 1 << 16, (rows, cols), dtype=np.uint16)
    lo = rng.integers(1, 1 << 16, (rows, cols), dtype=np.uint16)
    img = R.encode_mn(hi, lo, tile)
    idx = R.mn_index(rows, cols, tile)
    assert len(np.unique(idx)) == idx.size                   # the offset formula is injective
    assert np.count_nonzero(img) == 2 * rows * cols
    h2, l2 = R.decode_mn(img, rows, cols, tile)
    assert np.array_equal(h2, hi) and np.array_equal(l2, lo)


def test_offsets_stay_inside_their_plane():
    """Each 16-byte chunk of a k-block lands inside the plane the kernel sizes for it (plane_bytes)."""
    for w in (32, 64, 96, 128, 160, 256):
        r, c = np.meshgrid(np.arange(w), np.arange(4), indexing='ij')
        o = R.kmajor_sw64_offset(r, c)
        assert o.max() + 16 <= R.plane_bytes(w, False) and len(np.unique(o)) == o.size
        k, m = np.meshgrid(np.arange(R.BK), np.arange(w // 8), indexing='ij')
        o = R.mnmajor_sw128_offset(k, m)
        assert o.max() + 16 <= R.plane_bytes(w, True) and len(np.unique(o)) == o.size


def test_split_identity_bound():
    """x in [2^e, 2^(e+1)): truncation leaves r = x - hi in [0, 2^(e-7)), so r's exponent is at most e - 8 and rounding r
    to 8 significant bits errs by at most half an ulp, 2^(e-8-8) <= 2^-16 |x|.  The bound is reached: the worst case
    over a dense sample is above 2^-17 |x|.  (Below 2^-110 the residual's bf16 is denormal and the bound is absolute,
    2^-134.)"""
    rng = np.random.default_rng(0)
    x = (rng.standard_normal(1 << 20) * np.exp2(rng.integers(-100, 100, 1 << 20))).astype(np.float32)
    x = np.concatenate([x, np.float32(1.0) + np.arange(1 << 16, dtype=np.float32) * np.float32(2.0 ** -23)])
    hi, lo = R.split_bf16(x)
    err = np.abs(x.astype(np.float64) - hi.astype(np.float64) - lo.astype(np.float64))
    ratio = err / np.abs(x.astype(np.float64))
    assert ratio.max() <= 2.0 ** -16
    assert ratio.max() > 2.0 ** -17
    # hi is the truncation, lo the nearest bf16 (ties away from zero) of the exact residual
    assert np.array_equal(_bits(hi), _bits(x) & np.uint32(0xFFFF0000))
    r = x.astype(np.float64) - hi
    assert np.all(np.abs(r - lo) <= np.abs(r) * 2.0 ** -8)
    assert np.all((lo == 0) | (np.sign(lo) == np.sign(r)))


def test_split_product_error():
    """hi*hi + hi*lo + lo*hi drops lo*lo (|lo| < 2^-7 |x|: up to 2^-14 |a b|) and keeps the two split residuals
    (2^-16 each): |a b - P| <= (2^-14 + 2 * 2^-16 + 2^-31) |a b|.  1 pass: (2 * 2^-7 + 2^-14) |a b|."""
    rng = np.random.default_rng(1)
    A = rng.standard_normal((64, 256)).astype(np.float32)
    B = rng.standard_normal((48, 256)).astype(np.float32)
    P3 = R.split_product(A, B, 3)
    P1 = R.split_product(A, B, 1)
    mag = np.abs(A).astype(np.float64) @ np.abs(B).astype(np.float64).T
    exact = A.astype(np.float64) @ B.astype(np.float64).T
    assert np.all(np.abs(P3 - exact) <= (2.0 ** -14 + 2 * 2.0 ** -16 + 2.0 ** -31) * mag)
    assert np.all(np.abs(P1 - exact) <= (2 * 2.0 ** -7 + 2.0 ** -14) * mag)
    assert np.abs(P3 - exact).max() > 0 and np.abs(P1 - exact).max() > np.abs(P3 - exact).max()


def test_split_special_values():
    """The values the kernel's unsigned arithmetic gives for signed zeros, denormals, the largest finite value, inf and
    NaN (where x - hi is NaN the GPU produces 0x7FFFFFFF, whose rounded top half is 0x8000 = -0)."""
    tiny = np.float32(1.5e-41)                     # denormal
    x = np.array([0.0, -0.0, tiny, -tiny, np.finfo(np.float32).max, -np.finfo(np.float32).max, np.inf, -np.inf, np.nan,
                  np.float32(2.0 ** -149)], dtype=np.float32)
    hb, lb = R.split_bits(x)
    assert list(hb[:2]) == [0x0000, 0x8000] and list(lb[:2]) == [0, 0]
    # a denormal keeps its top 16 bits in hi and the next in lo, whose ulp is 2^-133: hi + lo errs by at most 2^-134
    # (1.5e-41 < 2^-133 is lost entirely, 1e-39 is not)
    d = np.array([tiny, -tiny, 1e-39, -1e-39], dtype=np.float32)
    h, l = R.split_bf16(d)
    assert np.all(np.abs(d.astype(np.float64) - h - l) <= 2.0 ** -134)
    assert np.array_equal(h[:2] + l[:2], [0, 0]) and np.all(h[2:] != 0)
    assert hb[4] == 0x7F7F and R.bf16_to_f32(lb[4]) > 0 and np.isfinite(R.bf16_to_f32(lb[4]))
    assert hb[5] == 0xFF7F and R.bf16_to_f32(lb[5]) < 0
    assert list(hb[6:8]) == [0x7F80, 0xFF80] and list(lb[6:9]) == [0x8000] * 3
    assert hb[8] == 0x7FC0
    assert hb[9] == 0 and lb[9] == 0                # the smallest denormal rounds away entirely
    # a NaN whose payload sits in the low half truncates to inf: the kernel does the same
    nan_low = np.array([0x7F800001], dtype=np.uint32).view(np.float32)
    hb, lb = R.split_bits(nan_low)
    assert hb[0] == 0x7F80 and lb[0] == 0x8000


def _loop_ref(A, B, segs=None, tile_group=None, num_m_tiles=None):
    """Plain integer loops: the definition of each schedule."""
    M, K = A.shape
    N = B.shape[1]
    if segs is not None:
        D = np.zeros((len(segs[0]), M, N))
        for g, (b, e) in enumerate(zip(*segs)):
            if e <= b:
                D[g] = np.nan          # no k-block: the tiles are skipped and D keeps what it held
                continue
            D[g] = A[:, b:e].astype(np.float64) @ B[g if len(B) > 1 else 0][:, b:e].T.astype(np.float64)
        return D
    D = np.full((1, M, N), np.nan)
    for m in range(M):
        t = m // 128
        if tile_group is not None and t >= num_m_tiles:
            continue
        g = tile_group[t] if tile_group is not None else 0
        D[0, m] = A[m].astype(np.float64) @ B[g].T.astype(np.float64)
    return D


def test_gemm_ref_schedules_and_epilogue():
    rng = np.random.default_rng(2)
    M, N, K, G = 300, 64, 80, 3
    A = rng.integers(-3, 4, (M, K)).astype(np.float32)
    B = rng.integers(-3, 4, (G, N, K)).astype(np.float32)
    tg = np.array([2, 0, 7])                      # third tile out of range: num_m_tiles = 2
    for passes in (1, 3):
        D, mag, _, _ = R.gemm_ref(A, B, passes=passes, tile_group=tg, num_m_tiles=2)
        assert np.array_equal(D, _loop_ref(A, B, tile_group=tg, num_m_tiles=2), equal_nan=True)
        segs = (np.array([0, 32, 40]), np.array([32, 32, 77]))
        D, mag, _, _ = R.gemm_ref(A, B, passes=passes, segs=segs)
        assert np.array_equal(D, _loop_ref(A, B, segs=segs), equal_nan=True)
        assert np.all(np.isnan(D) | (mag >= np.abs(D)))
    # gathers: -1 rows of A and -1 k of B contribute zero
    ri = rng.integers(-1, M, 200)
    ki = rng.integers(-1, K, 50)
    D, _, _, _ = R.gemm_ref(A[:, :50], B[:1], a_row_index=ri, b_k_index=ki)
    Ag = np.where((ri >= 0)[:, None], A[np.maximum(ri, 0), :50], 0)
    Bg = B[0][:, np.maximum(ki, 0)] * (ki >= 0)
    assert np.array_equal(D[0], Ag.astype(np.float64) @ Bg.T.astype(np.float64))
    # epilogue order: bias -> aux -> gelu -> col scale -> row scale -> resid -> colsum
    bias, cs, rs = rng.standard_normal(N), rng.standard_normal(N), rng.standard_normal(M)
    resid = rng.standard_normal((M, N))
    epi = R.EPI_BIAS | R.EPI_GELU | R.EPI_COLSCALE | R.EPI_ROWSCALE | R.EPI_RESID | R.EPI_COLSUM
    D, _, aux, colsum = R.gemm_ref(A, B[:1], epi=epi, bias=bias, col_scale=cs, row_scale=rs, resid=resid)
    P = A.astype(np.float64) @ B[0].T.astype(np.float64) + bias
    want = R.gelu64(P) * cs * rs[:, None] + resid
    assert np.allclose(D[0], want, rtol=1e-14, atol=1e-12) and np.array_equal(aux[0], P)
    assert np.allclose(colsum[0], want.sum(0), rtol=1e-12, atol=1e-9)


def test_gelu64_matches_torch():
    import torch
    x = np.linspace(-12, 12, 4001)
    t = torch.from_numpy(x).requires_grad_(True)
    y = torch.nn.functional.gelu(t)
    y.sum().backward()
    assert np.allclose(R.gelu64(x), y.detach().numpy(), rtol=1e-13, atol=1e-15)
    assert np.allclose(R.gelu_grad64(x), t.grad.numpy(), rtol=1e-13, atol=1e-15)
