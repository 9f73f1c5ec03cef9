"""CPU reference for the split-bf16 GEMM (csrc/gemm_tc.cuh) and the fused FFN (csrc/ffn_fused.cu).

Needs numpy only, so the CPU suite can check it without a GPU (tests/test_gemm_ref.py).

- `split_bf16` is the kernels' hi/lo split, bit for bit: hi = the fp32 bits truncated to bf16, lo = the fp32 residual
  x - hi rounded to bf16 by adding 0x8000 to its bits (a carry may ripple into the exponent, which is still correct
  rounding).  The library is built without fast-math, so x - hi is an IEEE subtraction with denormals, as numpy's.
- `decode_k` / `decode_mn` read the bf16 hi|lo tile images of `pack_b`, `pack_act`, `act_pack` and
  `layernorm_fwd_img` through the same offset formulas as the kernels (`kmajor_sw64_offset`, `mnmajor_sw128_offset`).
- `gemm_ref` is the exact (float64) product of the split operands, hi*hi + hi*lo + lo*hi for 3 passes and hi*hi for
  1 pass, followed by the kernel's epilogue in the kernel's order.  It also returns sum_k |a_k b_k|, the scale every
  rounding error of the fp32 accumulation is measured against.
"""
import math

import numpy as np

BK = 32          # k per k-block of every image
BM = 128         # rows of the A tile
GPU_NAN = np.uint32(0x7FFFFFFF)   # the canonical NaN an sm_90 FADD returns (payloads are not propagated)

EPI_BIAS, EPI_GELU, EPI_DGELU, EPI_COLSCALE, EPI_ROWSCALE, EPI_RESID, EPI_ATOMIC, EPI_AUXSTORE, EPI_COLSUM = (
    1, 2, 4, 8, 16, 32, 64, 128, 256)


# ---- the split ------------------------------------------------------------------------------------------------------
def split_bits(x):
    """(hi, lo) bf16 bit patterns (uint16 arrays) of the fp32 array x, as the kernels compute them."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    u = x.view(np.uint32)
    hi32 = u & np.uint32(0xFFFF0000)
    with np.errstate(invalid='ignore', over='ignore'):
        r = x - hi32.view(np.float32)
    rb = r.view(np.uint32).copy()
    rb[np.isnan(r)] = GPU_NAN                      # inf - inf and NaN - NaN: the GPU's canonical NaN, not x86's
    lo32 = rb + np.uint32(0x8000)                  # uint32 wrap-around, as the kernel's unsigned add
    return (hi32 >> 16).astype(np.uint16), (lo32 >> 16).astype(np.uint16)


def bf16_to_f32(bits):
    return (np.asarray(bits, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32)


def split_bf16(x):
    """(hi, lo) as float32 arrays: hi + lo = x to within 2^-16 |x| for finite x (see tests/test_gemm_ref.py)."""
    h, l = split_bits(x)
    return bf16_to_f32(h), bf16_to_f32(l)


# ---- canonical layouts (csrc/gemm_tc.cuh) -------------------------------------------------------------------------
def kmajor_sw64_offset(row, chunk):
    row, chunk = np.asarray(row, dtype=np.int64), np.asarray(chunk, dtype=np.int64)
    return (row >> 3) * 512 + (row & 7) * 64 + ((chunk ^ ((row >> 1) & 3)) << 4)


def mnmajor_sw128_offset(k, mn_chunk):
    k, mn_chunk = np.asarray(k, dtype=np.int64), np.asarray(mn_chunk, dtype=np.int64)
    g, cc = mn_chunk >> 3, mn_chunk & 7
    return (g * 4 + (k >> 3)) * 1024 + (k & 7) * 128 + ((cc ^ (k & 7)) << 4)


def plane_bytes(width, mn_major):
    return ((width + 63) // 64) * 4096 if mn_major else width * 64


def packed_act_elems(rows, cols, mn_major, tile):
    """bf16 elements of a pack_act image (gemm_tc.cu: packed_act_elems)."""
    if not mn_major:
        return -(-rows // tile) * -(-cols // BK) * 2 * tile * BK
    return -(-cols // tile) * -(-rows // BK) * 2 * (plane_bytes(tile, True) // 2)


def _u16(img):
    """uint16 view of an image given as a numpy array or a (CPU or CUDA) int16 torch tensor."""
    if hasattr(img, 'cpu'):
        img = img.detach().cpu().numpy()
    return np.ascontiguousarray(img).view(np.uint16).reshape(-1)


def k_index(rows, cols, tile):
    """bf16 element index of (row, k) in a K-major image of `tile`-row tiles (hi plane; lo is + tile*32)."""
    r = np.arange(rows, dtype=np.int64)[:, None]
    c = np.arange(cols, dtype=np.int64)[None, :]
    kblocks = -(-cols // BK)
    byte = ((r // tile) * kblocks + c // BK) * (tile * 128) + kmajor_sw64_offset(r % tile, (c % BK) // 8) + (c % 8) * 2
    return byte // 2


def mn_index(rows, cols, tile):
    """bf16 element index of (k = row, mn = col) in an MN-major image of `tile`-column tiles (lo is + plane/2)."""
    r = np.arange(rows, dtype=np.int64)[:, None]
    c = np.arange(cols, dtype=np.int64)[None, :]
    kblocks = -(-rows // BK)
    pb = plane_bytes(tile, True)
    byte = ((c // tile) * kblocks + r // BK) * (2 * pb) + mnmajor_sw128_offset(r % BK, (c % tile) // 8) + (c % 8) * 2
    return byte // 2


def decode_k(img, rows, cols, tile=BM):
    """(hi, lo) uint16 [rows, cols] of a K-major SWIZZLE_64B image; rows/cols may include the zero padding."""
    u = _u16(img)
    i = k_index(rows, cols, tile)
    return u[i], u[i + tile * BK]


def decode_mn(img, rows, cols, tile):
    """(hi, lo) uint16 [rows = reduction index, cols] of an MN-major SWIZZLE_128B image."""
    u = _u16(img)
    i = mn_index(rows, cols, tile)
    return u[i], u[i + plane_bytes(tile, True) // 2]


def encode_k(hi, lo, tile=BM):
    """Inverse of decode_k for [rows, cols] padded to whole tiles / k-blocks (the CPU round-trip check)."""
    rows, cols = hi.shape
    out = np.zeros(packed_act_elems(rows, cols, False, tile), dtype=np.uint16)
    i = k_index(rows, cols, tile)
    out[i] = hi
    out[i + tile * BK] = lo
    return out


def encode_mn(hi, lo, tile):
    rows, cols = hi.shape
    out = np.zeros(packed_act_elems(rows, cols, True, tile), dtype=np.uint16)
    i = mn_index(rows, cols, tile)
    out[i] = hi
    out[i + plane_bytes(tile, True) // 2] = lo
    return out


def decode_k_image(img, T, C):
    """fp32 torch [T, C] value hi + lo of a K-major operand image with 128-row tiles."""
    import torch
    h, l = decode_k(img, T, C)
    return torch.from_numpy(bf16_to_f32(h) + bf16_to_f32(l))


# ---- GELU ---------------------------------------------------------------------------------------------------------
def gelu64(x):
    x = np.asarray(x, dtype=np.float64)
    return 0.5 * x * (1.0 + _erf(x / math.sqrt(2.0)))


def gelu_grad64(x):
    x = np.asarray(x, dtype=np.float64)
    return 0.5 * (1.0 + _erf(x / math.sqrt(2.0))) + x * np.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


def _erf(x):
    from scipy.special import erf
    return erf(x)


# ---- the GEMM -----------------------------------------------------------------------------------------------------
def split_product(A, B, passes):
    """float64 [M, N] = exact sum over k of the split products of fp32 A[M, K] and B[N, K]."""
    ah, al = (t.astype(np.float64) for t in split_bf16(A))
    bh, bl = (t.astype(np.float64) for t in split_bf16(B))
    if passes == 1:
        return ah @ bh.T
    return ah @ bh.T + ah @ bl.T + al @ bh.T


def _gather_rows(X, index):
    out = np.zeros((len(index),) + X.shape[1:], dtype=np.float32)
    ok = index >= 0
    out[ok] = X[index[ok]]
    return out


def gemm_ref(A, B, *, passes=3, a_row_index=None, b_k_index=None, tile_group=None, num_m_tiles=None, segs=None,
             epi=0, bias=None, aux_in=None, col_scale=None, row_scale=None, resid=None, d_init=None):
    """Emulation of one gemm launch on logical operands.

    A [rows_A, K] holds A(m, k) (rows gathered through a_row_index, -1 = zero row); B [G, N, K_src] holds B(n, k) of
    each group (G = 1: shared), gathered along k through b_k_index.  Schedules: dense (default); grouped, where m tile t
    < num_m_tiles uses group tile_group[t] and later tiles are not computed; split-K, where segs = (begin, end) arrays
    give group g the reduction range [begin[g], end[g]).  The epilogue operands are per group ([G, ...]) or shared.

    Returns (D, mag, aux, colsum): D [G, M, N] float64 after the epilogue (NaN where the kernel writes nothing), mag
    [G, M, N] = sum_k |a_k b_k| of the fp32 operands, aux = the value before GELU (EPI_AUXSTORE / EPI_GELU), colsum
    [G, N] of the final values (EPI_COLSUM).  Split-K without EPI_ATOMIC leaves the D of an empty segment unwritten."""
    A = np.asarray(A, dtype=np.float32)
    B = np.asarray(B, dtype=np.float32)
    if B.ndim == 2:
        B = B[None]
    if a_row_index is not None:
        A = _gather_rows(A, np.asarray(a_row_index))
    if b_k_index is not None:
        B = np.stack([_gather_rows(b.T, np.asarray(b_k_index)).T for b in B])
    M, K = A.shape
    N = B.shape[1]
    if segs is not None:
        G = len(segs[0])
        acc = np.zeros((G, M, N))
        mag = np.zeros((G, M, N))
        for g in range(G):
            b, e = int(segs[0][g]), int(segs[1][g])
            Bg = B[g if B.shape[0] > 1 else 0]
            if e > b:
                acc[g] = split_product(A[:, b:e], Bg[:, b:e], passes)
                mag[g] = np.abs(A[:, b:e]).astype(np.float64) @ np.abs(Bg[:, b:e]).astype(np.float64).T
            elif not epi & EPI_ATOMIC:
                acc[g] = np.nan            # an empty segment has no k-block: its tiles are skipped, D is not written
        groups_of_rows = None
    else:
        G = 1
        groups_of_rows = np.zeros(M, dtype=np.int64)
        live = np.ones(M, dtype=bool)
        if tile_group is not None:
            nt = int(num_m_tiles)
            t = np.arange(M) // BM
            live = t < nt
            groups_of_rows = np.where(live, np.asarray(tile_group)[np.minimum(t, len(tile_group) - 1)], -1)
        acc = np.full((1, M, N), np.nan)
        mag = np.zeros((1, M, N))
        for g in np.unique(groups_of_rows[live]):
            rows = groups_of_rows == g
            Bg = B[g if B.shape[0] > 1 else 0]
            acc[0, rows] = split_product(A[rows], Bg, passes)
            mag[0, rows] = np.abs(A[rows]).astype(np.float64) @ np.abs(Bg).astype(np.float64).T

    x = acc.copy()
    if epi & EPI_BIAS:
        bias = np.asarray(bias, dtype=np.float64)
        if segs is not None:
            x += bias.reshape(-1, N)[:, None, :] if bias.size > N else bias.reshape(1, 1, N)
        elif bias.size > N:
            bb = bias.reshape(-1, N)[np.maximum(groups_of_rows, 0)]
            x += bb[None]
        else:
            x += bias.reshape(1, 1, N)
    aux = x.copy() if epi & (EPI_AUXSTORE | EPI_GELU) else None
    if epi & EPI_GELU:
        x = gelu64(x)
    if epi & EPI_DGELU:
        x = x * gelu_grad64(np.asarray(aux_in, dtype=np.float64).reshape(x.shape))
    scale = np.ones((1, 1, N))
    if epi & EPI_COLSCALE:
        scale = scale * np.asarray(col_scale, dtype=np.float64).reshape(1, 1, N)
    if epi & EPI_ROWSCALE:
        scale = scale * np.asarray(row_scale, dtype=np.float64).reshape(1, M, 1)
    x = x * scale
    mag = mag * np.abs(scale)
    if epi & EPI_RESID:
        x = x + np.asarray(resid, dtype=np.float64).reshape(x.shape)
    colsum = None
    if epi & EPI_COLSUM:
        if segs is not None:
            colsum = np.nansum(x, axis=1)
        else:
            ng = int(np.max(groups_of_rows)) + 1 if (groups_of_rows >= 0).any() else 1
            colsum = np.zeros((ng, N))
            for g in range(ng):
                colsum[g] = x[0, groups_of_rows == g].sum(axis=0)
    if epi & EPI_ATOMIC:
        if d_init is not None:
            x = x + np.asarray(d_init, dtype=np.float64).reshape(x.shape)
    return x, mag, aux, colsum
