"""Thin, allocation-only wrappers around the C-ABI kernels (one Python function per entry point).

PyTorch is used here for device memory (``torch.empty``), the current CUDA stream and nothing else;
all arithmetic happens in ``libsm3det_b200.so``.  Every wrapper validates that its tensors are
fp32/int32, contiguous and on the current CUDA device, then passes raw pointers.
"""
import ctypes as C
import ctypes as _ct      # the fused-FFN wrappers take a keyword argument named C (channels)
from typing import Optional

import torch

from . import _lib

SCHED_DENSE, SCHED_GROUPED, SCHED_SPLITK = 0, 1, 2
EPI_BIAS, EPI_GELU, EPI_DGELU, EPI_COLSCALE, EPI_ROWSCALE, EPI_RESID, EPI_ATOMIC, EPI_AUXSTORE, EPI_COLSUM = 1, 2, 4, 8, 16, 32, 64, 128, 256
LN_NHWC, LN_PATCH2, LN_NCHW = 0, 1, 2


# GEMM operand precision: 3 = split-bf16 hi*hi + hi*lo + lo*hi (fp32-accurate; what every parity test and bench.py use),
# 1 = hi*hi only (plain bf16 operands, fp32 accumulate) -- the mixed-precision recipe.  The precision is a per-call
# property carried by a thread-local scope: a backbone forward opens `precision_scope(passes)` around its kernels, every
# autograd Function decorated with `@captures_precision` remembers the scope it was RECORDED under and re-opens it for
# its backward -- so an interleaved forward of another model (EMA / teacher / validation hook) can no longer change the
# precision of a pending backward, and two Python threads do not see each other's mode.
import contextlib
import threading

_tls = threading.local()


def current_passes() -> int:
    return getattr(_tls, 'passes', 3)


@contextlib.contextmanager
def precision_scope(passes: int):
    if passes not in (1, 3):
        raise ValueError('mma passes must be 3 (fp32-accurate split-bf16) or 1 (bf16 operands)')
    prev = current_passes()
    _tls.passes = passes
    try:
        yield
    finally:
        _tls.passes = prev


def autocast_passes(module=None) -> int:
    """1 under torch.autocast (or when `module.amp` is set), else 3."""
    import torch as _t
    return 1 if (getattr(module, 'amp', False) or _t.is_autocast_enabled()) else 3


def captures_precision(cls):
    """Class decorator for torch.autograd.Function subclasses: backward runs at the GEMM precision of its own forward."""
    fwd, bwd = cls.forward, cls.backward

    def forward(ctx, *args, **kwargs):
        ctx._mma_passes = current_passes()
        return fwd(ctx, *args, **kwargs)

    def backward(ctx, *grads):
        with precision_scope(ctx._mma_passes):
            return bwd(ctx, *grads)

    cls.forward = staticmethod(forward)
    cls.backward = staticmethod(backward)
    return cls


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _p(t: Optional[torch.Tensor], dtype=torch.float32):
    if t is None:
        return None
    if not t.is_cuda:
        raise RuntimeError('sm3det_b200 ops need CUDA tensors (no CPU fallback exists)')
    if t.dtype != dtype:
        raise TypeError(f'expected {dtype}, got {t.dtype}')
    if not t.is_contiguous():
        raise ValueError('expected a contiguous tensor')
    return t.data_ptr()


def _pi(t):
    return _p(t, torch.int32)


def _pick_bn(n: int) -> int:
    """Tile width of an n-column GEMM output, as gemm::pick_bn: the largest of 128/96/64/32 dividing n; for any other
    n % 8 == 0 the last tile runs padded and masked, with the fewest tiles and then the least padding."""
    for bn in (128, 96, 64, 32):
        if n % bn == 0:
            return bn
    if n > 0 and n % 8 == 0:
        return min((128, 96, 64, 32), key=lambda bn: (-(-n // bn), -(-n // bn) * bn))
    raise ValueError(f'N={n} has no GEMM tile width (multiple of 8)')


def _n_tiles(n: int) -> int:
    return -(-n // _pick_bn(n))


def num_sms() -> int:
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def gemm(*, A, a_smn, a_sk, B, b_smn, b_sk, M, N, K, D, ldd, b_group_stride=0, a_row_index=None, b_k_index=None,
         sched=SCHED_DENSE, k_splits=1, num_groups=1, tile_group=None, num_m_tiles=None, seg_begin=None,
         seg_end=None, d_group_stride=0, bias=None, bias_group_stride=0, epilogue=0, aux_out=None, aux_in=None,
         ld_aux=0, col_scale=None, row_scale=None, resid=None, ld_resid=0, tile_n=0, b_packed=None,
         b_packed_group_stride=0, colsum=None, colsum_group_stride=0, a_packed=None):
    lib = _lib.load()
    a = _lib.GemmArgs()
    a.A = _p(A); a.a_stride_mn = a_smn; a.a_stride_k = a_sk
    a.b_packed = None if b_packed is None else _p(b_packed, torch.int16); a.b_packed_group_stride = b_packed_group_stride
    a.a_packed = None if a_packed is None else _p(a_packed, torch.int16)
    a.B = _p(B); a.b_stride_mn = b_smn; a.b_stride_k = b_sk; a.b_group_stride = b_group_stride
    a.a_row_index = _pi(a_row_index); a.b_k_index = _pi(b_k_index)
    a.M, a.N, a.K = M, N, K
    a.tile_n = tile_n; a.sched = sched; a.k_splits = k_splits; a.num_groups = num_groups
    a.tile_group = _pi(tile_group); a.num_m_tiles = _pi(num_m_tiles)
    a.seg_begin = _pi(seg_begin); a.seg_end = _pi(seg_end)
    a.D = _p(D); a.ldd = ldd; a.d_group_stride = d_group_stride
    a.bias = _p(bias); a.bias_group_stride = bias_group_stride
    a.epilogue = epilogue
    a.aux_out = _p(aux_out); a.aux_in = _p(aux_in); a.ld_aux = ld_aux
    a.col_scale = _p(col_scale); a.row_scale = _p(row_scale)
    a.resid = _p(resid); a.ld_resid = ld_resid
    a.colsum = _p(colsum); a.colsum_group_stride = colsum_group_stride
    a.mma_passes = current_passes()
    _lib.check(lib.sm3_gemm(C.byref(a), _stream()), 'sm3_gemm')
    return D


def pack_weight(w, *, transposed: bool, groups: int = 1, out=None, tile: int = 0):
    """bf16 hi/lo tile image of a weight for the GEMM's B operand (sm3_gemm_pack_b) -> (buffer, elems_per_group).
    tile > 0: explicit tile width (the fused FFN kernels stream weight chunks of their own width).  The image holds N
    padded to whole tiles of _pick_bn(N) rows (zeros past N), so a column tail (N % 32 != 0) takes the packed path too.

    w: [N,K] (or the first of `groups` adjacent [N,K] expert weights).  transposed=False packs B(n,k) = w[n,k]
    (forward);  transposed=True packs B(n=k', k=n') = w[n',k'] (dgrad).  Callers cache the result per parameter
    version (sm3det_b200.backbone.PackCache); this function never caches.
    """
    lib = _lib.load()
    n_, k_ = w.shape[-2], w.shape[-1]
    if transposed:
        N, K, s_mn, s_k = k_, n_, 1, k_
    else:
        N, K, s_mn, s_k = n_, k_, k_, 1
    per = lib.sm3_gemm_packed_elems(N, K)
    if out is None or out.numel() != groups * per:
        out = torch.empty((groups * per,), device=w.device, dtype=torch.int16)
    if tile:
        _lib.check(lib.sm3_gemm_pack_b_tile(_p(w), s_mn, s_k, n_ * k_, groups, N, K, tile, out.data_ptr(), _stream()),
                   'sm3_gemm_pack_b_tile')
    else:
        _lib.check(lib.sm3_gemm_pack_b(_p(w), s_mn, s_k, n_ * k_, groups, N, K, out.data_ptr(), _stream()), 'sm3_gemm_pack_b')
    return out, per


def pack_act(x, *, rows, cols, mn_major, tile=128, row_index=None, ld=None):
    """Pre-split an activation operand (sm3_gemm_pack_act).  mn_major=False: x[rows, cols=K] -> K-major A tiles
    (row_index = MoE dispatch gather).  mn_major=True: x[rows = reduction index, cols] -> MN-major tiles of `tile` cols."""
    lib = _lib.load()
    n = lib.sm3_gemm_packed_act_elems(rows, cols, 1 if mn_major else 0, tile)
    out = torch.empty((n,), device=x.device, dtype=torch.int16)
    _lib.check(lib.sm3_gemm_pack_act(_p(x), cols if ld is None else ld, _pi(row_index), rows, cols, 1 if mn_major else 0, tile,
                                     out.data_ptr(), _stream()), 'sm3_gemm_pack_act')
    return out


ACT_GELU, ACT_DGELU, ACT_COPY, ACT_BWD = 0, 1, 2, 3


# ---- fused dense FFN (narrow stages): the [T,4C] hidden tensor never leaves the SM --------------------------------------
FFN_FWD, FFN_BWD_DX, FFN_BWD_IMG, FFN_BWD_IMG_H = 0, 1, 2, 3


def ffn_chunk(mode: int, C: int) -> int:
    """hidden chunk width of sm3_ffn_fused for (mode, C); 0 = not supported (use the GEMM -> act_pack -> GEMM path).
    SM3_FUSED_FFN=0 disables every mode; SM3_FUSED_FFN_BWD=0 only the backward modes that emit the weight-gradient
    operands (2, 3), so the dense blocks' backward takes dgrad -> act_pack -> dgrad again (A/B in one process)."""
    import os
    if os.environ.get('SM3_FUSED_FFN', '1') == '0':
        return 0
    if mode >= FFN_BWD_IMG and os.environ.get('SM3_FUSED_FFN_BWD', '1') == '0':
        return 0
    return int(_lib.load().sm3_ffn_fused_chunk(mode, C))


def _ffn_args(*, T, C, chunk, mode, a1, wa1, b1, a2=None, wa2=None, wb=None):
    a = _lib.FfnArgs()
    a.a1 = _p(a1, torch.int16); a.a2 = None if a2 is None else _p(a2, torch.int16)
    a.wa1 = _p(wa1, torch.int16); a.wa2 = None if wa2 is None else _p(wa2, torch.int16)
    a.wb = None if wb is None else _p(wb, torch.int16)
    a.bias1 = _p(b1)
    a.M, a.C, a.H4, a.chunk, a.mma_passes, a.mode = T, C, 4 * C, chunk, current_passes(), mode
    return a


def ffn_fused_fwd(v_img, w1_img, w2_img, b1, b2, *, T, C, chunk, gamma=None, row_scale=None, resid=None, want_aux=False,
                  want_h=False):
    """out[T,C] = resid + row_scale * gamma * (gelu(v W1^T + b1) W2^T + b2); aux = the value before gamma (y2);
    want_h: also return the hidden pre-activation h [T,4C] (-> (out, aux, h))."""
    lib = _lib.load()
    out = torch.empty((T, C), device=b1.device, dtype=torch.float32)
    aux = torch.empty((T, C), device=b1.device, dtype=torch.float32) if want_aux else None
    h = torch.empty((T, 4 * C), device=b1.device, dtype=torch.float32) if want_h else None
    a = _ffn_args(T=T, C=C, chunk=chunk, mode=FFN_FWD, a1=v_img, wa1=w1_img, b1=b1, wb=w2_img)
    a.bias2 = _p(b2); a.col_scale = _p(gamma); a.row_scale = _p(row_scale); a.resid = _p(resid)
    a.out = _p(out); a.aux_out = _p(aux); a.h_out = _p(h)
    _lib.check(lib.sm3_ffn_fused(_ct.byref(a), _stream()), 'sm3_ffn_fused(fwd)')
    return (out, aux, h) if want_h else (out, aux)


def ffn_fused_bwd(v_img, dz_img, w1_img, w2gt_img, w1t_img, b1, *, T, C, chunk, want_wgrad_images=False, db1=None, h=None):
    """dv[T,C] = ((dz (gamma W2)) * gelu'(v W1^T + b1)) W1   (hidden pre-activation recomputed from v).

    want_wgrad_images: also return the two weight-gradient operands, (dv, dh_mn, a_mn): the MN-major images (tile 128) of
    dh = (dz (gamma W2)) * gelu'(h) and of gelu(h) that linear_wgrad takes as dy_packed / x_packed, and add the column
    sums of dh into db1 [4C] (required).  h: the forward's saved pre-activation [T,4C]; given, the kernel reads it instead of
    recomputing it (mode 3; v_img and w1_img are then unused).  chunk = ffn_chunk(2 or 3, C) accordingly."""
    lib = _lib.load()
    out = torch.empty((T, C), device=b1.device, dtype=torch.float32)
    if not want_wgrad_images:
        a = _ffn_args(T=T, C=C, chunk=chunk, mode=FFN_BWD_DX, a1=v_img, a2=dz_img, wa1=w1_img, wa2=w2gt_img, b1=b1, wb=w1t_img)
        a.out = _p(out)
        _lib.check(lib.sm3_ffn_fused(_ct.byref(a), _stream()), 'sm3_ffn_fused(bwd)')
        return out
    if db1 is None:
        raise ValueError('ffn_fused_bwd: want_wgrad_images needs db1')
    n = lib.sm3_gemm_packed_act_elems(T, 4 * C, 1, 128)
    dh_mn = torch.empty((n,), device=b1.device, dtype=torch.int16)
    a_mn = torch.empty((n,), device=b1.device, dtype=torch.int16)
    mode = FFN_BWD_IMG if h is None else FFN_BWD_IMG_H
    a = _ffn_args(T=T, C=C, chunk=chunk, mode=mode, a1=v_img if h is None else dz_img, a2=dz_img,
                  wa1=w1_img if h is None else w2gt_img, wa2=w2gt_img, b1=b1, wb=w1t_img)
    a.out = _p(out); a.dh_mn = dh_mn.data_ptr(); a.act_mn = a_mn.data_ptr(); a.db1 = _p(db1); a.h_in = _p(h)
    _lib.check(lib.sm3_ffn_fused(_ct.byref(a), _stream()), 'sm3_ffn_fused(bwd)')
    return out, dh_mn, a_mn


def fused_cost(name, *a, **kw):
    """(algorithmic FLOPs, algorithmic HBM bytes, shape) of a fused-FFN call, for bench.py's roofline (recomputation of the
    hidden pre-activation is NOT counted: FLOPs are those of the GEMMs the algorithm needs)."""
    T, Cc = kw['T'], kw['C']
    unit = 2.0 * T * Cc * 4 * Cc
    wbytes = 2 * 4.0 * 4 * Cc * Cc
    if name == 'ffn_fused_fwd':
        return 2 * unit, (3 + (1 if kw.get('want_aux') else 0) + (4 if kw.get('want_h') else 0)) * 4.0 * T * Cc + wbytes, (T, Cc, 'fwd')
    if not kw.get('want_wgrad_images'):
        return 2 * unit, 3 * 4.0 * T * Cc + 2 * wbytes, (T, Cc, 'bwd-dv')
    # bytes per token x channel: dz image + dv (4 + 4), the v image (4, mode 2) or the saved fp32 h (16, mode 3), and the
    # two [T,4C] hi|lo images (16 + 16)
    h = kw.get('h') is not None
    return 2 * unit, (8 + (16 if h else 4) + 32) * float(T * Cc) + 2 * wbytes, (T, Cc, 'bwd-img-h' if h else 'bwd-img')


def act_pack(h, *, rows, width, mode, da=None, want_k=False, mn_tile=0, want_f32=False, colsum=None, live_tiles=None,
             tile_group=None, mn_tile2=0):
    """Fused activation + pre-split (sm3_act_pack).  Returns (pack_k, pack_mn, out_f32); absent outputs are None.
    mode=ACT_BWD (needs mn_tile2): one pass over h emits da*gelu'(h) as pack_k / pack_mn AND gelu(h) as a second MN image;
    returns (pack_k, pack_mn, pack_mn2)."""
    lib = _lib.load()
    dev = h.device
    a = _lib.ActPackArgs()
    pk = pm = of = None
    if want_k:
        pk = torch.empty((lib.sm3_gemm_packed_act_elems(rows, width, 0, 128),), device=dev, dtype=torch.int16)
    if mn_tile:
        pm = torch.empty((lib.sm3_gemm_packed_act_elems(rows, width, 1, mn_tile),), device=dev, dtype=torch.int16)
    if want_f32:
        of = torch.empty((rows, width), device=dev, dtype=torch.float32)
    a.h = _p(h); a.da = _p(da); a.R = rows; a.W = width; a.mode = mode
    a.live_tiles = _pi(live_tiles); a.tile_group = _pi(tile_group)
    a.out_f32 = _p(of); a.pack_k = None if pk is None else pk.data_ptr(); a.pack_mn = None if pm is None else pm.data_ptr()
    a.mn_tile = mn_tile; a.colsum = _p(colsum)
    pm2 = None
    if mode == ACT_BWD:
        pm2 = torch.empty((lib.sm3_gemm_packed_act_elems(rows, width, 1, mn_tile2),), device=dev, dtype=torch.int16)
        a.pack_mn2 = pm2.data_ptr(); a.mn_tile2 = mn_tile2
    _lib.check(lib.sm3_act_pack(C.byref(a), _stream()), 'sm3_act_pack')
    if mode == ACT_BWD:
        return pk, pm, pm2
    return pk, pm, of


# When is an extra pack pass (8 B/element of HBM traffic) cheaper than splitting the operand inside the GEMM?  The
# in-kernel split is repeated for every tile column that re-reads the operand and is latency/issue bound; the packed
# main loop runs at the tensor-pipe rate.
import os as _os
PACK_A_MIN_K = int(_os.environ.get('SM3_PACK_A_MIN_K', '96'))
PACK_W_MIN_TILES = int(_os.environ.get('SM3_PACK_W_MIN_TILES', '2'))


def _pack_a_pays(N, K):
    return K >= PACK_A_MIN_K and _n_tiles(N) >= 2 or K >= 4 * PACK_A_MIN_K


def linear_fwd(x, w, bias=None, *, epilogue=0, out=None, aux_out=None, col_scale=None, row_scale=None, resid=None,
               row_index=None, rows=None, grouped=None, w_group_stride=0, bias_group_stride=0, packed=None,
               a_packed=None):
    """out[M,N] = epi(x[M,K] @ w[N,K]^T).  grouped = (tile_group, num_m_tiles) for expert segments.
    a_packed: an already pre-split K-major image of x (then x may be None and `rows` is required)."""
    K = w.shape[-1]
    N = w.shape[-2]
    M = rows if rows is not None else x.shape[0]
    if out is None:
        out = torch.empty((M, N), device=w.device, dtype=torch.float32)
    epi = epilogue | (EPI_BIAS if bias is not None else 0)
    kw = {}
    if grouped is not None:
        kw = dict(sched=SCHED_GROUPED, tile_group=grouped[0], num_m_tiles=grouped[1])
    if packed is not None:
        kw.update(b_packed=packed[0], b_packed_group_stride=packed[1])
        if a_packed is not None:
            kw.update(a_packed=a_packed)
            row_index = None
        elif _pack_a_pays(N, K):
            kw.update(a_packed=pack_act(x, rows=M, cols=K, mn_major=False, row_index=row_index))
            row_index = None
    gemm(A=x, a_smn=K, a_sk=1, B=w, b_smn=K, b_sk=1, b_group_stride=w_group_stride, M=M, N=N, K=K, D=out, ldd=N,
         a_row_index=row_index, bias=bias, bias_group_stride=bias_group_stride, epilogue=epi, aux_out=aux_out,
         ld_aux=N, col_scale=col_scale, row_scale=row_scale, resid=resid, ld_resid=N, **kw)
    return out


def linear_dgrad(dy, w, *, epilogue=0, out=None, aux_in=None, row_scale=None, resid=None, grouped=None,
                 w_group_stride=0, packed=None, colsum=None, colsum_group_stride=0, a_packed=None, rows=None):
    """dx[M,K] = epi(dy[M,N] @ w[N,K])   (w used as an MN-major B operand; no transposed copy).
    a_packed: pre-split K-major image of dy (then dy may be None and `rows` is required)."""
    N = w.shape[-2]
    M = rows if rows is not None else dy.shape[0]
    K = w.shape[-1]
    if out is None:
        out = torch.empty((M, K), device=w.device, dtype=torch.float32)
    kw = {}
    if grouped is not None:
        kw = dict(sched=SCHED_GROUPED, tile_group=grouped[0], num_m_tiles=grouped[1])
    if packed is not None:
        kw.update(b_packed=packed[0], b_packed_group_stride=packed[1])
        if a_packed is not None:
            kw.update(a_packed=a_packed)
        elif _pack_a_pays(K, N):
            kw.update(a_packed=pack_act(dy, rows=M, cols=N, mn_major=False))
    gemm(A=dy, a_smn=N, a_sk=1, B=w, b_smn=1, b_sk=K, b_group_stride=w_group_stride, M=M, N=K, K=N, D=out, ldd=K,
         epilogue=epilogue | (EPI_COLSUM if colsum is not None else 0), aux_in=aux_in, ld_aux=K, row_scale=row_scale,
         resid=resid, ld_resid=K, colsum=colsum, colsum_group_stride=colsum_group_stride, **kw)
    return out


def linear_wgrad(dy, x, dw, *, rows=None, x_row_index=None, row_scale=None, segs=None, num_groups=1, dy_packed=None,
                 x_packed=None):
    """dw[g][N,K] += dy[rows_g, N]^T @ x[rows_g, K]  (split-K with fp32 atomics; dw must be pre-zeroed).

    row_scale (optional, [N]) scales the rows of dw (e.g. layer-scale gamma folded into the epilogue).
    segs = (seg_begin, seg_end) device int32 arrays selecting each group's row range.  When the operands are packed
    (dy_packed / x_packed given, or chosen below) the kernel reads whole 32-row blocks: every seg_begin must be a
    multiple of 32, and the rows [seg_end, ceil32(seg_end)) must be zero in dy or in x (gathered -1 rows are zero).
    """
    R = rows if rows is not None else dy.shape[0]
    N = dw.shape[-2]
    K = dw.shape[-1]
    tiles = ((N + 127) // 128) * _n_tiles(K) * num_groups
    # ~3 work items per SM (the per-expert segments are unequal), but at least 1024 reduction rows per split
    splits = -(-3 * num_sms() // max(1, tiles))
    splits = max(1, min(64 if tiles > 1 else 2 * num_sms(), splits, max(1, (R // num_groups) // 1024)))
    epi = EPI_ATOMIC | (EPI_ROWSCALE if row_scale is not None else 0)
    kw = {}
    if dy_packed is not None or x_packed is not None or ((N + 127) // 128) * _n_tiles(K) >= PACK_W_MIN_TILES:
        # both operands are re-read by several output tiles: split them once (MN-major images), gather included
        if dy_packed is None:
            dy_packed = pack_act(dy, rows=R, cols=N, mn_major=True, tile=128)
        if x_packed is None:
            x_packed = pack_act(x, rows=R, cols=K, mn_major=True, tile=_pick_bn(K), row_index=x_row_index)
        kw = dict(a_packed=dy_packed, b_packed=x_packed)
        x_row_index = None
    gemm(A=dy, a_smn=1, a_sk=N, B=x, b_smn=1, b_sk=K, M=N, N=K, K=R, D=dw, ldd=K, d_group_stride=N * K,
         b_k_index=x_row_index, **kw, sched=SCHED_SPLITK, k_splits=splits, num_groups=num_groups,
         seg_begin=None if segs is None else segs[0], seg_end=None if segs is None else segs[1],
         epilogue=epi, row_scale=row_scale)
    return dw


def layernorm_fwd(x, w, b, eps, *, tokens, C, out=None, out_mode=LN_NHWC, H=0, W=0, save_stats=False):
    lib = _lib.load()
    if out is None:
        out = torch.empty_like(x)
    stats = torch.empty((tokens, 2), device=x.device, dtype=torch.float32) if save_stats else None
    _lib.check(lib.sm3_layernorm_fwd(_p(x), _p(w), _p(b), _p(out), _p(stats), tokens, C, float(eps), out_mode, H, W,
                                     _stream()), 'sm3_layernorm_fwd')
    return out, stats


def layernorm_fwd_img(x, w, b, eps, *, tokens, C, save_stats=False, want_f32=False):
    """LayerNorm whose output is the K-major bf16 hi|lo operand image of the next GEMM -> (img, v_f32 | None, stats | None)."""
    lib = _lib.load()
    img = torch.empty((lib.sm3_gemm_packed_act_elems(tokens, C, 0, 128),), device=x.device, dtype=torch.int16)
    y = torch.empty((tokens, C), device=x.device, dtype=torch.float32) if want_f32 else None
    stats = torch.empty((tokens, 2), device=x.device, dtype=torch.float32) if save_stats else None
    _lib.check(lib.sm3_layernorm_fwd_img(_p(x), _p(w), _p(b), img.data_ptr(), _p(y), _p(stats), tokens, C, float(eps), _stream()),
               'sm3_layernorm_fwd_img')
    return img, y, stats


def layernorm_bwd(dy, x, stats, w, dw, db, *, tokens, C, in_mode=LN_NHWC, H=0, W=0, dx=None, accumulate=False):
    lib = _lib.load()
    if dx is None:
        dx = torch.empty((tokens, C), device=x.device, dtype=torch.float32)
    _lib.check(lib.sm3_layernorm_bwd(_p(dy), _p(x), _p(stats), _p(w), _p(dx), _p(dw), _p(db), tokens, C, in_mode, H, W,
                                     1 if accumulate else 0, _stream()), 'sm3_layernorm_bwd')
    return dx


def stem_fwd(x, wt, bias, lnw, lnb, eps, ps, *, save=False):
    lib = _lib.load()
    N, Cin, H, W = x.shape
    C0 = wt.shape[1]
    y = torch.empty((N, H // ps, W // ps, C0), device=x.device, dtype=torch.float32)
    conv = torch.empty_like(y) if save else None
    stats = torch.empty((N * (H // ps) * (W // ps), 2), device=x.device, dtype=torch.float32) if save else None
    _lib.check(lib.sm3_stem_fwd(_p(x), _p(wt), _p(bias), _p(lnw), _p(lnb), _p(y), _p(conv), _p(stats), N, Cin, H, W,
                                ps, C0, float(eps), _stream()), 'sm3_stem_fwd')
    return y, conv, stats


def stem_wgrad(x, du, dwt, dbias, ps):
    lib = _lib.load()
    N, Cin, H, W = x.shape
    _lib.check(lib.sm3_stem_wgrad(_p(x), _p(du), _p(dwt), _p(dbias), N, Cin, H, W, ps, dwt.shape[1], _stream()),
               'sm3_stem_wgrad')


def dwconv7(x, wt, bias=None, resid=None, out=None):
    lib = _lib.load()
    N, H, W, Cc = x.shape
    if out is None:
        out = torch.empty_like(x)
    _lib.check(lib.sm3_dwconv7_fwd(_p(x), _p(wt), _p(bias), _p(resid), _p(out), N, H, W, Cc, _stream()), 'sm3_dwconv7_fwd')
    return out


def dwconv7_ln(x, wt, bias, lnw, lnb, eps, *, want_u=False, want_stats=False, want_v=False, want_img=False):
    """Block front in one pass (sm3_dwconv7_ln_fwd): u = dwconv7(x) + bias and its LayerNorm v.  Returns (u, stats, v, img),
    absent outputs None.  Bit-identical to dwconv7 -> layernorm_fwd, or -> layernorm_fwd_img when want_img."""
    lib = _lib.load()
    N, H, W, Cc = x.shape
    T = N * H * W
    dev = x.device
    u = torch.empty((N, H, W, Cc), device=dev, dtype=torch.float32) if want_u else None
    stats = torch.empty((T, 2), device=dev, dtype=torch.float32) if want_stats else None
    v = torch.empty((T, Cc), device=dev, dtype=torch.float32) if want_v else None
    img = torch.empty((lib.sm3_gemm_packed_act_elems(T, Cc, 0, 128),), device=dev, dtype=torch.int16) if want_img else None
    _lib.check(lib.sm3_dwconv7_ln_fwd(_p(x), _p(wt), _p(bias), _p(lnw), _p(lnb), _p(u), _p(stats), _p(v),
                                      None if img is None else img.data_ptr(), N, H, W, Cc, float(eps), _stream()),
               'sm3_dwconv7_ln_fwd')
    return u, stats, v, img


def dwconv7_wgrad(x, dy, dwt, dbias):
    lib = _lib.load()
    N, H, W, Cc = x.shape
    _lib.check(lib.sm3_dwconv7_wgrad(_p(x), _p(dy), _p(dwt), _p(dbias), N, H, W, Cc, _stream()), 'sm3_dwconv7_wgrad')


def moe_router(v, wp, bp, sim, tau, *, T, Cc, E, k, w_noise=None, noise=None, save=False):
    lib = _lib.load()
    P = wp.shape[0]
    dev = v.device
    a = _lib.RouterArgs()
    top_idx = torch.empty((T, k), device=dev, dtype=torch.int32)
    top_gate = torch.empty((T, k), device=dev, dtype=torch.float32)
    logits = torch.empty((T, E), device=dev, dtype=torch.float32) if save else None
    p_out = torch.empty((T, P), device=dev, dtype=torch.float32) if save else None
    m = min(k + 1, E)
    noisy_save = save and noise is not None
    top_vals = torch.empty((T, m), device=dev, dtype=torch.float32) if noisy_save else None
    top_idx_m = torch.empty((T, m), device=dev, dtype=torch.int32) if noisy_save else None
    sigma = torch.empty((T, E), device=dev, dtype=torch.float32) if noisy_save else None
    nb = lib.sm3_moe_router_blocks(T)
    partials = torch.empty((nb, 3 * E), device=dev, dtype=torch.float32)
    a.v = _p(v); a.proj_weight = _p(wp); a.proj_bias = _p(bp); a.sim_matrix = _p(sim); a.temperature = _p(tau)
    a.w_noise = _p(w_noise) if noise is not None else None
    a.noise = _p(noise)
    a.T, a.C, a.P, a.E, a.k = T, Cc, P, E, k
    a.top_idx = _pi(top_idx); a.top_gate = _p(top_gate); a.logits = _p(logits); a.top_vals = _p(top_vals)
    a.p_out = _p(p_out); a.partials = _p(partials); a.sigma = _p(sigma); a.top_idx_m = _pi(top_idx_m)
    _lib.check(lib.sm3_moe_router(C.byref(a), _stream()), 'sm3_moe_router')
    return dict(top_idx=top_idx, top_gate=top_gate, logits=logits, p=p_out, top_vals=top_vals, partials=partials,
                sigma=sigma, top_idx_m=top_idx_m)


def moe_plan(partials, *, T, E, k):
    lib = _lib.load()
    dev = partials.device
    max_tiles = (T * k + 127) // 128 + E
    f = torch.empty(2 * E + 1, device=dev, dtype=torch.float32)
    i = torch.empty(4 * E + max_tiles + 1, device=dev, dtype=torch.int32)
    importance, load, loss = f[:E], f[E:2 * E], f[2 * E:2 * E + 1]
    counts, seg_begin, seg_end, cursor = i[:E], i[E:2 * E], i[2 * E:3 * E], i[3 * E:4 * E]
    tile_group = i[4 * E:4 * E + max_tiles]
    num_m_tiles = i[4 * E + max_tiles:]
    a = _lib.PlanArgs()
    a.partials = _p(partials); a.T, a.E, a.k, a.max_m_tiles = T, E, k, max_tiles
    a.importance = importance.data_ptr(); a.load = load.data_ptr(); a.loss = loss.data_ptr()
    a.counts = counts.data_ptr(); a.seg_begin = seg_begin.data_ptr(); a.seg_end = seg_end.data_ptr()
    a.cursor = cursor.data_ptr(); a.tile_group = tile_group.data_ptr(); a.num_m_tiles = num_m_tiles.data_ptr()
    _lib.check(lib.sm3_moe_plan(C.byref(a), _stream()), 'sm3_moe_plan')
    return dict(importance=importance, load=load, loss=loss, counts=counts, seg_begin=seg_begin, seg_end=seg_end,
                cursor=cursor, tile_group=tile_group, num_m_tiles=num_m_tiles, max_rows=max_tiles * 128)


def moe_assign(top_idx, plan, *, T, E, k):
    lib = _lib.load()
    dev = top_idx.device
    slot_of = torch.empty((T, k), device=dev, dtype=torch.int32)
    pair_token = torch.full((plan['max_rows'],), -1, device=dev, dtype=torch.int32)
    _lib.check(lib.sm3_moe_assign(_pi(top_idx), T, k, E, plan['seg_begin'].data_ptr(), plan['cursor'].data_ptr(),
                                  _pi(slot_of), _pi(pair_token), _stream()), 'sm3_moe_assign')
    return slot_of, pair_token


def moe_combine(o, slot_of, top_idx, gate, gamma, resid, row_scale, *, T, Cc, k, want_y=False):
    lib = _lib.load()
    out = torch.empty((T, Cc), device=o.device, dtype=torch.float32)
    y = torch.empty((T, Cc), device=o.device, dtype=torch.float32) if want_y else None
    _lib.check(lib.sm3_moe_combine(_p(o), _pi(slot_of), _pi(top_idx), _p(gate), _p(gamma), _p(resid), _p(row_scale),
                                   _p(out), _p(y), T, Cc, k, _stream()), 'sm3_moe_combine')
    return out, y


def moe_combine_bwd(dout, o, slot_of, top_idx, gate, gamma, row_scale, d_o, dgamma, *, T, Cc, k):
    lib = _lib.load()
    dgate = torch.empty((T, k), device=o.device, dtype=torch.float32)
    _lib.check(lib.sm3_moe_combine_bwd(_p(dout), _p(o), _pi(slot_of), _pi(top_idx), _p(gate), _p(gamma), _p(row_scale),
                                       _p(d_o), _p(dgate), _p(dgamma), T, Cc, k, _stream()), 'sm3_moe_combine_bwd')
    return dgate


def moe_router_bwd(p, sim, tau, top_idx, top_gate, dgate, logits, importance, loss_scale, dsim, dtau, *, T, E, k,
                   noisy=None):
    """noisy = dict(noise, sigma, top_vals, top_idx_m, load) for noisy gating; returns (dp, dr) with dr [T,32] or None."""
    lib = _lib.load()
    P = p.shape[1]
    dp = torch.empty_like(p)
    dr = None
    dsim_hat = torch.zeros((P, E), device=p.device, dtype=torch.float32)
    a = _lib.RouterBwdArgs()
    a.p = _p(p); a.sim_matrix = _p(sim); a.temperature = _p(tau); a.top_idx = _pi(top_idx); a.top_gate = _p(top_gate)
    a.dgate = _p(dgate); a.logits = _p(logits); a.importance = importance.data_ptr(); a.loss_scale = _p(loss_scale)
    a.T, a.P, a.E, a.k = T, P, E, k
    a.dp = _p(dp); a.dsim_hat = _p(dsim_hat); a.dtemperature = _p(dtau)
    if noisy is not None:
        dr = torch.empty((T, 32), device=p.device, dtype=torch.float32)
        a.noise = _p(noisy['noise']); a.sigma = _p(noisy['sigma']); a.top_vals = _p(noisy['top_vals'])
        a.top_idx_m = _pi(noisy['top_idx_m']); a.load = noisy['load'].data_ptr(); a.dr = _p(dr)
    _lib.check(lib.sm3_moe_router_bwd(C.byref(a), _stream()), 'sm3_moe_router_bwd')
    _lib.check(lib.sm3_moe_router_bwd_finalize(_p(dsim_hat), _p(sim), _p(dsim), P, E, _stream()),
               'sm3_moe_router_bwd_finalize')
    return dp, dr


def colsum(a, out, *, rows, Cc, b=None, row_scale=None, segs=None, groups=1):
    lib = _lib.load()
    _lib.check(lib.sm3_colsum(_p(a), _p(b), _p(row_scale), None if segs is None else segs[0].data_ptr(),
                              None if segs is None else segs[1].data_ptr(), groups, _p(out), rows, Cc, _stream()),
               'sm3_colsum')
    return out


def gather_sum(src, slot_of, add, *, T, Cc, k, out=None):
    lib = _lib.load()
    if out is None:
        out = torch.empty((T, Cc), device=src.device, dtype=torch.float32)
    _lib.check(lib.sm3_gather_sum(_p(src), _pi(slot_of), _p(add), _p(out), T, Cc, k, _stream()), 'sm3_gather_sum')
    return out


def scale_rows(x, row_scale=None, col_scale=None, out=None):
    lib = _lib.load()
    Cc = x.shape[-1]
    rows = x.numel() // Cc
    if out is None:
        out = torch.empty_like(x)
    _lib.check(lib.sm3_scale_rows(_p(x), _p(row_scale), _p(col_scale), _p(out), rows, Cc, _stream()), 'sm3_scale_rows')
    return out


# ---- LSKNet-MoE (BASELINE config 5) ---------------------------------------------------------------------------
def dwconv(x, wt, bias=None, resid=None, *, ks, dil=1, out=None):
    """Depthwise ks x ks conv (dilation dil, "same" padding) on NHWC x; wt = taps [ks*ks, C]."""
    lib = _lib.load()
    N, H, W, Cc = x.shape
    if out is None:
        out = torch.empty_like(x)
    _lib.check(lib.sm3_dwconv_fwd(_p(x), _p(wt), _p(bias), _p(resid), _p(out), N, H, W, Cc, ks, dil, _stream()), 'sm3_dwconv_fwd')
    return out


def dwconv_wgrad(x, dy, dwt, dbias, *, ks, dil=1):
    lib = _lib.load()
    N, H, W, Cc = x.shape
    _lib.check(lib.sm3_dwconv_wgrad(_p(x), _p(dy), _p(dwt), _p(dbias), N, H, W, Cc, ks, dil, _stream()), 'sm3_dwconv_wgrad')


def colstat(x, *, rows, Cc, sh1=None, y=None, sh2=None, sc2=None, want_s1=True, want_s2=True):
    """(s1, s2): s1[c] = sum_r (x-sh1), s2[c] = sum_r (x-sh1) * (y ? (y-sh2)*sc2 : (x-sh1))."""
    lib = _lib.load()
    s = torch.zeros((2, Cc), device=x.device, dtype=torch.float32)
    _lib.check(lib.sm3_colstat(_p(x), _p(sh1), _p(y), _p(sh2), _p(sc2), s[0].data_ptr() if want_s1 else None,
                               s[1].data_ptr() if want_s2 else None, rows, Cc, _stream()), 'sm3_colstat')
    return s[0], s[1]


def affine(x1, a1=None, x2=None, a2=None, b=None, add=None, out=None):
    """out = a1[c]*x1 + a2[c]*x2 + b[c] + add  (channels-last; None operands skipped)."""
    lib = _lib.load()
    Cc = x1.shape[-1]
    rows = x1.numel() // Cc
    if out is None:
        out = torch.empty_like(x1)
    _lib.check(lib.sm3_affine(_p(x1), _p(a1), _p(x2), _p(a2), _p(b), _p(add), _p(out), rows, Cc, _stream()), 'sm3_affine')
    return out


def mul(a, b, add=None, out=None):
    lib = _lib.load()
    if out is None:
        out = torch.empty_like(a)
    _lib.check(lib.sm3_mul(_p(a), _p(b), _p(add), _p(out), a.numel(), _stream()), 'sm3_mul')
    return out


def dropout(x, p, seed):
    """seed: python int, or an int64 device tensor [1] (read by the kernel: CUDA-graph safe)."""
    lib = _lib.load()
    out = torch.empty_like(x)
    if torch.is_tensor(seed):
        assert seed.is_cuda and seed.dtype == torch.int64 and seed.numel() == 1
        _lib.check(lib.sm3_dropout_dev(_p(x), _p(out), x.numel(), float(p), seed.data_ptr(), _stream()), 'sm3_dropout_dev')
    else:
        _lib.check(lib.sm3_dropout(_p(x), _p(out), x.numel(), float(p), int(seed), _stream()), 'sm3_dropout')
    return out


def _drop_seed(seed):
    """(host seed, device seed pointer) of a dropout seed: a python int, or an int64 device tensor [1]."""
    if torch.is_tensor(seed):
        assert seed.is_cuda and seed.dtype == torch.int64 and seed.numel() == 1
        return 0, seed.data_ptr()
    return int(seed), None


def mlp_mid_fwd(h, wt, bias, *, p=0.0, seed=0, mask=None):
    """a = dropout(gelu(dwconv3x3(h) + bias)) on NHWC h (sm3_mlp_mid_fwd); wt = taps [9, C].  ``mask`` (pre-scaled keep
    mask, h's shape) replaces the hashed mask of ``seed``; p = 0 without a mask is no dropout."""
    lib = _lib.load()
    N, H, W, Cc = h.shape
    out = torch.empty_like(h)
    s, sdev = _drop_seed(seed)
    _lib.check(lib.sm3_mlp_mid_fwd(_p(h), _p(wt), _p(bias), _p(mask), _p(out), N, H, W, Cc, float(p), s, sdev, _stream()),
               'sm3_mlp_mid_fwd')
    return out


def mlp_mid_bwd(h, wt, bias, da, dwt, dbias, *, p=0.0, seed=0, mask=None):
    """dh of mlp_mid_fwd; dwt [9, C] and dbias [C] are accumulated."""
    lib = _lib.load()
    N, H, W, Cc = h.shape
    dh = torch.empty_like(h)
    s, sdev = _drop_seed(seed)
    _lib.check(lib.sm3_mlp_mid_bwd(_p(h), _p(wt), _p(bias), _p(da), _p(mask), _p(dh), _p(dwt), _p(dbias), N, H, W, Cc,
                                   float(p), s, sdev, _stream()), 'sm3_mlp_mid_bwd')
    return dh


def lsk_agg(a1, a2, *, T, Ch, want_idx=True):
    lib = _lib.load()
    agg = torch.empty((T, 2), device=a1.device, dtype=torch.float32)
    amax = torch.empty((T,), device=a1.device, dtype=torch.int32) if want_idx else None
    _lib.check(lib.sm3_lsk_agg(_p(a1), _p(a2), _p(agg), _pi(amax), T, Ch, _stream()), 'sm3_lsk_agg')
    return agg, amax


def conv7_c2(x, w, b, *, N, H, W, act):
    lib = _lib.load()
    y = torch.empty((N * H * W, 2), device=x.device, dtype=torch.float32)
    _lib.check(lib.sm3_conv7_c2(_p(x), _p(w), _p(b), _p(y), N, H, W, act, _stream()), 'sm3_conv7_c2')
    return y


def conv7_c2_wgrad(x, dpre, dw, db, *, N, H, W):
    lib = _lib.load()
    _lib.check(lib.sm3_conv7_c2_wgrad(_p(x), _p(dpre), _p(dw), _p(db), N, H, W, _stream()), 'sm3_conv7_c2_wgrad')


def lsk_mix(a1, a2, sig, *, T, Ch):
    lib = _lib.load()
    out = torch.empty((T, Ch), device=a1.device, dtype=torch.float32)
    _lib.check(lib.sm3_lsk_mix(_p(a1), _p(a2), _p(sig), _p(out), T, Ch, _stream()), 'sm3_lsk_mix')
    return out


def lsk_mix_bwd_sig(dout, a1, a2, sig, *, T, Ch):
    lib = _lib.load()
    dpre = torch.empty((T, 2), device=a1.device, dtype=torch.float32)
    _lib.check(lib.sm3_lsk_mix_bwd_sig(_p(dout), _p(a1), _p(a2), _p(sig), _p(dpre), T, Ch, _stream()), 'sm3_lsk_mix_bwd_sig')
    return dpre


def lsk_mix_bwd_in(dout, sig, dagg, amax, *, T, Ch):
    lib = _lib.load()
    da1 = torch.empty((T, Ch), device=dout.device, dtype=torch.float32)
    da2 = torch.empty((T, Ch), device=dout.device, dtype=torch.float32)
    _lib.check(lib.sm3_lsk_mix_bwd_in(_p(dout), _p(sig), _p(dagg), _pi(amax), _p(da1), _p(da2), T, Ch, _stream()),
               'sm3_lsk_mix_bwd_in')
    return da1, da2


def im2col(x, *, N, H, W, Cin, ks, stride, pad, Kp, nchw):
    lib = _lib.load()
    Ho, Wo = (H + 2 * pad - ks) // stride + 1, (W + 2 * pad - ks) // stride + 1
    col = torch.empty((N * Ho * Wo, Kp), device=x.device, dtype=torch.float32)
    _lib.check(lib.sm3_im2col(_p(x), _p(col), N, H, W, Cin, ks, stride, pad, Kp, 1 if nchw else 0, _stream()), 'sm3_im2col')
    return col, Ho, Wo


def col2im(dcol, *, N, H, W, Cin, ks, stride, pad, Kp, nchw=False):
    lib = _lib.load()
    dx = torch.empty((N, Cin, H, W) if nchw else (N, H, W, Cin), device=dcol.device, dtype=torch.float32)
    _lib.check(lib.sm3_col2im(_p(dcol), _p(dx), N, H, W, Cin, ks, stride, pad, Kp, 1 if nchw else 0, _stream()), 'sm3_col2im')
    return dx


def gather_rows_peer(bases, src_rank, src_row, *, rows, Cc, token_lists=None, scale=None, out=None):
    """out[r] = scale[r] * peer_buffer[src_rank[r]][row]  (bases / token_lists: int64 device tensors of peer pointers)."""
    lib = _lib.load()
    if out is None:
        out = torch.empty((rows, Cc), device=src_rank.device, dtype=torch.float32)
    _lib.check(lib.sm3_gather_rows_peer(_p(bases, torch.int64), None if token_lists is None else _p(token_lists, torch.int64),
                                        _pi(src_rank), _pi(src_row), _p(scale), _p(out), rows, Cc, _stream()),
               'sm3_gather_rows_peer')
    return out


# ---- MultitaskFPN ------------------------------------------------------------------------------------------------
def upsample_add(a, b):
    """a[N,H,W,C] + nearest-upsampled b[N,h,w,C]."""
    lib = _lib.load()
    N, H, W, Cc = a.shape
    out = torch.empty_like(a)
    _lib.check(lib.sm3_upsample_add(_p(a), _p(b), _p(out), N, H, W, b.shape[1], b.shape[2], Cc, _stream()), 'sm3_upsample_add')
    return out


def upsample_add_bwd(d, h, w):
    lib = _lib.load()
    N, H, W, Cc = d.shape
    db = torch.empty((N, h, w, Cc), device=d.device, dtype=torch.float32)
    _lib.check(lib.sm3_upsample_add_bwd(_p(d), _p(db), N, H, W, h, w, Cc, _stream()), 'sm3_upsample_add_bwd')
    return db


def transpose_batched(x, B, R, Cc, out_shape):
    """out[b,c,r] = x[b,r,c] (x viewed as [B,R,Cc])."""
    lib = _lib.load()
    out = torch.empty(out_shape, device=x.device, dtype=torch.float32)
    _lib.check(lib.sm3_transpose_batched(_p(x), _p(out), B, R, Cc, _stream()), 'sm3_transpose_batched')
    return out
