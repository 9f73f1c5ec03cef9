"""ctypes binding of the C-ABI CUDA library (include/sm3det_b200.h).

The library is built in-tree (``make`` or ``__graft_entry__.build()``) as
``sm3det_b200/lib/libsm3det_b200.so``.  There is NO fallback: if the library is missing or the
device is not sm_90, calling any op raises -- the product path never silently runs on PyTorch/CPU.
"""
import ctypes as C
import os
import threading

_LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'lib', 'libsm3det_b200.so')
_lock = threading.Lock()
_lib = None
LAUNCHES = 0   # number of C-ABI kernel-launching calls made (bench.py reports it as gpu_launches)

c_f32p = C.c_void_p      # device pointers travel as integers
c_i32p = C.c_void_p
c_stream = C.c_void_p


class GemmArgs(C.Structure):
    _fields_ = [
        ('A', c_f32p), ('a_stride_mn', C.c_int64), ('a_stride_k', C.c_int64),
        ('B', c_f32p), ('b_stride_mn', C.c_int64), ('b_stride_k', C.c_int64), ('b_group_stride', C.c_int64),
        ('a_row_index', c_i32p), ('b_k_index', c_i32p), ('b_packed', C.c_void_p), ('b_packed_group_stride', C.c_int64), ('a_packed', C.c_void_p),
        ('M', C.c_int32), ('N', C.c_int32), ('K', C.c_int32),
        ('tile_n', C.c_int32), ('sched', C.c_int32), ('k_splits', C.c_int32), ('num_groups', C.c_int32),
        ('tile_group', c_i32p), ('num_m_tiles', c_i32p), ('seg_begin', c_i32p), ('seg_end', c_i32p),
        ('D', c_f32p), ('ldd', C.c_int64), ('d_group_stride', C.c_int64),
        ('bias', c_f32p), ('bias_group_stride', C.c_int64),
        ('epilogue', C.c_int32),
        ('aux_out', c_f32p), ('aux_in', c_f32p), ('ld_aux', C.c_int64),
        ('col_scale', c_f32p), ('row_scale', c_f32p),
        ('resid', c_f32p), ('ld_resid', C.c_int64),
        ('colsum', c_f32p), ('colsum_group_stride', C.c_int64),
        ('mma_passes', C.c_int32),
    ]


class RouterArgs(C.Structure):
    _fields_ = [
        ('v', c_f32p), ('proj_weight', c_f32p), ('proj_bias', c_f32p), ('sim_matrix', c_f32p),
        ('temperature', c_f32p), ('w_noise', c_f32p), ('noise', c_f32p),
        ('T', C.c_int32), ('C', C.c_int32), ('P', C.c_int32), ('E', C.c_int32), ('k', C.c_int32),
        ('top_idx', c_i32p), ('top_gate', c_f32p), ('logits', c_f32p), ('top_vals', c_f32p), ('p_out', c_f32p),
        ('sigma', c_f32p), ('top_idx_m', c_i32p),
        ('partials', c_f32p),
    ]


class PlanArgs(C.Structure):
    _fields_ = [
        ('partials', c_f32p), ('T', C.c_int32), ('E', C.c_int32), ('k', C.c_int32), ('max_m_tiles', C.c_int32),
        ('importance', c_f32p), ('load', c_f32p), ('loss', c_f32p),
        ('counts', c_i32p), ('seg_begin', c_i32p), ('seg_end', c_i32p), ('cursor', c_i32p),
        ('tile_group', c_i32p), ('num_m_tiles', c_i32p),
    ]


class FfnArgs(C.Structure):
    _fields_ = [
        ('a1', C.c_void_p), ('a2', C.c_void_p), ('wa1', C.c_void_p), ('wa2', C.c_void_p), ('wb', C.c_void_p),
        ('bias1', c_f32p), ('bias2', c_f32p), ('col_scale', c_f32p), ('row_scale', c_f32p), ('resid', c_f32p),
        ('out', c_f32p), ('aux_out', c_f32p), ('h_out', c_f32p),
        ('M', C.c_int32), ('C', C.c_int32), ('H4', C.c_int32), ('chunk', C.c_int32), ('mma_passes', C.c_int32),
        ('mode', C.c_int32),
        ('dh_mn', C.c_void_p), ('act_mn', C.c_void_p), ('db1', c_f32p), ('h_in', c_f32p),
    ]


class EpPlanArgs(C.Structure):
    _fields_ = [
        ('allm', c_i32p), ('tile_group_s', c_i32p), ('num_tiles_s', c_i32p), ('pair_token', c_i32p),
        ('W', C.c_int32), ('me', C.c_int32), ('E', C.c_int32), ('R_s', C.c_int32), ('cap', C.c_int32),
        ('src_rank', c_i32p), ('src_slot', c_i32p), ('tile_group', c_i32p), ('num_tiles', c_i32p),
        ('seg_begin', c_i32p), ('seg_end', c_i32p), ('comb_rank', c_i32p), ('comb_row', c_i32p), ('overflow', c_i32p),
    ]


# name -> argtypes (restype is always int unless listed in _RESTYPES); mirrors include/sm3det_b200.h
_I32, _I64, _F32, _P = C.c_int32, C.c_int64, C.c_float, C.c_void_p
SIGNATURES = {
    'sm3_abi_version': [],
    'sm3_last_error': [],
    'sm3_device_supported': [],
    'sm3_gemm': [C.POINTER(GemmArgs), _P],
    'sm3_gemm_packed_elems': [_I32, _I32],
    'sm3_gemm_pack_b': [_P, _I64, _I64, _I64, _I32, _I32, _I32, _P, _P],
    'sm3_gemm_packed_act_elems': [_I64, _I32, _I32, _I32],
    'sm3_gemm_pack_act': [_P, _I64, _P, _I64, _I32, _I32, _I32, _P, _P],
    'sm3_gemm_tile_n': [_I32],
    'sm3_gemm_pack_b_tile': [_P, _I64, _I64, _I64, _I32, _I32, _I32, _I32, _P, _P],
    'sm3_gemm_workspace_bytes': [C.POINTER(GemmArgs)],
    'sm3_ffn_fused_chunk': [_I32, _I32],
    'sm3_ffn_fused': [C.POINTER(FfnArgs), _P],
    'sm3_ffn_fused_workspace_bytes': [C.POINTER(FfnArgs)],
    'sm3_moe_router_workspace_bytes': [C.POINTER(RouterArgs)],
    'sm3_moe_plan_workspace_bytes': [C.POINTER(PlanArgs)],
    'sm3_layernorm_fwd': [_P, _P, _P, _P, _P, _I64, _I32, _F32, _I32, _I32, _I32, _P],
    'sm3_layernorm_fwd_img': [_P, _P, _P, _P, _P, _P, _I64, _I32, _F32, _P],
    'sm3_layernorm_bwd': [_P, _P, _P, _P, _P, _P, _P, _I64, _I32, _I32, _I32, _I32, _I32, _P],
    'sm3_stem_fwd': [_P, _P, _P, _P, _P, _P, _P, _P, _I32, _I32, _I32, _I32, _I32, _I32, _F32, _P],
    'sm3_stem_wgrad': [_P, _P, _P, _P, _I32, _I32, _I32, _I32, _I32, _I32, _P],
    'sm3_dwconv7_fwd': [_P, _P, _P, _P, _P, _I32, _I32, _I32, _I32, _P],  # x, wt, bias, resid, y, N, H, W, C, stream
    'sm3_dwconv7_wgrad': [_P, _P, _P, _P, _I32, _I32, _I32, _I32, _P],
    # x, wt, bias, ln_weight, ln_bias, u, stats, v, img, N, H, W, C, eps, stream
    'sm3_dwconv7_ln_fwd': [_P, _P, _P, _P, _P, _P, _P, _P, _P, _I32, _I32, _I32, _I32, _F32, _P],
    'sm3_moe_router_bwd_finalize': [_P, _P, _P, _I32, _I32, _P],
    'sm3_moe_router_blocks': [_I32],
    'sm3_moe_router': [C.POINTER(RouterArgs), _P],
    'sm3_moe_plan': [C.POINTER(PlanArgs), _P],
    'sm3_moe_assign': [_P, _I32, _I32, _I32, _P, _P, _P, _P, _P],
    'sm3_moe_combine': [_P, _P, _P, _P, _P, _P, _P, _P, _P, _I32, _I32, _I32, _P],
    'sm3_moe_combine_bwd': [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I32, _I32, _I32, _P],
    'sm3_colsum': [_P, _P, _P, _P, _P, _I32, _P, _I64, _I32, _P],
    'sm3_gather_sum': [_P, _P, _P, _P, _I32, _I32, _I32, _P],
    'sm3_scale_rows': [_P, _P, _P, _P, _I64, _I32, _P],
    'sm3_moe_router_bwd': [_P, _P],
    'sm3_ep_plan': [C.POINTER(EpPlanArgs), _P],
    'sm3_gather_rows_peer': [_P, _P, _P, _P, _P, _P, _I64, _I32, _P],
    'sm3_upsample_add': [_P, _P, _P, _I32, _I32, _I32, _I32, _I32, _I32, _P],
    'sm3_upsample_add_bwd': [_P, _P, _I32, _I32, _I32, _I32, _I32, _I32, _P],
    'sm3_transpose_batched': [_P, _P, _I32, _I32, _I32, _P],
    # in / din, host array of L+1 level pointers, N, H, W, C, L, stream
    'sm3_fpn_export_pool': [_P, _P, _I32, _I32, _I32, _I32, _I32, _P],
    'sm3_fpn_export_pool_bwd': [_P, _P, _I32, _I32, _I32, _I32, _I32, _P],
    # OrientedRPNHead: host shape array [L][3] = (N, H, W), host arrays of level pointers
    'sm3_rpn_head_rows': [_P, _I32],
    # x, cls, reg, shapes, L, Cin, wconv_img, bconv, whead_img, bhead, ncls, nreg, h_out, mma_passes, stream
    'sm3_rpn_head_fwd': [_P, _P, _P, _P, _I32, _I32, _P, _P, _P, _P, _I32, _I32, _P, _I32, _P],
    # h, dcls, dreg, shapes, L, whead, ncls, nreg, dpre, dwhead, dbhead, dbconv, stream
    'sm3_rpn_head_mid_bwd': [_P, _P, _P, _P, _I32, _P, _I32, _I32, _P, _P, _P, _P, _P],
    # dpre, dx, shapes, L, Cin, wdx_img, mma_passes, stream
    'sm3_rpn_head_dx': [_P, _P, _P, _I32, _I32, _P, _I32, _P],
    'sm3_rpn_head_tap_index': [_P, _I32, _P, _P],
    # LSKNet-MoE
    'sm3_dwconv_fwd': [_P, _P, _P, _P, _P, _I32, _I32, _I32, _I32, _I32, _I32, _P],
    'sm3_dwconv_wgrad': [_P, _P, _P, _P, _I32, _I32, _I32, _I32, _I32, _I32, _P],
    'sm3_colstat': [_P, _P, _P, _P, _P, _P, _P, _I64, _I32, _P],
    'sm3_affine': [_P, _P, _P, _P, _P, _P, _P, _I64, _I32, _P],
    'sm3_mul': [_P, _P, _P, _P, _I64, _P],
    'sm3_dropout': [_P, _P, _I64, _F32, C.c_uint64, _P],
    'sm3_dropout_dev': [_P, _P, _I64, _F32, _P, _P],
    # h, weight_t, bias, mask, a, N, H, W, C, p, seed, seed_dev, stream
    'sm3_mlp_mid_fwd': [_P, _P, _P, _P, _P, _I32, _I32, _I32, _I32, _F32, C.c_uint64, _P, _P],
    # h, weight_t, bias, da, mask, dh, dweight_t, dbias, N, H, W, C, p, seed, seed_dev, stream
    'sm3_mlp_mid_bwd': [_P, _P, _P, _P, _P, _P, _P, _P, _I32, _I32, _I32, _I32, _F32, C.c_uint64, _P, _P],
    'sm3_lsk_agg': [_P, _P, _P, _P, _I64, _I32, _P],
    'sm3_conv7_c2': [_P, _P, _P, _P, _I32, _I32, _I32, _I32, _P],
    'sm3_conv7_c2_wgrad': [_P, _P, _P, _P, _I32, _I32, _I32, _P],
    'sm3_lsk_mix': [_P, _P, _P, _P, _I64, _I32, _P],
    'sm3_lsk_mix_bwd_sig': [_P, _P, _P, _P, _P, _I64, _I32, _P],
    'sm3_lsk_mix_bwd_in': [_P, _P, _P, _P, _P, _P, _I64, _I32, _P],
    'sm3_im2col': [_P, _P, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _P],
    'sm3_col2im': [_P, _P, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _P],
}
_RESTYPES = {'sm3_last_error': C.c_char_p, 'sm3_gemm_packed_elems': C.c_int64, 'sm3_gemm_packed_act_elems': C.c_int64, 'sm3_rpn_head_rows': C.c_int64,
             'sm3_gemm_workspace_bytes': C.c_size_t, 'sm3_ffn_fused_workspace_bytes': C.c_size_t,
             'sm3_moe_router_workspace_bytes': C.c_size_t, 'sm3_moe_plan_workspace_bytes': C.c_size_t}


class ActPackArgs(C.Structure):
    _fields_ = [
        ('h', c_f32p), ('da', c_f32p), ('R', C.c_int64), ('W', C.c_int32), ('mode', C.c_int32),
        ('live_tiles', c_i32p), ('tile_group', c_i32p),
        ('out_f32', c_f32p), ('pack_k', C.c_void_p), ('pack_mn', C.c_void_p), ('mn_tile', C.c_int32), ('colsum', c_f32p),
        ('pack_mn2', C.c_void_p), ('mn_tile2', C.c_int32),
    ]


class RouterBwdArgs(C.Structure):
    _fields_ = [
        ('p', c_f32p), ('sim_matrix', c_f32p), ('temperature', c_f32p),
        ('top_idx', c_i32p), ('top_gate', c_f32p), ('dgate', c_f32p), ('logits', c_f32p),
        ('importance', c_f32p), ('loss_scale', c_f32p),
        ('T', C.c_int32), ('P', C.c_int32), ('E', C.c_int32), ('k', C.c_int32),
        ('dp', c_f32p), ('dsim_hat', c_f32p), ('dtemperature', c_f32p),
        ('noise', c_f32p), ('sigma', c_f32p), ('top_vals', c_f32p), ('top_idx_m', c_i32p), ('load', c_f32p),
        ('dr', c_f32p),
    ]


SIGNATURES['sm3_moe_router_bwd'] = [C.POINTER(RouterBwdArgs), _P]
SIGNATURES['sm3_act_pack'] = [C.POINTER(ActPackArgs), _P]


def library_path() -> str:
    return _LIB_PATH


def load():
    """Load (once) and return the ctypes handle; raises if the CUDA library has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.isfile(_LIB_PATH):
            raise RuntimeError(
                f'sm3det_b200: CUDA library not built ({_LIB_PATH} missing). Run `make` at the repo root or '
                f'`python -c "import __graft_entry__ as g; g.build()"`. There is no CPU/PyTorch fallback.')
        lib = C.CDLL(_LIB_PATH)
        for name, argtypes in SIGNATURES.items():
            fn = getattr(lib, name)   # AttributeError here = header/library mismatch: fail loudly
            fn.argtypes = argtypes
            fn.restype = _RESTYPES.get(name, C.c_int)
        if lib.sm3_abi_version() != 1:
            raise RuntimeError('sm3det_b200: ABI version mismatch')
        _lib = lib
    return _lib


def check(rc: int, what: str):
    global LAUNCHES
    LAUNCHES += 1
    if rc != 0:
        msg = load().sm3_last_error()
        raise RuntimeError(f'sm3det_b200: {what} failed (rc={rc}): {msg.decode() if msg else "?"}')
