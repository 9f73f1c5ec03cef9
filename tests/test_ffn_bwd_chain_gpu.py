"""The fused dense-FFN backward that emits the weight-gradient operands (`ffn_chain_kernel` modes 2 and 3,
csrc/ffn_fused.cu) against a float64 reference, and the dense block's backward on it against the GEMM sequence.

Mode 2 (C <= 128) recomputes h = v W1^T + b1 from the v image; mode 3 (C = 192) reads the saved fp32 h.  Both form
d = dzs (gamma W2) and dh = d * gelu'(h) on chip and write dv = dh W1, db1 += sum_t dh, and the MN-major images (128-column
tiles, act_pack's layout) of dh and gelu(h) that the two split-K weight-gradient GEMMs read.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

import gemm_ref as R
from test_gemm_gpu import U, gelu_bound, gelu_grad_bound, split_err, tau

pytestmark = pytest.mark.gpu

SENT16 = 0x7A11          # int16 sentinel of the image buffers
SENT32 = 0x7FA11A11      # fp32 NaN payload of the dv / db1 buffers
GUARD = 4096             # sentinel elements before and after every output


@pytest.fixture(scope='module')
def ops():
    from sm3det_b200 import ops as o
    return o


def _guarded(n, dtype, fill):
    buf = torch.full((GUARD + n + GUARD,), fill, dtype=torch.int32 if dtype == torch.float32 else dtype, device='cuda')
    return buf if dtype != torch.float32 else buf.view(torch.float32)


def _run_chain(ops, mode, *, M, C, chunk, v_img, dz_img, w1c, w2gt, w1tn, b1, h):
    """One launch through the C ABI into sentinel-guarded outputs -> (dv, dh_mn, a_mn, db1, guard_ok)."""
    from sm3det_b200 import _lib
    lib = _lib.load()
    n_img = lib.sm3_gemm_packed_act_elems(M, 4 * C, 1, 128)
    dv = _guarded(M * C, torch.float32, SENT32)
    dh, am = _guarded(n_img, torch.int16, SENT16), _guarded(n_img, torch.int16, SENT16)
    db1 = _guarded(4 * C, torch.float32, SENT32)
    db1[GUARD:GUARD + 4 * C] = 0.0
    a = ops._ffn_args(T=M, C=C, chunk=chunk, mode=mode, a1=v_img if mode == 2 else dz_img, a2=dz_img,
                      wa1=w1c if mode == 2 else w2gt, wa2=w2gt, b1=b1, wb=w1tn)
    a.out = dv[GUARD:].data_ptr()
    a.dh_mn = dh[GUARD:].data_ptr(); a.act_mn = am[GUARD:].data_ptr()
    a.db1 = db1[GUARD:].data_ptr(); a.h_in = None if h is None else h.data_ptr()
    _lib.check(lib.sm3_ffn_fused(ctypes.byref(a), torch.cuda.current_stream().cuda_stream), 'sm3_ffn_fused')
    torch.cuda.synchronize()
    ok = True
    for buf, n in ((dv, M * C), (db1, 4 * C)):
        bits = buf.view(torch.int32)
        ok &= bool((bits[:GUARD] == SENT32).all()) and bool((bits[GUARD + n:] == SENT32).all())
    for buf in (dh, am):
        ok &= bool((buf[:GUARD] == SENT16).all()) and bool((buf[GUARD + n_img:] == SENT16).all())
    return (dv[GUARD:GUARD + M * C].view(M, C).cpu().numpy().astype(np.float64), dh[GUARD:GUARD + n_img].cpu(),
            am[GUARD:GUARD + n_img].cpu(), db1[GUARD:GUARD + 4 * C].cpu().numpy().astype(np.float64), ok)


def _cases():
    out = []
    for C in (32, 64, 96, 128, 192):
        Ms = [300, 512] + ([2 * 132 * 128 + 2 * 128 + 77] if C in (96, 192) else [])
        for M in Ms:
            for passes in (1, 3):
                for drop in (False, True):
                    if M > 1000 and (passes == 1 or not drop):
                        continue
                    out.append(pytest.param(C, M, passes, drop, id=f'C{C}-M{M}-p{passes}-{"drop" if drop else "nodrop"}'))
    return out


@pytest.mark.parametrize('C,M,passes,drop', _cases())
def test_ffn_bwd_chain_against_float64(ops, C, M, passes, drop):
    from sm3det_b200.ops import precision_scope
    mode = 2 if C <= 128 else 3
    cb = ops.ffn_chunk(mode, C)
    assert cb > 0 and ops.ffn_chunk(5 - mode, C) == 0
    if M > 1000:
        assert -(-M // 128) > 2 * ops.num_sms()
    rng = np.random.default_rng(C * 7 + M + passes + drop)
    H4 = 4 * C
    v = rng.standard_normal((M, C)).astype(np.float32)
    dz = rng.standard_normal((M, C)).astype(np.float32)
    if drop:                                     # drop-path: the caller packs dzs = row_scale * dz
        rs = np.exp2(rng.integers(-1, 2, M)).astype(np.float32)
        rs[::5] = 0
        dz = (dz * rs[:, None]).astype(np.float32)
    W1 = (rng.standard_normal((H4, C)) / math.sqrt(C)).astype(np.float32)
    b1 = (rng.standard_normal(H4) * 0.2).astype(np.float32)
    W2g = (rng.standard_normal((C, H4)) / math.sqrt(H4)).astype(np.float32)
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()
    v_img = ops.pack_act(dev(v), rows=M, cols=C, mn_major=False)
    dz_img = ops.pack_act(dev(dz), rows=M, cols=C, mn_major=False)
    w1c, _ = ops.pack_weight(dev(W1), transposed=False, tile=cb)
    w2gt, _ = ops.pack_weight(dev(W2g), transposed=True, tile=cb)
    w1tn, _ = ops.pack_weight(dev(W1), transposed=True, tile=C)
    v64, dz64, W164, W2g64 = (x.astype(np.float64) for x in (v, dz, W1, W2g))
    s = split_err(passes) + tau(C, passes)
    if mode == 2:
        h = v64 @ W164.T + b1
        eh = s * (np.abs(v64) @ np.abs(W164).T) + U * np.abs(h)
        h_dev = None
    else:                                        # mode 3 reads h as given: its reference is that fp32 tensor
        h32 = (v @ W1.T + b1).astype(np.float32)
        h, eh = h32.astype(np.float64), np.zeros((M, H4))
        h_dev = dev(h32)
    with precision_scope(passes):
        dv, dh_img, a_img, db1, guard_ok = _run_chain(ops, mode, M=M, C=C, chunk=cb, v_img=v_img, dz_img=dz_img, w1c=w1c,
                                                      w2gt=w2gt, w1tn=w1tn, b1=dev(b1), h=h_dev)
    assert guard_ok, 'a byte outside an output changed'
    d = dz64 @ W2g64
    ed = s * (np.abs(dz64) @ np.abs(W2g64)) + U * np.abs(d)
    y = d * R.gelu_grad64(h)
    ey = 1.13 * ed + (np.abs(d) + ed) * (0.8 * eh + gelu_grad_bound(h)) + U * np.abs(y)
    a = R.gelu64(h)
    ea = 1.13 * eh + gelu_bound(h)
    # dv (as mode 1)
    want = y @ W164
    ev = ey @ np.abs(W164) + (split_err(passes) + tau(H4, passes)) * ((np.abs(y) + ey) @ np.abs(W164))
    assert np.all(np.abs(dv - want) <= ev), f'dv: worst {np.max(np.abs(dv - want) / ev):.3g} of the bound'
    # the images: rows up to ceil32(M) decoded; hi + lo is the fp32 value to within 2^-16 of its magnitude
    Rm = -(-M // 32) * 32
    for img, ref, err, what in ((dh_img, y, ey, 'dh'), (a_img, a, ea, 'gelu(h)')):
        hi, lo = R.decode_mn(img.numpy(), Rm, H4, 128)
        assert not (hi[M:].any() or lo[M:].any()), f'{what}: padding rows {M}..{Rm} are not zero'
        got = R.bf16_to_f32(hi[:M]).astype(np.float64) + R.bf16_to_f32(lo[:M])
        bound = err + 2.0 ** -16 * (np.abs(ref) + err) + 1e-37
        assert np.all(np.abs(got - ref) <= bound), f'{what}: worst {np.max(np.abs(got - ref) / bound):.3g} of the bound'
    # db1: M fp32 values per column, each within ey, summed in fp32
    want_b = y.sum(0)
    eb = ey.sum(0) + M * U * (np.abs(y) + ey).sum(0)
    assert np.all(np.abs(db1 - want_b) <= eb), f'db1: worst {np.max(np.abs(db1 - want_b) / eb):.3g} of the bound'


def test_ffn_chunk_modes(ops):
    """Mode 2 exists exactly where v and dz tiles fit (C <= 128), mode 3 at C = 192; SM3_FUSED_FFN_BWD=0 disables both."""
    import os
    for C in range(32, 257, 32):
        assert (ops.ffn_chunk(2, C) > 0) == (C <= 128), C
        assert (ops.ffn_chunk(3, C) > 0) == (C == 192), C
    old = os.environ.get('SM3_FUSED_FFN_BWD')
    os.environ['SM3_FUSED_FFN_BWD'] = '0'
    try:
        assert ops.ffn_chunk(2, 96) == 0 and ops.ffn_chunk(3, 192) == 0 and ops.ffn_chunk(1, 96) > 0
    finally:
        if old is None:
            del os.environ['SM3_FUSED_FFN_BWD']
        else:
            os.environ['SM3_FUSED_FFN_BWD'] = old


@pytest.mark.parametrize('C', [96, 192])
@pytest.mark.parametrize('with_cp', [False, True])
@pytest.mark.parametrize('drop', [False, True])
def test_dense_block_fused_bwd_matches_gemm_sequence(monkeypatch, C, with_cp, drop):
    """DenseBlockFn: the same inputs through the chain-kernel backward and through dgrad -> act_pack -> dgrad.  The
    forward is bit-identical; every gradient agrees to 2e-3 of its largest magnitude (only accumulation orders differ)."""
    from test_checkpoint_gpu import _block, _inject, _run_block
    from sm3det_b200 import ops
    blk = _block(C, drop=0.1 if drop else 0.0, seed=C + 1)
    x = torch.randn((3, 20, 28, C), device='cuda')                  # T = 1680, not a multiple of 128
    if drop:
        _inject(blk, x, drop=True)
    up = torch.randn_like(x)
    names = {}
    res = {}
    for env in ('1', '0'):
        monkeypatch.setenv('SM3_FUSED_FFN_BWD', env)
        calls = []
        orig = ops.ffn_fused_bwd
        monkeypatch.setattr(ops, 'ffn_fused_bwd', lambda *a, **k: calls.append(k.get('want_wgrad_images')) or orig(*a, **k))
        res[env] = _run_block(blk, x, up, True, with_cp)
        monkeypatch.setattr(ops, 'ffn_fused_bwd', orig)
        names[env] = calls
    assert names['1'] == [True] and names['0'] == []
    (o1, _, g1), (o0, _, g0) = res['1'], res['0']
    assert torch.equal(o1, o0)
    assert set(g0) == set(g1)
    worst = 0.0
    for n in g0:
        scale = float(g0[n].abs().max())
        err = float((g0[n] - g1[n]).abs().max())
        worst = max(worst, err / (scale + 1e-30))
        assert err <= 2e-3 * scale, (n, err, scale)
    print(f'C={C} cp={with_cp} drop={drop}: worst gradient difference {worst:.3g} of its max')
