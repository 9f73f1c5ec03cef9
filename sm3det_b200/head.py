"""mmrotate ``OrientedRPNHead`` convolutions on the sm3det_b200 CUDA library.

Reference (mmrotate/models/dense_heads/rotated_rpn_head.py:43-49, oriented_rpn_head.py:18-24): per pyramid level,
``rpn_conv`` (3x3, in_channels -> feat_channels, pad 1), ReLU, then ``rpn_cls`` and ``rpn_reg`` (1x1).  Here every level
runs in one launch of one kernel: the 3x3 conv is an implicit GEMM that gathers its operand rows straight from the NCHW
maps (no im2col buffer), and its 128 x 256 ReLU tile feeds the [rpn_cls; rpn_reg] GEMM in shared memory; cls and reg
leave in NCHW.  The backward is three kernels and the library's split-K weight-gradient GEMM (csrc/rpn_head.cu).

``SM3RPNHeadMixin`` replaces only ``forward(feats)`` of a head class that builds ``rpn_conv`` / ``rpn_cls`` / ``rpn_reg``
(mmrotate's ``OrientedRPNHead``; INTEGRATION.md shows the binding).  ``OrientedRPNHeadConvs`` is a standalone module with
the same layers and ``state_dict`` keys, for use without mmrotate.  Losses, anchors, targets and proposals stay with
mmrotate.
"""
import torch
import torch.nn as nn
from torch.autograd import Function

from . import ops
from .registry import BaseModule

FEAT_CHANNELS = 256      # one 128 x 256 tile holds the whole hidden row, so the head GEMM stays on chip
MAX_HEAD_WIDTH = 32      # rpn_cls + rpn_reg output channels: one wgmma N


@ops.captures_precision
class RPNHeadFn(Function):
    """(L, want_grad, x_0 .. x_{L-1}, rpn_conv.weight, rpn_conv.bias, rpn_cls.weight, rpn_cls.bias, rpn_reg.weight,
    rpn_reg.bias) -> (cls_0 .. cls_{L-1}, reg_0 .. reg_{L-1}), all NCHW fp32."""

    @staticmethod
    def forward(ctx, L, want_grad, *args):
        xs = [a.contiguous().float() for a in args[:L]]
        wc, bc, wcls, bcls, wreg, breg = (t.float() for t in args[L:])
        ncls, nreg, Cin = wcls.shape[0], wreg.shape[0], wc.shape[1]
        wc_img, _ = ops.pack_weight(wc.permute(0, 2, 3, 1).reshape(FEAT_CHANNELS, 9 * Cin).contiguous(), transposed=False,
                                    tile=FEAT_CHANNELS)
        wh = torch.cat([wcls.reshape(ncls, FEAT_CHANNELS), wreg.reshape(nreg, FEAT_CHANNELS)]).contiguous()
        whp = torch.zeros((MAX_HEAD_WIDTH, FEAT_CHANNELS), device=wh.device, dtype=torch.float32)
        whp[:ncls + nreg] = wh
        wh_img, _ = ops.pack_weight(whp, transposed=False, tile=MAX_HEAD_WIDTH)
        bh = torch.cat([bcls, breg]).contiguous()
        cls, reg, h = ops.rpn_head_fwd(xs, wc_img, bc.contiguous(), wh_img, bh, ncls=ncls, nreg=nreg, want_h=want_grad)
        if want_grad:
            ctx.save_for_backward(*xs, wc, wh, h)
            ctx.geom = (L, Cin, ncls, nreg, [(x.shape[0], x.shape[2], x.shape[3]) for x in xs])
        return tuple(cls) + tuple(reg)

    @staticmethod
    def backward(ctx, *grads):
        L, Cin, ncls, nreg, shapes = ctx.geom
        saved = ctx.saved_tensors
        xs, wc, wh, h = saved[:L], saved[L], saved[L + 1], saved[L + 2]
        dev = h.device

        def g(i, c):
            n, hh, ww = shapes[i % L]
            return grads[i].contiguous().float() if grads[i] is not None else torch.zeros((n, c, hh, ww), device=dev)

        dcls = [g(i, ncls) for i in range(L)]
        dreg = [g(L + i, nreg) for i in range(L)]
        dwh = torch.zeros((ncls + nreg, FEAT_CHANNELS), device=dev, dtype=torch.float32)
        dbh = torch.zeros((ncls + nreg,), device=dev, dtype=torch.float32)
        dbc = torch.zeros((FEAT_CHANNELS,), device=dev, dtype=torch.float32)
        dpre = ops.rpn_head_mid_bwd(h, dcls, dreg, wh, dwh, dbh, dbc, ncls=ncls, nreg=nreg)

        dx = [None] * L
        if any(ctx.needs_input_grad[2:2 + L]):
            # dx = conv3x3(dpre) with the weight flipped 180 degrees and in/out-transposed: rows c (padded to 256), k = tap*256 + o
            wd = torch.zeros((FEAT_CHANNELS, 9 * FEAT_CHANNELS), device=dev, dtype=torch.float32)
            wd[:Cin] = wc.flip(2, 3).permute(1, 2, 3, 0).reshape(Cin, 9 * FEAT_CHANNELS)
            wd_img, _ = ops.pack_weight(wd, transposed=False, tile=FEAT_CHANNELS)
            dx = ops.rpn_head_dx(dpre, shapes, Cin, wd_img)

        dwc = None
        if ctx.needs_input_grad[2 + L]:
            # dW[o, c, ky, kx] = sum over positions of dpre[p, o] * x[c, p shifted by (ky-1, kx-1)]: one split-K GEMM per tap
            # on the NHWC rows of the input, gathered through the tap's neighbour index (-1 = zero row)
            R = h.shape[0]
            xr = ops.rpn_head_nhwc_rows(xs, R)
            idx = ops.rpn_head_tap_index(shapes, dev)
            dy_packed = ops.pack_act(dpre, rows=R, cols=FEAT_CHANNELS, mn_major=True, tile=128)
            dw9 = torch.zeros((9, FEAT_CHANNELS, Cin), device=dev, dtype=torch.float32)
            for tap in range(9):
                ops.linear_wgrad(dpre, xr, dw9[tap], rows=R, x_row_index=idx[tap], dy_packed=dy_packed)
            dwc = dw9.view(3, 3, FEAT_CHANNELS, Cin).permute(2, 3, 0, 1).contiguous()
        return (None, None, *dx, dwc, dbc, dwh[:ncls].reshape(ncls, FEAT_CHANNELS, 1, 1), dbh[:ncls],
                dwh[ncls:].reshape(nreg, FEAT_CHANNELS, 1, 1), dbh[ncls:])


def check_head_layers(rpn_conv, rpn_cls, rpn_reg, name='OrientedRPNHead'):
    """NotImplementedError for layer configurations the kernels do not cover."""
    c = rpn_conv
    if (c.kernel_size != (3, 3) or c.padding != (1, 1) or c.stride != (1, 1) or c.dilation != (1, 1) or c.groups != 1
            or c.bias is None or getattr(c, 'padding_mode', 'zeros') != 'zeros'):
        raise NotImplementedError(f'sm3det_b200 {name}: rpn_conv must be a biased 3x3 conv, stride 1, padding 1')
    if c.out_channels != FEAT_CHANNELS:
        raise NotImplementedError(f'sm3det_b200 {name}: feat_channels must be {FEAT_CHANNELS}, got {c.out_channels}')
    if c.in_channels % 32 or not 32 <= c.in_channels <= 256:
        raise NotImplementedError(f'sm3det_b200 {name}: in_channels must be a multiple of 32 in [32, 256], got {c.in_channels}')
    for m in (rpn_cls, rpn_reg):
        if m.kernel_size != (1, 1) or m.stride != (1, 1) or m.padding != (0, 0) or m.groups != 1 or m.bias is None \
                or m.in_channels != FEAT_CHANNELS:
            raise NotImplementedError(f'sm3det_b200 {name}: rpn_cls / rpn_reg must be biased 1x1 convs from {FEAT_CHANNELS} channels')
    if rpn_cls.out_channels + rpn_reg.out_channels > MAX_HEAD_WIDTH:
        raise NotImplementedError(f'sm3det_b200 {name}: rpn_cls + rpn_reg out channels must be <= {MAX_HEAD_WIDTH}, got '
                                  f'{rpn_cls.out_channels} + {rpn_reg.out_channels}')


def rpn_head_forward(rpn_conv, rpn_cls, rpn_reg, feats, *, amp=False):
    """(cls_scores, bbox_preds): two lists with one NCHW map per level, as mmdet's multi_apply(forward_single, feats)."""
    check_head_layers(rpn_conv, rpn_cls, rpn_reg)
    feats = list(feats)
    if not 1 <= len(feats) <= ops.RPN_MAX_LEVELS:
        raise NotImplementedError(f'sm3det_b200 OrientedRPNHead: 1 to {ops.RPN_MAX_LEVELS} levels, got {len(feats)}')
    for f in feats:
        if not f.is_cuda:
            raise RuntimeError('sm3det_b200 OrientedRPNHead runs on CUDA (sm_90a) only; there is no CPU path')
        if f.dim() != 4 or f.shape[1] != rpn_conv.in_channels:
            raise ValueError(f'sm3det_b200 OrientedRPNHead: expected [N, {rpn_conv.in_channels}, H, W] maps, got {tuple(f.shape)}')
    params = (rpn_conv.weight, rpn_conv.bias, rpn_cls.weight, rpn_cls.bias, rpn_reg.weight, rpn_reg.bias)
    want_grad = torch.is_grad_enabled() and any(t.requires_grad for t in (*feats, *params))
    L = len(feats)
    with ops.precision_scope(1 if (amp or torch.is_autocast_enabled()) else 3):   # bf16 operands under autocast
        outs = RPNHeadFn.apply(L, want_grad, *feats, *params)
    return list(outs[:L]), list(outs[L:])


class SM3RPNHeadMixin:
    """Mixin for a head class that builds ``rpn_conv`` / ``rpn_cls`` / ``rpn_reg`` (mmrotate's OrientedRPNHead): only
    ``forward(feats)`` is replaced; everything else (losses, anchors, get_bboxes) is the host class's."""

    def forward(self, feats):
        return rpn_head_forward(self.rpn_conv, self.rpn_cls, self.rpn_reg, feats, amp=getattr(self, 'amp', False))


class OrientedRPNHeadConvs(SM3RPNHeadMixin, BaseModule):
    """The layers of mmrotate's ``OrientedRPNHead`` (``_init_layers``, same parameter names and shapes, so the same
    ``state_dict`` keys) with the CUDA forward.  rpn_cls has num_anchors * cls_out_channels outputs (sigmoid
    classification: cls_out_channels = 1), rpn_reg num_anchors * 6."""

    def __init__(self, in_channels=256, feat_channels=256, num_anchors=3, cls_out_channels=1,
                 init_cfg=dict(type='Normal', layer='Conv2d', std=0.01)):
        super().__init__(init_cfg)
        self.in_channels = in_channels
        self.feat_channels = feat_channels
        self.num_anchors = num_anchors
        self.cls_out_channels = cls_out_channels
        self.rpn_conv = nn.Conv2d(in_channels, feat_channels, 3, padding=1)
        self.rpn_cls = nn.Conv2d(feat_channels, num_anchors * cls_out_channels, 1)
        self.rpn_reg = nn.Conv2d(feat_channels, num_anchors * 6, 1)
        check_head_layers(self.rpn_conv, self.rpn_cls, self.rpn_reg, 'OrientedRPNHeadConvs')
