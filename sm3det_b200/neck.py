"""Drop-in MultitaskFPN (SURVEY.md 8(f) rank 1) on the sm3det_b200 CUDA library.

Same class name, constructor kwargs, ``state_dict`` keys (``lateral_convs.{i}.conv.*``, ``fpn_convs.{i}.conv.*``) and
``forward(inputs, start_level=None, add_extra_convs=None)`` contract as the reference
(mmrotate/models/necks/Multitask_FPN.py:14-162): consumes the backbone's tuple of NCHW maps, returns a tuple of NCHW maps.
Inside, everything is NHWC: the 1x1 laterals read the NCHW inputs through im2col, the top-down path is one fused
nearest-upsample + add kernel per level, the 3x3 (stride 1 / 2) output convolutions are im2col + wgmma GEMM, and only the
returned levels are transposed back to NCHW.

``FPN`` is mmdet's neck of the same name (the single-dataset LSKNet, VAN and ConvNeXt configs) on the same pyramid code, with
mmdet's conv indexing; its max-pool extra levels leave through one export kernel together with the top level.
"""
import torch
import torch.nn as nn
from torch.autograd import Function

from . import lsk_functional as LF
from . import ops
from .registry import BaseModule, Registry

ROTATED_NECKS = Registry('neck')


class ConvModule(nn.Module):
    """mmcv.cnn.ConvModule reduced to what MultitaskFPN builds with norm_cfg=None, act_cfg=None: a biased Conv2d."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, conv_cfg=None, norm_cfg=None, act_cfg=None,
                 inplace=False):
        super().__init__()
        if conv_cfg is not None or norm_cfg is not None or act_cfg is not None:
            raise NotImplementedError('sm3det_b200 MultitaskFPN: conv_cfg / norm_cfg / act_cfg are not implemented '
                                      '(every SM3Det config leaves them None)')
        self.conv = nn.Conv2d(in_channels, out_channels, kernel_size, stride=stride, padding=padding)


@ops.captures_precision
class UpsampleAddFn(Function):
    @staticmethod
    def forward(ctx, a, b):
        ctx.hw = (b.shape[1], b.shape[2])
        return ops.upsample_add(a.contiguous(), b.contiguous())

    @staticmethod
    def backward(ctx, d):
        d = d.contiguous()
        return d, ops.upsample_add_bwd(d, *ctx.hw)


@ops.captures_precision
class ToNCHWFn(Function):
    @staticmethod
    def forward(ctx, x):
        N, H, W, C = x.shape
        return ops.transpose_batched(x.contiguous(), N, H * W, C, (N, C, H, W))

    @staticmethod
    def backward(ctx, d):
        N, C, H, W = d.shape
        return ops.transpose_batched(d.contiguous(), N, C, H * W, (N, H, W, C))


@ops.captures_precision
class ToNCHWPoolFn(Function):
    """x [N,H,W,C] -> (x as NCHW, then L levels of F.max_pool2d(., 1, stride=2), each applied to the one before), one
    kernel each way."""

    @staticmethod
    def forward(ctx, x, L):
        return ops.fpn_export_pool(x.contiguous(), L)

    @staticmethod
    def backward(ctx, *ds):
        return ops.fpn_export_pool_bwd([d.contiguous() for d in ds]), None


def _conv(m, x, nchw):
    c = m.conv
    return LF.PatchEmbedFn.apply(x, c.weight, c.bias, c.stride[0], nchw)


class _PyramidNeck(BaseModule):
    """Constructor checks, conv layout and NHWC pyramid shared by MultitaskFPN and FPN.  Lateral and output convs are built
    for the inputs start_level .. backbone_end_level-1; num_outs - backbone_end_level + extra_level stride-2 extra convs
    follow when add_extra_convs is set."""

    def __init__(self, in_channels, out_channels, num_outs, start_level, end_level, add_extra_convs, relu_before_extra_convs,
                 no_norm_on_lateral, conv_cfg, norm_cfg, act_cfg, upsample_cfg, init_cfg, extra_level):
        super().__init__(init_cfg)
        name = type(self).__name__
        assert isinstance(in_channels, list)
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.num_ins = len(in_channels)
        self.num_outs = num_outs
        self.relu_before_extra_convs = relu_before_extra_convs
        self.no_norm_on_lateral = no_norm_on_lateral
        self.fp16_enabled = False
        self.upsample_cfg = upsample_cfg.copy()
        if self.upsample_cfg.get('mode', 'nearest') != 'nearest' or 'scale_factor' in self.upsample_cfg:
            raise NotImplementedError(f"sm3det_b200 {name}: only upsample_cfg=dict(mode='nearest') (size-based) is implemented")
        if relu_before_extra_convs:
            raise NotImplementedError(f'sm3det_b200 {name}: relu_before_extra_convs is not implemented')
        if end_level == -1 or end_level == self.num_ins - 1:
            self.backbone_end_level = self.num_ins
            assert num_outs >= self.num_ins - start_level
        else:
            self.backbone_end_level = end_level + 1
            assert end_level < self.num_ins
            assert num_outs == end_level - start_level + 1
        self.start_level = start_level
        self.end_level = end_level
        self.add_extra_convs = add_extra_convs
        assert isinstance(add_extra_convs, (str, bool))
        if isinstance(add_extra_convs, str):
            assert add_extra_convs in ('on_input', 'on_lateral', 'on_output')
        elif add_extra_convs:
            self.add_extra_convs = 'on_input'
        self.lateral_convs = nn.ModuleList()
        self.fpn_convs = nn.ModuleList()
        for i in range(self.start_level, self.backbone_end_level):
            self.lateral_convs.append(ConvModule(in_channels[i], out_channels, 1, conv_cfg=conv_cfg,
                                                 norm_cfg=norm_cfg if not self.no_norm_on_lateral else None, act_cfg=act_cfg))
            self.fpn_convs.append(ConvModule(out_channels, out_channels, 3, padding=1, conv_cfg=conv_cfg, norm_cfg=norm_cfg,
                                             act_cfg=act_cfg))
        extra_levels = num_outs - self.backbone_end_level + extra_level
        if self.add_extra_convs and extra_levels >= 1:
            for i in range(extra_levels):
                cin = self.in_channels[self.backbone_end_level - 1] if (i == 0 and self.add_extra_convs == 'on_input') else out_channels
                self.fpn_convs.append(ConvModule(cin, out_channels, 3, stride=2, padding=1, conv_cfg=conv_cfg, norm_cfg=norm_cfg,
                                                 act_cfg=act_cfg))
        for c in list(in_channels) + [out_channels]:
            if c % 32:
                raise NotImplementedError(f'sm3det_b200 {name}: channel count {c} unsupported (multiple of 32)')

    def _pyramid(self, inputs, start_level, conv_offset, add_extra_convs):
        """NHWC outputs: lateral i = lateral_convs[i + conv_offset](inputs[i + start_level]) over the remaining lateral convs,
        the nearest top-down path, output i = fpn_convs[i + conv_offset](lateral i), then the stride-2 conv extra levels up
        to num_outs.  Without add_extra_convs it stops at the backbone levels."""
        if not inputs[0].is_cuda:
            raise RuntimeError(f'sm3det_b200 {type(self).__name__} runs on CUDA (sm_90a) only; there is no CPU path')
        laterals = [_conv(self.lateral_convs[i + conv_offset], inputs[i + start_level], True)
                    for i in range(len(self.lateral_convs) - conv_offset)]
        used = len(laterals)
        for i in range(used - 1, 0, -1):
            laterals[i - 1] = UpsampleAddFn.apply(laterals[i - 1], laterals[i])
        outs = [_conv(self.fpn_convs[i + conv_offset], laterals[i], False) for i in range(used)]
        if self.num_outs > len(outs) and add_extra_convs:
            if add_extra_convs == 'on_input':
                src, nchw = inputs[self.backbone_end_level - 1], True
            elif add_extra_convs == 'on_lateral':
                src, nchw = laterals[-1], False
            elif add_extra_convs == 'on_output':
                src, nchw = outs[-1], False
            else:
                raise NotImplementedError
            outs.append(_conv(self.fpn_convs[used + conv_offset], src, nchw))
            for i in range(used + 1, self.num_outs):
                outs.append(_conv(self.fpn_convs[i + conv_offset], outs[-1], False))
        return outs


@ROTATED_NECKS.register_module()
class MultitaskFPN(_PyramidNeck):
    def __init__(self, in_channels, out_channels, num_outs, start_level=0, end_level=-1, extra_level=0, add_extra_convs=False,
                 relu_before_extra_convs=False, no_norm_on_lateral=False, conv_cfg=None, norm_cfg=None, act_cfg=None,
                 upsample_cfg=dict(mode='nearest'), init_cfg=dict(type='Xavier', layer='Conv2d', distribution='uniform')):
        super().__init__(in_channels, out_channels, num_outs, start_level, end_level, add_extra_convs, relu_before_extra_convs,
                         no_norm_on_lateral, conv_cfg, norm_cfg, act_cfg, upsample_cfg, init_cfg, extra_level=extra_level)
        self.extra_level = extra_level

    def forward(self, inputs, start_level=None, add_extra_convs=None):
        with ops.precision_scope(ops.autocast_passes(self)):      # per-call GEMM precision (bf16 under autocast)
            return self._forward(inputs, start_level, add_extra_convs)

    def _forward(self, inputs, start_level=None, add_extra_convs=None):
        if start_level is None:
            start_level = self.start_level
        if add_extra_convs is None:
            add_extra_convs = self.add_extra_convs
        outs = self._pyramid(inputs, start_level, start_level, add_extra_convs)
        if self.num_outs > len(outs):
            raise NotImplementedError('sm3det_b200 MultitaskFPN: max-pool extra levels (add_extra_convs=False) are not implemented')
        return tuple(ToNCHWFn.apply(o) for o in outs)


@ROTATED_NECKS.register_module()
class FPN(_PyramidNeck):
    """mmdet 2.x ``FPN`` (as mmrotate 0.3 builds it) on the CUDA library, for norm_cfg = act_cfg = conv_cfg = None.

    Same kwargs and ``state_dict`` keys as mmdet's: lateral and output convs exist for inputs start_level ..
    backbone_end_level-1 only and are indexed from 0, followed by num_outs - backbone_end_level + start_level extra
    levels.  ``forward(inputs)`` takes the backbone's full tuple.  With add_extra_convs=False the extra levels are
    F.max_pool2d(outs[-1], 1, stride=2), chained; they are written by the kernel that exports the top level to NCHW."""

    def __init__(self, in_channels, out_channels, num_outs, start_level=0, end_level=-1, add_extra_convs=False,
                 relu_before_extra_convs=False, no_norm_on_lateral=False, conv_cfg=None, norm_cfg=None, act_cfg=None,
                 upsample_cfg=dict(mode='nearest'), init_cfg=dict(type='Xavier', layer='Conv2d', distribution='uniform')):
        if conv_cfg is not None or norm_cfg is not None or act_cfg is not None:
            raise NotImplementedError('sm3det_b200 FPN: conv_cfg / norm_cfg / act_cfg are not implemented '
                                      '(every FPN config of the LSKNet, VAN and ConvNeXt detectors leaves them None)')
        super().__init__(in_channels, out_channels, num_outs, start_level, end_level, add_extra_convs, relu_before_extra_convs,
                         no_norm_on_lateral, conv_cfg, norm_cfg, act_cfg, upsample_cfg, init_cfg, extra_level=start_level)

    def forward(self, inputs):
        assert len(inputs) == len(self.in_channels)
        with ops.precision_scope(ops.autocast_passes(self)):      # per-call GEMM precision (bf16 under autocast)
            outs = self._pyramid(inputs, self.start_level, 0, self.add_extra_convs)
            pool = self.num_outs - len(outs)
            if pool <= 0:
                return tuple(ToNCHWFn.apply(o) for o in outs)
            return tuple(ToNCHWFn.apply(o) for o in outs[:-1]) + ToNCHWPoolFn.apply(outs[-1], pool)
