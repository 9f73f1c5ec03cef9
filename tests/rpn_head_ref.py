"""CPU oracle for mmrotate ``OrientedRPNHead``'s convolutions (sm3det_b200.head).  TEST INFRASTRUCTURE.

A restatement of RotatedRPNHead.forward_single (mmrotate/models/dense_heads/rotated_rpn_head.py:43-49) over a list of
levels, with the layer shapes of OrientedRPNHead._init_layers (oriented_rpn_head.py:18-24).  tests/test_rpn_head.py checks
it bit for bit against the unmodified reference when the reference tree is present; tools/gen_golden_rpn_head.py writes
the fixtures under tests/golden/rpn_head.  Works in float32 and float64.
"""
import torch
import torch.nn.functional as F

# Fixtures: seeded fp32 CPU runs.  'pyramid' is batch 2 over the 40/20/10/5/3 levels; 'odd' a non-square pyramid with a
# 2x1 and a 1x1 level.  feat_channels = 256 and 3 anchors as in every SM3Det config; in_channels 32 / 64 keep the files small.
GOLDEN_CASES = {
    'pyramid': dict(batch=2, sizes=[(40, 40), (20, 20), (10, 10), (5, 5), (3, 3)], in_channels=32, seed=3),
    'odd': dict(batch=1, sizes=[(9, 14), (5, 7), (2, 1), (1, 1)], in_channels=64, seed=4),
}


def rpn_head_param_shapes(in_channels=256, feat_channels=256, num_anchors=3, cls_out_channels=1):
    return {
        'rpn_conv.weight': (feat_channels, in_channels, 3, 3), 'rpn_conv.bias': (feat_channels,),
        'rpn_cls.weight': (num_anchors * cls_out_channels, feat_channels, 1, 1), 'rpn_cls.bias': (num_anchors * cls_out_channels,),
        'rpn_reg.weight': (num_anchors * 6, feat_channels, 1, 1), 'rpn_reg.bias': (num_anchors * 6,),
    }


def make_params(in_channels=256, seed=0, dtype=torch.float32):
    """Seeded parameters with O(1) activations at every stage (weights ~ N(0, 1/fan_in), biases ~ N(0, 0.1))."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, s in rpn_head_param_shapes(in_channels).items():
        fan_in = s[1] * s[2] * s[3] if len(s) == 4 else 1
        sd[k] = (torch.randn(s, generator=g) * (fan_in ** -0.5 if len(s) == 4 else 0.1)).to(dtype)
    return sd


def make_feats(batch, sizes, in_channels, seed, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed + 1000)
    return [torch.randn(batch, in_channels, h, w, generator=g).to(dtype) for h, w in sizes]


def forward_single(sd, x):
    """rotated_rpn_head.py:43-49."""
    x = F.conv2d(x, sd['rpn_conv.weight'], sd['rpn_conv.bias'], padding=1)
    x = F.relu(x)
    return F.conv2d(x, sd['rpn_cls.weight'], sd['rpn_cls.bias']), F.conv2d(x, sd['rpn_reg.weight'], sd['rpn_reg.bias'])


def rpn_head_forward(sd, feats):
    """mmdet BaseDenseHead.forward: multi_apply(forward_single, feats) -> (cls_scores, bbox_preds)."""
    outs = [forward_single(sd, x) for x in feats]
    return [o[0] for o in outs], [o[1] for o in outs]


def load_reference_heads():
    """The unmodified reference oriented_rpn_head.py (and rotated_rpn_head.py, its base) executed through oracle/ref_shim.py,
    with stand-ins for the mmcv / mmdet names they import; None when the reference tree is absent.  The AnchorHead stand-in
    keeps only what _init_layers reads: in/feat channels, num_anchors = len(scales) * len(ratios), and
    cls_out_channels = num_classes (sigmoid classification, mmdet's default for the RPN)."""
    import sys
    import types

    import torch.nn as nn
    from oracle import ref_shim
    if not ref_shim.reference_available():
        return None

    def mod(name, **attrs):
        m = sys.modules.get(name)
        if m is None:
            m = types.ModuleType(name)
            m.__path__ = []
            sys.modules[name] = m
        for k, v in attrs.items():
            setattr(m, k, v)
        return m

    class AnchorHead(nn.Module):
        def __init__(self, num_classes, in_channels, feat_channels=256, anchor_generator=None, init_cfg=None, **kw):
            super().__init__()
            self.num_classes, self.in_channels, self.feat_channels = num_classes, in_channels, feat_channels
            ag = anchor_generator or dict(scales=[8], ratios=[0.5, 1.0, 2.0])
            self.num_anchors = len(ag['scales']) * len(ag['ratios'])
            self.cls_out_channels = num_classes
            self._init_layers()

    stub = lambda *a, **k: None
    mod('mmcv'); mod('mmcv.ops', batched_nms=stub)
    mod('mmcv.runner', force_fp32=lambda *a, **k: (lambda f: f))
    mod('mmdet'); mod('mmdet.core', anchor_inside_flags=stub, images_to_levels=stub, multi_apply=stub, unmap=stub)
    mod('mmdet.models'); mod('mmdet.models.dense_heads'); mod('mmdet.models.dense_heads.anchor_head', AnchorHead=AnchorHead)
    mod('mmrotate'); mod('mmrotate.core', obb2xyxy=stub); mod('mmrotate.models'); mod('mmrotate.models.dense_heads')
    mod('mmrotate.models.builder', ROTATED_HEADS=ref_shim._REGISTRY)
    ref_shim.load_reference_module('rotated_rpn_head', 'dense_heads')
    return ref_shim.load_reference_module('oriented_rpn_head', 'dense_heads')
