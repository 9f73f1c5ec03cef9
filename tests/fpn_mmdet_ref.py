"""CPU oracle for mmdet 2.x ``FPN`` (the neck of the single-dataset LSKNet, VAN and ConvNeXt configs).  TEST INFRASTRUCTURE.

mmdet is not part of the reference tree, so the oracle is pinned through the reference's modified copy of it,
mmrotate/models/necks/Multitask_FPN.py, by one identity (tools/gen_golden_fpn.py checks it bit for bit):

    FPN(start_level=s, **kw)(inputs)
      == MultitaskFPN(start_level=0, extra_level=s, **kw)(inputs, start_level=s)
    with FPN lateral_convs.j <-> MultitaskFPN lateral_convs.(j+s) and FPN fpn_convs.j <-> MultitaskFPN fpn_convs.(j+s).

MultitaskFPN(start_level=0) builds lateral and output convs for every input; called with start_level=s it uses those from
s on, and extra_level=s gives it the num_outs - backbone_end_level + s extra convs mmdet's FPN builds.  Its convs 0..s-1 are
unused.  norm_cfg = act_cfg = conv_cfg = None throughout (ConvModule = biased Conv2d), size-based nearest upsampling.
"""
import torch
import torch.nn.functional as F

# The fixtures of tests/golden/fpn_mmdet (tools/gen_golden_fpn.py): the three FPN modes of the shipped configs, batch 2,
# input maps 24/12/6/3 so that P5 is 3x3 and the max-pool P6 2x2.  out_channels=64 keeps the files small; nothing in the
# neck depends on the width beyond the conv shapes.
T_WIDTHS, CONVNEXT_T_WIDTHS = [32, 64, 160, 256], [96, 192, 384, 768]
GOLDEN_CASES = {
    'maxpool_t': dict(in_channels=T_WIDTHS, out_channels=64, num_outs=5),
    'on_output_t': dict(in_channels=T_WIDTHS, out_channels=64, num_outs=5, start_level=1, add_extra_convs='on_output'),
    'on_input_convnext_t': dict(in_channels=CONVNEXT_T_WIDTHS, out_channels=64, num_outs=5, start_level=1,
                                add_extra_convs='on_input'),
}
GOLDEN_BATCH, GOLDEN_SIZES, GOLDEN_SEED, GOLDEN_SD_SEED = 2, (24, 12, 6, 3), 21, 5


def fpn_inputs(in_channels, n, sizes, seed):
    """Seeded backbone maps [n, c_i, s_i, s_i] (CPU, fp32)."""
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(n, c, s, s, generator=g) for c, s in zip(in_channels, sizes)]


def _extra_src(add_extra_convs):
    return 'on_input' if add_extra_convs is True else add_extra_convs


def fpn_mmdet_param_shapes(in_channels, out_channels, num_outs, start_level=0, add_extra_convs=False):
    """state_dict shapes of mmdet's FPN (end_level=-1): lateral / output convs 0 .. num_ins-start_level-1 read inputs
    start_level .., then the stride-2 extra convs when add_extra_convs is set."""
    sh = {}
    used = len(in_channels) - start_level
    for j in range(used):
        sh[f'lateral_convs.{j}.conv.weight'] = (out_channels, in_channels[j + start_level], 1, 1)
        sh[f'lateral_convs.{j}.conv.bias'] = (out_channels,)
        sh[f'fpn_convs.{j}.conv.weight'] = (out_channels, out_channels, 3, 3)
        sh[f'fpn_convs.{j}.conv.bias'] = (out_channels,)
    extra = num_outs - used
    if add_extra_convs and extra >= 1:
        for i in range(extra):
            cin = in_channels[-1] if (i == 0 and _extra_src(add_extra_convs) == 'on_input') else out_channels
            sh[f'fpn_convs.{used + i}.conv.weight'] = (out_channels, cin, 3, 3)
            sh[f'fpn_convs.{used + i}.conv.bias'] = (out_channels,)
    return sh


def to_multitask_key(key, start_level):
    """The MultitaskFPN(start_level=0, extra_level=s) key of an FPN(start_level=s) key: the conv index moves up by s."""
    kind, idx, rest = key.split('.', 2)
    return f'{kind}.{int(idx) + start_level}.{rest}'


def from_multitask_state_dict(mt_sd, start_level):
    """FPN(start_level=s) state_dict of a MultitaskFPN(start_level=0, extra_level=s) one: convs 0..s-1 dropped, the rest
    re-indexed from 0."""
    out = {}
    for k, v in mt_sd.items():
        kind, idx, rest = k.split('.', 2)
        if int(idx) >= start_level:
            out[f'{kind}.{int(idx) - start_level}.{rest}'] = v
    return out


def fpn_forward_mmdet(sd, inputs, num_outs, start_level=0, add_extra_convs=False):
    """mmdet 2.x FPN.forward with end_level=-1 and no relu_before_extra_convs, on torch CPU ops."""
    conv = lambda k, x, **kw: F.conv2d(x, sd[k + '.conv.weight'], sd[k + '.conv.bias'], **kw)
    num_ins = len(inputs)
    laterals = [conv(f'lateral_convs.{j}', inputs[j + start_level]) for j in range(num_ins - start_level)]
    used = len(laterals)
    for i in range(used - 1, 0, -1):
        laterals[i - 1] = laterals[i - 1] + F.interpolate(laterals[i], size=laterals[i - 1].shape[2:], mode='nearest')
    outs = [conv(f'fpn_convs.{i}', laterals[i], padding=1) for i in range(used)]
    if num_outs > len(outs):
        if not add_extra_convs:
            for _ in range(num_outs - used):
                outs.append(F.max_pool2d(outs[-1], 1, stride=2))
        else:
            src = {'on_input': inputs[num_ins - 1], 'on_lateral': laterals[-1],
                   'on_output': outs[-1]}[_extra_src(add_extra_convs)]
            outs.append(conv(f'fpn_convs.{used}', src, stride=2, padding=1))
            for i in range(used + 1, num_outs):
                outs.append(conv(f'fpn_convs.{i}', outs[-1], stride=2, padding=1))
    return tuple(outs)
