"""LSKNet-T drop-in contract on the CPU (no GPU compute): the SM3Det_lsk_t backbone dicts and LSKNet_moe()'s defaults build
through the registry with the reference's state_dict layout, and the oracle reproduces the tests/golden/lsk_t fixtures."""
import glob
import os

import pytest
import torch

import test_lsk_oracle as O

GOLD_T = os.path.join(os.path.dirname(__file__), 'golden', 'lsk_t')
# configs/SM3Det/SM3Det_lsk_t.py:14-25 (identical in local_configs/SM3Det_lsk_t.py)
LSK_T_BACKBONE = dict(type='LSKNet_moe_MultiInput', MoE_Block_inds_fc1=[[], [0, 2], [i * 2 for i in range(5)], [0]],
                      MoE_Block_inds_fc2=[[], [0, 2], [i * 2 for i in range(5)], [0]], datasets=None, num_experts=4,
                      top_k=2, embed_dims=[32, 64, 160, 256], drop_rate=0.1, drop_path_rate=0.1, depths=[3, 3, 5, 2],
                      norm_cfg=dict(type='SyncBN', requires_grad=True),
                      init_cfg=dict(type='Pretrained', checkpoint='../data/pretrained/lsk_t_backbone.pth.tar'))


def test_lsk_t_registry_build_matches_reference_layout():
    from sm3det_b200 import build_backbone
    layout = torch.load(os.path.join(GOLD_T, 'layout.pt'), weights_only=False)
    net = build_backbone(dict(LSK_T_BACKBONE))
    sd = net.state_dict()
    assert list(sd) == layout['keys']
    assert {k: tuple(v.shape) for k, v in sd.items()} == layout['shapes']
    # the 16- / 80-wide halves of the LSK attention branch
    assert tuple(sd['block1.0.attn.spatial_gating_unit.conv1.weight'].shape) == (16, 32, 1, 1)
    assert tuple(sd['block3.0.attn.spatial_gating_unit.conv.weight'].shape) == (160, 80, 1, 1)


def test_lsk_net_moe_defaults_build():
    """LSKNet_moe()'s default embed_dims are the T widths."""
    from sm3det_b200 import LSKNet_moe, build_backbone
    from oracle.lsk_moe_oracle import LskConfig, lsk_param_shapes
    for net in (LSKNet_moe(), build_backbone(dict(type='LSKNet_moe'))):
        assert net.embed_dims == [32, 64, 160, 256]
        shapes = lsk_param_shapes(LskConfig(multi_input=False))
        assert {k: tuple(v.shape) for k, v in net.state_dict().items()} == {k: tuple(s) for k, s in shapes.items()}


@pytest.mark.parametrize('path', sorted(p for p in glob.glob(os.path.join(GOLD_T, '*.pt')) if not p.endswith('layout.pt')),
                         ids=lambda p: os.path.basename(p)[:-3])
def test_oracle_reproduces_lsk_t_golden(path):
    O.test_oracle_reproduces_reference_golden(path)
