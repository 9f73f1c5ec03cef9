"""sm3det_b200 -- H100-native (sm_90a) implementation of SM3Det's grid-level sparse-MoE ConvNeXt backbone."""
from .backbone import ConvNeXt_DA_MultiInput, ConvNeXt_moe, ConvNeXt_moe_MultiInput  # noqa: F401
from .lsk_backbone import LSKNet, LSKNet_moe, LSKNet_moe_MultiInput, VAN, VAN_moe, VAN_moe_MultiInput  # noqa: F401
from .registry import ROTATED_BACKBONES, build_backbone, register_into_mmrotate  # noqa: F401

__all__ = ['ConvNeXt_moe', 'ConvNeXt_moe_MultiInput', 'ConvNeXt_DA_MultiInput', 'LSKNet_moe', 'LSKNet_moe_MultiInput', 'VAN_moe', 'VAN_moe_MultiInput', 'LSKNet', 'VAN', 'ROTATED_BACKBONES', 'build_backbone', 'register_into_mmrotate']
