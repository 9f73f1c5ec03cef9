"""Generate tests/golden/lsk_t/: the LSKNet-T / VAN-T fixtures (configs/SM3Det/SM3Det_lsk_t.py, SM3Det_van_t.py).

    python tools/gen_golden_lsk_t.py [case ...]      (needs the reference tree, SM3DET_REFERENCE_ROOT)

Every case runs the UNMODIFIED reference lsk_moe.py / van_moe.py and asserts that the oracle reproduces it bit-for-bit
(oracle/gen_golden.py: run_lsk_case), exactly as the LSK-S fixtures are pinned.  The fixtures live in their own
subdirectory so the tests that glob tests/golden/*.pt do not pick them up.  layout.pt records the reference's
state_dict keys and shapes for the SM3Det_lsk_t backbone dict.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, 'tests', 'golden', 'lsk_t')

# configs/SM3Det/SM3Det_lsk_t.py:14-24 (MoE in stages 2-4; stage 3 lists [0, 2, 4, 6, 8] of its 5 blocks)
LSK_T_KW = dict(embed_dims=[32, 64, 160, 256], depths=[3, 3, 5, 2], MoE_Block_inds_fc1=[[], [0, 2], [0, 2, 4, 6, 8], [0]],
                MoE_Block_inds_fc2=[[], [0, 2], [0, 2, 4, 6, 8], [0]], num_experts=4, top_k=2)
# configs/SM3Det/SM3Det_van_t.py:14-24
VAN_T_KW = dict(embed_dims=[32, 64, 160, 256], depths=[3, 3, 5, 2], MoE_Block_inds_fc1=[[], [0, 2], [0, 2, 4], [0]],
                MoE_Block_inds_fc2=[[], [0, 2], [0, 2, 4], [0]], num_experts=8, top_k=2)

# name -> spec of oracle/gen_golden.py:run_lsk_case.  Training fixtures use batch 2 (oracle/cases.py: torch 2.11's CPU
# autograd is wrong for this op sequence at batch 1).  'full' cases keep strided samples and gradient digests (<= 1 MB).
LSK_T_CASES = {
    'lsk_t_1024_eval': dict(kw=dict(LSK_T_KW), img=(1, 1024, 1024), mode='eval', full=True, stride=8),
    'lsk_t_b2_512_train_noisy_drop': dict(kw=dict(LSK_T_KW, drop_rate=0.1), img=(2, 512, 512), mode='train_noisy',
                                          full=True, stride=8),
    # short depth, the same widths (the 16- and 80-wide LSK attention branch) and an expert layer in every stage: small
    # enough for full gradients and bit-exact routing
    'lsk_t_short_e4k2_train_noisy_drop': dict(kw=dict(embed_dims=[32, 64, 160, 256], depths=[1, 1, 2, 1],
                                                      MoE_Block_inds_fc1=[[0], [0], [0, 1], [0]],
                                                      MoE_Block_inds_fc2=[[], [0], [1], [0]], num_experts=4, top_k=2,
                                                      drop_rate=0.1),
                                              img=(2, 96, 96), mode='train_noisy'),
    'van_t_512_eval': dict(kw=dict(VAN_T_KW), img=(1, 512, 512), mode='eval', full=True, stride=4, unit='lka'),
}

# the SM3Det_lsk_t backbone dict without its pretrained init_cfg
LSK_T_BACKBONE = dict(type='LSKNet_moe_MultiInput', datasets=None, drop_rate=0.1, drop_path_rate=0.1,
                      norm_cfg=dict(type='SyncBN', requires_grad=True), **LSK_T_KW)


def run_layout():
    from oracle import ref_shim
    mod = ref_shim.load_reference_module('lsk_moe')
    kw = {k: v for k, v in LSK_T_BACKBONE.items() if k != 'type'}
    torch.manual_seed(0)
    sd = mod.LSKNet_moe_MultiInput(**kw).state_dict()
    os.makedirs(OUT, exist_ok=True)
    torch.save(dict(kw=kw, keys=list(sd), shapes={k: tuple(v.shape) for k, v in sd.items()}), os.path.join(OUT, 'layout.pt'))
    print(f'layout: {len(sd)} keys')


if __name__ == '__main__':
    from oracle import gen_golden
    torch.set_num_threads(8)
    gen_golden.OUT = OUT
    names = sys.argv[1:] or (list(LSK_T_CASES) + ['layout'])
    for nm in names:
        if nm == 'layout':
            run_layout()
        else:
            gen_golden.run_lsk_case(nm, LSK_T_CASES[nm])
