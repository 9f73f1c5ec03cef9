"""Generate tests/golden/fpn_mmdet/: forward fixtures of mmdet's FPN in its three modes (max-pool extra levels, 'on_output'
and 'on_input' extra convs).

    python tools/gen_golden_fpn.py [case ...]      (needs the reference tree, SM3DET_REFERENCE_ROOT)

mmdet is not in the reference tree.  Every case runs the UNMODIFIED reference Multitask_FPN.py through oracle/ref_shim.py as
MultitaskFPN(start_level=0, extra_level=s, **kw).forward(inputs, start_level=s), loaded with the FPN(start_level=s) state
dict re-indexed (lateral_convs.j / fpn_convs.j -> index j+s; its convs 0..s-1 keep their own values and are unused), and
asserts that tests/fpn_mmdet_ref.py:fpn_forward_mmdet reproduces it bit for bit.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
OUT = os.path.join(ROOT, 'tests', 'golden', 'fpn_mmdet')


def run_case(name, kw):
    import fpn_mmdet_ref as M
    from oracle import ref_shim
    from oracle.cases import save_golden
    from sm3det_b200.synth import make_state_dict
    s = kw.get('start_level', 0)
    mode = kw.get('add_extra_convs', False)
    shapes = M.fpn_mmdet_param_shapes(kw['in_channels'], kw['out_channels'], kw['num_outs'], s, mode)
    sd = make_state_dict(shapes, M.GOLDEN_SD_SEED, True)
    mod = ref_shim.load_reference_module('Multitask_FPN', 'necks')
    torch.manual_seed(0)
    ref_kw = {k: v for k, v in kw.items() if k != 'start_level'}
    ref = mod.MultitaskFPN(start_level=0, extra_level=s, **ref_kw)
    rsd = ref.state_dict()
    mapped = {M.to_multitask_key(k, s): v for k, v in sd.items()}
    assert set(mapped) <= set(rsd), set(mapped) - set(rsd)
    assert M.from_multitask_state_dict(rsd, s).keys() == sd.keys()
    for k, v in mapped.items():
        assert rsd[k].shape == v.shape, k
    rsd.update(mapped)
    ref.load_state_dict(rsd, strict=True)
    xs = M.fpn_inputs(kw['in_channels'], M.GOLDEN_BATCH, M.GOLDEN_SIZES, M.GOLDEN_SEED)
    with torch.no_grad():
        want = ref(xs, start_level=s)
        got = M.fpn_forward_mmdet(sd, xs, kw['num_outs'], s, mode)
    assert len(want) == len(got) == kw['num_outs']
    for a, b in zip(want, got):
        assert torch.equal(a, b), f'{name}: oracle differs from the reference by {(a - b).abs().max()}'
    gold = dict(name=name, kw=kw, batch=M.GOLDEN_BATCH, sizes=M.GOLDEN_SIZES, seed=M.GOLDEN_SEED, sd_seed=M.GOLDEN_SD_SEED,
                keys=sorted(sd), outs=[o.clone() for o in want])
    save_golden(gold, os.path.join(OUT, name + '.pt'))
    print(f'{name}: ok, ' + ', '.join('x'.join(map(str, o.shape[2:])) for o in want))


if __name__ == '__main__':
    import fpn_mmdet_ref
    for nm in sys.argv[1:] or list(fpn_mmdet_ref.GOLDEN_CASES):
        run_case(nm, fpn_mmdet_ref.GOLDEN_CASES[nm])
