"""Generate tests/golden/rpn_head/: seeded fp32 CPU forward fixtures of OrientedRPNHead's convolutions.

    python tools/gen_golden_rpn_head.py [case ...]

Each case (tests/rpn_head_ref.py:GOLDEN_CASES) stores the level maps, the parameters and the cls / reg outputs of the
oracle.  When the reference tree is present (SM3DET_REFERENCE_ROOT) the UNMODIFIED reference OrientedRPNHead is loaded with
the same parameters and its forward_single must reproduce every output bit for bit.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
OUT = os.path.join(ROOT, 'tests', 'golden', 'rpn_head')


def run_case(name, case):
    import rpn_head_ref as M
    sd = M.make_params(case['in_channels'], seed=case['seed'])
    feats = M.make_feats(case['batch'], case['sizes'], case['in_channels'], seed=case['seed'])
    with torch.no_grad():
        cls, reg = M.rpn_head_forward(sd, feats)
        ref = M.load_reference_heads()
        if ref is not None:
            head = ref.OrientedRPNHead(in_channels=case['in_channels'])
            head.load_state_dict(sd, strict=True)
            for x, c, r in zip(feats, cls, reg):
                rc, rr = head.forward_single(x.clone())
                assert torch.equal(rc, c) and torch.equal(rr, r), f'{name}: oracle differs from the reference'
        else:
            print(f'{name}: reference tree absent, fixture not cross-checked')
    from oracle.cases import save_golden          # files over the fixture size limit keep their large entries in parts/
    save_golden(dict(case=case, params=sd, feats=feats, cls=cls, reg=reg), os.path.join(OUT, name + '.pt'))
    print(name, [tuple(c.shape) for c in cls])


def main(names):
    import rpn_head_ref as M
    for name in names or list(M.GOLDEN_CASES):
        run_case(name, M.GOLDEN_CASES[name])


if __name__ == '__main__':
    main(sys.argv[1:])
