"""LSKNet-T / VAN-T (configs/SM3Det/SM3Det_lsk_t.py, SM3Det_van_t.py) on the GPU: widths [32, 64, 160, 256], so the
LSK attention branch's 1x1 convs are 16 and 80 channels wide and run on the GEMM's column tail.

Each fixture of tests/golden/lsk_t/ (generated from the unmodified reference by tools/gen_golden_lsk_t.py) is checked
with the machinery and tolerances of the LSK-S fixtures (tests/test_lsk_gpu.py): forward <= 1e-3 relative (2e-3 for the
1024^2 eval case, see FORWARD_TOL), routing and
LSK channel-argmax flips only at numerical ties (teacher-forced oracle), every parameter gradient <= 3e-3 against the
forced oracle (full-size cases) or the fixture (short case), BatchNorm running statistics and the gate loss.
"""
import glob
import os

import pytest
import torch

import test_lsk_gpu as L

pytestmark = pytest.mark.gpu
GOLD_T = os.path.join(os.path.dirname(__file__), 'golden', 'lsk_t')
FIXTURES = sorted(p for p in glob.glob(os.path.join(GOLD_T, '*.pt')) if os.path.basename(p) != 'layout.pt')


def test_fixtures_present():
    assert {os.path.basename(p)[:-3] for p in FIXTURES} == {
        'lsk_t_1024_eval', 'lsk_t_b2_512_train_noisy_drop', 'lsk_t_short_e4k2_train_noisy_drop', 'van_t_512_eval'}


# LSK-T in eval mode at 1x1024^2 is ill-conditioned at stage 3: the oracle in fp32 and in fp64 (same routing and channel
# argmax) differ by 2.5e-5 there, about 400x the fp32 unit roundoff, so the split-bf16 GEMMs' ~1e-5 relative error per
# product shows as ~1.2e-3 (measured on an H100; the training case at 2x512^2 shows 3e-5 at every stage).  That one
# fixture's forward is held to 2e-3; every other bound is the LSK-S one.
FORWARD_TOL = {'lsk_t_1024_eval': 2e-3}


@pytest.mark.parametrize('path', FIXTURES, ids=lambda p: os.path.basename(p)[:-3])
def test_lsk_t_backbone_matches_reference_golden(path, monkeypatch):
    monkeypatch.setattr(L, 'TOL', FORWARD_TOL.get(os.path.basename(path)[:-3], L.TOL))
    L.test_lsk_backbone_matches_reference_golden(path)


def test_graphed_lsk_t_step_matches_eager():
    """A CUDA-graph-captured LSK-T training step (gating noise and dropout off) replays to the eager loss and gradients."""
    from oracle.cases import load_golden
    from sm3det_b200.graphed import GraphedStep
    from sm3det_b200.synth import make_images
    from test_graph_gpu import fwd_bwd, grads, rel
    kw = dict(load_golden(os.path.join(GOLD_T, 'lsk_t_short_e4k2_train_noisy_drop.pt'))['kw'], noisy_gating=False,
              drop_rate=0.0)
    _, _, net = L.build(kw)
    net.train()
    x = make_images(2, 96, 96, seed=6).cuda()
    step = fwd_bwd(net)
    rm0 = {k: v.clone() for k, v in net.state_dict().items() if 'running_' in k}
    ref = step(x).clone()
    gr = grads(net)
    net.zero_grad(set_to_none=True)
    net.load_state_dict(rm0, strict=False)                       # BatchNorm running statistics advance on every pass
    g = GraphedStep(step, [x], net.parameters(), warmup=1)
    net.load_state_dict(rm0, strict=False)
    got = g(x)
    torch.cuda.synchronize()
    assert abs(got.item() - ref.item()) <= 2e-5 * abs(ref.item())
    now = grads(net)
    assert set(now) == set(gr)
    # w_gate.temperature: a scalar sum over all tokens with heavy cancellation; atomics reorder it between runs
    worst = max((rel(now[k], gr[k]) / (5.0 if k.endswith('temperature') else 1.0), k) for k in gr if float(gr[k].abs().max()) > 1e-8)
    assert worst[0] < 5e-4, worst
