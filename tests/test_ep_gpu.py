"""Expert-parallel MoE over NVLink peer memory (BASELINE config 4 mechanism): one rank, and two GPUs of one box."""
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('n', [pytest.param(n, marks=pytest.mark.skipif(torch.cuda.device_count() < n,
                                                                         reason=f'needs >= {n} GPUs')) for n in (1, 2)])
def test_expert_parallel_matches_local_experts(n):
    r = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', str(n),
                        '--master-addr', '127.0.0.1', '--master-port', '29543',
                        os.path.join(ROOT, 'tests', 'dist', 'ep_gpu_worker.py'), ROOT],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    assert r.stdout.count('ep ok') == n, r.stdout[-2000:]
