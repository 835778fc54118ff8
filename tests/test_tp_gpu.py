"""Tensor-parallel decode (SURVEY §8e) on real GPUs: G ranks, one GPU each, against the CPU oracle.
Skipped when the box has fewer than two GPUs."""
import json
import os
import subprocess
import sys

import pytest

from util import ROOT

pytestmark = pytest.mark.gpu


def _gpus():
    import torch
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.parametrize("world,L,E,steps", [
    (2, 2, 1024, 5),   # 512 channels per rank over 132 CTAs: 3-4 per CTA
    (2, 2, 4096, 4),   # 7B width
    (4, 1, 5120, 3),   # 14B width on four ranks
    (4, 3, 768, 6),    # 169M width: 192 channels per rank, one or two per CTA
    (8, 2, 4096, 3),   # 7B width on eight ranks: 512-byte row segments
    (8, 1, 5120, 3),   # 14B width on eight ranks
])
def test_tp_matches_oracle(pkg, make_model, tmp_path, world, L, E, steps):
    if _gpus() < world:
        pytest.skip("needs %d GPUs" % world)
    path = make_model(L, E)
    out = str(tmp_path / "tp.json")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", str(29500 + world),
           os.path.join(ROOT, "tests", "helpers", "tp_worker.py"), path, str(steps), out]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, "tp worker failed:\n" + r.stdout[-3000:] + r.stderr[-3000:]
    res = json.load(open(out))
    print(res)
    assert res["worst_vs_oracle"] < 1e-3
    assert res["worst_vs_single_gpu"] < 1e-4
    assert res["ranks_agree"] and res["greedy_agree"]
