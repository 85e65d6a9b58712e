"""-m gpu, needs >= 2 GPUs (skipped on a single-GPU box): training through the key shards on NCCL with one rank per GPU
(tools/dist_train_check.py) — a cross_attention_sharded step with attention dropout plus reduce_shard_grads, on all key
shards and on the rank grid, against the one-GPU CrossAttention step.  The host-side protocol is covered on CPU by
tests/test_shard_train_cpu.py (gloo), the kernels by tests/test_gpu_shard_train.py."""
import os
import subprocess
import sys

import pytest
import torch

from conftest import ROOT

pytestmark = pytest.mark.gpu


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs at least two GPUs on the box")
def test_sharded_training_step_agrees_with_one_gpu():
    n = min(torch.cuda.device_count(), 8)
    n = 1 << (n.bit_length() - 1)   # 2, 4 or 8 ranks
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}",
                        "--master-addr", "127.0.0.1", "--master-port", "29573",
                        os.path.join(ROOT, "tools", "dist_train_check.py")],
                       capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0 and "DIST_TRAIN_CHECK OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
