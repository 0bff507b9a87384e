"""Row-sharded solves with the normal-equation Anderson variants over 2 GPUs (NCCL inside the engine).  Skipped on
single-GPU boxes; the sharded Gram pass is emulated on CPU by tests/test_sharding_aa_variants_cpu.py."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_row_sharded_variant_solves_match_oracle():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", "29612", os.path.join(ROOT, "tests", "run_sharded_aa_variants_check.py")]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    print(res.stdout[-3000:])
    print(res.stderr[-3000:])
    assert res.returncode == 0
    assert "MISMATCH" not in res.stdout and res.stdout.count(" OK") == 4
