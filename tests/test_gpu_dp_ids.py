"""-m gpu (needs 2 GPUs): the same sample list decoded by 1 rank and by 2 ranks (torchrun, NCCL,
dp.shard_range + dp.gather_ids -- the code bench.py runs) returns IDENTICAL token ids in the same order.  This holds bit for
bit because no kernel's result depends on where a sample sits in the batch: attention tiles restart at every image / prompt,
the channel-attention Gram and the HFRE sums are reduced in an order-independent way, GEMM rows are independent."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(world, out):
    script = os.path.join(REPO, "scripts", "dp_ids.py")
    if world == 1:
        cmd = [sys.executable, script, "--out", out]
    else:
        with socket.socket() as s:
            s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
               "--master-port", str(port), script, "--out", out]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=REPO)
    assert r.returncode == 0, r.stderr[-3000:]
    return np.load(out)


def test_one_rank_and_two_ranks_return_identical_ids(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    one = _run(1, str(tmp_path / "ids1.npy"))
    two = _run(2, str(tmp_path / "ids2.npy"))
    assert one.shape == two.shape and one.shape[0] == 6
    assert np.array_equal(one, two), (one, two)
