"""walk() under torchrun on 2 GPUs (SURVEY.md §8e): frames of every clip sharded over the ranks, gathered to rank 0
over NCCL, rank 0 the only writer — the files must equal the single-process walk's, including the remainder split
(5 and 4 frames over 2 ranks with batch_size 2).  Needs 2 GPUs; skipped on a single-GPU machine."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from PIL import Image

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_sharded_walk_equals_single_process_walk(tmp_path):
    worker = os.path.join(HERE, "_walk_worker.py")
    env = dict(os.environ)
    r1 = subprocess.run([sys.executable, worker, str(tmp_path), "one"], env=env, capture_output=True, text=True, timeout=600)
    assert r1.returncode == 0, r1.stderr[-3000:]
    r2 = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                         "--master-addr", "127.0.0.1", "--master-port", "29731", worker, str(tmp_path), "two"],
                        env=env, capture_output=True, text=True, timeout=600)
    assert r2.returncode == 0, r2.stderr[-3000:]
    one = sorted(p.relative_to(tmp_path / "one").as_posix() for p in (tmp_path / "one").glob("**/*.png"))
    two = sorted(p.relative_to(tmp_path / "two").as_posix() for p in (tmp_path / "two").glob("**/*.png"))
    assert [f.replace("one_", "") for f in one] == [f.replace("two_", "") for f in two] and len(one) == 9
    for a, b in zip(one, two):
        x = np.asarray(Image.open(tmp_path / "one" / a)).astype(np.int32)
        y = np.asarray(Image.open(tmp_path / "two" / b)).astype(np.int32)
        assert np.abs(x - y).max() <= 1, (a, int(np.abs(x - y).max()))
    assert (tmp_path / "two" / "prompt_config.json").exists()
