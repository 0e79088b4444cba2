"""train.py --resume of a data-parallel run on 2 GPUs (torchrun, NCCL): tests/resume_ddp_check.py.  Skipped with fewer than 2
GPUs."""
import os
import subprocess
import sys

import pytest
import torch

from helpers import free_port

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B, H, W = 2, 128, 416


def torchrun(tmp_path, tag, argv):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(free_port()), os.path.join(ROOT, "tests", "resume_ddp_check.py"), str(tmp_path), tag, "--"] + argv
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=str(tmp_path))
    print(out.stdout[-3000:])
    assert out.returncode == 0, out.stderr[-4000:]
    return [torch.load(tmp_path / ("%s_rank%d.pt" % (tag, r))) for r in range(2)]


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_data_parallel_run_resumes_with_every_ranks_own_streams(tmp_path):
    """A world-2 run of one epoch, resumed for a second: each rank's resumed draws are the ones its own saved streams give (and
    the two ranks' differ), and after the resumed step the two ranks' parameter arenas are equal."""
    import random

    import numpy as np
    from scsfm.augment import Draw
    base = ["synthetic", "--name", "ddp", "-b", str(B), "--synthetic-size", str(H), str(W), "--epoch-size", "1", "--gpu-augment",
            "1", "--learn-intrinsics", "1"]
    first = torchrun(tmp_path, "first", base + ["--epochs", "1"])
    run = tmp_path / "checkpoints" / "ddp"
    run = run / os.listdir(run)[0]
    state = torch.load(run / "training_state.pth.tar", weights_only=False)
    assert state["world_size"] == 2 and len(state["rng"]) == 2
    want = []
    for r in range(2):                       # the draws rank r's saved streams give next
        random.setstate(state["rng"][r]["python"])
        np.random.set_state(state["rng"][r]["numpy"])
        want.append([(d.flip, float(d.x_scaling), float(d.y_scaling), d.offset_x, d.offset_y)
                     for d in (Draw.random(H, W) for _ in range(B))])
    assert want[0] != want[1]
    resumed = torchrun(tmp_path, "resumed", base + ["--epochs", "2", "--resume", str(run)])
    for r in range(2):
        assert len(first[r]["draws"]) == B and first[r]["draws"] != first[1 - r]["draws"]
        assert resumed[r]["draws"] == want[r], r
    for a, b in zip(resumed[0]["arenas"], resumed[1]["arenas"]):
        assert torch.equal(a, b)
    for a, b in zip(first[0]["arenas"], resumed[0]["arenas"]):
        assert not torch.equal(a, b)             # the resumed step moved them
