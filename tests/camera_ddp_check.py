"""Launched by tests/test_camera_gpu.py under torchrun (2 ranks, one GPU each): the data-parallel Trainer with a learned camera,
--cameras 1 (one camera) or --cameras 2 (a bank of two, rank r's shard using camera r only).

  eager  theta is bit-identical across the replicas after a step, and its all-reduced gradient is the mean of the gradients that
         a single-GPU Trainer computes on each rank's shard (same weights, records and indices).  With a bank each row is half
         of the one rank that uses that camera: the other rank's shard gives it exact zeros.
  graph  the captured data-parallel step (the camera gradient all-reduced inside the graph) tracks an eager data-parallel one
         (losses, the first step's dtheta, theta within 3 steps x 2 lr) and keeps the replicas' theta and dtheta bit-identical;
         with a bank its first gradient is the mean above as well.
Prints "CAMERA_DDP_OK <mode>" per passed mode on rank 0; any failure raises.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "sc-sfmlearner-release_b200"), os.path.join(ROOT, "tests", "golden"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import models  # noqa: E402
from golden_util import det_weights  # noqa: E402
from scsfm import synth  # noqa: E402
from scsfm.augment import Draw  # noqa: E402
from scsfm.camera import LearnedCamera, records  # noqa: E402
from scsfm.trainer import Trainer  # noqa: E402


def same_on_all_ranks(t):
    other = t.clone()
    dist.broadcast(other, 0)
    return torch.equal(t, other)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cameras", type=int, choices=[1, 2], default=1)
    bank = ap.parse_args().cameras == 2
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    per, H, W = 2, 128, 160
    tgt, refs, K = synth.triplet(31, per * world, H, W)
    draws = [Draw.given(H, W, i % 2 == 0, 1.0 + 0.03 * i, 1.1 - 0.02 * i, i, 2 * i) for i in range(per * world)]
    sl = slice(rank * per, (rank + 1) * per)
    args = (tgt[sl].to(dev), [r[sl].to(dev) for r in refs])
    rec = records(draws[sl], W, dev)
    fx, fy, cx, cy = float(K[0, 0, 0]), float(K[0, 1, 1]), float(K[0, 0, 2]), float(K[0, 1, 2])
    th0 = [fx * 1.1, fy * 0.9, cx + 3, cy - 2]
    ix = {}
    if bank:
        th0 = [th0, [fx * 0.9, fy * 1.1, cx - 3, cy + 2]]
        ix = {"camera_index": torch.full((per,), rank % 2, dtype=torch.int32, device=dev)}      # rank r's shard: camera r only

    def make(distributed, mode="tf32x3"):
        d, p = models.DispResNet(18, False), models.PoseResNet(18, False)
        for net in (d, p):
            net.load_state_dict(det_weights(net.state_dict()))
        camera = LearnedCamera.bank(th0, H, W) if bank else LearnedCamera(*th0, H, W)
        return Trainer(d.to(dev).train(), p.to(dev).train(), lr=1e-4, distributed=distributed, conv_mode=mode, camera=camera.to(dev))

    def check_mean(got, want, what):
        err = float((got - want).norm() / want.norm())
        print("rank %d %s: all-reduced dtheta %s, mean of the per-shard gradients %s, rel %.2e" % (rank, what, got.tolist(), want.tolist(),
                                                                                                    err), flush=True)
        assert err < 1e-4, (what, err)

    # ---- eager: replicas identical, gradient = mean of the per-shard single-GPU gradients -----------------------------------
    local_tr = make(False)
    local_tr.step(*args, aug=rec, **ix)
    g_local = local_tr.camera.theta.grad.clone()
    if bank:
        assert torch.equal(g_local[1 - rank % 2], torch.zeros(4, device=dev))      # the other camera gets nothing from this shard
    gathered = [torch.zeros_like(g_local) for _ in range(world)]
    dist.all_gather(gathered, g_local)
    want = sum(gathered) / world
    tr = make(True)
    tr.step(*args, aug=rec, **ix)
    torch.cuda.synchronize()
    check_mean(tr.camera.theta.grad, want, "eager")
    assert same_on_all_ranks(tr.camera.theta.detach()), "theta diverged"
    assert same_on_all_ranks(tr.camera.theta.grad), "dtheta differs between the ranks"
    if rank == 0:
        print("CAMERA_DDP_OK eager", flush=True)

    # ---- captured data-parallel step: its first replay starts from the state above's ------------------------------------------
    eager, graphed = make(True), make(True)
    graphed.capture(*args, allow_distributed=True, aug=rec, **ix)
    for it in range(3):
        a = [float(v) for v in eager.step(*args, aug=rec, **ix)]
        b = [float(v) for v in graphed.step(*args, aug=rec, **ix)]
        for x, y in zip(a, b):
            assert abs(x - y) <= (2e-4 if it == 0 else 5e-3) * abs(x) + 1e-6, (it, a, b)
        torch.cuda.synchronize()
        g_e, g_g = eager.camera.theta.grad, graphed.camera.theta.grad        # all-reduced inside the graph / eagerly
        if it == 0:                                                          # identical states: the same gradient
            err = float((g_g - g_e).norm() / g_e.norm())
            assert err < 1e-4, (it, err)
            if bank:
                check_mean(g_g, want, "graph")
        assert same_on_all_ranks(g_g), "graphed dtheta differs between the ranks"
        assert same_on_all_ranks(graphed.camera.theta.detach()), "graphed theta diverged"
    torch.cuda.synchronize()
    # 3 steps x 2 lr, the bound of the single-GPU test: Adam may step a noise-level gradient component either way
    assert float((graphed.camera.theta - eager.camera.theta).abs().max()) <= 3 * 2 * eager.camera_lr + 1e-4
    if rank == 0:
        print("CAMERA_DDP_OK graph", flush=True)
    dist.barrier()
    torch.cuda.synchronize()
    sys.stdout.flush()
    os._exit(0)          # (a process group must not be torn down while captured graphs still hold its NCCL kernels)


if __name__ == "__main__":
    main()
