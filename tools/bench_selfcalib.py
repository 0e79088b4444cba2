"""Self-calibrating training step speed: kitti_r18 Trainer steps (B=4, 256x832, 2 refs) in frames/s and library launches per step.

    python tools/bench_selfcalib.py [--steps 20] [--conv-mode tf32x3] [--cameras C]

Runs: captured without a camera (bench.py's step) | captured with a learned camera (Trainer(camera=...), augmentation records
in place of K) | eager with the learned camera | eager with a caller-owned K: theta as a torch parameter, the per-sample K
restated in torch from the records, the Trainer's K gradient and torch.optim.Adam on theta (the only option before the Trainer
owned the camera).  --cameras C > 1 adds a captured run with a bank of C learned cameras (LearnedCamera.bank, seeded random camera
indices per sample).  Each timed step starts from the same seeded state, with the L2 cache flushed before it; eager steps are
timed with their host work (the graph replays are not host-bound).  The card's name and power limit are printed with the numbers."""
import argparse
import json
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "sc-sfmlearner-release_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

RUNS = ("captured_no_camera", "captured_camera", "eager_camera", "eager_caller_k")


def torch_k(theta, rec):
    """The caller's restatement of the augmentation's intrinsics update, per sample, in torch ops."""
    xs, ys, flip, ox, oy, in_w = rec.to(theta.dtype).unbind(1)
    fx, fy, cx, cy = theta.unbind(0)
    cxb = torch.where(flip != 0, in_w - cx, cx)
    zero, one = torch.zeros_like(xs), torch.ones_like(xs)
    return torch.stack([torch.stack([fx * xs, zero, cxb * xs - ox], 1), torch.stack([zero, fy * ys, cy * ys - oy], 1),
                        torch.stack([zero, zero, one], 1)], 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--conv-mode", default="tf32x3", choices=["fp32", "tf32", "tf32x3"])
    ap.add_argument("--cameras", type=int, default=1, help="C > 1: also time a captured step with a bank of C cameras")
    args = ap.parse_args()
    import models
    from bench_finetune import card
    from scsfm import lib as L
    from scsfm import synth
    from scsfm.augment import Draw
    from scsfm.camera import LearnedCamera, records
    from scsfm.trainer import Trainer
    if not torch.cuda.is_available():
        raise SystemExit("bench_selfcalib needs a GPU")
    L.load()
    dev = torch.device("cuda", 0)
    B, H, W = 4, 256, 832
    tgt, refs, K = synth.triplet(1234, B, H, W, 2, "kitti")
    tgt, refs, K = tgt.to(dev), [r.to(dev) for r in refs], K.to(dev)
    random.seed(0)
    np.random.seed(0)
    rec = records([Draw.random(H, W) for _ in range(B)], W, dev)
    th0 = [float(K[0, 0, 0]), float(K[0, 1, 1]), float(K[0, 0, 2]), float(K[0, 1, 2])]
    C = max(1, args.cameras)
    gen = torch.Generator().manual_seed(0)
    bank0 = torch.tensor([th0] * C) * (1 + 0.05 * (torch.rand(C, 4, generator=gen) - 0.5))
    index = torch.randint(0, C, (B,), generator=gen, dtype=torch.int32).to(dev)
    runs = RUNS + (("captured_bank",) if C > 1 else ())
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    results = {}
    for run in runs:
        torch.manual_seed(0)
        disp, pose = models.DispResNet(18, False).to(dev).train(), models.PoseResNet(18, False).to(dev).train()
        cam = LearnedCamera(*th0, H, W).to(dev) if run in ("captured_camera", "eager_camera") else None
        if run == "captured_bank":
            cam = LearnedCamera.bank(bank0, H, W).to(dev)
        ix = {"camera_index": index} if run == "captured_bank" else {}
        tr = Trainer(disp, pose, lr=1e-4, num_scales=1, with_ssim=1, with_mask=1, with_auto_mask=1, padding_mode="zeros",
                     distributed=False, conv_mode=args.conv_mode, camera=cam)
        theta = torch.nn.Parameter(torch.tensor(th0, device=dev)) if run == "eager_caller_k" else None
        opt = torch.optim.Adam([theta], lr=0.1) if theta is not None else None
        initial = (tr.optimizer.snapshot(), tr._camera_snapshot(), None if theta is None else theta.detach().clone())

        def step():
            if cam is not None:
                return tr.step(tgt, refs, aug=rec, **ix)
            if theta is None:
                return tr.step(tgt, refs, K)
            out = tr.step(tgt, refs, torch_k(theta, rec))
            opt.step()
            opt.zero_grad()
            return out

        def reset():
            tr.optimizer.restore(initial[0])
            tr._camera_restore(initial[1])
            if theta is not None:
                theta.data.copy_(initial[2])
            for n in tr.optimizer.nets:
                n.refresh_operand_weights()
        for _ in range(2):
            step()
        if run.startswith("captured"):
            tr.capture(tgt, refs, K if cam is None else None, aug=rec if cam is not None else None, **ix)
        for _ in range(2):
            reset()
            step()
        torch.cuda.synchronize()
        total, launches = 0.0, 0
        for _ in range(args.steps):
            reset()
            flush.zero_()
            torch.cuda.synchronize()
            n0 = L.launch_count()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            step()
            e1.record()
            torch.cuda.synchronize()
            launches = tr.launches_per_step if run.startswith("captured") else L.launch_count() - n0
            total += e0.elapsed_time(e1)
        ms = total / args.steps
        results[run] = {"frames_per_s": round(B / (ms * 1e-3), 2), "ms_per_step": round(ms, 3), "launches_per_step": launches}
        if cam is not None:
            results[run]["theta"] = [round(v, 4) for v in cam.theta.reshape(-1).tolist()]
        if run == "captured_bank":
            results[run]["cameras"] = C
            results[run]["index"] = index.tolist()
        print(run, json.dumps(results[run]), flush=True)
        del tr, disp, pose
        torch.cuda.empty_cache()
    print(json.dumps({"card": card(), "config": "kitti_r18 B=%d %dx%d 2 refs %s, L2 flushed before each step" % (B, H, W, args.conv_mode),
                      "steps": args.steps, "results": results}), flush=True)


if __name__ == "__main__":
    main()
