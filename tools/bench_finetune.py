"""Fine-tuning step speed: kitti_r18 Trainer steps (B=4, 256x832, 2 refs, tf32x3, one CUDA-graph replay per step) with parts of
the networks frozen, in frames/s and library launches per step, beside the fully trainable step bench.py measures.

    python tools/bench_finetune.py [--steps 20] [--conv-mode tf32x3]

Patterns: all trainable | DispResNet encoder frozen and in eval mode | PoseResNet frozen | decoder-only (both encoders frozen and
in eval mode, PoseResNet's head still trained).  Each timed step starts from the same seeded state (as in bench.py), with the
L2 cache flushed before it; the card's name and power limit are printed with the numbers."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "sc-sfmlearner-release_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402


def freeze(disp, pose, pattern):
    if pattern in ("disp_encoder_frozen_eval", "decoder_only"):
        disp.encoder.requires_grad_(False)
        disp.encoder.eval()
    if pattern == "pose_frozen":
        pose.requires_grad_(False)
    if pattern == "decoder_only":
        pose.encoder.requires_grad_(False)
        pose.encoder.eval()


PATTERNS = ("all_trainable", "disp_encoder_frozen_eval", "pose_frozen", "decoder_only")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        out = ""
    return out or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--conv-mode", default="tf32x3", choices=["fp32", "tf32", "tf32x3"])
    args = ap.parse_args()
    import models
    from scsfm import lib as L
    from scsfm import synth
    from scsfm.trainer import Trainer
    if not torch.cuda.is_available():
        raise SystemExit("bench_finetune needs a GPU")
    L.load()
    dev = torch.device("cuda", 0)
    B, H, W = 4, 256, 832
    tgt, refs, K = synth.triplet(1234, B, H, W, 2, "kitti")
    tgt, refs, K = tgt.to(dev), [r.to(dev) for r in refs], K.to(dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    results = {}
    for pattern in PATTERNS:
        torch.manual_seed(0)
        disp, pose = models.DispResNet(18, False).to(dev).train(), models.PoseResNet(18, False).to(dev).train()
        freeze(disp, pose, pattern)
        tr = Trainer(disp, pose, lr=1e-4, num_scales=1, with_ssim=1, with_mask=1, with_auto_mask=1, padding_mode="zeros",
                     distributed=False, conv_mode=args.conv_mode)
        initial = tr.optimizer.snapshot()
        for _ in range(2):
            tr.step(tgt, refs, K)
        tr.capture(tgt, refs, K)

        def reset():
            tr.optimizer.restore(initial)
            for n in tr.optimizer.nets:
                n.refresh_operand_weights()
        for _ in range(2):
            reset()
            tr.step(tgt, refs, K)
        torch.cuda.synchronize()
        total = 0.0
        for _ in range(args.steps):
            reset()
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            tr.step(tgt, refs, K)
            e1.record()
            torch.cuda.synchronize()
            total += e0.elapsed_time(e1)
        ms = total / args.steps
        results[pattern] = {"frames_per_s": round(B / (ms * 1e-3), 2), "ms_per_step": round(ms, 3),
                            "launches_per_step": tr.launches_per_step}
        print(pattern, json.dumps(results[pattern]), flush=True)
        del tr, disp, pose
        torch.cuda.empty_cache()
    print(json.dumps({"card": card(), "config": "kitti_r18 B=%d %dx%d 2 refs %s, CUDA graph, L2 flushed before each step" % (
        B, H, W, args.conv_mode), "steps": args.steps, "results": results}), flush=True)


if __name__ == "__main__":
    main()
