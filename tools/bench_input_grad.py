"""Forward+backward throughput of DispResNet18 / PoseResNet18 with eval-mode and input-image gradients, and the stem
input-gradient kernel against the composition it replaces.  One JSON line per measurement; the first line names the card and
its power limit.

    python tools/bench_input_grad.py [--H 256 --W 832 --batches 1,4,16 --modes tf32x3,tf32 --iters 10 --warmup 3]

Arms (images/s for DispResNet, pairs/s for PoseResNet; forward + backward of one call, CUDA events):
  train_params       train mode, parameter gradients, images without gradient (the training step's network call)
  eval_params        eval mode, parameter gradients (frozen BatchNorm statistics)
  eval_input_only    eval mode, every parameter frozen, gradient of the input image(s) only
  cudnn_*            the same three on stock PyTorch / cuDNN (oracle.nets; TF32 convolutions on in mode tf32, off otherwise)
Stem: scsfm_stem_dgrad against the CUDA-core conv2d_dgrad + nhwc_to_nchw on the same dy (ms per call, CUDA events).
"""
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


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], text=True)
        power = out.strip()
    except (OSError, subprocess.CalledProcessError):
        power = "unknown"
    return name, power


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters      # ms


def loss_of(kind, out):
    if kind == "disp":
        outs = out if isinstance(out, (list, tuple)) else [out]
        return sum((1.0 / o).mean() for o in outs)
    return out.square().sum()


def net_arms(kind, B, H, W, mode, iters, warmup):
    import models
    from oracle import nets as N
    n_img = 1 if kind == "disp" else 2
    imgs = [torch.randn(B, 3, H, W, device="cuda") for _ in range(n_img)]
    res = {}

    def arm(net, training, params, img_grad):
        net.train(training)
        net.requires_grad_(params)

        def step():
            xs = [i.detach().requires_grad_(img_grad) for i in imgs]
            loss_of(kind, net(*xs)).backward()
        return timed(step, iters, warmup)

    net = (models.DispResNet(18, False) if kind == "disp" else models.PoseResNet(18, False)).cuda().set_conv_mode(mode)
    res["train_params"] = arm(net, True, True, False)
    res["eval_params"] = arm(net, False, True, False)
    res["eval_input_only"] = arm(net, False, False, True)
    del net
    torch.backends.cudnn.allow_tf32 = mode == "tf32"
    torch.backends.cuda.matmul.allow_tf32 = mode == "tf32"
    ref = (N.DispResNet(18) if kind == "disp" else N.PoseResNet(18)).cuda()
    res["cudnn_train_params"] = arm(ref, True, True, False)
    res["cudnn_eval_params"] = arm(ref, False, True, False)
    res["cudnn_eval_input_only"] = arm(ref, False, False, True)
    del ref
    torch.cuda.empty_cache()
    return {k: round(B * 1000.0 / ms, 1) for k, ms in res.items()}


def stem_arms(Cin, B, H, W, iters, warmup):
    from scsfm import nnops as O
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    dy = torch.randn(B, Ho, Wo, 64, device="cuda")
    w = torch.randn(64, 7, 7, Cin, device="cuda") * 0.05
    need = (True,) if Cin == 3 else (True, True)
    cx = O.ConvCtx("fp32")
    kern = timed(lambda: O.stem_dgrad(dy, w, H, W, need), iters, warmup)
    comp = timed(lambda: O.nhwc_to_nchw(cx.conv_dgrad(dy, w, (B, H, W, Cin), 2, 3)), iters, warmup)
    a = O.stem_dgrad(dy, w, H, W, need)
    b = O.nhwc_to_nchw(cx.conv_dgrad(dy, w, (B, H, W, Cin), 2, 3))
    diff = max(float((a[k] - b[:, 3 * k:3 * k + 3]).abs().max()) for k in range(len(need))) / float(b.abs().max())
    gflop = 2.0 * B * H * W * Cin * 64 * 49 / 4 / 1e9
    return dict(stem_dgrad_ms=round(kern, 4), simt_dgrad_plus_layout_ms=round(comp, 4), speedup=round(comp / kern, 2),
                stem_dgrad_tflops=round(gflop / kern, 2), max_rel_diff=diff)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--H", type=int, default=256)
    ap.add_argument("--W", type=int, default=832)
    ap.add_argument("--batches", default="1,4,16")
    ap.add_argument("--modes", default="tf32x3,tf32")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--skip-nets", action="store_true")
    a = ap.parse_args()
    name, power = card()
    print(json.dumps(dict(gpu=name, power_limit=power, H=a.H, W=a.W)), flush=True)
    batches = [int(b) for b in a.batches.split(",")]
    for Cin in (3, 6):
        for B in batches:
            print(json.dumps(dict(kind="stem", Cin=Cin, B=B, **stem_arms(Cin, B, a.H, a.W, a.iters, a.warmup))), flush=True)
    if a.skip_nets:
        return
    for kind in ("disp", "pose"):
        for mode in a.modes.split(","):
            for B in batches:
                r = net_arms(kind, B, a.H, a.W, mode, a.iters, a.warmup)
                print(json.dumps(dict(kind=kind, mode=mode, B=B, unit="images/s" if kind == "disp" else "pairs/s", **r)), flush=True)


if __name__ == "__main__":
    main()
