"""Inference throughput at 256x832: DispResNet images/s and PoseResNet pairs/s, four arms per configuration:
  recording  net.eval() with autograd on (the activation-recording path: conv, then bn_apply)
  fused      net.eval() under torch.no_grad() (BatchNorm in the convolution epilogues), eager
  predictor  scsfm.infer.Predictor (the fused forward replayed from a CUDA graph)
  cudnn      stock PyTorch/cuDNN on oracle.nets in eval mode, cuDNN TF32 at its default (cudnn_tf32) and off (cudnn_fp32)
Peak torch.cuda.max_memory_allocated above the resident weights per arm; the outputs of recording / fused / predictor are
compared bitwise in the same run.  One JSON line per configuration, with the card's name and power limit read in the same
process.  Needs a GPU.

    python tools/bench_infer.py [--layers 18 50] [--batch 1 16] [--modes tf32x3 tf32] [--kinds disp pose] [--iters 20]
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
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    name, _, power = q.stdout.strip().partition(", ")
    return name or torch.cuda.get_device_name(0), power or "unknown"


def timed(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return out, e0.elapsed_time(e1) / iters, (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def run(kind, layers, B, mode, iters):
    import models
    from oracle import nets as ON
    from scsfm.infer import Predictor
    torch.manual_seed(0)
    net = (models.DispResNet(layers, False) if kind == "disp" else models.PoseResNet(layers, False)).cuda().set_conv_mode(mode).eval()
    imgs = [torch.randn(B, 3, 256, 832, device="cuda") for _ in range(1 if kind == "disp" else 2)]
    res = {}

    def recording():
        with torch.enable_grad():
            return net(*imgs).detach()

    def fused():
        with torch.no_grad():
            return net(*imgs)

    pred = Predictor(net)
    outs = {}
    for name, fn in (("recording", recording), ("fused", fused), ("predictor", lambda: pred(*imgs))):
        outs[name], ms, mb = timed(fn, iters)
        res[name] = {"ms": round(ms, 3), "per_s": round(B * 1000.0 / ms, 1), "peak_mb": round(mb, 1)}
    del pred
    ref = (ON.DispResNet(layers) if kind == "disp" else ON.PoseResNet(layers)).cuda().eval()
    ref.load_state_dict(net.state_dict())
    for name, tf32 in (("cudnn_tf32", True), ("cudnn_fp32", False)):
        torch.backends.cudnn.allow_tf32 = tf32
        with torch.no_grad():
            _, ms, mb = timed(lambda: ref(*imgs), iters)
        res[name] = {"ms": round(ms, 3), "per_s": round(B * 1000.0 / ms, 1), "peak_mb": round(mb, 1)}
    torch.backends.cudnn.allow_tf32 = True
    bits = lambda a, b: torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))  # noqa: E731
    equal = bits(outs["recording"], outs["fused"]) and bits(outs["fused"], outs["predictor"])
    return res, equal


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, nargs="*", default=[18, 50])
    ap.add_argument("--batch", type=int, nargs="*", default=[1, 16])
    ap.add_argument("--modes", nargs="*", default=["tf32x3", "tf32"])
    ap.add_argument("--kinds", nargs="*", default=["disp", "pose"])
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_infer.py needs a CUDA device")
    name, power = card()
    for kind in args.kinds:
        for layers in args.layers:
            for B in args.batch:
                for mode in args.modes:
                    res, equal = run(kind, layers, B, mode, args.iters)
                    print(json.dumps({"net": "%sResNet%d" % (kind.capitalize(), layers), "unit": "images/s" if kind == "disp" else "pairs/s",
                                      "B": B, "H": 256, "W": 832, "conv_mode": mode, "arms": res, "outputs_bitwise_equal": equal,
                                      "card": name, "power_limit": power}), flush=True)
                    torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
