"""Offline evaluation throughput, one JSON line per configuration, with the card's name and power limit read in the same process.

  eval_depth  KITTI-sized synthetic data (697 images, 256x832 float64 predictions, float32 ground truth of the four Eigen sizes
              375x1242 / 370x1226 / 374x1238 / 376x1241 at ~5 % density) and NYU-sized data (654 images, 256x320 predictions,
              dense 480x640 ground truth): images/s of scsfm.loss_ops.eval_depth from arrays in host memory (packing, copies,
              kernel, read-back), the summed device time of the scsfm_eval_depth launches (CUDA events), and images/s of the
              reference's per-image numpy computation (cv2.resize when cv2 is installed, else the oracle's restated resize) on the
              first --host-images images.
  test_pose   snippets/s of PoseResNet18 on a --frames-frame synthetic sequence at 256x832: every consecutive pair once, in
              batches of --pose-batch through the Predictor (test_pose.py), against 4 batch-1 calls per snippet (the reference's
              call pattern); pose_vec2mat on the device, composition and errors on the host in both arms.

    python tools/bench_eval.py [--host-images 40] [--frames 200] [--pose-batch 16]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "sc-sfmlearner-release_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_infer import card  # noqa: E402

KITTI_SIZES = [(375, 1242), (370, 1226), (374, 1238), (376, 1241)]


def depth_data(dataset, n, seed=0):
    g = np.random.default_rng(seed)
    if dataset == "kitti":
        preds = np.exp(g.normal(2.5, 0.5, (n, 256, 832)))
        gts = []
        for k in range(n):
            H, W = KITTI_SIZES[k % 4]
            gt = np.zeros((H, W), np.float32)
            m = g.random((H, W)) < 0.05
            gt[m] = g.uniform(0.5, 90, int(m.sum()))
            gts.append(gt)
    else:
        preds = np.exp(g.normal(1.0, 0.4, (n, 256, 320)))
        gts = g.uniform(0.3, 11, (n, 480, 640)).astype(np.float32)
    return preds, gts


def host_rate(preds, gts, dataset, n):
    from oracle import evaluation as E
    try:
        import cv2
        resize, which = (lambda s, H, W: cv2.resize(s, (W, H))), "cv2"
    except ImportError:
        resize, which = E.resize_linear, "numpy"
    t = time.perf_counter()
    for i in range(n):
        E.eval_depth_image(preds[i], gts[i], dataset, resize)
    return n / (time.perf_counter() - t), which


def bench_depth(dataset, n, host_images):
    from scsfm import lib as L
    from scsfm import loss_ops
    preds, gts = depth_data(dataset, n)
    loss_ops.eval_depth(preds[:8], gts, dataset)                       # warm-up: module load, pinned buffers
    torch.cuda.synchronize()
    runs = []
    for _ in range(2):
        t = time.perf_counter()
        rows = loss_ops.eval_depth(preds, gts, dataset)
        runs.append(time.perf_counter() - t)
    L.PROF.update(enabled=True, only={"eval"}, events=[])
    loss_ops.eval_depth(preds, gts, dataset)
    torch.cuda.synchronize()
    kernel_ms = sum(e0.elapsed_time(e1) for _, _, e0, e1, _ in L.PROF["events"])
    L.PROF.update(enabled=False, events=[])
    hr, which = host_rate(preds, gts, dataset, host_images)
    return {"bench": "eval_depth", "dataset": dataset, "images": n, "images_per_s": round(n / min(runs), 1),
            "wall_s": [round(r, 3) for r in runs], "kernel_ms_total": round(kernel_ms, 3), "kernel_us_per_image": round(1000 * kernel_ms / n, 2),
            "host_images_per_s": round(hr, 2), "host_resize": which, "host_images_timed": host_images,
            "mean_n": round(float(rows[:, 0].mean()), 1)}


def bench_pose(frames_n, batch, mode="tf32x3"):
    import models
    from inverse_warp import pose_vec2mat
    from scsfm import inference_io as io
    from scsfm.infer import Predictor
    g = np.random.default_rng(1)
    frames = [g.integers(0, 256, (256, 832, 3), dtype=np.uint8) for _ in range(frames_n)]
    gt = np.tile(np.eye(4)[:3], (frames_n, 1, 1))
    gt[:, :, 3] = np.cumsum(g.normal(0, 1, (frames_n, 3)), 0)
    torch.manual_seed(0)
    net = models.PoseResNet(18, False).cuda().set_conv_mode(mode).eval()
    pred = Predictor(net)
    snippets = io.snippet_indices(frames_n)

    def batched():
        mats = []
        for i0, i1 in io.batches(frames_n - 1, batch):
            mats.append(pose_vec2mat(pred(io.network_input(np.stack(frames[i0:i1])), io.network_input(np.stack(frames[i0 + 1:i1 + 1])))).cpu().numpy())
        mats = np.concatenate(mats)
        return [io.pose_error(io.compensated_poses(gt, idx), io.integrate(mats[idx[0]:idx[-1]]).reshape(5, 3, 4)) for idx in snippets]

    def per_snippet():
        out = []
        for idx in snippets:
            ims = [io.network_input(frames[a][None]) for a in idx]
            mats = [pose_vec2mat(pred(ims[k], ims[k + 1])).cpu().numpy()[0] for k in range(4)]
            out.append(io.pose_error(io.compensated_poses(gt, idx), io.integrate(np.stack(mats)).reshape(5, 3, 4)))
        return out

    res = {}
    with torch.no_grad():
        for name, fn in (("batched_dedup", batched), ("per_snippet_b1", per_snippet)):
            fn()
            torch.cuda.synchronize()
            t = time.perf_counter()
            errs = fn()
            res[name] = round(len(snippets) / (time.perf_counter() - t), 1)
            res[name + "_errors"] = np.array(errs)
    diff = float(np.max(np.abs(res.pop("batched_dedup_errors") - res.pop("per_snippet_b1_errors"))))
    return {"bench": "test_pose", "frames": frames_n, "snippets": len(snippets), "pose_batch": batch, "conv_mode": mode,
            "snippets_per_s": res, "max_abs_error_difference": diff}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--host-images", type=int, default=40)
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--pose-batch", type=int, default=16)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval.py needs a CUDA device")
    name, power = card()
    for dataset, n in (("kitti", 697), ("nyu", 654)):
        print(json.dumps(dict(bench_depth(dataset, n, args.host_images), card=name, power_limit=power)), flush=True)
    print(json.dumps(dict(bench_pose(args.frames, args.pose_batch), card=name, power_limit=power)), flush=True)


if __name__ == "__main__":
    main()
