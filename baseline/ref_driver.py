"""Drives the UNMODIFIED reference training loop (reference train.py:235-299, `train.train()`) on synthetic batches.

The reference sources are not part of this repository: SCSFM_REFERENCE_DIR names a checkout of the original project
(default: the git-ignored oracle/_ref/ that __graft_entry__.build() installs).  This script puts baseline/stubs (stand-ins for path / tensorboardX /
blessings / progressbar / matplotlib / imageio, which are not installed and cannot be installed offline) and that
checkout on sys.path, imports the reference's own `train` module and
calls its `train()` function with the reference's own models, losses and torch.optim.Adam -- none of this repository's
kernels, models or engine are imported.  Only the DataLoader is replaced by an in-memory synthetic one (same tuple
layout as datasets/sequence_folders.py:55-65 / pair_folders.py:42-57).

    python baseline/ref_driver.py --device cpu|cuda --steps K --warmup W [--config kitti_r18|kitti_r50|nyu_r18]
                                  [--batch B] [--threads T] [--anomaly 0|1] [--cudnn-benchmark 0|1] [--tf32 0|1]

Prints ONE JSON line: {"ms_per_step", "frames_per_s", ...}.  Step time = wall clock between two consecutive batches
being handed to the loop (every reference iteration ends with loss.item() host syncs, train.py:277-290, so the wall
clock is the device time plus the reference's own host overheads, as shipped).
"""
import argparse
import json
import os
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("SCSFM_REFERENCE_DIR") or os.path.join(os.path.dirname(HERE), "oracle", "_ref")

CONFIGS = {  # name: (disp layers, pose layers, H, W, n_ref, per-GPU batch, intrinsics kind)
    "kitti_r18": (18, 18, 256, 832, 2, 4, "kitti"),
    "kitti_r50": (50, 50, 256, 832, 2, 2, "kitti"),
    "nyu_r18": (18, 18, 256, 320, 1, 8, "nyu"),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--device", choices=["cpu", "cuda"], default="cpu")
    ap.add_argument("--config", choices=sorted(CONFIGS), default="kitti_r18")
    ap.add_argument("--batch", type=int, default=0)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--threads", type=int, default=0)
    ap.add_argument("--anomaly", type=int, default=1, help="1 = as shipped (train.py:67 turns autograd anomaly detection on)")
    ap.add_argument("--cudnn-benchmark", type=int, default=1, help="1 = as train.py:82-83")
    ap.add_argument("--tf32", type=int, default=1, help="cuDNN/cuBLAS TF32 (torch's default for convolutions)")
    ap.add_argument("--budget-s", type=float, default=0.0, help="stop timing early once this many seconds of timed steps have run")
    args = ap.parse_args()

    if not os.path.isdir(REF) or not os.path.exists(os.path.join(REF, "train.py")):
        print(json.dumps({"unavailable": "no checkout of the original project (set SCSFM_REFERENCE_DIR)"}))
        return 0
    if args.device == "cpu":
        os.environ["CUDA_VISIBLE_DEVICES"] = ""       # the reference picks cuda whenever it is visible (train.py:66)
    sys.dont_write_bytecode = True
    sys.path[:0] = [REF, os.path.join(HERE, "stubs"), os.path.join(os.path.dirname(HERE), "sc-sfmlearner-release_b200", "scsfm")]
    import torch
    if args.threads > 0:
        torch.set_num_threads(args.threads)
    import synth                                     # seeded synthetic inputs only (pure torch, shared with the parity tests)
    sys.argv = ["train.py", "synthetic", "--name", "bench"]      # train.py builds its parser at import time
    # the reference's `datasets/` has no __init__.py; an installed package of the same name (HuggingFace datasets) would
    # shadow it, so bind the name to the reference directory explicitly
    import types
    ds = types.ModuleType("datasets")
    ds.__path__ = [os.path.join(REF, "datasets")]
    sys.modules["datasets"] = ds
    import train as T                                # the reference module, unmodified
    import models as M                               # the reference's own models package (oracle/_ref/models)
    assert os.path.dirname(os.path.abspath(M.__file__)).startswith(REF), "wrong `models` package on sys.path"
    torch.autograd.set_detect_anomaly(bool(args.anomaly))
    torch.backends.cudnn.allow_tf32 = bool(args.tf32)
    torch.backends.cuda.matmul.allow_tf32 = bool(args.tf32)
    if args.device == "cuda":
        torch.backends.cudnn.deterministic = True     # train.py:82-83
        torch.backends.cudnn.benchmark = bool(args.cudnn_benchmark)
    dl, pl, H, W, n_ref, batch, kind = CONFIGS[args.config]
    if args.batch > 0:
        batch = args.batch
    device = T.device
    assert device.type == args.device, (device, args.device)

    torch.manual_seed(0)
    disp_net = M.DispResNet(dl, False).to(device)
    pose_net = M.PoseResNet(pl, False).to(device)
    disp_net = torch.nn.DataParallel(disp_net)       # train.py:168-169 (identity on CPU / one GPU)
    pose_net = torch.nn.DataParallel(pose_net)
    optimizer = torch.optim.Adam([{"params": disp_net.parameters(), "lr": 1e-4}, {"params": pose_net.parameters(), "lr": 1e-4}],
                                 betas=(0.9, 0.999), weight_decay=0)
    tgt, refs, K = synth.triplet(1234, batch, H, W, n_ref, kind)
    if args.device == "cuda":
        tgt, refs, K = tgt.pin_memory(), [r.pin_memory() for r in refs], K.pin_memory()
    total = args.warmup + args.steps
    stamps, early = [], []

    class Loader:
        """In-memory stand-in for the DataLoader: the same batch `total` times; stamps the hand-over times."""

        def __len__(self):
            return total

        def __iter__(self):
            for i in range(total):
                if args.device == "cuda":
                    torch.cuda.synchronize()
                stamps.append(time.perf_counter())
                if args.budget_s > 0 and i > args.warmup and stamps[-1] - stamps[args.warmup] > args.budget_s:
                    early.append(1)
                    return
                yield tgt, refs, K, torch.inverse(K)

    save = T.Path(tempfile.mkdtemp(prefix="scsfm_ref_"))
    targs = argparse.Namespace(photo_loss_weight=1.0, smooth_loss_weight=0.1, geometry_consistency_weight=0.5, print_freq=10,
                               num_scales=1, with_ssim=1, with_mask=1, with_auto_mask=1, padding_mode="zeros", batch_size=batch,
                               save_path=save, log_full="progress_log_full.csv")
    open(save / targs.log_full, "w").close()
    logger = T.TermLogger(n_epochs=1, train_size=total, valid_size=0)
    T.train(targs, Loader(), disp_net, pose_net, optimizer, total, logger, T.SummaryWriter(save))
    if args.device == "cuda":
        torch.cuda.synchronize()
    if not early:
        stamps.append(time.perf_counter())
    steps = len(stamps) - 1 - args.warmup
    dt = stamps[-1] - stamps[args.warmup]
    print(json.dumps({"ms_per_step": round(1e3 * dt / steps, 3), "frames_per_s": round(batch * steps / dt, 4), "steps": steps,
                      "warmup": args.warmup, "batch": batch, "config": args.config, "device": args.device,
                      "threads": torch.get_num_threads(), "anomaly": args.anomaly, "tf32": args.tf32,
                      "cudnn_benchmark": args.cudnn_benchmark, "torch": torch.__version__,
                      "what": "unmodified reference train.train() (train.py:235-299) on a synthetic in-memory loader"}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
