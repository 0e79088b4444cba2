"""Training entry with the reference's command line (reference train.py:24-61) on the H100 path.

    python train.py DIR --name EXP [--resnet-layers 18 -b 4 -s 0.1 -c 0.5 --with-auto-mask 1 ...]
    torchrun --nproc-per-node 8 train.py DIR --name EXP ...        # data parallel, one process per GPU

What is different from the reference loop (train.py:235-299), by design:
  * the per-iteration step (train.py:254-282) is scsfm.trainer.Trainer.step: stacked network calls, fused loss
    kernels, arena Adam, no host synchronisation; losses are read back every --print-freq iterations only
    (the reference calls .item() 5-9 times per iteration and appends a CSV row each time);
  * multi-GPU is one process per GPU with a NCCL gradient all-reduce instead of nn.DataParallel
    (train.py:168-169); -b is the per-GPU batch size;
  * `torch.autograd.set_detect_anomaly(True)` (train.py:67) is not enabled.
DIR may be the literal word `synthetic` (seeded KITTI-shaped batches, no files needed); otherwise the
reference's dataset classes (datasets/sequence_folders.py, pair_folders.py, validation_folders.py and
custom_transforms.py -- host-side I/O, out of scope of this repo) must be importable from PYTHONPATH.
Checkpoints keep the reference's file names and layout (utils.py:57-66): {'epoch', 'state_dict'}.
"""
import argparse
import csv
import datetime
import os
import shutil
import time

import numpy as np

import torch
import torch.distributed as dist

import models
from loss_functions import compute_errors, compute_photo_and_geometry_loss, compute_smooth_loss
from scsfm import nnops, synth
from scsfm.trainer import Trainer, compute_depth, compute_pose_with_inv

parser = argparse.ArgumentParser(description="SC-SfMLearner training on KITTI / NYU (H100 path)",
                                 formatter_class=argparse.ArgumentDefaultsHelpFormatter)
parser.add_argument("data", metavar="DIR", help="path to dataset, or 'synthetic'")
parser.add_argument("--folder-type", type=str, choices=["sequence", "pair"], default="sequence", help="the dataset dype to train")
parser.add_argument("--sequence-length", type=int, metavar="N", help="sequence length for training", default=3)
parser.add_argument("-j", "--workers", default=4, type=int, metavar="N", help="number of data loading workers")
parser.add_argument("--epochs", default=200, type=int, metavar="N", help="number of total epochs to run")
parser.add_argument("--epoch-size", default=0, type=int, metavar="N", help="manual epoch size (will match dataset size if not set)")
parser.add_argument("-b", "--batch-size", default=4, type=int, metavar="N", help="mini-batch size (per GPU)")
parser.add_argument("--lr", "--learning-rate", default=1e-4, type=float, metavar="LR", help="initial learning rate")
parser.add_argument("--momentum", default=0.9, type=float, metavar="M", help="momentum for sgd, alpha parameter for adam")
parser.add_argument("--beta", default=0.999, type=float, metavar="M", help="beta parameters for adam")
parser.add_argument("--weight-decay", "--wd", default=0, type=float, metavar="W", help="weight decay")
parser.add_argument("--print-freq", default=10, type=int, metavar="N", help="print frequency")
parser.add_argument("--seed", default=0, type=int, help="seed for random functions, and network initialization")
parser.add_argument("--log-summary", default="progress_log_summary.csv", metavar="PATH", help="csv where to save per-epoch train and valid stats")
parser.add_argument("--log-full", default="progress_log_full.csv", metavar="PATH", help="csv where to save per-gradient descent train stats")
parser.add_argument("--log-output", action="store_true", help="accepted for compatibility (tensorboard image logging is out of scope)")
parser.add_argument("--resnet-layers", type=int, default=18, choices=[18, 50], help="number of ResNet layers for depth estimation.")
parser.add_argument("--num-scales", "--number-of-scales", type=int, help="the number of scales", metavar="W", default=1)
parser.add_argument("-p", "--photo-loss-weight", type=float, help="weight for photometric loss", metavar="W", default=1)
parser.add_argument("-s", "--smooth-loss-weight", type=float, help="weight for disparity smoothness loss", metavar="W", default=0.1)
parser.add_argument("-c", "--geometry-consistency-weight", type=float, help="weight for depth consistency loss", metavar="W", default=0.5)
parser.add_argument("--with-ssim", type=int, default=1, help="with ssim or not")
parser.add_argument("--with-mask", type=int, default=1, help="with the the mask for moving objects and occlusions or not")
parser.add_argument("--with-auto-mask", type=int, default=0, help="with the the mask for stationary points")
parser.add_argument("--with-pretrain", type=int, default=0,
                    help="with or without imagenet pretrain for resnet.  The reference defaults to 1 and downloads the torchvision "
                         "weights; there is no network here, so the default is 0 and 1 loads resnet{18,50}-*.pth from "
                         "$SCSFM_PRETRAINED_DIR or the torch hub cache (clear error if absent)")
parser.add_argument("--dataset", type=str, choices=["kitti", "nyu"], default="kitti", help="the dataset to train")
parser.add_argument("--pretrained-disp", dest="pretrained_disp", default=None, metavar="PATH", help="path to pre-trained dispnet model")
parser.add_argument("--pretrained-pose", dest="pretrained_pose", default=None, metavar="PATH", help="path to pre-trained Pose net model")
parser.add_argument("--name", dest="name", type=str, required=True, help="name of the experiment, checkpoints are stored in checpoints/name")
parser.add_argument("--padding-mode", type=str, choices=["zeros", "border"], default="zeros", help="padding mode for image warping")
parser.add_argument("--with-gt", action="store_true", help="use ground truth for validation (npy depth maps, see the reference's data/kitti_raw_loader.py)")
# additions of this implementation
parser.add_argument("--conv-mode", choices=["fp32", "tf32", "tf32x3"], default="tf32x3",
                    help="tf32x3 = wgmma tensor cores with split-accumulate operands (fp32-level results, the parity mode); tf32 = "
                         "wgmma single TF32 product (cuDNN's default arithmetic, fastest); fp32 = exact CUDA-core convolutions")
parser.add_argument("--cuda-graph", type=int, default=1, help="capture the training step in a CUDA graph (single GPU)")
parser.add_argument("--overlap", type=int, default=1, help="run PoseResNet next to DispResNet and the weight gradients on side streams")
parser.add_argument("--synthetic-size", type=int, nargs=2, default=[256, 832], metavar=("H", "W"))
parser.add_argument("--gpu-augment", type=int, default=None, choices=[0, 1],
                    help="1: the training transforms (flip, zoom-crop, to-tensor, normalise: custom_transforms.py) run on the GPU on uint8 "
                         "frames (scsfm.augment.GpuAugment, bit-identical to the host chain for equal random draws); 0: the reference's "
                         "host-side chain inside the loader workers.  Default: 1 for real datasets, 0 for DIR = synthetic")

best_error = -1
n_iter = 0


class SyntheticLoader:
    """Seeded KITTI/NYU-shaped batches in the dataset's return convention (tgt_img, ref_imgs, K, K_inv); raw=True: the frames
    as decoded uint8 images [B, n_img, H, W, 3] plus K (what RawFrames below delivers for a real dataset)."""

    def __init__(self, length, batch, H, W, n_ref, kind, seed, raw=False):
        self.length, self.args, self.seed, self.raw = length, (batch, H, W, n_ref, kind), seed, raw

    def __len__(self):
        return self.length

    def __iter__(self):
        b, H, W, n_ref, kind = self.args
        for i in range(self.length):
            tgt, refs, K = synth.triplet(self.seed + i, b, H, W, n_ref, kind)
            if self.raw:
                frames = torch.stack([tgt] + list(refs), 1).permute(0, 1, 3, 4, 2)          # [B, n_img, H, W, 3], normalised
                yield ((frames * 0.225 + 0.45) * 255).round().clamp(0, 255).to(torch.uint8), K
            else:
                yield tgt, refs, K, torch.linalg.inv(K)


class RawFrames(torch.utils.data.Dataset):
    """A reference dataset built with transform=None (datasets/sequence_folders.py:55-66, pair_folders.py): sample -> (frames
    uint8 [n_img, H, W, 3] with the target first, intrinsics).  uint8 is exact for decoded JPEG/PNG frames and a quarter of the
    bytes through the worker pipes and PCIe."""

    def __init__(self, ds):
        self.ds = ds

    def __len__(self):
        return len(self.ds)

    def __getitem__(self, i):
        tgt, refs, K, _ = self.ds[i]
        return np.stack([tgt] + list(refs)).astype(np.uint8), np.asarray(K, np.float32)


class GpuAugmentLoader:
    """Wraps a loader of (frames uint8 [B, n_img, H, W, 3], K [B, 3, 3]) batches: upload, device-side transforms, and the
    loop's (tgt_img, ref_imgs, intrinsics, intrinsics_inv) tuple comes out resident on the GPU."""

    def __init__(self, loader, device, train=True):
        from scsfm.augment import GpuAugment
        self.loader, self.device = loader, device
        self.aug = GpuAugment(mean=(0.45, 0.45, 0.45), std=(0.225, 0.225, 0.225), train=train, device=device)
        self.sampler = getattr(loader, "sampler", None)

    def __len__(self):
        return len(self.loader)

    def __iter__(self):
        for frames, K in self.loader:
            frames = frames.to(self.device, non_blocking=True).transpose(0, 1).contiguous()     # image slot major
            imgs, K = self.aug(frames, K)
            yield imgs[0], imgs[1:], K, torch.linalg.inv(K)


def _reference_dataset_module(name):
    """datasets/<name>.py of the reference, loaded by file path from the first sys.path entry that holds it.  The reference's
    datasets/ directory has no __init__.py (a namespace package), so a plain `import datasets.<name>` resolves to any installed
    regular package called `datasets` (HuggingFace's) instead -- regular packages win over namespace packages whatever the
    path order.  The module is registered under a private name (picklable for loader workers); sys.modules['datasets'] is left alone."""
    import importlib.util
    import sys
    key = "scsfm_reference_datasets_" + name
    if key in sys.modules:
        return sys.modules[key]
    for entry in sys.path:
        f = os.path.join(entry or ".", "datasets", name + ".py")
        if os.path.isfile(f):
            spec = importlib.util.spec_from_file_location(key, f)
            mod = importlib.util.module_from_spec(spec)
            sys.modules[key] = mod
            try:
                spec.loader.exec_module(mod)
            except BaseException:
                del sys.modules[key]
                raise
            return mod
    raise ImportError("datasets/%s.py not found on sys.path" % name)


def make_loaders(args, rank, world, device="cuda"):
    gpu_aug = args.gpu_augment if args.gpu_augment is not None else (0 if args.data == "synthetic" else 1)
    if args.data == "synthetic":
        H, W = args.synthetic_size
        n_ref = 1 if args.folder_type == "pair" else args.sequence_length - 1
        n = args.epoch_size if args.epoch_size > 0 else 100
        train_loader = SyntheticLoader(n, args.batch_size, H, W, n_ref, args.dataset, 1000 * rank, raw=bool(gpu_aug))
        if gpu_aug:
            train_loader = GpuAugmentLoader(train_loader, device, train=True)
        return train_loader, SyntheticLoader(max(1, n // 10), args.batch_size, H, W, n_ref, args.dataset, 7777 + rank)
    try:
        import custom_transforms
        PairFolder = _reference_dataset_module("pair_folders").PairFolder
        SequenceFolder = _reference_dataset_module("sequence_folders").SequenceFolder
    except ImportError as e:
        raise SystemExit("real datasets need the reference's host-side loaders (datasets/*.py, custom_transforms.py) on "
                         "PYTHONPATH -- they are out of scope of this repo (%s); or pass DIR = synthetic" % e)
    normalize = custom_transforms.Normalize(mean=[0.45, 0.45, 0.45], std=[0.225, 0.225, 0.225])
    train_tf = custom_transforms.Compose([custom_transforms.RandomHorizontalFlip(), custom_transforms.RandomScaleCrop(),
                                          custom_transforms.ArrayToTensor(), normalize])
    valid_tf = custom_transforms.Compose([custom_transforms.ArrayToTensor(), normalize])
    if gpu_aug:
        train_tf = None                      # the datasets hand out the decoded frames; the transforms run on the GPU per batch
    if args.folder_type == "sequence":
        train_set = SequenceFolder(args.data, transform=train_tf, seed=args.seed, train=True,
                                   sequence_length=args.sequence_length, dataset=args.dataset)
    else:
        train_set = PairFolder(args.data, seed=args.seed, train=True, transform=train_tf)
    if gpu_aug:
        train_set = RawFrames(train_set)
    if args.with_gt:
        ValidationSet = _reference_dataset_module("validation_folders").ValidationSet
        val_set = ValidationSet(args.data, transform=valid_tf, dataset=args.dataset)
    else:
        val_set = SequenceFolder(args.data, transform=None if gpu_aug else valid_tf, seed=args.seed, train=False,
                                 sequence_length=args.sequence_length, dataset=args.dataset)
        if gpu_aug:
            val_set = RawFrames(val_set)     # (the ground-truth validation set above keeps the host chain: it also returns depth maps)
    sampler = torch.utils.data.distributed.DistributedSampler(train_set, world, rank, shuffle=True, seed=args.seed) if world > 1 else None
    train_loader = torch.utils.data.DataLoader(train_set, batch_size=args.batch_size, shuffle=sampler is None, sampler=sampler,
                                               num_workers=args.workers, pin_memory=True, drop_last=True)
    val_loader = torch.utils.data.DataLoader(val_set, batch_size=args.batch_size, shuffle=False, num_workers=args.workers,
                                             pin_memory=True)
    if gpu_aug:
        train_loader = GpuAugmentLoader(train_loader, device, train=True)
        if not args.with_gt:
            val_loader = GpuAugmentLoader(val_loader, device, train=False)      # ArrayToTensor + Normalize only
    return train_loader, val_loader


def save_checkpoint(save_path, dispnet_state, exp_pose_state, is_best, filename="checkpoint.pth.tar"):
    """Same files as the reference's utils.save_checkpoint (utils.py:57-66); tensors are detached from the arena."""
    for prefix, state in (("dispnet", dispnet_state), ("exp_pose", exp_pose_state)):
        state = dict(state, state_dict={k: v.detach().clone().contiguous().cpu() for k, v in state["state_dict"].items()})
        torch.save(state, os.path.join(save_path, "{}_{}".format(prefix, filename)))
        if is_best:
            shutil.copyfile(os.path.join(save_path, "{}_{}".format(prefix, filename)),
                            os.path.join(save_path, "{}_model_best.pth.tar".format(prefix)))


def main():
    global best_error, n_iter
    args = parser.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        raise SystemExit("train.py drives the H100 kernels: a CUDA device is required (no CPU fallback)")
    torch.cuda.set_device(local)
    device = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=device)

    timestamp = datetime.datetime.now().strftime("%m-%d-%H:%M")
    args.save_path = os.path.join("checkpoints", args.name, timestamp)
    if rank == 0:
        print("=> will save everything to {}".format(args.save_path))
        os.makedirs(args.save_path, exist_ok=True)
    torch.manual_seed(args.seed)

    train_loader, val_loader = make_loaders(args, rank, world, device)
    if args.epoch_size == 0:
        args.epoch_size = len(train_loader)

    if rank == 0:
        print("=> creating model")
    try:
        disp_net = models.DispResNet(args.resnet_layers, args.with_pretrain).to(device)
        pose_net = models.PoseResNet(18, args.with_pretrain).to(device)      # train.py:155 hard-codes 18 for the pose net
    except FileNotFoundError as e:
        raise SystemExit("--with-pretrain 1: %s" % e)
    if args.pretrained_disp:
        disp_net.load_state_dict(torch.load(args.pretrained_disp, map_location=device)["state_dict"], strict=False)
    if args.pretrained_pose:
        pose_net.load_state_dict(torch.load(args.pretrained_pose, map_location=device)["state_dict"], strict=False)

    trainer = Trainer(disp_net, pose_net, lr=args.lr, betas=(args.momentum, args.beta), weight_decay=args.weight_decay,
                      num_scales=args.num_scales, with_ssim=args.with_ssim, with_mask=args.with_mask,
                      with_auto_mask=args.with_auto_mask, padding_mode=args.padding_mode, w1=args.photo_loss_weight,
                      w2=args.smooth_loss_weight, w3=args.geometry_consistency_weight, distributed=world > 1, conv_mode=args.conv_mode, overlap_nets=bool(args.overlap), overlap_wgrad=bool(args.overlap))
    if rank == 0:
        with open(os.path.join(args.save_path, args.log_summary), "w") as f:
            csv.writer(f, delimiter="\t").writerow(["train_loss", "validation_loss"])
        with open(os.path.join(args.save_path, args.log_full), "w") as f:
            csv.writer(f, delimiter="\t").writerow(["train_loss", "photo_loss", "smooth_loss", "geometry_consistency_loss"])

    for epoch in range(args.epochs):
        sampler = getattr(train_loader, "sampler", None)
        if hasattr(sampler, "set_epoch"):
            sampler.set_epoch(epoch)           # DistributedSampler: a different shuffle every epoch
        train_loss = train(args, train_loader, trainer, device, rank, world)
        if args.with_gt:
            errors, names = validate_with_gt(args, val_loader, disp_net, device)
        else:
            errors, names = validate_without_gt(args, val_loader, disp_net, pose_net, device)
        if rank == 0:
            print(" * epoch {} train loss {:.4f} | ".format(epoch, train_loss) +
                  ", ".join("{} : {:.3f}".format(n, e) for n, e in zip(names, errors)))
            decisive = errors[1]
            if best_error < 0:
                best_error = decisive
            is_best = decisive < best_error
            best_error = min(best_error, decisive)
            save_checkpoint(args.save_path, {"epoch": epoch + 1, "state_dict": disp_net.state_dict()},
                            {"epoch": epoch + 1, "state_dict": pose_net.state_dict()}, is_best)
            with open(os.path.join(args.save_path, args.log_summary), "a") as f:
                csv.writer(f, delimiter="\t").writerow([train_loss, decisive])
    if world > 1:
        dist.destroy_process_group()


def train(args, train_loader, trainer, device, rank, world):
    """One epoch of train.py:235-299.  Returns the mean total loss of the logged iterations."""
    global n_iter
    trainer.disp_net.train()
    trainer.pose_net.train()
    end = time.time()
    shown, total, rows = 0.0, 0, []
    for i, (tgt_img, ref_imgs, intrinsics, _) in enumerate(train_loader):
        tgt_img = tgt_img.to(device, non_blocking=True)
        ref_imgs = [img.to(device, non_blocking=True) for img in ref_imgs]
        intrinsics = intrinsics.to(device, non_blocking=True)
        if args.cuda_graph and world == 1 and trainer._graph is None and i == 0 and n_iter == 0:
            trainer.capture(tgt_img, ref_imgs, intrinsics)
        out = trainer.step(tgt_img, ref_imgs, intrinsics)
        rows.append(torch.stack(out))
        if i % args.print_freq == 0 or i >= args.epoch_size - 1:
            vals = torch.stack(rows).cpu()            # one read-back per print interval (train.py:270-277,288-290)
            rows = []
            if rank == 0:
                with open(os.path.join(args.save_path, args.log_full), "a") as f:
                    w = csv.writer(f, delimiter="\t")
                    for v in vals.tolist():
                        w.writerow(v)
                dt = time.time() - end
                print("Train: iter {} ({:.1f} frames/s/GPU) Loss {:.4f} photo {:.4f} smooth {:.4f} geo {:.4f}".format(
                    i, args.batch_size * vals.shape[0] / max(dt, 1e-9), *vals[-1].tolist()))
            shown += float(vals[:, 0].sum())
            total += vals.shape[0]
            end = time.time()
        n_iter += 1
        if i >= args.epoch_size - 1:
            break
    return shown / max(total, 1)


@torch.no_grad()
def validate_without_gt(args, val_loader, disp_net, pose_net, device):
    """train.py:302-362: eval-mode networks, the same losses, auto-mask forced off."""
    disp_net.eval()
    pose_net.eval()
    acc, n = torch.zeros(4, device=device), 0
    for tgt_img, ref_imgs, intrinsics, _ in val_loader:
        tgt_img = tgt_img.to(device)
        ref_imgs = [img.to(device) for img in ref_imgs]
        intrinsics = intrinsics.to(device)
        tgt_depth = [1 / disp_net(tgt_img)]
        ref_depths = [[1 / disp_net(r)] for r in ref_imgs]
        poses = [pose_net(tgt_img, r) for r in ref_imgs]
        poses_inv = [pose_net(r, tgt_img) for r in ref_imgs]
        l1, l3 = compute_photo_and_geometry_loss(tgt_img, ref_imgs, intrinsics, tgt_depth, ref_depths, poses, poses_inv,
                                                 args.num_scales, args.with_ssim, args.with_mask, False, args.padding_mode)
        l2 = compute_smooth_loss(tgt_depth, tgt_img, ref_depths, ref_imgs)
        acc += torch.stack([l1, l1, l2, l3])
        n += 1
    return (acc / max(n, 1)).tolist(), ["Total loss", "Photo loss", "Smooth loss", "Consistency loss"]


@torch.no_grad()
def validate_with_gt(args, val_loader, disp_net, device):
    """train.py:365-423."""
    disp_net.eval()
    names = ["abs_diff", "abs_rel", "sq_rel", "a1", "a2", "a3"]
    acc, n = [0.0] * 6, 0
    for tgt_img, depth in val_loader:
        tgt_img, depth = tgt_img.to(device), depth.to(device)
        if depth.nelement() == 0:
            continue
        output_depth = 1 / disp_net(tgt_img)[:, 0]
        if depth.nelement() != output_depth.nelement():
            b, h, w = depth.size()
            output_depth = torch.nn.functional.interpolate(output_depth.unsqueeze(1), [h, w]).squeeze(1)
        acc = [a + e for a, e in zip(acc, compute_errors(depth, output_depth, args.dataset))]
        n += 1
    return [a / max(n, 1) for a in acc], names


if __name__ == "__main__":
    main()
