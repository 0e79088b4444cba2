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

--learn-intrinsics 1 learns the camera (self-calibration): one fx, fy, cx, cy shared by every training scene, seen by each sample
through its own flip / zoom / crop (scsfm.camera.LearnedCamera), trained with the networks inside the captured / data-parallel
step.  It needs the GPU transforms.  The camera is saved as camera_checkpoint.pth.tar {'epoch', 'state_dict'} next to the
networks' files (camera_model_best.pth.tar with the same best-copy rule).
--camera-groups calibration | scene learns a bank of cameras instead: one per distinct cam.txt (KITTI raw's recording days,
Cityscapes' sequences) or one per training scene (uncalibrated video), each sample seeing its own group's camera.  The
checkpoint then holds theta [C,4] and a top-level 'groups' list of the cameras' labels.

At the end of every epoch rank 0 also writes training_state.pth.tar beside the checkpoints: the networks, both Adams, the camera,
the epoch, n_iter, best_error, the command line, the logs' row counts and every rank's random streams.  --resume RUN_DIR continues
that run in RUN_DIR at the next epoch, as if it had not stopped.
"""
import argparse
import csv
import datetime
import os
import random
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
parser.add_argument("--learn-intrinsics", type=int, default=0, choices=[0, 1],
                    help="1: learn the camera intrinsics fx, fy, cx, cy (self-calibration) with the networks; needs --gpu-augment 1 and "
                         "one camera for all training scenes, or --camera-groups")
parser.add_argument("--intrinsics-init", type=float, nargs=4, default=None, metavar=("FX", "FY", "CX", "CY"),
                    help="initial camera, in pixels at the training resolution.  Default: the first training scene's cam.txt "
                         "(DIR = synthetic: the synthetic K)")
parser.add_argument("--intrinsics-lr", type=float, default=0.1,
                    help="Adam learning rate of the learned intrinsics (pixels per step at most, roughly): 0.1 recovers fx, fy to "
                         "1%% from 20%% off in a few hundred steps (tests/test_camera_gpu.py)")
parser.add_argument("--camera-groups", choices=["one", "calibration", "scene"], default="one",
                    help="with --learn-intrinsics 1: one camera shared by every training scene (one); one camera per distinct cam.txt "
                         "matrix, per sample's intrinsics file with --folder-type pair (calibration: KITTI raw's recording days, "
                         "Cityscapes' sequences); one camera per training scene (scene: uncalibrated video).  Each camera starts from "
                         "its group's cam.txt, or every one from --intrinsics-init")
parser.add_argument("--resume", default=None, metavar="RUN_DIR",
                    help="continue the run saved in RUN_DIR (its training_state.pth.tar) at the epoch after the last one it finished, "
                         "in RUN_DIR.  The other flags come from this command line; --resnet-layers, --learn-intrinsics, "
                         "--camera-groups and the number of processes must be the run's")

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
    bytes through the worker pipes and PCIe.  With groups (one camera index per sample, see CameraTable): (frames, K, group)."""

    def __init__(self, ds, groups=None):
        self.ds, self.groups = ds, groups

    def __len__(self):
        return len(self.ds)

    def __getitem__(self, i):
        tgt, refs, K, _ = self.ds[i]
        out = np.stack([tgt] + list(refs)).astype(np.uint8), np.asarray(K, np.float32)
        return out if self.groups is None else out + (self.groups[i],)


class GpuAugmentLoader:
    """Wraps a loader of (frames uint8 [B, n_img, H, W, 3], K [B, 3, 3]) batches: upload, device-side transforms, and the
    loop's (tgt_img, ref_imgs, intrinsics, intrinsics_inv) tuple comes out resident on the GPU.  records=True appends the
    augmentation records; groups=True reads (frames, K, group) batches (RawFrames with groups) and appends the camera index of
    every sample, int32 [B] on the device."""

    def __init__(self, loader, device, train=True, records=False, groups=False):
        from scsfm.augment import GpuAugment
        self.loader, self.device, self.records, self.groups = loader, device, records, groups
        self.aug = GpuAugment(mean=(0.45, 0.45, 0.45), std=(0.225, 0.225, 0.225), train=train, device=device)
        self.sampler = getattr(loader, "sampler", None)

    def __len__(self):
        return len(self.loader)

    def __iter__(self):
        for batch in self.loader:
            frames, K = batch[:2]
            frames = frames.to(self.device, non_blocking=True).transpose(0, 1).contiguous()     # image slot major
            if self.records:                   # + the augmentation records a learned camera builds each sample's K from
                imgs, K, rec = self.aug(frames, K, return_records=True)
                out = imgs[0], imgs[1:], K, torch.linalg.inv(K), rec
            else:
                imgs, K = self.aug(frames, K)
                out = imgs[0], imgs[1:], K, torch.linalg.inv(K)
            if self.groups:                    # + each sample's camera in a bank of learned cameras
                out += (batch[2].to(self.device, torch.int32, non_blocking=True),)
            yield out


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


def gpu_augment_on(args):
    return args.gpu_augment if args.gpu_augment is not None else (0 if args.data == "synthetic" else 1)


def _read_intrinsics(path):
    """A 3x3 float32 intrinsics file, read as the reference's SequenceFolder / PairFolder read it."""
    return np.genfromtxt(path).astype(np.float32).reshape(3, 3)


def _training_scenes(root, split="train.txt"):
    with open(os.path.join(root, split)) as f:
        return [line.strip() for line in f if line.strip()]


def _intrinsics_files(scene_dir, folder_type):
    """The intrinsics files the reference's loader reads in one scene, in its order: cam.txt (SequenceFolder), or one sorted
    *.txt per image pair (PairFolder, datasets/pair_folders.py:37-42)."""
    if folder_type != "pair":
        return [os.path.join(scene_dir, "cam.txt")]
    names = sorted(os.listdir(scene_dir))
    imgs = [n for n in names if n.endswith(".jpg")]
    txts = [os.path.join(scene_dir, n) for n in names if n.endswith(".txt") and os.path.isfile(os.path.join(scene_dir, n))]
    return [txts[i // 2] for i in range(0, len(imgs) - 1, 2)]


class CameraTable:
    """The cameras of --camera-groups.  Camera c stands for a group of samples: keys[c] is the group's key (one, calibration: the
    float32 bytes of its intrinsics matrix; scene: its scene directory), labels[c] names it (the first intrinsics file of the
    group, relative to DIR, or the scene) and Ks[c] is the matrix it starts from.  Cameras are numbered in the order of the first
    train.txt scene that uses them, so every rank and every run builds the same table whatever the sample shuffle.  'one' groups
    as 'calibration' does, and learns a single camera (check_learn_intrinsics refuses more than one)."""

    def __init__(self, root, mode, folder_type="sequence"):
        if mode not in ("one", "calibration", "scene"):
            raise ValueError("camera groups: 'one', 'calibration' or 'scene', got %r" % (mode,))
        self.mode, self.keys, self.labels, self.Ks, self._index = mode, [], [], [], {}
        for scene in _training_scenes(root):
            d = os.path.join(root, scene)
            for f in _intrinsics_files(d, folder_type):
                K = _read_intrinsics(f)
                key = os.path.abspath(d) if mode == "scene" else K.tobytes()
                self._add(key, scene if mode == "scene" else os.path.relpath(f, root), K)

    @classmethod
    def single(cls, K, label):
        """One camera starting from K (DIR = synthetic)."""
        table = cls.__new__(cls)
        table.mode, table.keys, table.labels, table.Ks, table._index = "one", [], [], [], {}
        table._add(K.tobytes(), label, K)
        return table

    def _add(self, key, label, K):
        if key not in self._index:
            self._index[key] = len(self.keys)
            self.keys.append(key)
            self.labels.append(label)
            self.Ks.append(K)

    def __len__(self):
        return len(self.keys)

    def key(self, sample):
        """The group key of a reference dataset sample (an entry of SequenceFolder / PairFolder .samples)."""
        if self.mode != "scene":
            return np.asarray(sample["intrinsics"], np.float32).reshape(3, 3).tobytes()
        return os.path.abspath(os.path.dirname(str(sample["tgt"])))

    def index(self, sample):
        """The camera of a sample; -1 for a sample whose group no training scene has."""
        return self._index.get(self.key(sample), -1)

    def thetas(self, init=None):
        """[C][fx, fy, cx, cy]: each group's intrinsics, or init (--intrinsics-init) for every camera."""
        return [list(init) if init is not None else [float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])] for K in self.Ks]

    def camera(self, init, height, width):
        """The LearnedCamera of the table: one camera (theta [4]) for 'one', a bank (theta [C,4], labelled) otherwise."""
        from scsfm.camera import LearnedCamera
        if self.mode == "one":
            return LearnedCamera(*self.thetas(init)[0], height, width)
        return LearnedCamera.bank(self.thetas(init), height, width, groups=self.labels)


def check_learn_intrinsics(args):
    """--learn-intrinsics 1: the GPU transforms must be on (they hand out the augmentation records) and, with --camera-groups one,
    the training scenes must share one camera.  Returns the CameraTable of the cameras to learn (None without
    --learn-intrinsics); SystemExit with the reason otherwise."""
    groups = getattr(args, "camera_groups", "one")
    if groups != "one" and not args.learn_intrinsics:
        raise SystemExit("--camera-groups %s groups the cameras learned by --learn-intrinsics 1, which is off" % groups)
    if not args.learn_intrinsics:
        return None
    if not gpu_augment_on(args):
        raise SystemExit("--learn-intrinsics 1 needs the GPU transforms (--gpu-augment 1): the learned camera is built per sample "
                         "from the flip / zoom / crop records they hand out; learning K under the host-side chain is not supported")
    if args.data == "synthetic":
        if groups != "one":
            raise SystemExit("--camera-groups %s: DIR = synthetic has one camera (use --camera-groups one)" % groups)
        H, W = args.synthetic_size
        table = CameraTable.single(synth.intrinsics(1, H, W, args.dataset)[0].numpy(), "synthetic")
    else:
        table = CameraTable(args.data, groups, args.folder_type)
    if not len(table):
        raise SystemExit("--learn-intrinsics 1: %s/train.txt lists no scene with intrinsics" % args.data)
    if groups == "one" and len(table) > 1:
        raise SystemExit("--learn-intrinsics 1 learns ONE camera, but the training scenes have %d different intrinsics matrices "
                         "(e.g. %s differs from %s): several cameras are not supported (--camera-groups calibration learns one "
                         "camera per cam.txt)" % (len(table), table.labels[1], table.labels[0]))
    if args.intrinsics_init is not None:
        fx, fy = args.intrinsics_init[:2]
        if not (fx > 0 and fy > 0):
            raise SystemExit("--intrinsics-init: focal lengths must be positive, got fx %g fy %g" % (fx, fy))
    return table


def make_loaders(args, rank, world, device="cuda", cameras=None):
    """cameras: the CameraTable of --camera-groups calibration | scene (None otherwise): every sample then carries its camera
    index, -1 for a validation sample whose group is not a training camera's."""
    gpu_aug = gpu_augment_on(args)
    rec = {"records": True} if args.learn_intrinsics else {}       # the augmentation records, for a learned camera
    grp = {"groups": True} if cameras is not None else {}
    if args.data == "synthetic":
        H, W = args.synthetic_size
        n_ref = 1 if args.folder_type == "pair" else args.sequence_length - 1
        n = args.epoch_size if args.epoch_size > 0 else 100
        train_loader = SyntheticLoader(n, args.batch_size, H, W, n_ref, args.dataset, 1000 * rank, raw=bool(gpu_aug))
        if gpu_aug:
            train_loader = GpuAugmentLoader(train_loader, device, train=True, **rec)
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
        train_set = RawFrames(train_set, None if cameras is None else [cameras.index(s) for s in train_set.samples])
        if cameras is not None and -1 in train_set.groups:
            raise SystemExit("--camera-groups %s: a training sample belongs to no camera group" % args.camera_groups)
    if args.with_gt:
        ValidationSet = _reference_dataset_module("validation_folders").ValidationSet
        val_set = ValidationSet(args.data, transform=valid_tf, dataset=args.dataset)
    else:
        val_set = SequenceFolder(args.data, transform=None if gpu_aug else valid_tf, seed=args.seed, train=False,
                                 sequence_length=args.sequence_length, dataset=args.dataset)
        if gpu_aug:
            val_set = RawFrames(val_set)     # (the ground-truth validation set above keeps the host chain: it also returns depth maps)
            if cameras is not None:
                val_set.groups = [cameras.index(s) for s in val_set.ds.samples]
                if rank == 0:
                    n = sum(g >= 0 for g in val_set.groups)
                    print("=> validation: {} samples use their training group's learned camera, {} keep their dataset K".format(
                        n, len(val_set.groups) - n))
    sampler = torch.utils.data.distributed.DistributedSampler(train_set, world, rank, shuffle=True, seed=args.seed) if world > 1 else None
    train_loader = torch.utils.data.DataLoader(train_set, batch_size=args.batch_size, shuffle=sampler is None, sampler=sampler,
                                               num_workers=args.workers, pin_memory=True, drop_last=True)
    val_loader = torch.utils.data.DataLoader(val_set, batch_size=args.batch_size, shuffle=False, num_workers=args.workers,
                                             pin_memory=True)
    if gpu_aug:
        train_loader = GpuAugmentLoader(train_loader, device, train=True, **rec, **grp)
        if not args.with_gt:
            val_loader = GpuAugmentLoader(val_loader, device, train=False, **grp)      # ArrayToTensor + Normalize only
    return train_loader, val_loader


def save_checkpoint(save_path, dispnet_state, exp_pose_state, is_best, filename="checkpoint.pth.tar"):
    """Same files as the reference's utils.save_checkpoint (utils.py:57-66); tensors are detached from the arena."""
    for prefix, state in (("dispnet", dispnet_state), ("exp_pose", exp_pose_state)):
        state = dict(state, state_dict={k: v.detach().clone().contiguous().cpu() for k, v in state["state_dict"].items()})
        torch.save(state, os.path.join(save_path, "{}_{}".format(prefix, filename)))
        if is_best:
            shutil.copyfile(os.path.join(save_path, "{}_{}".format(prefix, filename)),
                            os.path.join(save_path, "{}_model_best.pth.tar".format(prefix)))


def save_camera_checkpoint(save_path, camera_state, is_best, filename="checkpoint.pth.tar"):
    """The learned camera next to the networks' files, with the same best-copy rule: camera_checkpoint.pth.tar
    {'epoch', 'state_dict': {'theta', 'height', 'width'}}, plus 'groups' (the labels of the cameras) for a bank."""
    state = dict(camera_state, state_dict={k: v.detach().clone().cpu() for k, v in camera_state["state_dict"].items()})
    torch.save(state, os.path.join(save_path, "camera_{}".format(filename)))
    if is_best:
        shutil.copyfile(os.path.join(save_path, "camera_{}".format(filename)), os.path.join(save_path, "camera_model_best.pth.tar"))


TRAINING_STATE = "training_state.pth.tar"


def rng_state(device):
    """This process's random streams: Python's `random` and numpy's (the augmentation draws), torch's CPU generator (the loaders'
    shuffle) and, on a CUDA device, its generator."""
    return {"python": random.getstate(), "numpy": np.random.get_state(), "torch": torch.get_rng_state(),
            "cuda": torch.cuda.get_rng_state(device) if device.type == "cuda" else None}


def set_rng_state(state, device):
    random.setstate(state["python"])
    np.random.set_state(state["numpy"])
    torch.set_rng_state(state["torch"])
    if state["cuda"] is not None:
        torch.cuda.set_rng_state(state["cuda"], device)


def gather_rng_states(world, device):
    """Every rank's rng_state, in RANK order.  A collective with world > 1: every rank calls it."""
    mine = rng_state(device)
    if world == 1:
        return [mine]
    states = [None] * world
    dist.all_gather_object(states, mine)
    return states


def log_rows(path):
    """The number of data rows of a CSV log (its lines after the header)."""
    with open(path, "rb") as f:
        return sum(1 for _ in f) - 1


def truncate_log(path, rows):
    """Keep the header and the first `rows` data rows of a CSV log: the rows of an epoch that was cut off go."""
    with open(path, "rb+") as f:
        for i in range(rows + 1):
            if not f.readline():
                raise SystemExit("--resume: %s has %d data rows, fewer than the %d the training state counts" % (path, max(i - 1, 0), rows))
        f.truncate(f.tell())


def save_training_state(save_path, state):
    """torch.save into a temporary file beside TRAINING_STATE, flushed to disk, then renamed over it: a run killed while
    saving keeps its previous state whole."""
    path = os.path.join(save_path, TRAINING_STATE)
    tmp = path + ".tmp"
    try:
        with open(tmp, "wb") as f:
            torch.save(state, f)
            f.flush()
            os.fsync(f.fileno())
        os.replace(tmp, path)
    except BaseException:
        if os.path.exists(tmp):
            os.remove(tmp)
        raise


def check_resume(args, cameras, world):
    """--resume RUN_DIR: the training state saved in RUN_DIR (on the CPU), once this command line is known to continue it; None
    without --resume.  SystemExit naming the flag otherwise.  Resuming with a different number of processes is not supported,
    and the flags that set the shapes of the state must be the run's."""
    if args.resume is None:
        return None
    if args.pretrained_disp or args.pretrained_pose:
        raise SystemExit("--resume continues a run from its own training state; it does not take --pretrained-disp / --pretrained-pose")
    path = os.path.join(args.resume, TRAINING_STATE)
    if not os.path.isfile(path):
        raise SystemExit("--resume %s: there is no %s in that directory (train.py writes it at the end of every epoch)"
                         % (args.resume, TRAINING_STATE))
    state = torch.load(path, map_location="cpu", weights_only=False)     # (the random streams and the command line are not tensors)
    if state["world_size"] != world:
        raise SystemExit("--resume: the run was trained by %d processes (WORLD_SIZE), this one has %d; resuming with a different "
                         "number of GPUs is not supported" % (state["world_size"], world))
    for name in ("resnet_layers", "learn_intrinsics", "camera_groups"):
        if getattr(args, name) != state["args"][name]:
            flag = "--" + name.replace("_", "-")
            raise SystemExit("--resume: %s %s, the run was trained with %s %s (it sets the shapes of the saved state)"
                             % (flag, getattr(args, name), flag, state["args"][name]))
    if cameras is not None:
        saved = state["trainer"]["camera"]["theta"].reshape(-1, 4).shape[0]
        if saved != len(cameras):
            raise SystemExit("--resume: the run learned %d cameras, the training scenes now give %d (--camera-groups %s)"
                             % (saved, len(cameras), args.camera_groups))
    return state


def training_size(args, train_loader):
    if args.data == "synthetic":
        return tuple(args.synthetic_size)
    frames = train_loader.loader.dataset[0][0]            # RawFrames: uint8 [n_img, H, W, 3]
    return tuple(frames.shape[1:3])


def main():
    global best_error, n_iter
    args = parser.parse_args()
    cameras = check_learn_intrinsics(args)
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    resume = check_resume(args, cameras, world)
    if not torch.cuda.is_available():
        raise SystemExit("train.py drives the H100 kernels: a CUDA device is required (no CPU fallback)")
    torch.cuda.set_device(local)
    device = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=device)

    if resume is None:
        timestamp = datetime.datetime.now().strftime("%m-%d-%H:%M")
        args.save_path = os.path.join("checkpoints", args.name, timestamp)
        if rank == 0:
            print("=> will save everything to {}".format(args.save_path))
            os.makedirs(args.save_path, exist_ok=True)
    else:
        args.save_path = args.resume
        if rank == 0:
            print("=> resuming {} at epoch {}".format(args.save_path, resume["epoch"]))
    # the reference's dataset classes seed Python's and numpy's streams with --seed as well (datasets/sequence_folders.py); seeding
    # them here makes the augmentation draws of DIR = synthetic repeatable too
    random.seed(args.seed)
    np.random.seed(args.seed)
    torch.manual_seed(args.seed)

    bank = cameras is not None and cameras.mode != "one"          # every sample then carries its camera index
    train_loader, val_loader = make_loaders(args, rank, world, device, cameras if bank else None)
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
    camera = None
    if cameras is not None:
        camera = cameras.camera(args.intrinsics_init, *training_size(args, train_loader)).to(device)
        if bank and rank == 0:
            print("=> learning {} cameras (--camera-groups {})".format(len(cameras), args.camera_groups))

    trainer = Trainer(disp_net, pose_net, lr=args.lr, betas=(args.momentum, args.beta), weight_decay=args.weight_decay,
                      num_scales=args.num_scales, with_ssim=args.with_ssim, with_mask=args.with_mask,
                      with_auto_mask=args.with_auto_mask, padding_mode=args.padding_mode, w1=args.photo_loss_weight,
                      w2=args.smooth_loss_weight, w3=args.geometry_consistency_weight, distributed=world > 1, conv_mode=args.conv_mode, overlap_nets=bool(args.overlap), overlap_wgrad=bool(args.overlap),
                      camera=camera, camera_lr=args.intrinsics_lr)
    logs = {"summary": os.path.join(args.save_path, args.log_summary), "full": os.path.join(args.save_path, args.log_full)}
    if resume is None:
        start_epoch, n_iter, best_error = 0, 0, -1
        if rank == 0:
            with open(logs["summary"], "w") as f:
                csv.writer(f, delimiter="\t").writerow(["train_loss", "validation_loss"])
            with open(logs["full"], "w") as f:
                csv.writer(f, delimiter="\t").writerow(["train_loss", "photo_loss", "smooth_loss", "geometry_consistency_loss"])
    else:
        trainer.load_state_dict(resume["trainer"])
        start_epoch, n_iter, best_error = resume["epoch"], resume["n_iter"], resume["best_error"]
        if rank == 0:
            for k, path in logs.items():
                truncate_log(path, resume["log_rows"][k])
        # last: building the datasets reseeds Python's and numpy's streams, and building the networks draws from torch's
        set_rng_state(resume["rng"][rank], device)
        resume = None                          # (the host copy of the state)

    for epoch in range(start_epoch, args.epochs):
        sampler = getattr(train_loader, "sampler", None)
        if hasattr(sampler, "set_epoch"):
            sampler.set_epoch(epoch)           # DistributedSampler: a different shuffle every epoch
        train_loss = train(args, train_loader, trainer, device, rank, world)
        if args.with_gt:
            errors, names = validate_with_gt(args, val_loader, disp_net, device)
        else:
            errors, names = validate_without_gt(args, val_loader, disp_net, pose_net, device, camera)
        if rank == 0:
            print(" * epoch {} train loss {:.4f} | ".format(epoch, train_loss) +
                  ", ".join("{} : {:.3f}".format(n, e) for n, e in zip(names, errors)))
            for c, th in enumerate([] if camera is None else camera.theta.reshape(-1, 4).tolist()):
                learned = "fx {:.3f} fy {:.3f} cx {:.3f} cy {:.3f}".format(*th)
                if camera.groups is None:
                    print(" * epoch {} learned camera {}".format(epoch, learned))
                else:                                   # a bank: each camera beside its group's cam.txt
                    K = cameras.Ks[c]
                    print(" * epoch {} camera {} {}: learned {} | cam.txt fx {:.3f} fy {:.3f} cx {:.3f} cy {:.3f}".format(
                        epoch, c, camera.groups[c], learned, K[0, 0], K[1, 1], K[0, 2], K[1, 2]))
            decisive = errors[1]
            if best_error < 0:
                best_error = decisive
            is_best = decisive < best_error
            best_error = min(best_error, decisive)
            save_checkpoint(args.save_path, {"epoch": epoch + 1, "state_dict": disp_net.state_dict()},
                            {"epoch": epoch + 1, "state_dict": pose_net.state_dict()}, is_best)
            if camera is not None:
                state = {"epoch": epoch + 1, "state_dict": camera.state_dict()}
                if camera.groups is not None:
                    state["groups"] = list(camera.groups)
                save_camera_checkpoint(args.save_path, state, is_best)
            with open(logs["summary"], "a") as f:
                csv.writer(f, delimiter="\t").writerow([train_loss, decisive])
        rng = gather_rng_states(world, device)
        if rank == 0:
            save_training_state(args.save_path, {
                "trainer": trainer.state_dict(), "epoch": epoch + 1, "n_iter": n_iter, "best_error": best_error, "args": vars(args),
                "log_rows": {k: log_rows(path) for k, path in logs.items()}, "world_size": world, "rng": rng})
    if world > 1:
        dist.destroy_process_group()


def train(args, train_loader, trainer, device, rank, world):
    """One epoch of train.py:235-299.  Returns the mean total loss of the logged iterations."""
    global n_iter
    trainer.disp_net.train()
    trainer.pose_net.train()
    end = time.time()
    shown, total, rows = 0.0, 0, []
    for i, batch in enumerate(train_loader):
        tgt_img, ref_imgs, intrinsics = batch[:3]
        tgt_img = tgt_img.to(device, non_blocking=True)
        ref_imgs = [img.to(device, non_blocking=True) for img in ref_imgs]
        intrinsics = intrinsics.to(device, non_blocking=True)
        inputs = dict(intrinsics=intrinsics) if trainer.camera is None else dict(aug=batch[4])    # a learned camera builds K itself
        if len(batch) > 5:
            inputs["camera_index"] = batch[5]        # a bank of cameras: each sample's
        if args.cuda_graph and world == 1 and trainer._graph is None:        # the first batch of the process
            trainer.capture(tgt_img, ref_imgs, **inputs)
            print("=> captured the training step in a CUDA graph ({} kernel launches per step)".format(trainer.launches_per_step))
        out = trainer.step(tgt_img, ref_imgs, **inputs)
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
def validate_without_gt(args, val_loader, disp_net, pose_net, device, camera=None):
    """train.py:302-362: eval-mode networks, the same losses, auto-mask forced off.  With a learned camera its K (the identity
    draw: the validation frames are not flipped, zoomed or cropped) replaces the dataset's.  With a bank of cameras only the
    samples of a training group (camera index >= 0) take their camera's K; the others keep the dataset's."""
    disp_net.eval()
    pose_net.eval()
    acc, n = torch.zeros(4, device=device), 0
    for batch in val_loader:
        tgt_img, ref_imgs, intrinsics = batch[:3]
        tgt_img = tgt_img.to(device)
        ref_imgs = [img.to(device) for img in ref_imgs]
        intrinsics = intrinsics.to(device)
        if camera is not None:
            from scsfm.camera import identity_records
            idx = batch[4] if len(batch) > 4 else None        # a bank's camera index
            K = camera(identity_records(tgt_img.shape[0], tgt_img.shape[-1], device), idx)
            # (an index of -1 builds a NaN K, which the where() drops)
            intrinsics = K if idx is None else torch.where((idx >= 0)[:, None, None], K, intrinsics)
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
