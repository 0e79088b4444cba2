"""Training-time image transforms on the GPU (csrc/augment.cu, include/scsfm.h: scsfm_augment_batch).

Replaces, for a whole batch, the per-sample chain the reference builds in train.py:88-101 and the dataset classes apply in
their __getitem__ (datasets/sequence_folders.py:59-62):

    custom_transforms.Compose([RandomHorizontalFlip(), RandomScaleCrop(), ArrayToTensor(), Normalize(mean, std)])    # train
    custom_transforms.Compose([ArrayToTensor(), Normalize(mean, std)])                                                # validation

The datasets are then built with transform=None (they return the decoded frames), the batch crosses PCIe as uint8 and one
kernel writes the normalised [B,3,H,W] float tensors.  The random numbers are drawn on the host, per sample, in the reference's
order (custom_transforms.py:52 random.random(); :71 np.random.uniform(1, 1.15, 2) -> x, y; :79-80 np.random.randint for the y
offset, then the x offset) and the intrinsics are updated with the reference's expressions, so equal RNG states give results
equal to the reference chain bit for bit (tests/test_augment_gpu.py).  There is no CPU fallback.
"""
import ctypes
import random

import numpy as np
import torch

from . import lib as L


class Draw:
    """The random draws of one sample: flip, zoom factors, crop offsets (offsets need the image size, hence the method)."""
    __slots__ = ("flip", "x_scaling", "y_scaling", "scaled_w", "scaled_h", "offset_x", "offset_y")

    def __init__(self, flip, x_scaling, y_scaling, scaled_w, scaled_h, offset_x, offset_y):
        self.flip, self.x_scaling, self.y_scaling = bool(flip), x_scaling, y_scaling
        self.scaled_w, self.scaled_h, self.offset_x, self.offset_y = int(scaled_w), int(scaled_h), int(offset_x), int(offset_y)

    @classmethod
    def random(cls, in_h, in_w):
        flip = random.random() < 0.5
        x_scaling, y_scaling = np.random.uniform(1, 1.15, 2)
        scaled_h, scaled_w = int(in_h * y_scaling), int(in_w * x_scaling)
        offset_y = np.random.randint(scaled_h - in_h + 1)
        offset_x = np.random.randint(scaled_w - in_w + 1)
        return cls(flip, x_scaling, y_scaling, scaled_w, scaled_h, offset_x, offset_y)

    @classmethod
    def identity(cls, in_h, in_w):
        return cls(False, 1.0, 1.0, in_w, in_h, 0, 0)

    @classmethod
    def given(cls, in_h, in_w, flip, x_scaling, y_scaling, offset_x, offset_y):
        return cls(flip, x_scaling, y_scaling, int(in_w * x_scaling), int(in_h * y_scaling), offset_x, offset_y)


def update_intrinsics(K, d, in_w):
    """The intrinsics side of RandomHorizontalFlip (custom_transforms.py:56-57) and RandomScaleCrop (:74-75, :83-84) for one
    3 x 3 numpy matrix; same expressions and order, so the result follows the installed numpy's casting rules like the reference's."""
    K = np.copy(K)
    if d.flip:
        K[0, 2] = in_w - K[0, 2]
    K[0] *= d.x_scaling
    K[1] *= d.y_scaling
    K[0, 2] -= d.offset_x
    K[1, 2] -= d.offset_y
    return K


class GpuAugment:
    """Callable on a batch: (images, intrinsics[, draws]) -> (list of [B,3,H,W] float32 CUDA tensors, [B,3,3] float32 CUDA tensor).

    images: uint8 tensor [n_img,B,H,W,3] (host, ideally pinned, or device) or a list of n_img [B,H,W,3] tensors; float tensors
    holding integer values 0..255 (what the reference's load_as_float returns) are accepted and converted on the host.
    train=True draws one Draw.random per sample unless `draws` is given; train=False is the validation chain.
    """

    def __init__(self, mean=(0.45, 0.45, 0.45), std=(0.225, 0.225, 0.225), train=True, device="cuda"):
        self.mean = (ctypes.c_float * 3)(*mean)
        self.std = (ctypes.c_float * 3)(*std)
        self.train = train
        self.device = torch.device(device)
        self._bound = False

    def _lib(self):
        lib = L.load()
        if not self._bound:
            P, I, LL = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong
            lib.scsfm_augment_workspace_ints.restype = LL
            lib.scsfm_augment_workspace_ints.argtypes = [I, I, I]
            lib.scsfm_augment_batch.argtypes = [P, P, I, I, I, I, P, P, P, P, LL, P]
            self._bound = True
        return lib

    def __call__(self, images, intrinsics, draws=None):
        if not torch.cuda.is_available():
            raise RuntimeError("GpuAugment needs a CUDA device: the H100 path has no CPU fallback")
        if isinstance(images, (list, tuple)):
            images = torch.stack([torch.as_tensor(im) for im in images])
        images = torch.as_tensor(images)
        if images.dim() != 5 or images.shape[-1] != 3:
            raise ValueError("GpuAugment expects images of shape [n_img,B,H,W,3], got %s" % (tuple(images.shape),))
        if images.dtype != torch.uint8:
            images = images.to(torch.uint8)               # integer-valued floats (load_as_float): exact
        n_img, B, H, W, _ = images.shape
        if draws is None:
            draws = [Draw.random(H, W) if self.train else Draw.identity(H, W) for _ in range(B)]
        if len(draws) != B:
            raise ValueError("GpuAugment: %d draws for a batch of %d" % (len(draws), B))
        for d in draws:
            if d.scaled_w < W or d.scaled_h < H or not (0 <= d.offset_x <= d.scaled_w - W) or not (0 <= d.offset_y <= d.scaled_h - H):
                raise ValueError("GpuAugment: zoomed size %dx%d / offset (%d, %d) do not contain a %dx%d crop"
                                 % (d.scaled_w, d.scaled_h, d.offset_x, d.offset_y, W, H))
        K = np.asarray(intrinsics.cpu() if torch.is_tensor(intrinsics) else intrinsics)
        if K.shape != (B, 3, 3):
            raise ValueError("GpuAugment expects intrinsics of shape [B,3,3], got %s" % (K.shape,))
        K_out = np.stack([update_intrinsics(K[b], draws[b], W) for b in range(B)]).astype(np.float32)
        params = torch.tensor([[int(d.flip), d.scaled_w, d.scaled_h, d.offset_x, d.offset_y] for d in draws], dtype=torch.int32)
        dev = self.device
        images = images.contiguous().to(dev, non_blocking=True)
        params = params.to(dev, non_blocking=True)
        lib = self._lib()
        nws = int(lib.scsfm_augment_workspace_ints(B, H, W))
        work = torch.empty(nws, dtype=torch.int32, device=dev)
        out = torch.empty(n_img, B, 3, H, W, dtype=torch.float32, device=dev)
        L.launch(lib.scsfm_augment_batch, "scsfm_augment_batch", "augment", 2, 15.0 * n_img * B * H * W, L.ptr(images), L.ptr(params), n_img, B,
                 H, W, ctypes.cast(self.mean, ctypes.c_void_p), ctypes.cast(self.std, ctypes.c_void_p), L.ptr(out), L.ptr(work), nws, L.stream())
        return [out[i] for i in range(n_img)], torch.from_numpy(K_out).to(dev, non_blocking=True)
