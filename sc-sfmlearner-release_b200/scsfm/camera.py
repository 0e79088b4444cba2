"""Learned cameras for self-calibration under the training transforms (csrc/camera.cu, include/scsfm.h: scsfm_camera_*).

A camera theta = (fx, fy, cx, cy) is in pixels at the training resolution (what cam.txt holds after preparation).  With the GPU
transforms every sample is flipped, zoomed and cropped (custom_transforms.py:46-89), so the intrinsics the losses see are one per
sample: K_b = aug_b(theta).  `records()` turns the random draws of a batch into device records; `LearnedCamera(records)` builds
the batch's K with the augmentation's own arithmetic and back-propagates into theta in one small deterministic kernel.  The K it
returns feeds the loss entry points unchanged (their intrinsics gradient supplies dK).

A dataset recorded with several cameras (KITTI raw: one calibration per recording day; Cityscapes: one per sequence; uncalibrated
video: one per clip) learns a bank of cameras instead: `LearnedCamera.bank(thetas [C,4], ...)` holds theta [C,4], and
`forward(aug, index)` gives sample b the view of camera index[b] through its own record.  One camera is the same kernels' bank of
one with a null index.
"""
import ctypes

import numpy as np
import torch

from . import lib as L

AUG_DOUBLES = 6          # SCSFM_CAMERA_AUG_DOUBLES: x_scale, y_scale, flip, offset_x, offset_y, in_w

_bound = False


def _lib():
    global _bound
    lib = L.load()
    if not _bound:
        P, I = ctypes.c_void_p, ctypes.c_int
        lib.scsfm_camera_build_indexed.argtypes = [P, I, P, P, I, P, P]
        lib.scsfm_camera_grad_indexed.argtypes = [P, P, P, I, I, P, P]
        _bound = True
    return lib


def _numpy_factor(scale):
    """The value update_intrinsics' `K[0] *= scale` multiplies a float32 row by under the installed numpy's casting rules: a
    float64 draw (np.random.uniform) promotes the product to float64, a Python float stays float32 (NumPy 2)."""
    row = np.ones(1, np.float32)
    return float(np.float32(scale)) if (row * scale).dtype == np.float32 else float(scale)


def record_rows(draws, in_w):
    """float64 numpy [B, AUG_DOUBLES]: one record per augment.Draw of a batch whose input images are in_w pixels wide."""
    return np.array([[_numpy_factor(d.x_scaling), _numpy_factor(d.y_scaling), float(bool(d.flip)), int(d.offset_x), int(d.offset_y),
                      int(in_w)] for d in draws], np.float64).reshape(len(draws), AUG_DOUBLES)


def records(draws, in_w, device="cuda"):
    """Device tensor float64 [B, AUG_DOUBLES] of the draws (the layout scsfm_camera_build reads)."""
    return torch.from_numpy(record_rows(draws, in_w)).to(device, non_blocking=True)


def identity_records(B, in_w, device="cuda"):
    """Records of the validation chain (no flip, zoom or crop): K_b = theta for every sample."""
    r = torch.zeros(B, AUG_DOUBLES, dtype=torch.float64)
    r[:, 0] = r[:, 1] = 1.0
    r[:, 5] = in_w
    return r.to(device)


class _DeviceError(TypeError, RuntimeError):
    """A camera input on the wrong device: a RuntimeError as torch reports device mismatches, and a TypeError as the Trainer
    reports its malformed step inputs."""


def _check_theta(theta):
    if not theta.is_cuda:
        raise _DeviceError("the learned camera runs on the GPU: theta must be a CUDA tensor (move the camera to the GPU first; "
                           "there is no CPU fallback)")
    if theta.dtype != torch.float32 or not (theta.shape == (4,) or (theta.dim() == 2 and theta.shape[1] == 4 and theta.shape[0] >= 1)):
        raise TypeError("theta must be float32 [4] (fx, fy, cx, cy) or [C,4] (a bank of C cameras), got %s %s"
                        % (theta.dtype, tuple(theta.shape)))


def _check(theta, aug, index=None, B=None):
    """Types, shapes and devices of a call, checked before any launch: records float64 [B, AUG_DOUBLES] on the GPU; theta [4]
    takes no index, theta [C,4] requires one, int32 or int64 [B] on theta's device.  B is the batch size (the records' own by
    default)."""
    _check_theta(theta)
    if not aug.is_cuda:
        raise _DeviceError("the learned camera runs on the GPU: the augmentation records must be a CUDA tensor (there is no CPU "
                           "fallback)")
    B = len(aug) if B is None else B
    if aug.dtype != torch.float64 or tuple(aug.shape) != (B, AUG_DOUBLES) or B < 1:
        raise TypeError("augmentation records must be float64 [%d, %d] (scsfm.camera.records), got %s %s"
                        % (B, AUG_DOUBLES, aug.dtype, tuple(aug.shape)))
    if theta.dim() == 1:
        if index is not None:
            raise TypeError("a camera index is for a bank of cameras (theta [C,4]); this is one camera, theta [4]")
        return
    if index is None:
        raise TypeError("a bank of %d cameras needs the camera index of every sample (int32 or int64 [%d] CUDA tensor)"
                        % (theta.shape[0], B))
    if not isinstance(index, torch.Tensor) or index.dtype not in (torch.int32, torch.int64) or tuple(index.shape) != (B,):
        raise TypeError("camera index must be an int32 or int64 CUDA tensor [%d], got %s" % (
            B, "%s %s" % (index.dtype, tuple(index.shape)) if isinstance(index, torch.Tensor) else type(index).__name__))
    if index.device != theta.device:
        raise _DeviceError("camera index must be an int32 or int64 CUDA tensor on the camera's device %s, got %s"
                           % (theta.device, index.device))


def _index32(index):
    return None if index is None else index.to(torch.int32).contiguous()


def build(theta, aug, index=None):
    """K [B,3,3] float32 of theta through every record (no autograd).  theta [C,4] with index [B]: sample b sees camera index[b]
    (an index outside [0, C) gives a NaN K)."""
    _check(theta, aug, index)
    theta, aug, index = theta.detach().contiguous(), aug.contiguous(), _index32(index)
    K = torch.empty(aug.shape[0], 3, 3, device=theta.device, dtype=torch.float32)
    L.launch(_lib().scsfm_camera_build_indexed, "scsfm_camera_build_indexed", "camera", 1, 0.0, L.ptr(theta), theta.numel() // 4,
             L.ptr(aug), L.ptr(index), aug.shape[0], L.ptr(K), L.stream())
    return K


def grad(aug, dK, dtheta, index=None):
    """dtheta [4] (or [C,4] with index [B]) += d(loss)/dtheta given dK = d(loss)/dK [B,3,3]."""
    if dK.dtype != torch.float32 or tuple(dK.shape) != (aug.shape[0], 3, 3):
        raise TypeError("dK must be float32 [%d,3,3], got %s %s" % (aug.shape[0], dK.dtype, tuple(dK.shape)))
    _check(dtheta, aug, index)
    if not dtheta.is_contiguous():
        raise TypeError("dtheta must be contiguous (the gradient is added in place)")
    dK, index = dK.contiguous(), _index32(index)
    L.launch(_lib().scsfm_camera_grad_indexed, "scsfm_camera_grad_indexed", "camera", 1, 0.0, L.ptr(aug), L.ptr(index), L.ptr(dK),
             aug.shape[0], dtheta.numel() // 4, L.ptr(dtheta), L.stream())
    return dtheta


class CameraBuild(torch.autograd.Function):
    """apply(theta [4] or [C,4], aug [B, AUG_DOUBLES], index None or [B]) -> K [B,3,3]; the backward is scsfm_camera_grad_indexed."""

    @staticmethod
    def forward(ctx, theta, aug, index=None):
        _check(theta, aug, index)
        index = _index32(index)
        ctx.save_for_backward(aug, index)
        ctx.theta_shape = tuple(theta.shape)
        return build(theta, aug, index)

    @staticmethod
    def backward(ctx, dK):
        aug, index = ctx.saved_tensors
        dtheta = torch.zeros(ctx.theta_shape, device=dK.device, dtype=torch.float32)
        return grad(aug, dK.to(torch.float32), dtheta, index), None, None


class LearnedCamera(torch.nn.Module):
    """One pinhole camera, theta = (fx, fy, cx, cy) float32 in pixels at the training resolution height x width, or a bank of C
    cameras (LearnedCamera.bank), theta [C,4] with one label per camera in `groups`.
    forward(aug) -> K [B,3,3] of every sample's view through its augmentation record, differentiable in theta; a bank takes
    forward(aug, index) with index [B] (int32 or int64 CUDA): sample b sees camera index[b].
    state_dict: {'theta', 'height', 'width'}."""

    def __init__(self, fx, fy, cx, cy, height=0, width=0):
        super().__init__()
        self.theta = torch.nn.Parameter(torch.tensor([fx, fy, cx, cy], dtype=torch.float32))
        self.register_buffer("height", torch.tensor(int(height), dtype=torch.int64))
        self.register_buffer("width", torch.tensor(int(width), dtype=torch.int64))
        self.groups = None

    @classmethod
    def bank(cls, thetas, height=0, width=0, groups=None):
        """C cameras: thetas [C,4] (fx, fy, cx, cy per row); groups: C labels (what each camera stands for, e.g. its cam.txt)."""
        thetas = torch.as_tensor(thetas, dtype=torch.float32)
        if thetas.dim() != 2 or thetas.shape[1] != 4 or thetas.shape[0] < 1:
            raise TypeError("a camera bank takes thetas [C,4] with C >= 1, got %s" % (tuple(thetas.shape),))
        groups = ["camera %d" % c for c in range(thetas.shape[0])] if groups is None else [str(g) for g in groups]
        if len(groups) != thetas.shape[0]:
            raise ValueError("%d group labels for %d cameras" % (len(groups), thetas.shape[0]))
        cam = cls(0.0, 0.0, 0.0, 0.0, height, width)
        cam.theta = torch.nn.Parameter(thetas.clone())
        cam.groups = groups
        return cam

    def forward(self, aug, index=None):
        return CameraBuild.apply(self.theta, aug, index)

    def extra_repr(self):
        rows = self.theta.detach().cpu().reshape(-1, 4).tolist()
        return "; ".join("fx, fy, cx, cy = %s" % ", ".join("%.3f" % v for v in r) for r in rows) + \
            " at %dx%d" % (int(self.height), int(self.width))
