"""Drop-in for the reference's `loss_functions` module (reference loss_functions.py), H100 path.

`compute_photo_and_geometry_loss`, `compute_pairwise_loss` and `compute_smooth_loss` keep the
reference signatures and return zero-dim autograd-connected tensors, but each is ONE fused
sm_90a kernel forward and one backward (csrc/warp_loss.cu, csrc/smooth.cu) instead of ~180
ATen ops per pair.  GPU tensors only: there is no CPU fallback.
"""
import torch
from torch import nn

from inverse_warp import inverse_warp, inverse_warp2  # noqa: F401  (re-exported like the reference)
from scsfm import loss_ops as _ops

device = torch.device("cuda") if torch.cuda.is_available() else torch.device("cpu")


class SSIM(nn.Module):
    """Stand-alone SSIM dissimilarity map clamp((1-SSIM)/2, 0, 1) (reference loss_functions.py:11-42).

    The training path never calls this module: the 3x3 SSIM statistics are computed inside the fused
    pairwise kernel on shared-memory tiles.  It is kept for scripts that use it directly.
    """

    def __init__(self):
        super().__init__()
        self.C1 = 0.01 ** 2
        self.C2 = 0.03 ** 2

    @staticmethod
    def _mean3(t):
        return nn.functional.avg_pool2d(nn.functional.pad(t, (1, 1, 1, 1), mode="reflect"), 3, 1)

    def forward(self, x, y):
        mx, my = self._mean3(x), self._mean3(y)
        vx = self._mean3(x * x) - mx * mx
        vy = self._mean3(y * y) - my * my
        cxy = self._mean3(x * y) - mx * my
        num = (2 * mx * my + self.C1) * (2 * cxy + self.C2)
        den = (mx * mx + my * my + self.C1) * (vx + vy + self.C2)
        return torch.clamp((1 - num / den) / 2, 0, 1)


compute_ssim_loss = SSIM().to(device)


def compute_photo_and_geometry_loss(tgt_img, ref_imgs, intrinsics, tgt_depth, ref_depths, poses, poses_inv,
                                    max_scales, with_ssim, with_mask, with_auto_mask, padding_mode):
    """Photometric and geometry-consistency losses summed over references, scales and both warp
    directions (reference loss_functions.py:50-92); one kernel launch for all of them."""
    return _ops.photo_and_geometry_loss(tgt_img, ref_imgs, intrinsics, tgt_depth, ref_depths, poses, poses_inv,
                                        max_scales, with_ssim, with_mask, with_auto_mask, padding_mode)


def compute_pairwise_loss(tgt_img, ref_img, tgt_depth, ref_depth, pose, intrinsic, with_ssim, with_mask,
                          with_auto_mask, padding_mode):
    """(reconstruction_loss, geometry_consistency_loss) of one warp direction (reference :95-119)."""
    return _ops.pairwise_loss(tgt_img, ref_img, tgt_depth, ref_depth, pose, intrinsic, with_ssim, with_mask,
                              with_auto_mask, padding_mode)


def mean_on_mask(diff, valid_mask):
    """Masked mean over the whole batch, constant 0 when the expanded mask sums to <= 10000
    (reference :123-129).  Evaluated on the device: no host synchronisation for the branch."""
    mask = valid_mask.expand_as(diff)
    total = mask.sum()
    mean = (diff * mask).sum() / total.clamp(min=1)
    return torch.where(total > 10000, mean, torch.zeros_like(mean))


def compute_smooth_loss(tgt_depth, tgt_img, ref_depths, ref_imgs):
    """Edge-aware smoothness of the scale-0 depth of the target and every reference (reference :132-159)."""
    return _ops.smooth_loss(tgt_depth, tgt_img, ref_depths, ref_imgs)


@torch.no_grad()
def compute_errors(gt, pred, dataset):
    """Validation metrics [abs_diff, abs_rel, sq_rel, a1, a2, a3] with the Garg (KITTI) / NYU crop and
    per-image median scaling (reference :163-205).  One median-select + one metrics launch for the whole batch
    (csrc/eval_ops.cu); the only host synchronisation is the final read of the six numbers."""
    batch_size, h, w = gt.size()
    if dataset == "kitti":
        (ya, yb), (xa, xb), max_depth = (0.40810811, 0.99189189), (0.03594771, 0.96405229), 80
    elif dataset == "nyu":
        (ya, yb), (xa, xb), max_depth = (0.09375, 0.98125), (0.0640625, 0.9390625), 10
    else:
        raise ValueError("dataset must be 'kitti' or 'nyu'")
    per_image = _ops.compute_errors(gt, pred, int(ya * h), int(yb * h), int(xa * w), int(xb * w), float(max_depth))
    return (per_image[:, :6].double().sum(0) / batch_size).tolist()
