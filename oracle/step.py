"""Oracle: one optimisation step of the reference training loop (restates reference
train.py:249-282, 426-444).  TEST INFRASTRUCTURE -- see oracle/__init__.py.
"""
import torch

from . import losses


def compute_depth(disp_net, tgt_img, ref_imgs):
    """depth = 1/disparity for every scale of the target and each reference (train.py:426-434)."""
    tgt_depth = [1 / d for d in disp_net(tgt_img)]
    ref_depths = [[1 / d for d in disp_net(r)] for r in ref_imgs]
    return tgt_depth, ref_depths


def compute_pose_with_inv(pose_net, tgt_img, ref_imgs):
    """Forward and backward relative poses, two separate network calls per reference (train.py:437-444), in the reference's
    order (tgt,ref0), (ref0,tgt), (tgt,ref1), ...: each call moves the BatchNorm running statistics, so with two or more
    references the order shows in them."""
    poses, poses_inv = [], []
    for r in ref_imgs:
        poses.append(pose_net(tgt_img, r))
        poses_inv.append(pose_net(r, tgt_img))
    return poses, poses_inv


def make_optimizer(disp_net, pose_net, lr=1e-4, betas=(0.9, 0.999), weight_decay=0.0):
    """Adam over two parameter groups (train.py:171-178)."""
    return torch.optim.Adam([{"params": disp_net.parameters(), "lr": lr},
                             {"params": pose_net.parameters(), "lr": lr}], betas=betas, weight_decay=weight_decay)


def train_step(disp_net, pose_net, optimizer, tgt_img, ref_imgs, intrinsics, *, num_scales=1,
               with_ssim=1, with_mask=1, with_auto_mask=1, padding_mode="zeros", w1=1.0, w2=0.1, w3=0.5):
    """Forward, losses, backward, Adam (train.py:259-282).  Returns the four scalar losses (detached)."""
    tgt_depth, ref_depths = compute_depth(disp_net, tgt_img, ref_imgs)
    poses, poses_inv = compute_pose_with_inv(pose_net, tgt_img, ref_imgs)
    photo, geo = losses.compute_photo_and_geometry_loss(tgt_img, ref_imgs, intrinsics, tgt_depth, ref_depths,
                                                        poses, poses_inv, num_scales, with_ssim, with_mask,
                                                        with_auto_mask, padding_mode)
    smooth = losses.compute_smooth_loss(tgt_depth, tgt_img, ref_depths, ref_imgs)
    loss = w1 * photo + w2 * smooth + w3 * geo
    optimizer.zero_grad()
    loss.backward()
    optimizer.step()
    return loss.detach(), photo.detach(), smooth.detach(), geo.detach()
