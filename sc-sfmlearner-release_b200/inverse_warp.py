"""Drop-in for the reference's `inverse_warp` module (reference inverse_warp.py), H100 path.

`inverse_warp2` and `pose_vec2mat` run hand-written sm_90a kernels from libscsfm
(csrc/warp_loss.cu) -- tensors must live on the GPU, there is no CPU fallback.  The small
geometric helpers that the training path no longer calls separately (they are fused inside
the loss kernel) are kept with the reference's names and argument meaning as thin device-side
torch expressions so that scripts importing them (test_pose.py:9, test_vo.py:10) keep working.
"""
import torch

from scsfm import lib as _L
from scsfm import loss_ops as _ops


def check_sizes(input, input_name, expected):
    """Same contract as reference inverse_warp.py:20-26: AssertionError naming the tensor."""
    ok = input.ndimension() == len(expected)
    for dim, sym in enumerate(expected):
        if ok and sym.isdigit():
            ok = input.size(dim) == int(sym)
    assert ok, "wrong size for {}, expected {}, got  {}".format(input_name, "x".join(expected), list(input.size()))


def _pixel_rays(b, h, w, like):
    ys, xs = torch.meshgrid(torch.arange(h, device=like.device, dtype=like.dtype),
                            torch.arange(w, device=like.device, dtype=like.dtype), indexing="ij")
    return torch.stack((xs, ys, torch.ones_like(xs)), 0).reshape(1, 3, h * w).expand(b, 3, h * w)


def pixel2cam(depth, intrinsics_inv):
    """[B,H,W] depth, [B,3,3] inverse intrinsics -> camera-frame points [B,3,H,W] (reference :29-44).
    No module-global grid cache: the call is re-entrant."""
    b, h, w = depth.size()
    return (intrinsics_inv @ _pixel_rays(b, h, w, depth)).reshape(b, 3, h, w) * depth.unsqueeze(1)


def _project(cam_coords, proj_c2p_rot, proj_c2p_tr):
    b, _, h, w = cam_coords.size()
    pts = cam_coords.reshape(b, 3, -1)
    if proj_c2p_rot is not None:
        pts = proj_c2p_rot @ pts
    if proj_c2p_tr is not None:
        pts = pts + proj_c2p_tr
    z = pts[:, 2].clamp(min=1e-3)
    xn = 2 * (pts[:, 0] / z) / (w - 1) - 1
    yn = 2 * (pts[:, 1] / z) / (h - 1) - 1
    return xn, yn, z


def cam2pixel(cam_coords, proj_c2p_rot, proj_c2p_tr, padding_mode):
    """Camera points -> [-1,1] sampling grid [B,H,W,2] (reference :47-74; padding_mode unused there too)."""
    b, _, h, w = cam_coords.size()
    xn, yn, _ = _project(cam_coords, proj_c2p_rot, proj_c2p_tr)
    return torch.stack([xn, yn], dim=2).reshape(b, h, w, 2)


def cam2pixel2(cam_coords, proj_c2p_rot, proj_c2p_tr, padding_mode):
    """As cam2pixel plus the clamped depth; 'zeros' rewrites out-of-range coordinates to 2 (reference :194-227)."""
    b, _, h, w = cam_coords.size()
    xn, yn, z = _project(cam_coords, proj_c2p_rot, proj_c2p_tr)
    if padding_mode == "zeros":
        xn = torch.where(((xn > 1) | (xn < -1)).detach(), torch.full_like(xn, 2.0), xn)
        yn = torch.where(((yn > 1) | (yn < -1)).detach(), torch.full_like(yn, 2.0), yn)
    return torch.stack([xn, yn], dim=2).reshape(b, h, w, 2), z.reshape(b, 1, h, w)


def euler2mat(angle):
    """[B,3] (rx,ry,rz) -> Rx.Ry.Rz [B,3,3] (reference :77-112), closed form of the product."""
    x, y, z = angle[:, 0], angle[:, 1], angle[:, 2]
    sx, cx, sy, cy, sz, cz = torch.sin(x), torch.cos(x), torch.sin(y), torch.cos(y), torch.sin(z), torch.cos(z)
    rows = [cy * cz, -cy * sz, sy,
            cx * sz + sx * sy * cz, cx * cz - sx * sy * sz, -sx * cy,
            sx * sz - cx * sy * cz, sx * cz + cx * sy * sz, cx * cy]
    return torch.stack(rows, dim=1).reshape(-1, 3, 3)


def quat2mat(quat):
    """[B,3] vector part, scalar part fixed to 1 then normalised -> rotation (reference :115-136)."""
    q = torch.cat([torch.ones_like(quat[:, :1]), quat], dim=1)
    q = q / q.norm(p=2, dim=1, keepdim=True)
    w, x, y, z = q.unbind(1)
    rows = [w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (w * y + x * z),
            2 * (w * z + x * y), w * w - x * x + y * y - z * z, 2 * (y * z - w * x),
            2 * (x * z - w * y), 2 * (w * x + y * z), w * w - x * x - y * y + z * z]
    return torch.stack(rows, dim=1).reshape(-1, 3, 3)


def pose_vec2mat(vec, rotation_mode="euler"):
    """(tx,ty,tz,rx,ry,rz) [B,6] -> [B,3,4] (reference :139-154).  CUDA kernel when no gradient is
    needed (test_pose.py / test_vo.py usage), differentiable device expression otherwise."""
    if vec.is_cuda and not (torch.is_grad_enabled() and vec.requires_grad):
        return _ops.pose_vec2mat(vec, rotation_mode)
    rot = euler2mat(vec[:, 3:]) if rotation_mode == "euler" else quat2mat(vec[:, 3:])
    return torch.cat([rot, vec[:, :3].unsqueeze(-1)], dim=2)


def inverse_warp2(img, depth, ref_depth, pose, intrinsics, padding_mode="zeros"):
    """Warp the source view into the target view (reference :230-269), one fused kernel.

    img [B,3,H,W], depth / ref_depth [B,1,H,W], pose [B,6], intrinsics [B,3,3] ->
    (projected_img, valid_mask, projected_depth, computed_depth).  Differentiable w.r.t.
    depth, ref_depth, pose and intrinsics through hand-written backward kernels.
    """
    check_sizes(img, "img", "B3HW")
    check_sizes(depth, "depth", "B1HW")
    check_sizes(ref_depth, "ref_depth", "B1HW")
    check_sizes(pose, "pose", "B6")
    check_sizes(intrinsics, "intrinsics", "B33")
    return _ops.InverseWarp2.apply(img, depth, ref_depth, pose, intrinsics, _ops._padding(padding_mode))


def inverse_warp(img, depth, pose, intrinsics, rotation_mode="euler", padding_mode="zeros"):
    """Legacy warp of SfMLearner (reference :157-191), unused by training: image only, boolean validity,
    no rewrite of out-of-range coordinates.  depth is [B,H,W]."""
    check_sizes(img, "img", "B3HW")
    check_sizes(depth, "depth", "BHW")
    check_sizes(pose, "pose", "B6")
    check_sizes(intrinsics, "intrinsics", "B33")
    if rotation_mode == "euler" and padding_mode == "border":
        d = depth.unsqueeze(1)
        warped, valid, _, _ = _ops.InverseWarp2.apply(img, d, d, pose, intrinsics, _L.PAD_BORDER)
        return warped, valid[:, 0] > 0.5
    cam = pixel2cam(depth, torch.linalg.inv(intrinsics))
    proj = intrinsics @ pose_vec2mat(pose, rotation_mode)
    grid = cam2pixel(cam, proj[:, :, :3], proj[:, :, -1:], padding_mode)
    warped = torch.nn.functional.grid_sample(img, grid, padding_mode=padding_mode, align_corners=False)
    return warped, grid.abs().max(dim=-1)[0] <= 1
