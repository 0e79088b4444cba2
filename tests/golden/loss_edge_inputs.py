"""Seeded inputs for the edge cases of the photometric / geometry loss backward (tests/test_loss_backward_edges_gpu.py) and
for the reference vectors that pin the oracle on them (make_golden_loss_edges.py, tests/test_loss_edges_cpu.py).

Pure torch on the CPU.  Unlike scsfm.synth (smoothed noise, |T - Iw| never above 1) the images are sharp: 8-pixel blocks
plus noise at the dataset normalisation (x - 0.45) / 0.225, with every reference the target's texture shifted a few pixels
plus its own noise, so that the L1 clamp saturates on a large share of the pixels as it does on real frames.  Every
sample has its own fx and cx.  Three motion levels:

  small   the synth pose scale;
  large   three times that: a clear share of the pixels leaves the frame;
  behind  the target depth holds a patch at depth 0.01 and the first pose is a pure translation with
          t_z = -0.01 + 5e-4, so the patch's points land at Zr = 5e-4 (behind the 1e-3 clamp of cam2pixel2).  t_x, t_y
          put a block of the patch inside the source image: with Z clamped to 1e-3 a patch pixel x projects to
          10 x + (fx t_x + cx t_z) / 1e-3, so about a tenth of the patch's width (and height) stays in view.
"""
import torch

from scsfm import synth

PATCH_DEPTH = 0.01
PATCH_ZR = 5e-4
SUB4 = (Ellipsis, slice(None, None, 4), slice(None, None, 4))     # loss_edges.npz keeps every fourth row and column of a map
# settings of loss_edges.npz -- name: (seed, B, H, W, n_ref, n_scales, motion, (ssim, mask, auto_mask), padding)
GOLDEN_SETTINGS = {
    "sharp_111_zeros": (21, 2, 128, 256, 2, 1, "small", (1, 1, 1), "zeros"),
    "sharp_000_border": (22, 2, 128, 256, 1, 2, "small", (0, 0, 0), "border"),
    "large_110_zeros": (23, 2, 128, 256, 1, 1, "large", (1, 1, 0), "zeros"),
    "behind_110_zeros": (24, 2, 128, 256, 1, 1, "behind", (1, 1, 0), "zeros"),
}


def sharp_images(gen, B, H, W, n_ref, block=8, noise=0.03):
    """Target and references: piecewise-constant texture in [0, 1] plus noise, normalised like the dataset."""
    pad = 4
    ny, nx = -(-(H + 2 * pad) // block), -(-(W + 2 * pad) // block)
    base = torch.rand(B, 3, ny, nx, generator=gen).repeat_interleave(block, 2).repeat_interleave(block, 3)

    def view(dy, dx):
        v = base[..., pad + dy:pad + dy + H, pad + dx:pad + dx + W]
        return ((v + noise * torch.randn(v.shape, generator=gen) - 0.45) / 0.225).contiguous()
    shifts = [(1, 2), (-1, -2), (0, 3)]
    return view(0, 0), [view(*shifts[i % 3]) for i in range(n_ref)]


def per_sample_intrinsics(gen, B, H, W):
    """synth.intrinsics with fx scaled by U(0.85, 1.15) and cx by U(0.9, 1.1) per sample."""
    K = synth.intrinsics(B, H, W).clone()
    K[:, 0, 0] *= 0.85 + 0.3 * torch.rand(B, generator=gen)
    K[:, 0, 2] *= 0.9 + 0.2 * torch.rand(B, generator=gen)
    return K.contiguous()


def behind_camera_pose(K, H, W):
    """Pure translation that puts the patch's points at Zr = PATCH_ZR and its block that stays in view near the image centre."""
    B = K.shape[0]
    tz = PATCH_ZR - PATCH_DEPTH
    r0, c0 = patch_origin(H, W)
    # pixel (r0, c0) of the patch lands at (1, 1) of the source image
    fx, cx, fy, cy = K[:, 0, 0], K[:, 0, 2], K[:, 1, 1], K[:, 1, 2]
    tx = ((1.0 - c0 * PATCH_DEPTH / 1e-3) * 1e-3 - cx * tz) / fx
    ty = ((1.0 - r0 * PATCH_DEPTH / 1e-3) * 1e-3 - cy * tz) / fy
    pose = torch.zeros(B, 6)
    pose[:, 0], pose[:, 1], pose[:, 2] = tx, ty, tz
    return pose


def patch_origin(H, W):
    return H // 3, W // 3


def loss_inputs(seed, B, H, W, n_ref=1, n_scales=1, motion="small", block=8, ref_depth_shifts=None):
    """(tgt_img, ref_imgs, intrinsics, tgt_depth[s], ref_depths[i][s], poses[i], poses_inv[i]) in the reference's
    conventions.  Depth scale s is H >> s by W >> s; ref_depth_shifts[s] overrides it for the reference depths (the
    loss upsamples every level to the image size, so the two sides of a pair may differ in resolution)."""
    g = torch.Generator().manual_seed(seed)
    tgt, refs = sharp_images(g, B, H, W, n_ref, block)
    K = per_sample_intrinsics(g, B, H, W)
    rsh = list(range(n_scales)) if ref_depth_shifts is None else list(ref_depth_shifts)
    tgt_depth = [synth.depth_map(g, B, H >> s, W >> s) for s in range(n_scales)]
    ref_depths = [[synth.depth_map(g, B, H >> s, W >> s) for s in rsh] for _ in range(n_ref)]
    scale = {"small": 1.0, "large": 3.0, "behind": 1.0}[motion]
    poses = [synth.pose(g, B) * scale for _ in range(n_ref)]
    poses_inv = [synth.pose(g, B) * scale for _ in range(n_ref)]
    if motion == "behind":
        r0, c0 = patch_origin(H, W)
        tgt_depth[0][:, :, r0:r0 + H // 10 + 2, c0:c0 + W // 10 + 2] = PATCH_DEPTH
        poses[0] = behind_camera_pose(K, H, W)
    return tgt, refs, K, tgt_depth, ref_depths, poses, poses_inv


def golden_setting(name):
    """(inputs, n_scales, flags, padding) of one setting of loss_edges.npz."""
    seed, B, H, W, n_ref, n_scales, motion, flags, pm = GOLDEN_SETTINGS[name]
    return loss_inputs(seed, B, H, W, n_ref, n_scales, motion), n_scales, flags, pm


def checksums(inputs):
    """sum |x| in float64 of every input tensor, in a fixed order: pins the inputs behind a stored fixture."""
    tgt, refs, K, td, rd, ps, pi = inputs
    return [float(x.double().abs().sum()) for x in [tgt, *refs, K, *td, *[x for r in rd for x in r], *ps, *pi]]
