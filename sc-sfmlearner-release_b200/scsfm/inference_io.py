"""Host side of the inference scripts (run_inference.py, test_disp.py, test_vo.py): image decoding, the network input on the
device, output naming, the colour maps of the reference's visualisation and the visual-odometry integration.

Images are decoded with PIL.  A frame that is not at network size is resized with Pillow BILINEAR on the uint8 frame -- a
documented deviation from the reference's skimage / scipy resize, which is not part of the parity contract.  The uint8
frames go to the device and are normalised by the validation chain of GpuAugment (identity draw): for frames already at
network size the network input is bit-identical to the reference's (img / 255 - 0.45) / 0.225.
"""
import os

import numpy as np
import torch


def load_frame(path, height, width, resize=True):
    """uint8 [H,W,3] of an image file; resized to height x width (Pillow BILINEAR) unless it has that size or resize=False."""
    from PIL import Image
    im = Image.open(path).convert("RGB")
    if resize and (im.height != height or im.width != width):
        im = im.resize((width, height), Image.BILINEAR)
    return np.asarray(im, dtype=np.uint8)


def network_input(frames, device="cuda"):
    """uint8 frames [B,H,W,3] (numpy or torch) -> the normalised network input [B,3,H,W] float32 on the device."""
    from .augment import GpuAugment
    fr = torch.as_tensor(np.ascontiguousarray(frames))
    B = fr.shape[0]
    out, _ = GpuAugment(train=False, device=device)(fr.unsqueeze(0), np.tile(np.eye(3, dtype=np.float32), (B, 1, 1)))
    return out[0]


def list_images(directory, exts):
    """Files of `directory` with one of the extensions, in the reference's order (one glob per extension, in order)."""
    out = []
    for ext in exts:
        out += sorted(os.path.join(directory, f) for f in os.listdir(directory) if f.endswith("." + ext) and
                      os.path.isfile(os.path.join(directory, f)))
    return out


def output_name(path, dataset_dir, suffix):
    """run_inference's file name: the path relative to dataset_dir with its parts joined by '-', then suffix + extension."""
    rel, ext = os.path.splitext(os.path.relpath(path, dataset_dir))
    parts = [p for p in rel.split(os.sep) if p not in ("", ".")]
    return "{}{}{}".format("-".join(parts), suffix, ext)


# --- colour maps (visualisation only) ----------------------------------------------------------------------------------
# opencv_rainbow: the reference's five control points (utils.py); bone: matplotlib's published segment data.
_RAINBOW = ((0.000, (1.00, 0.00, 0.00)), (0.400, (1.00, 1.00, 0.00)), (0.600, (0.00, 1.00, 0.00)), (0.800, (0.00, 0.00, 1.00)),
            (1.000, (0.60, 0.00, 1.00)))
_BONE = {"red": ((0.0, 0.0), (0.746032, 0.652778), (1.0, 1.0)),
         "green": ((0.0, 0.0), (0.365079, 0.319444), (0.746032, 0.777778), (1.0, 1.0)),
         "blue": ((0.0, 0.0), (0.365079, 0.444444), (1.0, 1.0))}


def _lut(name):
    """(N, 4) RGBA lookup table with the resolution the reference's COLORMAPS use (rainbow 1000, bone 10000)."""
    if name == "rainbow":
        n = 1000
        xs = [p for p, _ in _RAINBOW]
        ch = [[c[i] for _, c in _RAINBOW] for i in range(3)]
        x = np.linspace(0, 1, n)
        rgb = [np.interp(x, xs, c) for c in ch]
    elif name == "bone":
        n = 10000
        x = np.linspace(0, 1, n)
        rgb = [np.interp(x, [p for p, _ in _BONE[k]], [v for _, v in _BONE[k]]) for k in ("red", "green", "blue")]
    else:
        raise ValueError("colour map must be 'rainbow' or 'bone', got %r" % (name,))
    return np.stack(rgb + [np.ones(n)], axis=1)


_LUTS = {}


def colorize(values, max_value, name):
    """tensor2array of the reference for a single-channel map: RGBA float32 [H,W,4] of values / max_value through the colour
    map (below 0: the first colour, 1 and above: the last one, as a matplotlib colormap call)."""
    lut = _LUTS.get(name)
    if lut is None:
        lut = _LUTS[name] = _lut(name)
    n = lut.shape[0]
    x = np.asarray(values, dtype=np.float64) / float(max_value) * n
    x[x == n] = n - 1
    idx = np.clip(np.floor(np.nan_to_num(x, nan=-1.0)), 0, n - 1).astype(np.int64)
    return lut[idx].astype(np.float32)


def save_png_like(path, rgba):
    """(255 * rgba).astype(uint8) written with PIL in the format of the file extension (RGBA as the reference writes it)."""
    from PIL import Image
    Image.fromarray((255 * rgba).astype(np.uint8), mode="RGBA").save(path)


# --- visual odometry ---------------------------------------------------------------------------------------------------
def integrate(pose_mats):
    """The reference test_vo.py loop on the host in float64: global_pose = global_pose @ inv([pose_mat; 0 0 0 1]) per
    consecutive pair, in order.  pose_mats [N-1,3,4] -> [N,12] rows of global_pose[0:3, :] (the first row is the identity)."""
    global_pose = np.eye(4)
    poses = [global_pose[0:3, :].reshape(1, 12)]
    for m in pose_mats:
        pose_mat = np.vstack([m, np.array([0, 0, 0, 1])])
        global_pose = global_pose @ np.linalg.inv(pose_mat)
        poses.append(global_pose[0:3, :].reshape(1, 12))
    return np.concatenate(poses, axis=0)


def batches(n, batch_size):
    return [(i, min(n, i + batch_size)) for i in range(0, n, batch_size)]


# --- pose evaluation (test_pose.py) ------------------------------------------------------------------------------------
def kitti_sequences(dataset_dir, patterns):
    """Names of the directories under <dataset_dir>/sequences matching any of the fnmatch patterns, SORTED (the reference
    visits a set, whose order changes from process to process)."""
    import fnmatch
    root = os.path.join(dataset_dir, "sequences")
    return sorted({d for d in os.listdir(root) if os.path.isdir(os.path.join(root, d)) and any(fnmatch.fnmatch(d, p) for p in patterns)})


def read_poses(path):
    """KITTI odometry ground truth: one 3x4 matrix per line, 12 numbers -> float64 [N,3,4]."""
    return np.genfromtxt(path).astype(np.float64).reshape(-1, 3, 4)


def odom_intrinsics(calib_path, cam, src_hw, dst_hw):
    """K [3,3] float32 of camera `cam` (2 or 3: line P<cam> of a KITTI odometry calib.txt) for frames of size src_hw = (h, w)
    resized to dst_hw: row 0 scaled by dst_w / w and row 1 by dst_h / h, in float32 (what the odometry training set's cam.txt
    holds)."""
    with open(calib_path) as f:
        line = f.readlines()[int(cam)]
    K = np.array(line.split()[1:]).reshape(3, 4).astype(np.float32)[0:3, 0:3]
    K[0, :] *= dst_hw[1] / src_hw[1]
    K[1, :] *= dst_hw[0] / src_hw[0]
    return K


# --- meshes ------------------------------------------------------------------------------------------------------------
def write_ply(path, verts, faces, colors):
    """Binary little-endian PLY: vertices float32 x y z with uint8 red green blue, faces as a uchar count and int32 indices."""
    verts = np.ascontiguousarray(verts, dtype="<f4").reshape(-1, 3)
    colors = np.ascontiguousarray(colors, dtype=np.uint8).reshape(-1, 3)
    faces = np.asarray(faces).reshape(-1, 3)
    if len(colors) != len(verts):
        raise ValueError("%d colours for %d vertices" % (len(colors), len(verts)))
    if len(faces) and (faces.min() < 0 or faces.max() >= len(verts) or len(verts) > 2 ** 31 - 1):
        raise ValueError("face indices must lie in [0, %d) and fit int32" % len(verts))
    vrec = np.empty(len(verts), dtype=[("p", "<f4", 3), ("c", "u1", 3)])
    vrec["p"], vrec["c"] = verts, colors
    frec = np.empty(len(faces), dtype=[("n", "u1"), ("i", "<i4", 3)])
    frec["n"], frec["i"] = 3, faces
    header = ("ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\n"
              "property uchar red\nproperty uchar green\nproperty uchar blue\nelement face %d\n"
              "property list uchar int vertex_indices\nend_header\n" % (len(verts), len(faces)))
    with open(path, "wb") as f:
        f.write(header.encode("ascii"))
        f.write(vrec.tobytes())
        f.write(frec.tobytes())


def read_ply(path):
    """(verts float32 [V,3], faces int64 [F,3], colors uint8 [V,3]) of a PLY written by write_ply."""
    with open(path, "rb") as f:
        data = f.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    counts = {}
    for line in data[:end].decode("ascii").splitlines():
        p = line.split()
        if p[:1] == ["element"]:
            counts[p[1]] = int(p[2])
    nv, nf = counts["vertex"], counts["face"]
    v = np.frombuffer(data, dtype=[("p", "<f4", 3), ("c", "u1", 3)], count=nv, offset=end)
    fr = np.frombuffer(data, dtype=[("n", "u1"), ("i", "<i4", 3)], count=nf, offset=end + v.nbytes)
    if nf and not np.all(fr["n"] == 3):
        raise ValueError("%s: only triangle faces are read" % path)
    return v["p"].copy(), fr["i"].astype(np.int64), v["c"].copy()


def snippet_indices(n_imgs, seq_length=5):
    """[n_snippets, seq_length] frame indices: every target frame with (seq_length - 1) // 2 frames on each side."""
    demi = (seq_length - 1) // 2
    return np.arange(-demi, demi + 1).reshape(1, -1) + np.arange(demi, n_imgs - demi).reshape(-1, 1)


def compensated_poses(poses, idx):
    """Ground-truth poses [len(idx),3,4] of a snippet relative to its first frame: translations minus the first one, then
    inv(R_first) @ pose."""
    p = np.stack([poses[i] for i in idx])
    t0 = p[0, :, -1].copy()
    p[:, :, -1] -= t0
    return np.linalg.inv(p[0, :, :3]) @ p


def pose_error(gt, pred):
    """(ATE, RE) of one snippet [L,3,4]: ATE = |t_gt - s t_pred| / L with the least-squares scale s of the translations;
    RE = mean angle of gt_R @ inv(pred_R) (arctan2 of twice its sine and cosine)."""
    t_gt, t_pred = gt[:, :, -1], pred[:, :, -1]
    scale = np.sum(t_gt * t_pred) / np.sum(t_pred ** 2)
    ate = np.linalg.norm((t_gt - scale * t_pred).reshape(-1))
    re = 0
    for g, p in zip(gt, pred):
        R = g[:, :3] @ np.linalg.inv(p[:, :3])
        s = np.linalg.norm([R[0, 1] - R[1, 0], R[1, 2] - R[2, 1], R[0, 2] - R[2, 0]])
        re += np.arctan2(s, np.trace(R) - 1)
    return ate / gt.shape[0], re / gt.shape[0]
