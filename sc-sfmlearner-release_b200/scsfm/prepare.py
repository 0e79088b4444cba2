"""Training-set preparation: the reference's data/prepare_train_data.py and its three loaders (kitti_raw_loader.py,
kitti_odom_loader.py, cityscapes_loader.py), with the per-frame arithmetic on the device (csrc/prepare.cu).

The host crawls the dataset, parses calibration and OXTS records, selects frames, decodes PNGs and reads Velodyne .bin
files in a thread pool; batches of frames go to the device, where scsfm_resize_bilinear_u8 resizes them (Pillow BILINEAR,
what scipy.misc.imresize did, bit for bit) and scsfm_velo_depth projects the clouds into ground-truth depth maps
(generate_depth_map, bit for bit up to the last bit of the reference's BLAS projection); the pool then encodes and writes
the frames.  The files written are the reference's: <scene>/cam.txt (np.savetxt's default format, float64 for KITTI raw and
Cityscapes, float32 for odometry), <scene>/poses.txt (%.6e, 12 values a row), <scene>/<id>.jpg (Pillow's default JPEG
settings, as scipy.misc.imsave), <scene>/<id>.npy (float32 depth), then train.txt / val.txt.  Scene directories with fewer
than three frames are removed.  There is no CPU fallback: the device operations are `DeviceOps`.

Deviations, both documented in the command-line help: the KITTI raw test scenes come from a file the user names
(--test-scenes), and the validation split draws over the sorted scene prefixes, so it does not depend on PYTHONHASHSEED.
"""
import ctypes
import fnmatch
import json
import os
import shutil
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
from PIL import Image

from .inference_io import odom_intrinsics

MIN_SPEED = 2


# ----- calibration and poses --------------------------------------------------------------------------------------------------
def read_calib(path):
    """KITTI raw calibration text: every 'key: v v v' line whose values all parse as floats, as float64 arrays."""
    data = {}
    with open(path) as f:
        for line in f:
            if ":" not in line:
                continue
            key, value = line.split(":", 1)
            try:
                data[key] = np.array([float(x) for x in value.split()])
            except ValueError:
                pass
    return data


def rigid(R, t):
    """4 x 4 [R t; 0 0 0 1]."""
    return np.vstack((np.hstack([np.reshape(R, (3, 3)), np.reshape(t, (3, 1))]), [0, 0, 0, 1]))


def _rot(axis, a):
    c, s = np.cos(a), np.sin(a)
    if axis == 0:
        return np.array([[1, 0, 0], [0, c, -s], [0, s, c]])
    if axis == 1:
        return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])
    return np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]])


def oxts_pose(packet, scale):
    """SE(3) pose of one OXTS packet (lat, lon, alt, roll, pitch, yaw): Mercator translation with the first frame's scale,
    rotation Rz(yaw) Ry(pitch) Rx(roll)."""
    lat, lon, alt, roll, pitch, yaw = packet
    er = 6378137.
    ty = lat * np.pi * er / 180.
    tx = scale * lon * np.pi * er / 180.
    t = np.array([tx, ty, alt]).reshape(-1, 1)
    R = _rot(2, yaw).dot(_rot(1, pitch).dot(_rot(0, roll)))
    return rigid(R, t)


def p_velo2im(P_rect, cam2cam, velo2cam, ratio):
    """P_rect / ratio (rows 0 and 1) . R_rect_00 . Tr_velo_cam, with numpy's products in the reference's order."""
    P = np.copy(P_rect)
    P[0] /= ratio
    P[1] /= ratio
    R = np.eye(4)
    R[:3, :3] = cam2cam["R_rect_00"].reshape(3, 3)
    T = np.vstack((np.hstack((velo2cam["R"].reshape(3, 3), velo2cam["T"][..., np.newaxis])), np.array([0, 0, 0, 1.0])))
    return np.dot(np.dot(P, R), T)


def select_by_speed(speeds, min_speed=MIN_SPEED):
    """Indices kept by the cumulative-speed rule: add each frame's speed (a 3-vector, or a scalar broadcast over three
    components as Cityscapes' vehicle speed is) and keep the frame once the norm exceeds min_speed, then restart."""
    cum = np.zeros(3)
    keep = []
    for i, s in enumerate(speeds):
        cum += s
        if np.linalg.norm(cum) > min_speed:
            keep.append(i)
            cum *= 0
    return keep


def read_static_frames(path):
    """static_frames.txt: '<date> <drive> <frame>' lines -> {drive: set of 10-digit frame ids}."""
    out = {}
    with open(path) as f:
        for line in f:
            if line.strip():
                _, drive, frame = line.split(" ")
                out.setdefault(drive, set()).add("%.10d" % int(frame))
    return out


def _image_size(path):
    """(height, width) of a PNG without decoding it."""
    with Image.open(path) as im:
        return im.size[1], im.size[0]


def _dirs(path):
    return sorted(d for d in os.listdir(path) if os.path.isdir(os.path.join(path, d)))


class Frame:
    __slots__ = ("id", "img", "velo", "pose")

    def __init__(self, id, img, velo=None, pose=None):
        self.id, self.img, self.velo, self.pose = id, img, velo, pose


class Scene:
    """One output directory: rel_path, the intrinsics written to cam.txt, the selected frames, and for KITTI raw depth the
    frame-independent P_velo2im; crop_rows keeps the top rows after the resize (Cityscapes)."""

    def __init__(self, rel_path, intrinsics, frames, P=None, crop_rows=None):
        self.rel_path, self.intrinsics, self.frames, self.P, self.crop_rows = rel_path, intrinsics, frames, P, crop_rows


# ----- the three datasets -----------------------------------------------------------------------------------------------------
class KittiRaw:
    """KITTI raw: <root>/<date>/<drive>_sync/{image_02,image_03}/data/*.png, oxts/data/*.txt, velodyne_points/data/*.bin and
    <root>/<date>/calib_{cam_to_cam,velo_to_cam,imu_to_velo}.txt.  Every drive not named in the test scenes is a scene with
    one output directory per camera."""
    cam_ids = ("02", "03")
    dates = ("2011_09_26", "2011_09_28", "2011_09_29", "2011_09_30", "2011_10_03")

    def __init__(self, root, test_scenes_file, static_frames_file=None, img_height=128, img_width=416, get_depth=False,
                 get_pose=False, depth_size_ratio=1):
        self.root, self.h, self.w = root, img_height, img_width
        self.get_depth, self.get_pose, self.ratio = get_depth, get_pose, depth_size_ratio
        self.static = read_static_frames(static_frames_file) if static_frames_file is not None else None
        with open(test_scenes_file) as f:
            test = set(line.strip() for line in f)
        self.scenes = [os.path.join(root, date, d) for date in self.dates if os.path.isdir(os.path.join(root, date))
                       for d in _dirs(os.path.join(root, date)) if d[:-5] not in test]

    def collect(self, drive):
        calib_dir = os.path.dirname(drive)
        name = os.path.basename(drive)
        cam2cam = read_calib(os.path.join(calib_dir, "calib_cam_to_cam.txt"))
        velo2cam = read_calib(os.path.join(calib_dir, "calib_velo_to_cam.txt"))
        imu2velo = read_calib(os.path.join(calib_dir, "calib_imu_to_velo.txt"))
        imu2cam = rigid(cam2cam["R_rect_00"], np.zeros(3)) @ rigid(velo2cam["R"], velo2cam["T"]) @ rigid(imu2velo["R"], imu2velo["T"])
        oxts_dir = os.path.join(drive, "oxts", "data")
        oxts = sorted(f for f in os.listdir(oxts_dir) if f.endswith(".txt"))
        speeds, poses, scale, origin = [], [], None, None
        for f in oxts:
            m = np.genfromtxt(os.path.join(oxts_dir, f))
            speeds.append(m[8:11])
            if scale is None:
                scale = np.cos(m[0] * np.pi / 180.)
            pose = oxts_pose(m[:6], scale)
            if origin is None:
                origin = pose
            poses.append((imu2cam @ np.linalg.inv(origin) @ pose @ np.linalg.inv(imu2cam))[:3])
        ids = ["{:010d}".format(n) for n in range(len(oxts))]
        if self.static is None:
            keep = select_by_speed(speeds)
        else:
            static = self.static.get(name, ())
            keep = [i for i, fid in enumerate(ids) if fid not in static]
        scenes = []
        for c in self.cam_ids:
            img = lambda fid: os.path.join(drive, "image_" + c, "data", fid + ".png")   # noqa: E731
            if not ids or not os.path.isfile(img(ids[0])):
                return []
            h, w = _image_size(img(ids[0]))
            P_rect = np.reshape(cam2cam["P_rect_" + c], (3, 4))
            P_rect[0] *= self.w / w
            P_rect[1] *= self.h / h
            P = p_velo2im(P_rect, cam2cam, velo2cam, self.ratio) if self.get_depth else None
            frames = [Frame(ids[i], img(ids[i]),
                            os.path.join(drive, "velodyne_points", "data", ids[i] + ".bin") if self.get_depth else None,
                            poses[i] if self.get_pose else None) for i in keep]
            scenes.append(Scene(name + "_" + c, P_rect[:, :3], frames, P))
        return scenes


class KittiOdom:
    """KITTI odometry: <root>/sequences/<00..08>/{image_2,image_3}/*.png and calib.txt; every frame, no depth or pose."""
    cam_ids = ("2", "3")
    train_sets = ("00", "01", "02", "03", "04", "05", "06", "07", "08")

    def __init__(self, root, img_height=256, img_width=832):
        self.root, self.h, self.w = root, img_height, img_width
        seq = os.path.join(root, "sequences")
        self.scenes = [os.path.join(seq, d) for d in _dirs(seq) if d in self.train_sets]

    def collect(self, drive):
        scenes = []
        name = os.path.basename(drive)
        for c in self.cam_ids:
            img_dir = os.path.join(drive, "image_" + c)
            ids = sorted(f.split(".")[0] for f in os.listdir(img_dir))
            h, w = _image_size(os.path.join(img_dir, ids[0] + ".png"))
            K = odom_intrinsics(os.path.join(drive, "calib.txt"), c, (h, w), (self.h, self.w))
            scenes.append(Scene(name + "_" + c, K, [Frame(i, os.path.join(img_dir, i + ".png")) for i in ids]))
        return scenes


class Cityscapes:
    """Cityscapes: <root>/leftImg8bit_sequence/train/<city>/<city>_<scene>_<frame>_leftImg8bit.png, camera/train/<city>/
    *_camera.json, vehicle_sequence/train/<city>/*_vehicle.json.  Every run of consecutive frames of a scene gives two output
    directories, the even and the odd frames; frames are selected by speed and the bottom quarter is cropped after the
    resize (the car's bonnet)."""

    def __init__(self, root, split="train", img_height=171, img_width=416):
        self.root, self.split, self.h, self.w = root, split, img_height, img_width
        base = os.path.join(root, "leftImg8bit_sequence", split)
        self.scenes = [os.path.join(base, d) for d in _dirs(base)]

    def _intrinsics(self, city_dir, city, scene_id):
        cam_dir = os.path.join(self.root, "camera", self.split, city)
        cam_file = sorted(f for f in os.listdir(cam_dir) if fnmatch.fnmatch(f, "{}_{}_*_camera.json".format(city, scene_id)))[0]
        frame_id = cam_file.split("_")[2]
        with open(os.path.join(cam_dir, cam_file)) as f:
            c = json.load(f)["intrinsic"]
        K = np.array([[c["fx"], 0, c["u0"]], [0, c["fy"], c["v0"]], [0, 0, 1]])
        h, w = _image_size(os.path.join(city_dir, "{}_{}_{}_leftImg8bit.png".format(city, scene_id, frame_id)))
        K[0] *= self.w / w
        K[1] *= self.h / h
        return K

    def _speed(self, city, scene_id, frame_id):
        with open(os.path.join(self.root, "vehicle_sequence", self.split, city,
                               "{}_{}_{}_vehicle.json".format(city, scene_id, frame_id))) as f:
            return json.load(f)["speed"]

    def collect(self, city_dir):
        city = os.path.basename(city_dir)
        runs = {}
        for f in sorted(f for f in os.listdir(city_dir) if f.endswith(".png")):
            scene_id, frame_id = f.split("_")[1:3]
            r = runs.setdefault(scene_id, [])
            if not r or int(frame_id) - int(r[-1][-1]) > 1:
                r.append([])
            r[-1].append(frame_id)
        scenes = []
        for scene_id, subs in runs.items():
            K = self._intrinsics(city_dir, city, scene_id)
            for sub in subs:
                speeds = [self._speed(city, scene_id, fid) for fid in sub]
                for parity in (0, 1):
                    ids = sub[parity::2]
                    frames = [Frame(ids[i], os.path.join(city_dir, "{}_{}_{}_leftImg8bit.png".format(city, scene_id, ids[i])))
                              for i in select_by_speed(speeds[parity::2])]
                    scenes.append(Scene("{}_{}_{}_{}".format(city, scene_id, sub[0], parity), K, frames,
                                        crop_rows=int(self.h * 0.75)))
        return scenes


# ----- device operations ------------------------------------------------------------------------------------------------------
class DeviceOps:
    """The two kernels on lists of host arrays (results come back to the host for the writers)."""

    def __init__(self, device="cuda"):
        import torch
        if not torch.cuda.is_available():
            raise RuntimeError("data preparation needs a CUDA device: the H100 path has no CPU fallback")
        self.torch, self.device = torch, torch.device(device)
        from . import lib as L
        self.L = L
        lib = L.load()
        P, I, S = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t
        lib.scsfm_resize_bilinear_workspace_bytes.restype = S
        lib.scsfm_resize_bilinear_workspace_bytes.argtypes = [I, I, I, I, I]
        lib.scsfm_resize_bilinear_u8.argtypes = [P, I, I, I, I, I, P, P, S, P]
        lib.scsfm_velo_depth_workspace_bytes.restype = S
        lib.scsfm_velo_depth_workspace_bytes.argtypes = [I, I, I]
        lib.scsfm_velo_depth.argtypes = [P, P, P, P, I, I, I, P, P, S, P]
        self.lib = lib

    def resize_batch(self, frames, out_h, out_w):
        """frames: uint8 tensor [B,H,W,3] (host or device) -> device uint8 tensor [B,out_h,out_w,3]."""
        torch, L = self.torch, self.L
        x = torch.as_tensor(frames)
        if x.dtype != torch.uint8 or x.dim() != 4 or x.shape[-1] != 3:
            raise ValueError("resize_bilinear expects uint8 frames [B,H,W,3], got %s %s" % (x.dtype, tuple(x.shape)))
        B, H, W, _ = x.shape
        x = x.contiguous().to(self.device, non_blocking=True)
        out = torch.empty(B, out_h, out_w, 3, dtype=torch.uint8, device=self.device)
        nws = int(self.lib.scsfm_resize_bilinear_workspace_bytes(B, H, W, out_h, out_w))
        ws = torch.empty(max(nws, 16), dtype=torch.uint8, device=self.device)
        L.launch(self.lib.scsfm_resize_bilinear_u8, "scsfm_resize_bilinear_u8", "prepare", 4, 3.0 * B * (H * W + out_h * out_w),
                 L.ptr(x), B, H, W, out_h, out_w, L.ptr(out), L.ptr(ws), nws, L.stream())
        return out

    def resize(self, frames, out_h, out_w):
        """List of H x W x 3 uint8 arrays of any sizes -> list of out_h x out_w x 3 arrays; one launch per source size."""
        torch = self.torch
        out = [None] * len(frames)
        groups = {}
        for i, f in enumerate(frames):
            groups.setdefault(f.shape, []).append(i)
        for shape, idx in groups.items():
            batch = torch.from_numpy(np.stack([frames[i] for i in idx])).pin_memory()
            res = self.resize_batch(batch, out_h, out_w).cpu().numpy()
            for j, i in enumerate(idx):
                out[i] = res[j]
        return out

    def depth(self, clouds, Ps, Hd, Wd):
        """Clouds (N_b x 4 float32 arrays) with their 3 x 4 float64 P_velo2im -> list of Hd x Wd float32 depth maps."""
        torch, L = self.torch, self.L
        B = len(clouds)
        counts = [len(c) for c in clouds]
        offsets = np.zeros(B + 1, np.int64)
        offsets[1:] = np.cumsum(counts)
        pts = np.concatenate([np.asarray(c, np.float32).reshape(-1, 4) for c in clouds]) if offsets[-1] else np.zeros((1, 4), np.float32)
        d_pts = torch.from_numpy(pts).to(self.device)
        d_off = torch.from_numpy(offsets).to(self.device)
        d_P = torch.from_numpy(np.ascontiguousarray(np.stack(Ps), np.float64)).to(self.device)
        out = torch.empty(B, Hd, Wd, dtype=torch.float32, device=self.device)
        nws = int(self.lib.scsfm_velo_depth_workspace_bytes(B, Hd, Wd))
        ws = torch.empty(nws, dtype=torch.uint8, device=self.device)
        L.launch(self.lib.scsfm_velo_depth, "scsfm_velo_depth", "prepare", 3, 16.0 * int(offsets[-1]) + 20.0 * B * Hd * Wd,
                 L.ptr(d_pts), L.ptr(d_off), offsets.ctypes.data_as(ctypes.c_void_p), L.ptr(d_P), B, Hd, Wd, L.ptr(out), L.ptr(ws), nws,
                 L.stream())
        res = out.cpu().numpy()
        return [res[b] for b in range(B)]


# ----- the pipeline -----------------------------------------------------------------------------------------------------------
def decode(frame):
    """(H x W x 3 uint8 frame, N x 4 float32 cloud or None), on a pool thread."""
    with Image.open(frame.img) as im:
        img = np.asarray(im)
    if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 3:
        raise ValueError("%s: expected an 8-bit RGB image, got %s %s" % (frame.img, img.dtype, img.shape))
    velo = np.fromfile(frame.velo, dtype=np.float32).reshape(-1, 4) if frame.velo is not None else None
    return img, velo


def write(dump_dir, frame_id, img, depth):
    Image.fromarray(img).save(os.path.join(dump_dir, "{}.jpg".format(frame_id)))
    if depth is not None:
        np.save(os.path.join(dump_dir, "{}.npy".format(frame_id)), depth)


def dump(scenes, dump_root, height, width, depth_ratio, ops, num_threads=4, batch_size=64, stats=None):
    """Write every scene: cam.txt, the frames (and depth maps where the scene has P), poses.txt; then remove directories with
    fewer than 3 frames.  Frames are decoded and written on `num_threads` threads; `batch_size` frames at a time go through
    `ops` (DeviceOps).  stats, if a dict, receives the seconds spent waiting for decode, on the device and waiting for writes."""
    st = stats if stats is not None else {}
    for k in ("decode", "device", "encode", "frames"):
        st.setdefault(k, 0)
    Hd, Wd = height // depth_ratio, width // depth_ratio
    items = []
    for s in scenes:
        d = os.path.join(dump_root, s.rel_path)
        os.makedirs(d, exist_ok=True)
        np.savetxt(os.path.join(d, "cam.txt"), s.intrinsics)
        items += [(s, d, f) for f in s.frames]
    chunks = [items[i:i + batch_size] for i in range(0, len(items), batch_size)]
    writes = []
    with ThreadPoolExecutor(max(1, num_threads)) as pool:
        pending = [pool.submit(decode, f) for _, _, f in chunks[0]] if chunks else []
        for k, chunk in enumerate(chunks):
            t0 = time.perf_counter()
            decoded = [p.result() for p in pending]
            pending = [pool.submit(decode, f) for _, _, f in chunks[k + 1]] if k + 1 < len(chunks) else []
            t1 = time.perf_counter()
            imgs = ops.resize([img for img, _ in decoded], height, width)
            with_depth = [i for i, (s, _, _) in enumerate(chunk) if s.P is not None]
            depths = [None] * len(chunk)
            if with_depth:
                maps = ops.depth([decoded[i][1] for i in with_depth], [chunk[i][0].P for i in with_depth], Hd, Wd)
                for i, m in zip(with_depth, maps):
                    depths[i] = m
            st["device"] += time.perf_counter() - t1
            st["decode"] += t1 - t0
            for (s, d, f), img, dep in zip(chunk, imgs, depths):
                if s.crop_rows is not None:
                    img = np.ascontiguousarray(img[:s.crop_rows])
                writes.append(pool.submit(write, d, f.id, img, dep))
        t0 = time.perf_counter()
        for w in writes:
            w.result()
        st["encode"] += time.perf_counter() - t0
    st["frames"] += len(items)
    for s in scenes:
        d = os.path.join(dump_root, s.rel_path)
        poses = [f.pose.tolist() for f in s.frames if f.pose is not None]
        if poses:
            np.savetxt(os.path.join(d, "poses.txt"), np.array(poses).reshape(-1, 12), fmt="%.6e")
        if sum(1 for f in os.listdir(d) if f.endswith(".jpg")) < 3:
            shutil.rmtree(d)


def write_split(dump_root, remove_train_gt=False, seed=8964):
    """train.txt / val.txt: both cameras of a scene (directories sharing the name up to the last two characters) go to the
    same list; about 10 % of the prefixes, drawn in sorted order from np.random.seed(seed), go to validation.  With
    remove_train_gt the training scenes' .npy depth maps are deleted."""
    np.random.seed(seed)
    subdirs = _dirs(dump_root)
    prefixes = sorted(set(d[:-2] for d in subdirs))
    with open(os.path.join(dump_root, "train.txt"), "w") as tf, open(os.path.join(dump_root, "val.txt"), "w") as vf:
        for pr in prefixes:
            group = [d for d in subdirs if fnmatch.fnmatch(d, pr + "*")]
            if np.random.random() < 0.1:
                for s in group:
                    vf.write("{}\n".format(s))
            else:
                for s in group:
                    tf.write("{}\n".format(s))
                    if remove_train_gt:
                        for f in os.listdir(os.path.join(dump_root, s)):
                            if f.endswith(".npy"):
                                os.remove(os.path.join(dump_root, s, f))
