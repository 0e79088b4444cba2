"""Training-set preparation throughput (data/prepare_train_data.py), one JSON line with the card's name and power limit.

  resize   frames/s of scsfm_resize_bilinear_u8 on --frames 375x1242 frames -> 256x832 (kernel time from CUDA events, and the
           whole call from host memory including both copies), against Pillow's BILINEAR resize on one host thread.
  depth    depth maps/s of scsfm_velo_depth on --clouds 120k-point clouds -> 256x832 (kernel time, and the whole call from host
           memory), against the numpy oracle (oracle/prepare.py) and the reference's duplicate loop (Counter over the sub2ind
           keys, then one np.where over all points per duplicated key), both on one host thread.
  e2e      data/prepare_train_data.py on a synthetic KITTI raw drive of --e2e-frames 1242x375 frames per camera with 120k-point
           clouds (--with-depth --with-pose, 256x832): frames/s end to end (JPEG files written), and the seconds spent waiting
           for PNG decode, on the device and waiting for the JPEG writes, in --num-threads host threads.

    python tools/bench_prepare.py [--frames 64] [--clouds 32] [--e2e-frames 60] [--num-threads 8]
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time
from collections import Counter

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "sc-sfmlearner-release_b200"), os.path.join(ROOT, "sc-sfmlearner-release_b200", "data"),
          os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests", "golden")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402
from PIL import Image  # noqa: E402

from bench_infer import card  # noqa: E402


def timed_events(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3 / reps


def timed_host(fn, reps):
    fn()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t0) / reps


def loop_depth(velo, P, Hd, Wd):
    """The reference's duplicate resolution as an algorithm: last-point assignment, then per duplicated key a scan of all
    points for that key."""
    from oracle import prepare as OP
    with np.errstate(divide="ignore", invalid="ignore"):
        px, py, z = OP.project(velo, P)
        keep = (px >= 0) & (py >= 0) & (px < Wd) & (py < Hd)
    px, py, z = px[keep], py[keep], z[keep]
    depth = np.zeros((Hd, Wd), np.float32)
    depth[py.astype(int), px.astype(int)] = z
    keys = py * (Wd - 1) + px - 1
    for k in [k for k, c in Counter(keys).items() if c > 1]:
        pts = np.where(keys == k)[0]
        depth[int(py[pts[0]]), int(px[pts[0]])] = z[pts].min()
    depth[depth < 0] = 0
    return depth


def kitti_P():
    P = np.array([[721.5, 0, 609.6, 44.9], [0, 721.5, 172.9, 0.22], [0, 0, 1.0, 0.0027]])
    P[0] *= 832 / 1242
    P[1] *= 256 / 375
    Tr = np.array([[0, -1, 0, -0.004], [0, 0, -1, -0.076], [1, 0, 0, -0.27], [0, 0, 0, 1.0]])
    return P @ Tr


def make_drive(root, n, seed=0):
    """A KITTI raw drive at full size: calibration, OXTS (every frame selected by speed), PNGs and 120k-point clouds."""
    import prepare_trees as T
    g = np.random.RandomState(seed)
    date = os.path.join(root, "2011_09_26")
    drive = os.path.join(date, "2011_09_26_drive_0001_sync")
    fmt = lambda a: " ".join("%.6e" % v for v in np.ravel(a))   # noqa: E731
    P = np.array([[721.5, 0, 609.6, 44.9], [0, 721.5, 172.9, 0.22], [0, 0, 1.0, 0.0027]])
    texts = {"calib_cam_to_cam.txt": "R_rect_00: %s\nP_rect_02: %s\nP_rect_03: %s\n" % (fmt(np.eye(3)), fmt(P), fmt(P)),
             "calib_velo_to_cam.txt": "R: %s\nT: %s\n" % (fmt([[0, -1, 0], [0, 0, -1], [1, 0, 0]]), fmt([-0.004, -0.076, -0.27])),
             "calib_imu_to_velo.txt": "R: %s\nT: %s\n" % (fmt(np.eye(3)), fmt([-0.81, 0.32, -0.8]))}
    for d in ("2011_09_28", "2011_09_29", "2011_09_30", "2011_10_03"):
        os.makedirs(os.path.join(root, d))
    for sub in ("oxts/data", "image_02/data", "image_03/data", "velodyne_points/data"):
        os.makedirs(os.path.join(drive, sub))
    for k, v in texts.items():
        open(os.path.join(date, k), "w").write(v)
    base = T.image(seed, 375, 1242).astype(np.int16)
    for i in range(n):
        row = np.zeros(30)
        row[:6] = [49.0 + 1e-5 * i, 8.4 + 2e-5 * i, 110, 0, 0, 0.5]
        row[8] = 5.0
        open(os.path.join(drive, "oxts", "data", "%010d.txt" % i), "w").write(" ".join("%.10f" % v for v in row) + "\n")
        for c in ("02", "03"):
            img = np.clip(np.roll(base, 3 * i, axis=1) + g.randint(-8, 9, base.shape), 0, 255).astype(np.uint8)
            Image.fromarray(img).save(os.path.join(drive, "image_%s" % c, "data", "%010d.png" % i))
        T.cloud(seed + i, 120000, "scene").tofile(os.path.join(drive, "velodyne_points", "data", "%010d.bin" % i))
    open(os.path.join(root, "test_scenes.txt"), "w").write("2011_09_26_drive_0117\n")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--clouds", type=int, default=32)
    ap.add_argument("--e2e-frames", type=int, default=60)
    ap.add_argument("--num-threads", type=int, default=8)
    a = ap.parse_args()
    import prepare_trees as T
    from oracle import prepare as OP
    from scsfm import prepare as P
    ops = P.DeviceOps()
    name, power = card()
    out = {"metric": "prepare_throughput", "gpu": name, "power_limit": power}

    frames = np.stack([T.image(i, 375, 1242) for i in range(a.frames)])
    host = torch.from_numpy(frames).pin_memory()
    dev = host.cuda()
    out["resize_kernel_frames_per_s"] = a.frames / timed_events(lambda: ops.resize_batch(dev, 256, 832), 10)
    out["resize_call_frames_per_s"] = a.frames / timed_host(lambda: (ops.resize_batch(host, 256, 832).cpu()), 5)
    n_pil = min(16, a.frames)
    out["resize_pillow_frames_per_s"] = n_pil / timed_host(
        lambda: [Image.fromarray(f).resize((832, 256), Image.BILINEAR) for f in frames[:n_pil]], 2)

    Pk = kitti_P()
    clouds = [T.cloud(100 + i, 120000, "scene") for i in range(a.clouds)]
    pts = torch.from_numpy(np.concatenate(clouds)).cuda()
    offsets = np.arange(a.clouds + 1, dtype=np.int64) * 120000
    d_off = torch.from_numpy(offsets).cuda()
    d_P = torch.from_numpy(np.stack([Pk] * a.clouds)).cuda()
    d_out = torch.empty(a.clouds, 256, 832, device="cuda")
    nws = int(ops.lib.scsfm_velo_depth_workspace_bytes(a.clouds, 256, 832))
    ws = torch.empty(nws, dtype=torch.uint8, device="cuda")
    L = ops.L
    import ctypes
    kern = lambda: L.launch(ops.lib.scsfm_velo_depth, "scsfm_velo_depth", "prepare", 3, 0, L.ptr(pts), L.ptr(d_off),   # noqa: E731
                            offsets.ctypes.data_as(ctypes.c_void_p), L.ptr(d_P), a.clouds, 256, 832, L.ptr(d_out), L.ptr(ws), nws,
                            L.stream())
    out["depth_kernel_maps_per_s"] = a.clouds / timed_events(kern, 10)
    out["depth_call_maps_per_s"] = a.clouds / timed_host(lambda: ops.depth(clouds, [Pk] * a.clouds, 256, 832), 3)
    out["depth_oracle_maps_per_s"] = 4 / timed_host(lambda: [OP.depth_map(c, Pk, 256, 832) for c in clouds[:4]], 1)
    t0 = time.perf_counter()
    ref = loop_depth(clouds[0], Pk, 256, 832)
    out["depth_reference_loop_maps_per_s"] = 1 / (time.perf_counter() - t0)
    out["depth_reference_loop_equal"] = bool(np.array_equal(ref, ops.depth(clouds[:1], [Pk], 256, 832)[0]))

    import prepare_train_data as C
    tmp = tempfile.mkdtemp()
    try:
        make_drive(os.path.join(tmp, "raw"), a.e2e_frames)
        stats = {}
        argv = [os.path.join(tmp, "raw"), "--test-scenes", os.path.join(tmp, "raw", "test_scenes.txt"), "--with-depth", "--with-pose",
                "--height", "256", "--width", "832", "--dump-root", os.path.join(tmp, "dump"), "--num-threads", str(a.num_threads)]
        t0 = time.perf_counter()
        C.main(argv, ops=ops, stats=stats)
        wall = time.perf_counter() - t0
        out["e2e_frames"] = stats["frames"]
        out["e2e_frames_per_s"] = stats["frames"] / wall
        out["e2e_seconds"] = {"total": wall, "decode_wait": stats["decode"], "device": stats["device"], "encode_wait": stats["encode"]}
        out["num_threads"] = a.num_threads
    finally:
        shutil.rmtree(tmp)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
