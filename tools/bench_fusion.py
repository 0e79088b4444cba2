"""Benchmark of the TSDF fusion (scsfm.fusion.TSDFVolume) on a seeded synthetic street; prints one JSON line.

1000 depth maps of 256 x 832 are rendered analytically on the device (a ground plane, box facades along both sides and
spheres) along a 1 km path, and fused at 0.2 voxels (trunc 0.8, max depth 80) in passes of 16 frames.  Reported:
  * integrate frames/s and voxel updates/s (voxel-frame visits: touched voxels times the frames of their pass), and the
    same passes split by CUDA events into the allocation (kernel, counter read, pool growth) and the integration kernel;
  * bytes/s of the voxel traffic, 40 bytes (20 read, 20 written) per voxel of every touched brick, against 3.35 TB/s;
  * the time of mesh();
  * the same integration written as vectorised torch ops over the touched bricks of the first passes (baseline);
  * run_fusion.py's end-to-end frames/s on a written PNG sequence with a random-init DispResNet-18;
  * the card name and power limit, read in the same run.
Everything it writes goes to a temporary directory."""
import argparse
import json
import math
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "sc-sfmlearner-release_b200"))

H, W = 256, 832
HBM = 3.35e12


def scene(seed, length):
    rng = np.random.default_rng(seed)
    boxes = []
    for side in (-1, 1):
        z = -20.0
        while z < length + 100:
            d = rng.uniform(8, 25)
            x0 = side * rng.uniform(7, 10)
            boxes.append((min(x0, x0 + side * 12), -rng.uniform(6, 20), z, max(x0, x0 + side * 12), 1.6, z + d))
            z += d + rng.uniform(0.5, 6)
    sph = [(rng.uniform(-5, 5), 1.6 - r, rng.uniform(0, length), r) for r in rng.uniform(0.3, 1.2, 120)]
    return torch.tensor(boxes, dtype=torch.float64, device="cuda"), torch.tensor(sph, dtype=torch.float64, device="cuda")


def path(n, length):
    z = np.linspace(0, length, n)
    T = np.tile(np.eye(4), (n, 1, 1))
    yaw = 0.05 * np.sin(z / 60)
    T[:, 0, 0], T[:, 0, 2], T[:, 2, 0], T[:, 2, 2] = np.cos(yaw), np.sin(yaw), -np.sin(yaw), np.cos(yaw)
    T[:, 0, 3], T[:, 2, 3] = 1.5 * np.sin(z / 80), z
    return T


def render(K, T, boxes, sph):
    """Camera-z depth [H,W] float32 of the nearest of the ground plane y = 1.6, the boxes and the spheres (0: nothing)."""
    v, u = torch.meshgrid(torch.arange(H, device="cuda", dtype=torch.float64), torch.arange(W, device="cuda", dtype=torch.float64),
                          indexing="ij")
    dc = torch.stack([(u - K[0, 2]) / K[0, 0], (v - K[1, 2]) / K[1, 1], torch.ones_like(u)], -1).reshape(-1, 3)
    Tt = torch.as_tensor(T, device="cuda")
    d = dc @ Tt[:3, :3].T
    o = Tt[:3, 3]
    best = torch.where(d[:, 1] > 1e-9, (1.6 - o[1]) / d[:, 1], torch.full_like(d[:, 0], math.inf))
    inv = 1 / d
    t0 = (boxes[None, :, :3] - o) * inv[:, None, :]
    t1 = (boxes[None, :, 3:] - o) * inv[:, None, :]
    tn = torch.minimum(t0, t1).amax(-1)
    tf = torch.maximum(t0, t1).amin(-1)
    tb = torch.where((tn <= tf) & (tn > 0), tn, torch.full_like(tn, math.inf)).amin(-1)
    oc = o[None] - sph[:, :3]
    b = 2 * d @ oc.T
    a = (d * d).sum(-1, keepdim=True)
    c = (oc * oc).sum(-1)[None] - sph[:, 3][None] ** 2
    disc = b * b - 4 * a * c
    ts = torch.where(disc >= 0, (-b - disc.clamp(min=0).sqrt()) / (2 * a), torch.full_like(b, math.inf))
    ts = torch.where(ts > 0, ts, torch.full_like(ts, math.inf)).amin(-1)
    best = torch.minimum(torch.minimum(best, tb), ts)
    return torch.where(torch.isfinite(best), best, torch.zeros_like(best)).reshape(H, W).float()


def torch_integrate(vol, frames_depth, K, T, cells):
    """The integration of one pass as vectorised torch ops over the voxels of the listed cells (no colour)."""
    p = torch.as_tensor(vol.lo, dtype=torch.float32, device="cuda") + (vol._cell_voxels(cells).float() + 0.5) * vol.voxel_size
    fields = vol._cell_fields(cells)
    tsdf, w = fields[0], fields[1]
    for f in range(len(frames_depth)):
        inv = torch.as_tensor(np.linalg.inv(T[f]), dtype=torch.float32, device="cuda")
        pc = p @ inv[:3, :3].T + inv[:3, 3]
        z = pc[:, 2]
        iu = torch.floor(K[0, 0] * pc[:, 0] / z + K[0, 2] + 0.5)
        iv = torch.floor(K[1, 1] * pc[:, 1] / z + K[1, 2] + 0.5)
        ok = (z > 0) & (iu >= 0) & (iu < W) & (iv >= 0) & (iv < H)
        d = frames_depth[f].reshape(-1)[torch.where(ok, iv * W + iu, torch.zeros_like(iu)).long()]
        sdf = d - z
        upd = ok & (d > 0) & (d <= vol.max_depth) & (sdf.abs() <= vol.trunc)
        wn = w + 1
        tsdf = torch.where(upd, (tsdf * w + sdf / vol.trunc) / wn, tsdf)
        w = torch.where(upd, wn, w)
    fields[0], fields[1] = tsdf, w
    vol._set_cell_fields(cells, fields)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True,
                            text=True, timeout=30).stdout.strip()
        power = float(pl.splitlines()[0])
    except Exception:                            # noqa: BLE001 -- reported as unknown
        power = None
    return name, power


def end_to_end(n_frames, tmp):
    from PIL import Image
    import models
    import run_fusion
    T = path(n_frames, n_frames * 1.0)
    seq = os.path.join(tmp, "seqs", "00", "image_2")
    os.makedirs(seq)
    rng = np.random.default_rng(0)
    for i in range(n_frames):
        Image.fromarray(rng.integers(0, 256, (H, W, 3), dtype=np.uint8)).save(os.path.join(seq, "%06d.png" % i))
    np.savetxt(os.path.join(tmp, "poses.txt"), T[:, :3].reshape(-1, 12), fmt="%1.8e")
    torch.manual_seed(0)
    torch.save({"state_dict": models.DispResNet(18, False).state_dict()}, os.path.join(tmp, "disp.tar"))
    args = ["--pretrained-dispnet", os.path.join(tmp, "disp.tar"), "--dataset-dir", os.path.join(tmp, "seqs") + "/", "--sequence",
            "00", "--poses", os.path.join(tmp, "poses.txt"), "--voxel-size", "0.2", "--intrinsics", "360", "360", "415.5", "127.5",
            "--batch-size", "16", "--output", os.path.join(tmp, "m.ply")]
    run_fusion.main(args)                        # warm-up: graphs, allocator
    r = run_fusion.main(args)
    return r["frames"] / r["seconds"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1000)
    ap.add_argument("--length", type=float, default=1000.0)
    ap.add_argument("--baseline-passes", type=int, default=8)
    ap.add_argument("--e2e-frames", type=int, default=160)
    a = ap.parse_args()
    from scsfm import lib
    from scsfm.fusion import TSDFVolume
    lib.load()
    torch.manual_seed(0)
    boxes, sph = scene(0, a.length)
    T = path(a.frames, a.length)
    K = np.array([[360.0, 0, 415.5], [0, 360.0, 127.5], [0, 0, 1]])
    Kt = torch.as_tensor(K, device="cuda")
    depth = torch.stack([render(Kt, T[i], boxes, sph) for i in range(a.frames)])
    centres = T[:, :3, 3]
    lo, hi = centres.min(0) - 80, centres.max(0) + 80

    def fuse():
        vol = TSDFVolume(lo, hi, 0.2)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(0, a.frames, 16):
            vol.integrate(depth[i:i + 16], K, T[i:i + 16])
        torch.cuda.synchronize()
        return vol, time.perf_counter() - t0

    fuse()                                           # warm-up (pool growth, module loads)
    vol, dt = fuse()
    visits = vol.brick_visits
    # the same passes again, split: allocation (kernel, counter read, pool growth) and the integration kernel, by CUDA events
    Kb = np.broadcast_to(K, (a.frames, 3, 3))
    split = TSDFVolume(lo, hi, 0.2)
    alloc_ms = apply_ms = 0.0
    voxel_updates = 0                     # voxel-frame visits: each pass's bricks times its frame count
    for i in range(0, a.frames, 16):
        frames = split._frames(depth, Kb, T, None, i, min(16, a.frames - i))
        e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        e[0].record()
        touched = split._allocate(frames, H, W)
        e[1].record()
        split._apply(frames, H, W, touched)
        e[2].record()
        e[2].synchronize()
        alloc_ms += e[0].elapsed_time(e[1])
        apply_ms += e[1].elapsed_time(e[2])
        voxel_updates += touched * 512 * len(frames)
    del split
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    verts, faces, _ = vol.mesh()
    torch.cuda.synchronize()
    mesh_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    vol.mesh()
    torch.cuda.synchronize()
    mesh_s = min(mesh_s, time.perf_counter() - t0)

    # torch baseline over the listed bricks of the first passes (allocation by the library's kernel, untimed)
    base = TSDFVolume(lo, hi, 0.2)
    tb, nb_frames = 0.0, 0
    for p in range(a.baseline_passes):
        i = p * 16
        frames = base._frames(depth, Kb, T, None, i, min(16, a.frames - i))
        cells = base._listed(base._allocate(frames, H, W)).clone()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        torch_integrate(base, depth[i:i + len(frames)], K, T[i:i + len(frames)], cells)
        torch.cuda.synchronize()
        tb += time.perf_counter() - t0
        nb_frames += len(frames)

    name, power = card()
    with tempfile.TemporaryDirectory() as tmp:
        e2e = end_to_end(a.e2e_frames, tmp)
    bytes_moved = visits * 512 * 40
    print(json.dumps({
        "workload": "tsdf_fusion_street", "frames": a.frames, "size": [H, W], "voxel": 0.2, "trunc": 0.8, "max_depth": 80.0,
        "bricks": vol.num_bricks, "brick_visits": visits, "volume_mb": round(vol.memory_bytes() / 2 ** 20, 1),
        "integrate_s": round(dt, 4), "integrate_frames_per_s": round(a.frames / dt, 1),
        "voxel_updates_per_s": float("%.4g" % (voxel_updates / dt)),
        "allocate_ms": round(alloc_ms, 2), "integrate_kernel_ms": round(apply_ms, 2),
        "voxel_bytes_per_s": float("%.4g" % (bytes_moved / dt)), "fraction_of_3_35_TBps": round(bytes_moved / dt / HBM, 3),
        "mesh_s": round(mesh_s, 4), "mesh_vertices": len(verts), "mesh_faces": len(faces),
        "torch_baseline_frames_per_s": round(nb_frames / tb, 1) if tb else None,
        "run_fusion_frames_per_s": round(e2e, 1), "gpu": name, "power_limit_w": power}))


if __name__ == "__main__":
    main()
