"""Small synthetic KITTI raw, KITTI odometry and Cityscapes trees for the training-set preparation tests.

A tree is described by a JSON spec (stored in tests/golden/prepare.npz by make_golden_prepare.py): text files verbatim
(calibration, OXTS rows, Cityscapes JSONs, the lists), and images / Velodyne clouds by (seed, shape), drawn with numpy's
legacy RandomState, whose streams numpy keeps fixed.  `build(spec, root)` writes the tree; `make_specs(test_scenes)` draws
the specs (only the golden maker calls it).
"""
import json
import os

import numpy as np
from PIL import Image

RAW_HW, ODOM_HW, CITY_HW = (16, 48), (16, 40), (24, 40)       # --height/--width of the runs


def image(seed, h, w):
    return np.random.RandomState(seed).randint(0, 256, (h, w, 3)).astype(np.uint8)


def cloud(seed, n, kind="scene"):
    """N x 4 float32 Velodyne rows.  'scene': most points ahead, some behind, some barely ahead (negative depth after the
    camera offset); 'behind': every x < 0; 'dense': a narrow cone, many points per pixel."""
    g = np.random.RandomState(seed)
    if kind == "behind":
        x = -g.uniform(0.0, 30.0, n)
        y, z = g.uniform(-10, 10, n), g.uniform(-2, 2, n)
    elif kind == "dense":
        x = g.uniform(3.0, 40.0, n)
        y, z = x * g.uniform(-0.3, 0.3, n), x * g.uniform(-0.1, 0.05, n)
    else:
        x = g.uniform(-5.0, 40.0, n)
        x[: n // 10] = g.uniform(0.0, 0.4, n // 10)
        y, z = x * g.uniform(-0.8, 0.8, n), x * g.uniform(-0.3, 0.15, n) + g.uniform(-0.5, 0.5, n)
    r = g.uniform(0, 1, n)
    return np.stack([x, y, z, r], 1).astype(np.float32)


def build(spec, root):
    """Write the tree described by `spec` (a dict or its JSON text) under root."""
    if isinstance(spec, str):
        spec = json.loads(spec)
    for rel, text in spec["text"].items():
        p = os.path.join(root, rel)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        with open(p, "w") as f:
            f.write(text)
    for rel, (seed, h, w) in spec["images"].items():
        p = os.path.join(root, rel)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        Image.fromarray(image(seed, h, w)).save(p)
    for rel in spec.get("dirs", ()):
        os.makedirs(os.path.join(root, rel), exist_ok=True)
    for rel, (seed, n, kind) in spec["clouds"].items():
        p = os.path.join(root, rel)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        cloud(seed, n, kind).tofile(p)
    return root


def _fmt(a):
    return " ".join("%.6e" % v for v in np.ravel(a))


def _raw_spec(g, test_scenes):
    text, images, clouds = {}, {}, {}
    seed = [1000]

    def nxt():
        seed[0] += 1
        return seed[0]

    R_rect = np.eye(3) + g.normal(0, 0.01, (3, 3))
    for date in ("2011_09_26", "2011_09_28"):
        P2 = [[58.0, 0, 49.5, 4.4], [0, 58.0, 14.5, 0.02], [0, 0, 1, 0.003]]
        P3 = [[58.0, 0, 48.5, -31.0], [0, 58.0, 14.0, 0.3], [0, 0, 1, 0.004]]
        text[date + "/calib_cam_to_cam.txt"] = ("calib_time: 09-Jan-2012 13:57:47\ncorner_dist: 9.950000e-02\n"
                                               "R_rect_00: %s\nP_rect_00: %s\nP_rect_02: %s\nP_rect_03: %s\n"
                                               % (_fmt(R_rect), _fmt(P2), _fmt(P2), _fmt(P3)))
        Rv = np.array([[0, -1, 0], [0, 0, -1], [1, 0, 0]]) + g.normal(0, 0.01, (3, 3))
        text[date + "/calib_velo_to_cam.txt"] = ("calib_time: 15-Mar-2012 11:37:16\nR: %s\nT: %s\ndelta_f: 0 0\n"
                                                % (_fmt(Rv), _fmt([-0.004, -0.076, -0.27])))
        Ri = np.eye(3) + g.normal(0, 0.01, (3, 3))
        text[date + "/calib_imu_to_velo.txt"] = "calib_time: 25-May-2012 16:47:16\nR: %s\nT: %s\n" % (_fmt(Ri), _fmt([-0.81, 0.32, -0.8]))
    test_drive = next(t for t in test_scenes if t.startswith("2011_09_26"))
    # (date/drive, frames, image size, speed scale)
    drives = [("2011_09_26/2011_09_26_drive_0001_sync", 9, (30, 100), 3.5),
              ("2011_09_26/%s_sync" % test_drive, 3, (30, 100), 1.2),
              ("2011_09_28/2011_09_28_drive_0001_sync", 7, (31, 98), 2.5),
              ("2011_09_28/2011_09_28_drive_0099_sync", 4, (30, 100), 0.2)]
    for drive, n, (h, w), sp in drives:
        lat0, lon0 = 49.0 + g.uniform(0, 0.01), 8.4 + g.uniform(0, 0.01)
        for i in range(n):
            row = np.zeros(30)
            row[:6] = [lat0 + 1e-5 * i, lon0 + 2e-5 * i, 110 + 0.1 * i, g.normal(0, 0.02), g.normal(0, 0.02), 0.5 + g.normal(0, 0.05)]
            row[8:11] = [g.uniform(0, sp), g.normal(0, 0.2 * sp), g.normal(0, 0.05)]
            row[11:] = g.normal(0, 1, 19)
            text["%s/oxts/data/%010d.txt" % (drive, i)] = " ".join("%.10f" % v for v in row) + "\n"
            for c in ("02", "03"):
                images["%s/image_%s/data/%010d.png" % (drive, c, i)] = (nxt(), h, w)
            clouds["%s/velodyne_points/data/%010d.bin" % (drive, i)] = (nxt(), 1500 + 100 * i, "scene")
    # the other recording dates exist without drives
    return {"text": text, "images": images, "clouds": clouds, "dirs": ["2011_09_29", "2011_09_30", "2011_10_03"]}


def _odom_spec(g):
    text, images = {}, {}
    seed = [2000]
    for seq, n in (("00", 5), ("03", 2), ("09", 3)):
        lines = []
        for k in range(4):
            P = [[45.0 + k, 0, 50.2, -38.0 * k], [0, 45.0 + k, 15.1, 0.01 * k], [0, 0, 1, 0.002 * k]]
            lines.append("P%d: %s" % (k, " ".join("%.12e" % v for v in np.ravel(P))))
        lines.append("Tr: " + " ".join("%.12e" % v for v in g.normal(0, 1, 12)))
        text["sequences/%s/calib.txt" % seq] = "\n".join(lines) + "\n"
        for i in range(n):
            for c in ("2", "3"):
                seed[0] += 1
                images["sequences/%s/image_%s/%06d.png" % (seq, c, i)] = (seed[0], 37, 123)
    return {"text": text, "images": images, "clouds": {}}


def _city_spec(g):
    text, images = {}, {}
    seed = [3000]
    runs = {"000000": [list(range(19, 35)), list(range(40, 45))], "000001": [list(range(3, 17))]}
    for scene, subs in runs.items():
        first = subs[0][0]
        cam = {"extrinsic": {"baseline": 0.209}, "intrinsic": {"fx": 110.3 + g.uniform(0, 5), "fy": 111.1 + g.uniform(0, 5),
                                                              "u0": 50.7 + g.uniform(0, 1), "v0": 24.9 + g.uniform(0, 1)}}
        text["camera/train/aachen/aachen_%s_%06d_camera.json" % (scene, first)] = json.dumps(cam, indent=2)
        for sub in subs:
            for f in sub:
                seed[0] += 1
                images["leftImg8bit_sequence/train/aachen/aachen_%s_%06d_leftImg8bit.png" % (scene, f)] = (seed[0], 48, 96)
                text["vehicle_sequence/train/aachen/aachen_%s_%06d_vehicle.json" % (scene, f)] = json.dumps(
                    {"gpsHeading": 0.0, "speed": round(float(g.uniform(0.5, 1.6)), 4)})
    return {"text": text, "images": images, "clouds": {}}


def make_specs(test_scenes):
    g = np.random.RandomState(8)
    raw = _raw_spec(g, test_scenes)
    drive = "2011_09_26/2011_09_26_drive_0001_sync"
    raw["text"]["static_frames.txt"] = "".join("2011_09_26 2011_09_26_drive_0001_sync %010d\n" % i for i in (1, 2, 6)) + \
        "2011_09_28 2011_09_28_drive_0001_sync 0000000000\n"
    raw["text"]["test_scenes.txt"] = "".join(t + "\n" for t in test_scenes)
    # extra clouds for generate_depth_map alone (read through drive 0001's calibration)
    raw["clouds"][drive + "/velodyne_points/data/extra_empty.bin"] = (4001, 0, "scene")
    raw["clouds"][drive + "/velodyne_points/data/extra_behind.bin"] = (4002, 2000, "behind")
    raw["clouds"][drive + "/velodyne_points/data/extra_dense.bin"] = (4003, 30000, "dense")
    raw["clouds"][drive + "/velodyne_points/data/extra_sparse.bin"] = (4004, 300, "scene")
    return {"raw": raw, "odom": _odom_spec(g), "city": _city_spec(g)}


EXTRA_CLOUDS = ("extra_empty", "extra_behind", "extra_dense", "extra_sparse")

# (name, tree, command-line flags after the tree root; the dump root is appended)
RUNS = [("raw_static", "raw", ["--dataset-format", "kitti_raw", "--static-frames", "{root}/static_frames.txt", "--with-depth",
                               "--with-pose", "--height", "16", "--width", "48"]),
        ("raw_speed", "raw", ["--dataset-format", "kitti_raw", "--with-depth", "--with-pose", "--no-train-gt", "--height", "16",
                              "--width", "48", "--depth-size-ratio", "2"]),
        ("odom", "odom", ["--dataset-format", "kitti_odom", "--with-depth", "--with-pose", "--height", "16", "--width", "40"]),
        ("city", "city", ["--dataset-format", "cityscapes", "--with-depth", "--with-pose", "--height", "24", "--width", "40"])]


def dump_listing(dump_root):
    """{relative path: file bytes} of everything under a dump root."""
    out = {}
    for d, _, files in os.walk(dump_root):
        for f in files:
            p = os.path.join(d, f)
            with open(p, "rb") as fh:
                out[os.path.relpath(p, dump_root)] = fh.read()
    return out
