"""Training-set preparation on the host: the oracle resize against live Pillow, the oracle depth map against the unmodified
reference's generate_depth_map, and data/prepare_train_data.py end to end against the reference's files (golden:
tests/golden/prepare.npz, written by tests/golden/make_golden_prepare.py).  The two device operations are replaced by the
oracle functions here, in the test only."""
import json
import os
import sys

import numpy as np
import pytest
from PIL import Image

from oracle import augment as OA
from oracle import prepare as OP

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "sc-sfmlearner-release_b200")
GOLDEN = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, os.path.join(PKG, "data"))
sys.path.insert(0, GOLDEN)

import prepare_trees as T  # noqa: E402

# (source h, w) -> (target h, w): KITTI raw's four sizes and odometry to 256 x 832, Cityscapes to 256 x 832, an upscale,
# one axis only, identity
RESIZES = [((375, 1242), (256, 832)), ((376, 1241), (256, 832)), ((370, 1224), (256, 832)), ((370, 1226), (128, 416)),
           ((1024, 2048), (256, 832)), ((30, 40), (64, 100)), ((375, 1242), (375, 832)), ((375, 1242), (256, 1242)),
           ((37, 53), (37, 53))]


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "prepare.npz"))


class OracleOps:
    """The device operations' contract, computed by the oracle."""

    def resize(self, frames, out_h, out_w):
        return [OP.resize_bilinear_u8(f, out_w, out_h) for f in frames]

    def depth(self, clouds, Ps, Hd, Wd):
        return [OP.depth_map(c, P, Hd, Wd) for c, P in zip(clouds, Ps)]


def pillow(img, w, h):
    return np.asarray(Image.fromarray(img).resize((w, h), Image.BILINEAR))


@pytest.mark.parametrize("src,dst", RESIZES)
def test_oracle_resize_is_pillow_bilinear(src, dst):
    img = np.random.RandomState(src[0] * 7 + dst[1]).randint(0, 256, src + (3,)).astype(np.uint8)
    img[:20, :20] = 255                      # saturated and flat corners: the clip and the exact-1 taps
    img[-20:, -20:] = 0
    assert np.array_equal(OP.resize_bilinear_u8(img, dst[1], dst[0]), pillow(img, dst[1], dst[0]))


def test_tap_counts():
    assert OP.resample_coeffs(1242, 832)[1].shape[1] == 5
    assert OP.resample_coeffs(2048, 832)[1].shape[1] == 7
    assert OP.resample_coeffs(40, 100)[1].shape[1] == 3


@pytest.mark.parametrize("n_in,n_out", [(375, 431), (1242, 1300), (128, 147), (416, 417)])
def test_bicubic_coefficients_match_the_augment_oracle(n_in, n_out):
    a, b = OP.resample_coeffs(n_in, n_out, "bicubic"), OA.resample_coeffs(n_in, n_out)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def _rint_boundary_culprit(cloud, P):
    """Whether some kept point's u0/u2 or u1/u2 lies within a few ulps of a rint half-way point: the only way the reference's
    BLAS summation order can move a point to another pixel."""
    v = np.asarray(cloud, np.float32).reshape(-1, 4)
    v = v[v[:, 0] >= 0]
    u = (P @ np.c_[v[:, :3].astype(np.float64), np.ones(len(v))].T)
    for a in (u[0] / u[2], u[1] / u[2]):
        frac = np.abs(a - np.floor(a) - 0.5)
        if np.any(frac <= 8 * np.spacing(np.abs(a) + 1)):
            return True
    return False


def test_oracle_depth_is_the_reference(golden):
    """generate_depth_map on the extra clouds (empty, all behind, dense, sparse) and three drive frames, ratios 1 and 2; P is
    built here from the calibration text, as scsfm.prepare does."""
    import tempfile
    from scsfm import prepare as P
    with tempfile.TemporaryDirectory() as tmp:
        T.build(str(golden["spec_raw"]), tmp)
        drive = os.path.join(tmp, "2011_09_26", "2011_09_26_drive_0001_sync")
        for ratio in (1, 2):
            loader = P.KittiRaw(tmp, os.path.join(tmp, "test_scenes.txt"), img_height=16, img_width=48, get_depth=True,
                                depth_size_ratio=ratio)
            scene = loader.collect(drive)[0]
            assert np.array_equal(np.hstack([scene.intrinsics, golden["depth_r%d_P_rect" % ratio][:, 3:]]), golden["depth_r%d_P_rect" % ratio])
            for fid in T.EXTRA_CLOUDS + tuple("%010d" % i for i in range(3)):
                cloud = np.fromfile(os.path.join(drive, "velodyne_points", "data", fid + ".bin"), np.float32).reshape(-1, 4)
                want = golden["depth_r%d_%s" % (ratio, fid)]
                got = OP.depth_map(cloud, scene.P, 16 // ratio, 48 // ratio)
                assert got.dtype == np.float32 and got.shape == want.shape
                bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))
                for y, x in bad:
                    assert _rint_boundary_culprit(cloud, scene.P), (ratio, fid, y, x, got[y, x], want[y, x])


def test_depth_rule_on_constructed_collisions():
    """Points placed on chosen pixels: the last point wins a pixel, the pixel of a key's first point gets the key's minimum,
    the row-edge partner keeps its own value, a negative depth becomes 0."""
    Hd, Wd = 3, 4
    P = np.array([[0, 1.0, 0, 0], [0, 0, 1.0, 0], [1.0, 0, 0, -1.0]])     # u = (y, z, x - 1): depth x - 1

    def at(px, py, d):          # lands on (py, px) with depth d
        return [d + 1, (px + 1) * d, (py + 1) * d, 0]
    pts = np.array([at(1, 0, 5.0), at(1, 0, 3.0), at(1, 0, 4.0),      # one pixel: last is 4, the key's minimum 3 wins
                    at(3, 0, 9.0), at(0, 1, 2.0),                        # key shared by (0, 3) and (1, 0): first on (0, 3)
                    at(0, 2, 7.0), at(3, 1, 6.0), at(3, 1, 8.0),         # key shared by (1, 3) and (2, 0): first on (2, 0)
                    at(2, 2, -0.5),                                      # x = 0.5 is kept, its depth is negative
                    [-1.0, 2.0, 2.0, 0]], np.float32)                   # behind: dropped
    d = OP.depth_map(pts, P, Hd, Wd)
    assert d[0, 1] == 3.0
    assert d[0, 3] == 2.0 and d[1, 0] == 2.0
    assert d[2, 0] == 6.0 and d[1, 3] == 8.0
    assert d[2, 2] == 0.0
    assert np.count_nonzero(d) == 5
    d_neg = OP.depth_map(pts[8:9], P, Hd, Wd)
    assert np.count_nonzero(d_neg) == 0 and OP.project(pts[8:9], P)[2][0] == -0.5


def _run_cli(golden, name, tree, flags, tmp, ops):
    import prepare_train_data as C
    root = os.path.join(tmp, tree)
    if not os.path.isdir(root):
        T.build(str(golden["spec_" + tree]), root)
    dump = os.path.join(tmp, "dump_" + name)
    argv = [root] + [f.format(root=root) for f in flags] + ["--dump-root", dump, "--num-threads", "3", "--batch-size", "5"]
    if tree == "raw":
        argv += ["--test-scenes", os.path.join(root, "test_scenes.txt")]
    C.main(argv, ops=ops)
    return dump


def compare_dump(golden, name, dump):
    """Every file the reference wrote, with the same bytes (text files compared as text for a readable failure)."""
    import hashlib
    want = json.loads(str(golden[name + "_files"]))
    got = T.dump_listing(dump)
    assert sorted(got) == sorted(want)
    for k, v in got.items():
        if k.endswith(".txt"):
            assert v.decode() == str(golden[name + "_text_" + k]), k
        elif k.endswith(".npy"):
            assert np.array_equal(np.load(os.path.join(dump, k)).view(np.uint32), golden[name + "_npy_" + k].view(np.uint32)), k
        assert hashlib.sha256(v).hexdigest() == want[k], k


@pytest.mark.parametrize("name,tree,flags", T.RUNS, ids=[r[0] for r in T.RUNS])
def test_cli_writes_the_reference_files(golden, name, tree, flags, tmp_path):
    dump = _run_cli(golden, name, tree, flags, str(tmp_path), OracleOps())
    compare_dump(golden, name, dump)


def test_refusals(tmp_path, capsys):
    import prepare_train_data as C
    with pytest.raises(SystemExit):
        C.parse([str(tmp_path), "--dataset-format", "kitti_raw"])
    assert "--test-scenes" in capsys.readouterr().err
    for h, w, r in ((128, 416, 3), (126, 416, 4), (128, 2, 2), (128, 416, 0)):
        with pytest.raises(SystemExit):
            C.parse([str(tmp_path), "--dataset-format", "kitti_odom", "--height", str(h), "--width", str(w), "--depth-size-ratio", str(r)])
        assert "--depth-size-ratio" in capsys.readouterr().err
    args = C.parse([str(tmp_path), "--dataset-format", "kitti_odom"])
    assert (args.height, args.width, args.depth_size_ratio, args.num_threads, args.dump_root) == (128, 416, 1, 4, "dump")


def test_device_ops_have_no_cpu_fallback():
    import torch
    from scsfm import prepare as P
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        P.DeviceOps()


def test_kernel_entry_points_reject_bad_arguments_without_a_gpu():
    import ctypes
    from scsfm import lib
    L = lib.load()
    n0 = lib.launch_count()
    L.scsfm_resize_bilinear_workspace_bytes.restype = ctypes.c_size_t
    L.scsfm_velo_depth_workspace_bytes.restype = ctypes.c_size_t
    assert L.scsfm_resize_bilinear_u8(None, 1, 8, 8, 4, 4, None, None, ctypes.c_size_t(0), None) == -1
    assert b"resize_bilinear_u8" in L.scsfm_last_error()
    buf = ctypes.create_string_buffer(64)
    assert L.scsfm_resize_bilinear_u8(buf, 1, 8, 4000, 8, 4, buf, buf, ctypes.c_size_t(1 << 30), None) == -1
    assert b"31x" in L.scsfm_last_error()
    off = (ctypes.c_longlong * 2)(0, 10)
    assert L.scsfm_velo_depth(buf, buf, off, buf, 1, 8, 1, buf, buf, ctypes.c_size_t(1 << 20), None) == -1
    assert b"Wd >= 2" in L.scsfm_last_error()
    bad = (ctypes.c_longlong * 2)(0, -1)
    assert L.scsfm_velo_depth(buf, buf, bad, buf, 1, 8, 8, buf, buf, ctypes.c_size_t(1 << 20), None) == -1
    assert b"offsets" in L.scsfm_last_error()
    assert L.scsfm_velo_depth_workspace_bytes(2, 8, 24) == 2 * 8 * 24 * 16
    assert lib.launch_count() == n0
