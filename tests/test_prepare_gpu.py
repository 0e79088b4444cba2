"""Training-set preparation on the device (csrc/prepare.cu): the resize kernel against Pillow, the depth kernel against the
oracle and the unmodified reference's generate_depth_map (tests/golden/prepare.npz), data/prepare_train_data.py end to end
against the reference's files, and the dump in the reference's dataset classes and train.py --with-gt."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import prepare as OP
from test_prepare_cpu import RESIZES, _run_cli, compare_dump, pillow

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, GOLDEN)

import prepare_trees as T  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "prepare.npz"))


@pytest.fixture(scope="module")
def ops():
    from scsfm import prepare as P
    return P.DeviceOps()


def _frames(n, h, w, seed):
    g = np.random.RandomState(seed)
    f = g.randint(0, 256, (n, h, w, 3)).astype(np.uint8)
    f[0, :16, :16] = 255
    f[-1, -16:, -16:] = 0
    return f


@pytest.mark.parametrize("src,dst", RESIZES)
def test_resize_kernel_is_pillow(ops, src, dst):
    frames = _frames(3, src[0], src[1], src[0] + dst[1])
    out = ops.resize_batch(torch.from_numpy(frames), dst[0], dst[1]).cpu().numpy()
    for b in range(3):
        assert np.array_equal(out[b], pillow(frames[b], dst[1], dst[0])), b


def test_resize_mixed_batch(ops):
    sizes = [(375, 1242), (376, 1241), (370, 1224), (375, 1242), (370, 1226), (376, 1241)]
    frames = [_frames(1, h, w, 10 + i)[0] for i, (h, w) in enumerate(sizes)]
    out = ops.resize(frames, 256, 832)
    for f, o in zip(frames, out):
        assert np.array_equal(o, pillow(f, 832, 256))


def _P():
    P = np.array([[720.0, 0, 415.0, 45.0], [0, 720.0, 128.0, 0.2], [0, 0, 1.0, 0.003]]) / 1.5
    R = np.array([[0, -1, 0, -0.004], [0, 0, -1, -0.076], [1, 0, 0, -0.27], [0, 0, 0, 1.0]])
    return P @ R


def test_depth_kernel_is_the_oracle(ops):
    """An empty cloud, a cloud entirely behind, a 120k-point KITTI-like cloud at 256 x 832 and ratio 2; two runs bitwise equal."""
    P = _P()
    big = T.cloud(7, 120000, "scene")
    clouds = [T.cloud(1, 0), T.cloud(2, 5000, "behind"), big, T.cloud(3, 60000, "dense")]
    for Hd, Wd in ((256, 832), (128, 416)):
        Ps = [P / np.array([[256 / Hd], [256 / Hd], [1.0]])] * len(clouds)
        got = ops.depth(clouds, Ps, Hd, Wd)
        again = ops.depth(clouds, Ps, Hd, Wd)
        for c, Pb, g, a in zip(clouds, Ps, got, again):
            want = OP.depth_map(c, Pb, Hd, Wd)
            assert np.array_equal(g.view(np.uint32), want.view(np.uint32))
            assert np.array_equal(g.view(np.uint32), a.view(np.uint32))
        assert np.count_nonzero(got[0]) == 0 and np.count_nonzero(got[1]) == 0 and np.count_nonzero(got[2]) > 1000


def test_depth_kernel_is_the_reference(ops, golden, tmp_path):
    from scsfm import prepare as P
    T.build(str(golden["spec_raw"]), str(tmp_path))
    drive = os.path.join(str(tmp_path), "2011_09_26", "2011_09_26_drive_0001_sync")
    for ratio in (1, 2):
        loader = P.KittiRaw(str(tmp_path), os.path.join(str(tmp_path), "test_scenes.txt"), img_height=16, img_width=48,
                            get_depth=True, depth_size_ratio=ratio)
        scene = loader.collect(drive)[0]
        fids = T.EXTRA_CLOUDS + tuple("%010d" % i for i in range(3))
        clouds = [np.fromfile(os.path.join(drive, "velodyne_points", "data", f + ".bin"), np.float32).reshape(-1, 4) for f in fids]
        got = ops.depth(clouds, [scene.P] * len(clouds), 16 // ratio, 48 // ratio)
        for f, c, g in zip(fids, clouds, got):
            assert np.array_equal(g.view(np.uint32), OP.depth_map(c, scene.P, 16 // ratio, 48 // ratio).view(np.uint32)), f
            assert np.array_equal(g.view(np.uint32), golden["depth_r%d_%s" % (ratio, f)].view(np.uint32)), f


@pytest.mark.parametrize("name,tree,flags", T.RUNS, ids=[r[0] for r in T.RUNS])
def test_cli_end_to_end(golden, ops, name, tree, flags, tmp_path):
    dump = _run_cli(golden, name, tree, flags, str(tmp_path), ops)
    compare_dump(golden, name, dump)


@pytest.fixture(scope="module")
def train_dump(golden, ops, tmp_path_factory):
    """KITTI raw at 128 x 160 with depth; every scene is listed for validation as well, so the --with-gt validation has
    scenes whichever way the 10 % draw fell."""
    tmp = str(tmp_path_factory.mktemp("prep"))
    flags = ["--dataset-format", "kitti_raw", "--with-depth", "--with-pose", "--height", "128", "--width", "160"]
    dump = _run_cli(golden, "train", "raw", flags, tmp, ops)
    scenes = sorted(d for d in os.listdir(dump) if os.path.isdir(os.path.join(dump, d)))
    assert scenes
    for f in ("train.txt", "val.txt"):
        with open(os.path.join(dump, f), "w") as fh:
            fh.write("".join(s + "\n" for s in scenes))
    return dump


def test_dump_loads_in_the_reference_datasets(train_dump):
    import subprocess
    from helpers import reference_loader_env
    env = reference_loader_env()
    if env is None:
        pytest.skip("the original project's modules are not installed (oracle/_ref/, made by __graft_entry__.build())")
    from oracle import reference
    # the reference's datasets/ has no __init__.py, so an installed package of that name would win an import: load by path
    code = ("import importlib.util, os, sys\n"
            "def load(n):\n"
            "    spec = importlib.util.spec_from_file_location(n, os.path.join(sys.argv[2], 'datasets', n + '.py'))\n"
            "    m = importlib.util.module_from_spec(spec); spec.loader.exec_module(m); return m\n"
            "t = load('sequence_folders').SequenceFolder(sys.argv[1], transform=None, seed=0, train=True, sequence_length=3)\n"
            "v = load('validation_folders').ValidationSet(sys.argv[1], transform=None, dataset='kitti')\n"
            "tgt, refs, K, Kinv = t[0]\nimg, depth = v[0]\n"
            "print(len(t), len(v), tgt.shape, len(refs), K.shape, img.shape, tuple(depth.shape))\n")
    out = subprocess.run([sys.executable, "-c", code, train_dump, reference.installed()], capture_output=True, text=True, timeout=300, env=env)
    assert out.returncode == 0, out.stderr[-3000:]
    n_train, n_val = (int(v) for v in out.stdout.split()[:2])
    assert n_train > 0 and n_val > 0
    assert "(128, 160, 3)" in out.stdout and "(128, 160)" in out.stdout, out.stdout


def test_train_with_gt_on_the_dump(train_dump, tmp_path):
    import subprocess
    from helpers import reference_loader_env
    env = reference_loader_env()
    if env is None:
        pytest.skip("the original project's modules are not installed (oracle/_ref/, made by __graft_entry__.build())")
    cmd = [sys.executable, os.path.join(ROOT, "sc-sfmlearner-release_b200", "train.py"), train_dump, "--with-gt", "--name", "prep",
           "--epochs", "1", "--epoch-size", "2", "-b", "2", "-j", "0", "--resnet-layers", "18", "--num-scales", "1",
           "--with-pretrain", "0", "--print-freq", "1"]
    out = subprocess.run(cmd, cwd=str(tmp_path), capture_output=True, text=True, timeout=600, env=env)
    assert out.returncode == 0, out.stderr[-3000:]
    runs = os.listdir(tmp_path / "checkpoints" / "prep")
    import csv
    full = list(csv.reader(open(tmp_path / "checkpoints" / "prep" / runs[0] / "progress_log_summary.csv"), delimiter="\t"))
    assert len(full) >= 2 and all(np.isfinite(float(v)) for v in full[1]), full
