"""A bank of learned cameras, CPU side: the C ABI of scsfm_camera_build_indexed / scsfm_camera_grad_indexed (declared, exported,
argument errors reported without a launch), a numpy restatement of the indexed build against update_intrinsics of each sample's own
camera, train.py's --camera-groups (flags, refusals, the camera table) and the sample-to-camera mapping through the reference's
own SequenceFolder / PairFolder."""
import ctypes
import os
import random
import re
import subprocess
import sys

import numpy as np
import pytest

from camera_helpers import indexed_build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "sc-sfmlearner-release_b200")


def test_header_declares_and_library_exports_the_indexed_entries():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "scsfm.h")).read(), flags=re.S)
    assert re.search(r"\bscsfm_camera_build_indexed\s*\(\s*const float\s*\*\s*theta\s*,\s*int n_cams\s*,\s*const double\s*\*\s*aug\s*,"
                     r"\s*const int\s*\*\s*idx\s*,\s*int B\s*,\s*float\s*\*\s*K_out\s*,\s*void\s*\*\s*stream\s*\)", src)
    assert re.search(r"\bscsfm_camera_grad_indexed\s*\(\s*const double\s*\*\s*aug\s*,\s*const int\s*\*\s*idx\s*,\s*const float\s*\*\s*dK\s*,"
                     r"\s*int B\s*,\s*int n_cams\s*,\s*float\s*\*\s*dtheta\s*,\s*void\s*\*\s*stream\s*\)", src)
    from scsfm import lib
    L = lib.load()
    assert hasattr(L, "scsfm_camera_build_indexed") and hasattr(L, "scsfm_camera_grad_indexed")


def test_indexed_entries_reject_bad_arguments_without_a_launch():
    from scsfm import camera
    from scsfm import lib
    L = camera._lib()
    n0 = lib.launch_count()
    f = ctypes.c_void_p(16)               # never dereferenced: every call below fails its argument check first
    for args in ((None, 2, f, f, 1, f), (f, 2, None, f, 1, f), (f, 2, f, None, 1, f), (f, 2, f, f, 1, None)):
        assert L.scsfm_camera_build_indexed(*args, None) == -1
        assert b"camera_build_indexed" in L.scsfm_last_error() and b"null" in L.scsfm_last_error()
    assert L.scsfm_camera_build_indexed(f, 0, f, f, 1, f, None) == -1
    assert b"number of cameras" in L.scsfm_last_error()
    assert L.scsfm_camera_build_indexed(f, 3, f, f, 0, f, None) == -1
    assert b"batch size" in L.scsfm_last_error()
    for args in ((None, f, f, 1, 2, f), (f, None, f, 1, 2, f), (f, f, None, 1, 2, f), (f, f, f, 1, 2, None)):
        assert L.scsfm_camera_grad_indexed(*args, None) == -1
        assert b"camera_grad_indexed" in L.scsfm_last_error() and b"null" in L.scsfm_last_error()
    assert L.scsfm_camera_grad_indexed(f, f, f, 1, 0, f, None) == -1
    assert b"number of cameras" in L.scsfm_last_error()
    assert L.scsfm_camera_grad_indexed(f, f, f, -1, 4, f, None) == -1
    assert b"batch size" in L.scsfm_last_error()
    assert lib.launch_count() == n0


def test_python_bank_checks_before_any_launch():
    import torch
    from scsfm import camera
    from scsfm import lib
    n0 = lib.launch_count()
    rec = torch.zeros(3, 6, dtype=torch.float64)
    with pytest.raises(RuntimeError, match="CUDA"):
        camera.build(torch.zeros(2, 4), rec, torch.zeros(3, dtype=torch.int32))
    with pytest.raises(TypeError, match="bank"):
        camera.LearnedCamera.bank(torch.zeros(4))
    with pytest.raises(ValueError, match="labels"):
        camera.LearnedCamera.bank(torch.zeros(2, 4), groups=["a"])
    bank = camera.LearnedCamera.bank([[1, 2, 3, 4], [5, 6, 7, 8]], 10, 20, groups=["a", "b"])
    assert tuple(bank.theta.shape) == (2, 4) and bank.groups == ["a", "b"]
    assert sorted(bank.state_dict()) == ["height", "theta", "width"] and int(bank.width) == 20
    assert camera.LearnedCamera.bank([[1, 2, 3, 4]]).groups == ["camera 0"]
    assert lib.launch_count() == n0


@pytest.mark.parametrize("kind,H,W", [("kitti", 256, 832), ("nyu", 256, 320)])
@pytest.mark.parametrize("seed", [0, 1])
def test_indexed_build_restated_equals_update_intrinsics_of_each_samples_camera(kind, H, W, seed):
    from scsfm import synth
    from scsfm.augment import Draw, update_intrinsics
    from scsfm.camera import record_rows
    random.seed(seed)
    np.random.seed(seed)
    base = synth.intrinsics(1, H, W, kind)[0].numpy()
    Ks = [base, (base * np.array([[1.1, 1, 0.9], [1, 0.95, 1.05], [1, 1, 1]])).astype(np.float32),
          (base * np.array([[0.8, 1, 1.02], [1, 1.2, 0.97], [1, 1, 1]])).astype(np.float32)]
    thetas = [(K[0, 0], K[1, 1], K[0, 2], K[1, 2]) for K in Ks]
    draws = [Draw.random(H, W) for _ in range(60)]
    idx = np.random.randint(0, 3, len(draws))
    assert set(idx.tolist()) == {0, 1, 2}
    for d, r, c in zip(draws, record_rows(draws, W), idx):
        want = update_intrinsics(Ks[c], d, W).astype(np.float32)
        assert indexed_build(thetas, r, c).tobytes() == want.tobytes(), (c, d.flip, d.x_scaling)
    r = record_rows(draws[:1], W)[0]
    for bad in (-1, 3, 1 << 30):
        assert np.isnan(indexed_build(thetas, r, bad)).all()


# ---- train.py --camera-groups -------------------------------------------------------------------------------------------------
K_A = [[241.67, 0, 204.17], [0, 246.28, 59.0], [0, 0, 1]]
K_B = [[245.0, 0, 200.0], [0, 246.5, 61.0], [0, 0, 1]]


def _scenes(root, cams, val=()):
    """cams: ordered {scene: K} written as <scene>/cam.txt, train.txt listing them in that order; val: validation scenes."""
    os.makedirs(root, exist_ok=True)
    with open(os.path.join(root, "train.txt"), "w") as f:
        f.write("".join(s + "\n" for s in cams if s not in val))
    with open(os.path.join(root, "val.txt"), "w") as f:
        f.write("".join(s + "\n" for s in val))
    for s, K in cams.items():
        os.makedirs(os.path.join(root, s), exist_ok=True)
        np.savetxt(os.path.join(root, s, "cam.txt"), np.asarray(K, np.float32))
    return root


def _parse(*argv):
    import train as T
    return T.parser.parse_args(list(argv))


def _theta(K):
    K = np.asarray(K, np.float32)
    return [float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])]


# 4 scenes, 2 calibrations, listed B-first so that the table's order is the train.txt order, not the calibration's
FOUR = {"2011_09_28_drive_0001_sync_02": K_B, "2011_09_26_drive_0001_sync_02": K_A, "2011_09_26_drive_0002_sync_03": K_A,
        "2011_09_28_drive_0002_sync_03": K_B}


def test_camera_groups_default_to_a_one_camera_table():
    import train as T
    a = _parse("synthetic", "--name", "x")
    assert a.camera_groups == "one"
    assert T.check_learn_intrinsics(a) is None
    # with 'one' the table holds one camera, learned as theta [4] with no group labels
    a = _parse("synthetic", "--name", "x", "--learn-intrinsics", "1", "--gpu-augment", "1")
    t = T.check_learn_intrinsics(a)
    assert isinstance(t, T.CameraTable) and t.mode == "one" and len(t) == 1
    cam = t.camera(None, 256, 832)
    assert tuple(cam.theta.shape) == (4,) and cam.groups is None


def test_camera_groups_refusals(tmp_path):
    import train as T
    data = _scenes(str(tmp_path / "d"), FOUR)
    for g in ("calibration", "scene"):
        with pytest.raises(SystemExit, match="--learn-intrinsics 1"):
            T.check_learn_intrinsics(_parse(data, "--name", "x", "--camera-groups", g))
        with pytest.raises(SystemExit, match="--gpu-augment 1"):
            T.check_learn_intrinsics(_parse(data, "--name", "x", "--camera-groups", g, "--learn-intrinsics", "1", "--gpu-augment", "0"))
        with pytest.raises(SystemExit, match="synthetic has one camera"):
            T.check_learn_intrinsics(_parse("synthetic", "--name", "x", "--camera-groups", g, "--learn-intrinsics", "1", "--gpu-augment", "1"))
        with pytest.raises(SystemExit, match="positive"):
            T.check_learn_intrinsics(_parse(data, "--name", "x", "--camera-groups", g, "--learn-intrinsics", "1", "--intrinsics-init",
                                            "0", "1", "2", "3"))
    # 'one' keeps its refusal of several cameras, now with a hint
    with pytest.raises(SystemExit, match="ONE camera.*several cameras are not supported.*--camera-groups calibration"):
        T.check_learn_intrinsics(_parse(data, "--name", "x", "--learn-intrinsics", "1"))


def test_calibration_groups_follow_train_txt(tmp_path):
    import train as T
    data = _scenes(str(tmp_path / "d"), FOUR)
    t = T.check_learn_intrinsics(_parse(data, "--name", "x", "--learn-intrinsics", "1", "--camera-groups", "calibration"))
    assert isinstance(t, T.CameraTable) and len(t) == 2
    assert t.labels == ["2011_09_28_drive_0001_sync_02/cam.txt", "2011_09_26_drive_0001_sync_02/cam.txt"]
    assert t.thetas() == [_theta(K_B), _theta(K_A)]
    assert [K.tobytes() for K in t.Ks] == [np.asarray(K, np.float32).tobytes() for K in (K_B, K_A)]
    # a sample's key: its float32 intrinsics
    assert t.index({"intrinsics": np.asarray(K_A, np.float32), "tgt": "x"}) == 1
    assert t.index({"intrinsics": np.asarray(K_B, np.float64), "tgt": "x"}) == 0
    assert t.index({"intrinsics": np.eye(3, dtype=np.float32), "tgt": "x"}) == -1


def test_scene_groups_give_one_camera_per_scene(tmp_path):
    import train as T
    data = _scenes(str(tmp_path / "d"), FOUR)
    t = T.check_learn_intrinsics(_parse(data, "--name", "x", "--learn-intrinsics", "1", "--camera-groups", "scene"))
    assert len(t) == 4 and t.labels == list(FOUR)
    assert t.thetas() == [_theta(K) for K in FOUR.values()]
    for c, s in enumerate(FOUR):
        assert t.index({"intrinsics": np.eye(3), "tgt": os.path.join(data, s, "0000001.jpg")}) == c
    assert t.index({"intrinsics": np.eye(3), "tgt": os.path.join(data, "other", "0000001.jpg")}) == -1


def test_intrinsics_init_sets_every_camera(tmp_path):
    import train as T
    data = _scenes(str(tmp_path / "d"), FOUR)
    for g, n in (("calibration", 2), ("scene", 4)):
        a = _parse(data, "--name", "x", "--learn-intrinsics", "1", "--camera-groups", g, "--intrinsics-init", "240", "250", "200", "60")
        t = T.check_learn_intrinsics(a)
        assert t.thetas(a.intrinsics_init) == [[240.0, 250.0, 200.0, 60.0]] * n


def test_table_does_not_depend_on_the_shuffle_seed(tmp_path):
    import train as T
    data = _scenes(str(tmp_path / "d"), FOUR)
    tables = []
    for seed in ("0", "7"):
        t = T.check_learn_intrinsics(_parse(data, "--name", "x", "--learn-intrinsics", "1", "--camera-groups", "calibration",
                                            "--seed", seed))
        tables.append((t.keys, t.labels, t.thetas()))
    assert tables[0] == tables[1]


def test_pair_folder_groups_by_each_pairs_intrinsics_file(tmp_path):
    """--folder-type pair: one intrinsics file per image pair (datasets/pair_folders.py:37-42), so one scene may hold several
    calibrations; a file beyond the last pair is not read."""
    import train as T
    root = str(tmp_path / "p")
    layout = {"s1": [K_A, K_B], "s2": [K_B, K_A, np.eye(3)]}     # s2: 4 images -> 2 pairs, its third .txt is never read
    for s, Ks in layout.items():
        os.makedirs(os.path.join(root, s))
        for i in range(4):
            open(os.path.join(root, s, "%07d.jpg" % i), "wb").close()
        for i, K in enumerate(Ks):
            np.savetxt(os.path.join(root, s, "%07d.txt" % i), np.asarray(K, np.float32))
    with open(os.path.join(root, "train.txt"), "w") as f:
        f.write("s1\ns2\n")
    a = _parse(root, "--name", "x", "--learn-intrinsics", "1", "--camera-groups", "calibration", "--folder-type", "pair")
    t = T.check_learn_intrinsics(a)
    assert t.labels == [os.path.join("s1", "0000000.txt"), os.path.join("s1", "0000001.txt")]
    assert t.thetas() == [_theta(K_A), _theta(K_B)]
    t = T.check_learn_intrinsics(_parse(root, "--name", "x", "--learn-intrinsics", "1", "--camera-groups", "scene", "--folder-type", "pair"))
    assert t.labels == ["s1", "s2"] and t.thetas() == [_theta(K_A), _theta(K_B)]


def test_reference_loaders_map_every_sample_to_its_camera(tmp_path):
    """Through the reference's own SequenceFolder and PairFolder (two shuffle seeds): RawFrames with the table's groups hands out
    (frames, K, group) with K the group's intrinsics, the same index for a sample whatever the shuffle, and validation samples of
    an unseen calibration get -1."""
    from helpers import make_disk_dataset, reference_loader_env
    env = reference_loader_env()
    if env is None:
        pytest.skip("the original project's modules are not installed (oracle/_ref/, made by __graft_entry__.build())")
    data = make_disk_dataset(str(tmp_path / "data"), H=64, W=96, scenes=("a", "b", "c", "d", "v"), frames=3)
    Ks = {"a": K_B, "b": K_A, "c": K_A, "d": K_B, "v": [[100.0, 0, 48], [0, 100, 32], [0, 0, 1]]}
    for s, K in Ks.items():
        np.savetxt(os.path.join(data, s, "cam.txt"), np.asarray(K, np.float32))
    code = ("import sys, os; sys.path.insert(0, %r)\n"
            "import numpy as np, train as T\n"
            "SF = T._reference_dataset_module('sequence_folders').SequenceFolder\n"
            "for g in ('calibration', 'scene'):\n"
            "    table = T.CameraTable(%r, g)\n"
            "    by_tgt = []\n"
            "    for seed in (0, 5):\n"
            "        ds = SF(%r, seed=seed, train=True, sequence_length=3)\n"
            "        rf = T.RawFrames(ds, [table.index(s) for s in ds.samples])\n"
            "        m = {}\n"
            "        for i, s in enumerate(ds.samples):\n"
            "            frames, K, c = rf[i]\n"
            "            assert K.tobytes() == table.Ks[c].tobytes() or g == 'scene', (g, c)\n"
            "            assert g == 'calibration' or table.labels[c] == os.path.basename(os.path.dirname(s['tgt'])), (c, s['tgt'])\n"
            "            m[str(s['tgt'])] = c\n"
            "        by_tgt.append(m)\n"
            "    assert by_tgt[0] == by_tgt[1]\n"
            "    val = SF(%r, seed=0, train=False, sequence_length=3)\n"
            "    print('MAP', g, len(table), sorted(set(by_tgt[0].values())), sorted({table.index(s) for s in val.samples}))\n"
            "PF = T._reference_dataset_module('pair_folders').PairFolder\n"
            "table = T.CameraTable(%r, 'calibration', 'pair')\n"
            "ds = PF(%r, seed=3, train=True)\n"
            "print('PAIR', len(table), sorted({table.index(s) for s in ds.samples}))\n"
            % (PKG, data, data, data, data, data))
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600, env=env)
    assert out.returncode == 0, out.stderr[-3000:]
    lines = out.stdout.strip().splitlines()
    assert lines[0] == "MAP calibration 2 [0, 1] [-1]", lines
    assert lines[1] == "MAP scene 4 [0, 1, 2, 3] [-1]", lines
    # (PairFolder reads one .txt per pair: cam.txt is the only .txt of each scene, so every scene's single pair maps to it)
    assert lines[2] == "PAIR 2 [0, 1]", lines
