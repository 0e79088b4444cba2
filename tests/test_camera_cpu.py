"""The learned camera, CPU side: the C ABI (one build and one gradient entry, scsfm_camera_build_indexed /
scsfm_camera_grad_indexed, whose null camera index means one camera; argument errors reported without a launch), the augmentation
record derived from a Draw (a numpy restatement of the build kernel's arithmetic reproduces update_intrinsics bit for bit), and
train.py's --learn-intrinsics validation."""
import ctypes
import os
import random
import re

import numpy as np
import pytest

from camera_helpers import kernel_build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_and_library_have_only_the_indexed_camera_entries():
    """The indexed entries are the only camera entries: the one-camera entries scsfm_camera_build / scsfm_camera_grad are gone."""
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "scsfm.h")).read(), flags=re.S)
    for name in ("scsfm_camera_build_indexed", "scsfm_camera_grad_indexed"):
        assert re.search(r"\b%s\s*\(" % name, src), name
    for name in ("scsfm_camera_build", "scsfm_camera_grad"):
        assert not re.search(r"\b%s\s*\(" % name, src), name
    assert re.search(r"#define SCSFM_CAMERA_AUG_DOUBLES 6\b", src)
    from scsfm import camera
    from scsfm import lib
    assert camera.AUG_DOUBLES == 6
    L = lib.load()
    assert hasattr(L, "scsfm_camera_build_indexed") and hasattr(L, "scsfm_camera_grad_indexed")
    assert not hasattr(L, "scsfm_camera_build") and not hasattr(L, "scsfm_camera_grad")


def test_null_camera_index_means_one_camera_and_bad_arguments_launch_nothing():
    """A null camera index passes the argument checks with one camera (the call below then fails on its batch size) and is
    refused with more; the other refusals hold for one camera as well."""
    from scsfm import camera
    from scsfm import lib
    L = camera._lib()
    n0 = lib.launch_count()
    fake = ctypes.c_void_p(16)            # never dereferenced: every call below fails its argument check first
    assert L.scsfm_camera_build_indexed(fake, 1, fake, None, 0, fake, None) == -1
    assert b"batch size" in L.scsfm_last_error()
    assert L.scsfm_camera_build_indexed(fake, 2, fake, None, 1, fake, None) == -1
    assert b"camera_build_indexed" in L.scsfm_last_error() and b"null idx" in L.scsfm_last_error()
    assert L.scsfm_camera_grad_indexed(fake, None, fake, 0, 1, fake, None) == -1
    assert b"batch size" in L.scsfm_last_error()
    assert L.scsfm_camera_grad_indexed(fake, None, fake, 1, 2, fake, None) == -1
    assert b"camera_grad_indexed" in L.scsfm_last_error() and b"null idx" in L.scsfm_last_error()
    assert L.scsfm_camera_build_indexed(None, 1, fake, None, 1, fake, None) == -1
    assert b"camera_build" in L.scsfm_last_error() and b"theta" in L.scsfm_last_error()
    assert L.scsfm_camera_build_indexed(fake, 1, None, None, 1, fake, None) == -1
    assert L.scsfm_camera_build_indexed(fake, 1, fake, None, 1, None, None) == -1
    assert L.scsfm_camera_build_indexed(fake, 1, fake, None, 0, fake, None) == -1
    assert b"batch size" in L.scsfm_last_error()
    assert L.scsfm_camera_grad_indexed(None, None, fake, 1, 1, fake, None) == -1
    assert b"camera_grad" in L.scsfm_last_error()
    assert L.scsfm_camera_grad_indexed(fake, None, None, 1, 1, fake, None) == -1
    assert L.scsfm_camera_grad_indexed(fake, None, fake, 1, 1, None, None) == -1
    assert L.scsfm_camera_grad_indexed(fake, None, fake, -3, 1, fake, None) == -1
    assert b"batch size" in L.scsfm_last_error()
    with pytest.raises(ValueError, match="camera_grad"):
        lib.check(L.scsfm_camera_grad_indexed(None, None, None, 1, 1, None, None), "scsfm_camera_grad_indexed")
    assert lib.launch_count() == n0


def test_python_wrappers_check_types_before_any_launch():
    import torch
    from scsfm import camera
    with pytest.raises(RuntimeError, match="CUDA"):
        camera.build(torch.zeros(4), torch.zeros(2, 6, dtype=torch.float64))


@pytest.mark.parametrize("kind,H,W", [("kitti", 256, 832), ("nyu", 256, 320)])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_records_of_draws_reproduce_update_intrinsics(kind, H, W, seed):
    """Seeded random draws (float64 zoom factors), with and without flip, plus the identity draw and given Python-float factors
    (which numpy multiplies in float32): the kernel arithmetic on the record equals update_intrinsics on the float32 matrix."""
    from scsfm import synth
    from scsfm.augment import Draw, update_intrinsics
    from scsfm.camera import record_rows
    random.seed(seed)
    np.random.seed(seed)
    K = synth.intrinsics(1, H, W, kind)[0].numpy()
    draws = [Draw.random(H, W) for _ in range(64)]
    assert {d.flip for d in draws} == {False, True}
    draws += [Draw.identity(H, W), Draw.given(H, W, True, 1.1, 1.07, 3, 2), Draw.given(H, W, False, 1.149, 1.0001, 0, 1)]
    theta = (K[0, 0], K[1, 1], K[0, 2], K[1, 2])
    rows = record_rows(draws, W)
    assert rows.dtype == np.float64 and rows.shape == (len(draws), 6)
    for d, r in zip(draws, rows):
        want = update_intrinsics(K, d, W).astype(np.float32)
        got = kernel_build(theta, r)
        assert got.tobytes() == want.tobytes(), (d.flip, d.x_scaling, d.y_scaling, got, want)
    # the identity draw leaves the camera as it is
    assert kernel_build(theta, rows[64]).tobytes() == K.astype(np.float32).tobytes()


def test_float64_factor_is_not_rounded_to_float32_first():
    """The two roundings differ for some products: the record keeps the float64 draw, so the restatement follows numpy."""
    from scsfm.augment import Draw, update_intrinsics
    from scsfm.camera import record_rows
    K = np.array([[483.4, 0, 408.3], [0, 492.6, 118.0], [0, 0, 1]], np.float32)
    differ = 0
    rng = np.random.RandomState(5)
    for _ in range(2000):
        xs, ys = rng.uniform(1, 1.15, 2)
        d = Draw.given(256, 832, False, xs, ys, 0, 0)
        r = record_rows([d], 832)[0]
        assert kernel_build((K[0, 0], K[1, 1], K[0, 2], K[1, 2]), r).tobytes() == update_intrinsics(K, d, 832).tobytes()
        differ += np.float32(np.float64(K[0, 0]) * xs) != np.float32(K[0, 0] * np.float32(xs))
    assert differ > 0


def _args(*extra):
    import train as T
    return T.parser.parse_args(["synthetic", "--name", "x"] + list(extra))


def test_train_flags_defaults():
    a = _args()
    assert a.learn_intrinsics == 0 and a.intrinsics_init is None and a.intrinsics_lr == 0.1
    import train as T
    assert T.check_learn_intrinsics(a) is None


def test_learn_intrinsics_needs_the_gpu_transforms():
    import train as T
    for extra in ([], ["--gpu-augment", "0"]):              # synthetic defaults to the host chain
        with pytest.raises(SystemExit, match="--gpu-augment 1"):
            T.check_learn_intrinsics(_args("--learn-intrinsics", "1", *extra))
    with pytest.raises(SystemExit, match="--gpu-augment 1"):
        T.check_learn_intrinsics(T.parser.parse_args(["some/dir", "--name", "x", "--learn-intrinsics", "1", "--gpu-augment", "0"]))


def test_learn_intrinsics_initial_camera_table():
    import train as T
    from scsfm import synth
    t = T.check_learn_intrinsics(_args("--learn-intrinsics", "1", "--gpu-augment", "1", "--synthetic-size", "128", "416"))
    K = synth.intrinsics(1, 128, 416)[0]
    assert t.mode == "one" and t.thetas() == [[float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])]]
    a = _args("--learn-intrinsics", "1", "--gpu-augment", "1", "--intrinsics-init", "100", "110", "60", "30")
    assert T.check_learn_intrinsics(a).thetas(a.intrinsics_init) == [[100.0, 110.0, 60.0, 30.0]]
    with pytest.raises(SystemExit, match="positive"):
        T.check_learn_intrinsics(_args("--learn-intrinsics", "1", "--gpu-augment", "1", "--intrinsics-init", "-100", "110", "60", "30"))


def _scenes(root, cams):
    os.makedirs(root, exist_ok=True)
    with open(os.path.join(root, "train.txt"), "w") as f:
        f.write("\n".join(cams) + "\n")
    for s, K in cams.items():
        os.makedirs(os.path.join(root, s), exist_ok=True)
        np.savetxt(os.path.join(root, s, "cam.txt"), np.asarray(K, np.float32))


K1 = [[241.67, 0, 204.17], [0, 246.28, 59.0], [0, 0, 1]]
K2 = [[245.0, 0, 200.0], [0, 246.28, 59.0], [0, 0, 1]]


def _theta(K):
    K = np.asarray(K, np.float32)
    return [float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])]


def test_one_camera_table_reads_the_scenes_and_refuses_several_cameras(tmp_path):
    import train as T
    one = str(tmp_path / "one")
    _scenes(one, {"seq_a": K1, "seq_b": K1})
    args = T.parser.parse_args([one, "--name", "x", "--learn-intrinsics", "1"])        # real data: GPU transforms by default
    t = T.check_learn_intrinsics(args)
    assert len(t) == 1 and t.thetas() == [_theta(K1)]
    assert t.camera(None, 10, 20).groups is None and tuple(t.camera(None, 10, 20).theta.shape) == (4,)
    two = str(tmp_path / "two")
    _scenes(two, {"seq_a": K1, "seq_b": K2})
    with pytest.raises(SystemExit, match="ONE camera.*seq_b"):
        T.check_learn_intrinsics(T.parser.parse_args([two, "--name", "x", "--learn-intrinsics", "1"]))
    # an explicit initial camera does not lift the one-camera rule
    with pytest.raises(SystemExit, match="ONE camera"):
        T.check_learn_intrinsics(T.parser.parse_args([two, "--name", "x", "--learn-intrinsics", "1", "--intrinsics-init", "240", "240",
                                                      "200", "60"]))


def test_learn_intrinsics_of_a_pair_folder_reads_its_pair_files(tmp_path):
    """--folder-type pair with one camera: the intrinsics files PairFolder reads (one per image pair; there is no cam.txt) are the
    ones checked and the camera starts from them."""
    import train as T
    root = str(tmp_path / "p")
    for s, Ks in {"s1": [K1, K1], "s2": [K1, K2]}.items():
        os.makedirs(os.path.join(root, s))
        for i in range(4):
            open(os.path.join(root, s, "%07d.jpg" % i), "wb").close()
        for i, K in enumerate(Ks):
            np.savetxt(os.path.join(root, s, "%07d.txt" % i), np.asarray(K, np.float32))
    with open(os.path.join(root, "train.txt"), "w") as f:
        f.write("s1\n")
    args = T.parser.parse_args([root, "--name", "x", "--learn-intrinsics", "1", "--folder-type", "pair"])
    assert T.check_learn_intrinsics(args).thetas() == [_theta(K1)]
    with open(os.path.join(root, "train.txt"), "w") as f:
        f.write("s1\ns2\n")
    with pytest.raises(SystemExit, match="ONE camera.*" + re.escape(os.path.join("s2", "0000001.txt"))):
        T.check_learn_intrinsics(args)
