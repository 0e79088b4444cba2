"""Writes tests/golden/prepare.npz: what the UNMODIFIED reference's data/prepare_train_data.py writes for small synthetic
KITTI raw, KITTI odometry and Cityscapes trees (tests/golden/prepare_trees.py), and generate_depth_map on extra clouds.

    python tests/golden/make_golden_prepare.py /path/to/SC-SfMLearner-Release

The reference needs packages that no longer run on NumPy 2 / SciPy >= 1.3, so they are shimmed here and only here:
np.int -> int; scipy.misc.imread -> np.asarray(PIL.Image.open(path)), imresize(img, (h, w)) -> PIL BILINEAR resize to
(w, h) (what SciPy did for uint8 RGB arrays: bytescale leaves them unchanged), imsave -> PIL save (default JPEG settings);
path.Path -> a small str subclass with the methods the loaders call (listing in sorted order); pebble -> unused
(--num-threads 1).  The validation split: the reference iterates a set of scene prefixes, so its draws depend on
PYTHONHASHSEED; the run below gives its module a `set` that returns the sorted prefixes, the order this project uses.

Recorded per run: every written file's bytes for the text files (cam.txt, poses.txt, train.txt, val.txt), the .npy depth
maps as arrays and a SHA-256 of every file.  The trees are built in a directory without underscores in its path
(cityscapes_loader.py splits the camera file's full path on '_').
"""
import builtins
import hashlib
import io
import json
import os
import runpy
import shutil
import sys
import tempfile
import types

import numpy as np

sys.dont_write_bytecode = True
HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.path.abspath(sys.argv[1])
sys.path[:0] = [HERE, os.path.join(REF, "data")]

import prepare_trees as T  # noqa: E402
from PIL import Image  # noqa: E402


class Path(str):
    def __truediv__(self, o):
        return Path(os.path.join(str(self), str(o)))

    def __add__(self, o):
        return Path(str(self) + str(o))

    def realpath(self):
        return Path(os.path.realpath(self))

    def dirname(self):
        return Path(os.path.dirname(self))

    @property
    def parent(self):
        return self.dirname()

    @property
    def name(self):
        return Path(os.path.basename(self))

    def basename(self):
        return self.name

    def isfile(self):
        return os.path.isfile(self)

    def makedirs_p(self):
        os.makedirs(self, exist_ok=True)
        return self

    mkdir_p = makedirs_p

    def _list(self, pattern, want_dir):
        import fnmatch
        out = [Path(os.path.join(self, f)) for f in sorted(os.listdir(self)) if os.path.isdir(os.path.join(self, f)) == want_dir]
        return [p for p in out if pattern is None or fnmatch.fnmatch(os.path.basename(p), pattern)]

    def files(self, pattern=None):
        return self._list(pattern, False)

    def dirs(self, pattern=None):
        return self._list(pattern, True)

    def rmtree(self):
        shutil.rmtree(self)

    def remove_p(self):
        if os.path.exists(self):
            os.remove(self)


def install_shims():
    np.int = int
    sys.modules["path"] = types.SimpleNamespace(Path=Path)
    sys.modules["pebble"] = types.SimpleNamespace(ProcessPool=None)
    import scipy.misc
    scipy.misc.imread = lambda p: np.asarray(Image.open(p))
    scipy.misc.imresize = lambda img, size: np.asarray(Image.fromarray(img).resize((size[1], size[0]), Image.BILINEAR))
    scipy.misc.imsave = lambda p, img: Image.fromarray(img).save(p)


def record(out, name, dump_root):
    files = T.dump_listing(dump_root)
    out[name + "_files"] = np.array(json.dumps({k: hashlib.sha256(v).hexdigest() for k, v in sorted(files.items())}))
    for k, v in sorted(files.items()):
        if k.endswith(".txt"):
            out[name + "_text_" + k] = np.array(v.decode())
        elif k.endswith(".npy"):
            out[name + "_npy_" + k] = np.load(io.BytesIO(v))
    print(name, len(files), "files,", sum(k.endswith(".jpg") for k in files), "jpg,", sum(k.endswith(".npy") for k in files), "npy")


def main():
    install_shims()
    test_scenes = [t.strip() for t in open(os.path.join(REF, "data", "test_scenes.txt")) if t.strip()]
    specs = T.make_specs(test_scenes)
    out = {"test_scenes": np.array(test_scenes)}
    for k, s in specs.items():
        out["spec_" + k] = np.array(json.dumps(s))
    tmp = os.path.join(tempfile.gettempdir(), "scsfmgolden%d" % os.getpid())
    assert "_" not in tmp
    os.makedirs(tmp)
    try:
        for k, s in specs.items():
            T.build(s, os.path.join(tmp, k))
        script = os.path.join(REF, "data", "prepare_train_data.py")
        for name, tree, flags in T.RUNS:
            root = os.path.join(tmp, tree)
            dump = os.path.join(tmp, "dump" + name.replace("_", ""))
            flags = [f.format(root=root) for f in flags]
            sys.argv = ["prepare_train_data.py", root] + flags + ["--dump-root", dump, "--num-threads", "1"]
            np.random.seed(0)
            runpy.run_path(script, init_globals={"set": lambda it: sorted(builtins.set(it))}, run_name="__main__")
            record(out, name, dump)
        # generate_depth_map alone on the extra clouds, ratios 1 and 2, through drive 0001's camera 02
        from kitti_raw_loader import KittiRawLoader
        drive = Path(os.path.join(tmp, "raw", "2011_09_26", "2011_09_26_drive_0001_sync"))
        for ratio in (1, 2):
            loader = KittiRawLoader(os.path.join(tmp, "raw"), img_height=16, img_width=48, get_depth=True, depth_size_ratio=ratio)
            scene = loader.collect_scenes(drive)[0]
            scene["frame_id"] = list(T.EXTRA_CLOUDS) + ["%010d" % i for i in range(3)]
            for i, fid in enumerate(scene["frame_id"]):
                out["depth_r%d_%s" % (ratio, fid)] = loader.generate_depth_map(scene, i)
            out["depth_r%d_P_rect" % ratio] = scene["P_rect"]
    finally:
        shutil.rmtree(tmp)
    path = os.path.join(HERE, "prepare.npz")
    np.savez_compressed(path, **out)
    print("wrote prepare.npz", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
