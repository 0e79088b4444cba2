"""CPU-side checks of the inference additions: the eval-BatchNorm fields of the convolution descriptor, host-side argument
checks of the batched eval prepare (no launch on an error), the Predictor's input checks, and the host logic of the inference
scripts (flags and defaults, file discovery and output names, trajectory integration, colour maps)."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_conv_descriptor_eval_bn_fields_match_the_c_struct():
    from scsfm import nnops as O
    src = r'''
#include <stdio.h>
#include <stddef.h>
#include "scsfm.h"
int main(void) {
    printf("%zu %zu %zu %zu\n", sizeof(ScsfmConv), offsetof(ScsfmConv, bn_scale), offsetof(ScsfmConv, bn_shift),
           offsetof(ScsfmConv, out_lo));
    return 0;
}'''
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "t.c"), "-o", os.path.join(d, "t")])
        out = [int(v) for v in subprocess.check_output([os.path.join(d, "t")], text=True).split()]
    C = O.Conv
    assert out == [ctypes.sizeof(C), C.bn_scale.offset, C.bn_shift.offset, C.out_lo.offset]
    d = O.Conv()
    assert d.bn_scale is None and d.bn_shift is None and d.out_lo is None       # existing callers leave them NULL


def test_eval_prepare_rejects_bad_arguments_without_a_launch():
    from scsfm import lib
    from scsfm import nnops as O
    L = O._lib()
    n0 = lib.launch_count()
    assert L.scsfm_bn_eval_prepare_batched(None, 3, None) == -1 and b"bn_eval_prepare_batched" in L.scsfm_last_error()
    assert L.scsfm_bn_eval_prepare_batched(ctypes.c_void_p(256), 0, None) == -1
    assert lib.launch_count() == n0


def test_predictor_takes_only_this_package_s_networks():
    import torch
    from scsfm.infer import Predictor
    with pytest.raises(TypeError):
        Predictor(torch.nn.Conv2d(3, 3, 3))


# --- the inference scripts: flags and host logic -----------------------------------------------------------------------
def _script(name):
    import importlib
    return importlib.import_module(name)


def _defaults(parser, required):
    return vars(parser.parse_args(required))


def test_script_flags_keep_the_reference_defaults():
    ri = _defaults(_script("run_inference").parser, ["--pretrained", "w.tar", "--resnet-layers", "18"])
    assert ri == dict(output_disp=False, output_depth=False, pretrained="w.tar", img_height=256, img_width=832, no_resize=False,
                      dataset_list=None, dataset_dir=".", output_dir="output", img_exts=["png", "jpg", "bmp"], resnet_layers=18,
                      conv_mode="tf32x3", batch_size=1)
    td = _defaults(_script("test_disp").parser, ["--pretrained-dispnet", "d.tar", "--output-dir", "o", "--resnet-layers", "50"])
    assert td == dict(pretrained_dispnet="d.tar", img_height=256, img_width=832, min_depth=1e-3, max_depth=80, dataset_dir=".",
                      dataset_list=None, output_dir="o", resnet_layers=50, conv_mode="tf32x3", batch_size=1)
    tv = _defaults(_script("test_vo").parser, ["--pretrained-posenet", "p.tar"])
    assert tv == dict(pretrained_posenet="p.tar", img_height=256, img_width=832, no_resize=False, dataset_dir=None, output_dir=None,
                      img_exts=["png", "jpg", "bmp"], rotation_mode="euler", sequence="09", conv_mode="tf32x3", batch_size=1)
    for mod, req in (("run_inference", ["--pretrained", "w"]), ("test_disp", ["--pretrained-dispnet", "w", "--output-dir", "o"])):
        with pytest.raises(SystemExit):
            _script(mod).parser.parse_args(req)                    # --resnet-layers is required, as in the reference
    with pytest.raises(SystemExit):
        _script("test_vo").parser.parse_args(["--pretrained-posenet", "p", "--rotation-mode", "axis"])


def test_run_inference_without_an_output_kind_stops_before_loading(capsys):
    _script("run_inference").main(["--pretrained", "/nonexistent.tar", "--resnet-layers", "18"])
    assert "You must at least output one value !" in capsys.readouterr().out


def test_file_discovery_and_output_names(tmp_path):
    from scsfm import inference_io as io
    for n in ("b.png", "a.png", "c.jpg", "d.txt", "e.bmp"):
        (tmp_path / n).write_bytes(b"")
    (tmp_path / "sub.png").mkdir()
    got = [os.path.basename(p) for p in io.list_images(str(tmp_path), ["png", "jpg", "bmp"])]
    assert got == ["a.png", "b.png", "c.jpg", "e.bmp"]          # one glob per extension, in the order given
    assert io.output_name("/data/kitti/2011_09_26/0000000005.png", "/data/kitti", "_disp") == "2011_09_26-0000000005_disp.png"
    assert io.output_name("./x/y/z.jpg", ".", "_depth") == "x-y-z_depth.jpg"
    assert io.output_name("img.bmp", ".", "_disp") == "img_disp.bmp"
    assert io.batches(5, 2) == [(0, 2), (2, 4), (4, 5)]


def test_trajectory_integration_is_the_reference_loop():
    from scsfm import inference_io as io
    rng = np.random.default_rng(0)
    mats = []
    for _ in range(5):
        a = rng.normal(0, 0.05, 3)
        R = np.linalg.qr(np.eye(3) + np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]]))[0]
        mats.append(np.hstack([R * np.sign(np.diag(R)), rng.normal(0, 1, (3, 1))]).astype(np.float32))
    got = io.integrate(np.stack(mats))
    g, want = np.eye(4), [np.eye(4)[:3].reshape(12)]
    for m in mats:
        g = g @ np.linalg.inv(np.vstack([m, [0, 0, 0, 1]]))
        want.append(g[:3].reshape(12))
    assert got.shape == (6, 12) and got.dtype == np.float64
    np.testing.assert_array_equal(got, np.stack(want))
    assert io.integrate(np.zeros((0, 3, 4))).shape == (1, 12)


def test_colour_map_anchor_colours():
    from scsfm import inference_io as io
    rb = io.colorize(np.array([0.0, 0.4, 0.6, 0.8, 1.0, 3.0, -1.0]), 1.0, "rainbow")
    np.testing.assert_allclose(rb[:, :3], [[1, 0, 0], [1, 1, 0], [0, 1, 0], [0, 0, 1], [0.6, 0, 1], [0.6, 0, 1], [1, 0, 0]],
                               atol=6e-3)      # one step of the 1000-entry table, as matplotlib's lookup
    assert (rb[:, 3] == 1).all()
    bone = io.colorize(np.array([0.0, 1.0, 0.746032, 0.365079]), 1.0, "bone")
    np.testing.assert_allclose(bone[:, :3], [[0, 0, 0], [1, 1, 1], [0.652778, 0.777778, 0.746032 * 0.0 + 0.444444 + (1 - 0.444444) *
                                                                      (0.746032 - 0.365079) / (1 - 0.365079)],
                                              [0.365079 / 0.746032 * 0.652778, 0.319444, 0.444444]], atol=1e-3)
    with pytest.raises(ValueError):
        io.colorize(np.zeros(2), 1.0, "magma")
