"""The offline evaluation on the device: scsfm_eval_depth (through scsfm.loss_ops.eval_depth) against the numpy oracle per
image, chunk-size invariance, and eval_depth.py / test_pose.py end to end.  Needs a GPU."""
import os

import numpy as np
import pytest
import torch

from golden_util import det_weights

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KITTI_SIZES = [(375, 1242), (370, 1226), (374, 1238), (376, 1241)]


def _preds(g, n, h, w):
    p = np.exp(g.normal(2.5, 0.5, (n, h, w)))
    p[:, h // 2:h // 2 + 8, w // 8:w // 8 + 20] *= 1e-5          # below min_depth after scaling
    p[:, -12:-4, w // 2:w // 2 + 20] *= 1e5                      # above max_depth after scaling
    return p


def _kitti(g, dtype, n=4):
    preds = _preds(g, n, 256, 832)
    gts = []
    for k in range(n):
        H, W = KITTI_SIZES[k % 4]
        gt = np.where(g.random((H, W)) < 0.05, g.uniform(0.5, 90, (H, W)), 0).astype(dtype)
        gt[H - 20, 100:110] = np.float32(1e-3) if dtype == np.float32 else 1e-3          # excluded (not > 1e-3 in the dtype)
        gt[H - 19, 100:110] = np.nextafter(dtype(80), dtype(0))                          # kept: just below 80
        gts.append(gt)
    return preds, gts


def _nyu(g, dtype, n=2):
    preds = _preds(g, n, 256, 320)
    gts = [g.uniform(0.3, 11, (480, 640)).astype(dtype) for _ in range(n)]
    return preds, gts


def _small(g, dtype, counts):
    """16x20 ground truths with exactly `counts[k]` valid pixels (NYU mask: whole image)."""
    preds = _preds(g, len(counts), 8, 10)
    gts = []
    for c in counts:
        gt = np.zeros((16, 20), dtype)
        pos = g.choice(16 * 20, c, replace=False)
        gt.reshape(-1)[pos] = g.uniform(0.5, 9, c)
        gts.append(gt)
    return preds, gts


def _ties(g, dtype):
    preds, gts = _nyu(g, dtype, 2)
    preds = np.round(preds * 2) / 2 + 0.5
    return preds, [(np.round(x * 4) / 4).astype(dtype) for x in gts]


def _check(rows, preds, gts, dataset):
    from oracle import evaluation as E
    assert rows.shape == (len(preds), 12)
    for i in range(len(preds)):
        want = E.eval_depth_image(preds[i], gts[i], dataset)
        got = rows[i]
        if want[0] == 0:
            assert got[0] == 0 and np.isnan(got[1:]).all(), got
            continue
        # n, both medians and the ratio: bitwise
        assert got[:4].tobytes() == want[:4].tobytes(), (i, got[:4], want[:4])
        for c in ("abs_rel", "sq_rel", "rmse"):
            k = E.COLUMNS.index(c)
            assert abs(got[k] - want[k]) <= 1e-12 * abs(want[k]), (i, c, got[k], want[k])      # fp64 summation order
        for c in ("rmse_log", "log10"):
            # the device's and numpy's log of a float32 ground truth may differ by one float32 ulp (<= 4.8e-7 below 80): relative
            # 1e-6, with that ulp as a floor where the scaled prediction equals the ground truth (n = 1, 2: the metric is ulp noise)
            k = E.COLUMNS.index(c)
            floor = 4.8e-7 if gts[i].dtype == np.float32 else 1e-15
            assert abs(got[k] - want[k]) <= 1e-6 * abs(want[k]) + floor, (i, c, got[k], want[k])
        for c in ("a1", "a2", "a3"):
            k = E.COLUMNS.index(c)
            assert got[k] == want[k], (i, c, got[k], want[k])


CASES = {
    "kitti_f32_four_sizes": lambda g: ("kitti",) + _kitti(g, np.float32),
    "kitti_f64_four_sizes": lambda g: ("kitti",) + _kitti(g, np.float64),
    "nyu_f32": lambda g: ("nyu",) + _nyu(g, np.float32),
    "nyu_f64": lambda g: ("nyu",) + _nyu(g, np.float64),
    "n_0_1_2_odd_even_f32": lambda g: ("nyu",) + _small(g, np.float32, [0, 1, 2, 7, 8, 320]),
    "n_0_1_2_odd_even_f64": lambda g: ("nyu",) + _small(g, np.float64, [0, 1, 2, 31, 64, 319]),
    "ties_f32": lambda g: ("nyu",) + _ties(g, np.float32),
    "ties_f64": lambda g: ("nyu",) + _ties(g, np.float64),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_eval_depth_kernel_matches_the_oracle(case):
    from scsfm import loss_ops
    dataset, preds, gts = CASES[case](np.random.default_rng(sorted(CASES).index(case)))
    rows = loss_ops.eval_depth(preds, gts, dataset)
    _check(rows, preds, gts, dataset)


@pytest.mark.parametrize("name", ["kitti32", "kitti64", "nyu32", "nyu64"])
def test_eval_depth_kernel_on_the_golden_cases(name):
    from scsfm import loss_ops
    z = np.load(os.path.join(ROOT, "tests", "golden", "eval.npz"))
    preds = z[name + "_pred"]
    gts = [z[name + "_gt%d" % k] for k in range(len(preds))]
    keep = [i for i in range(len(preds)) if preds[i].mean() != -1]
    rows = loss_ops.eval_depth(preds, gts, name[:-2], indices=keep)
    _check(rows, preds[keep], [gts[i] for i in keep], name[:-2])


def test_results_do_not_depend_on_the_chunk_size():
    from scsfm import loss_ops
    g = np.random.default_rng(42)
    preds, gts = _kitti(g, np.float32, n=9)
    rows = [loss_ops.eval_depth(preds, gts, "kitti", chunk=c) for c in (1, 7, 9)]
    assert rows[0].tobytes() == rows[1].tobytes() == rows[2].tobytes()
    sub = loss_ops.eval_depth(preds, gts + [np.zeros((3, 3), np.float64)], "kitti", indices=[5, 2])    # extra ground truth ignored
    assert sub.tobytes() == rows[0][[5, 2]].tobytes()


def test_eval_depth_script_end_to_end(tmp_path, capsys):
    import eval_depth
    from oracle import evaluation as E
    g = np.random.default_rng(5)
    preds, gts = _kitti(g, np.float32, n=5)
    preds[3] = -1                                                    # skipped
    np.save(tmp_path / "pred.npy", preds)
    (tmp_path / "gt").mkdir()
    for k, gt in enumerate(gts + [gts[0]]):                          # one ground truth more than predictions: ignored
        np.save(tmp_path / "gt" / ("%010d.npy" % k), gt)
    eval_depth.main(["--dataset", "kitti", "--pred_depth", str(tmp_path / "pred.npy"), "--gt_depth", str(tmp_path / "gt"),
                     "--ratio_name", str(tmp_path / "ratios.txt")])
    out = capsys.readouterr().out
    rows, _ = E.eval_depth(preds, gts, "kitti")
    lines, ratios = eval_depth.report(rows, "kitti")
    assert out == "==> Evaluating depth result...\n" + "\n".join(lines) + "\n"
    np.savetxt(tmp_path / "want.txt", ratios, fmt='%.4f')
    assert open(tmp_path / "ratios.txt").read() == open(tmp_path / "want.txt").read()
    # NYU: one [N,H,W] file
    preds, gts = _nyu(g, np.float32, 3)
    np.save(tmp_path / "pn.npy", preds)
    np.save(tmp_path / "gn.npy", np.stack(gts))
    eval_depth.main(["--dataset", "nyu", "--pred_depth", str(tmp_path / "pn.npy"), "--gt_depth", str(tmp_path / "gn.npy")])
    rows, _ = E.eval_depth(preds, gts, "nyu")
    assert capsys.readouterr().out == "==> Evaluating depth result...\n" + "\n".join(eval_depth.report(rows, "nyu")[0]) + "\n"


def _pose_fixture(tmp_path, n=9):
    import models
    from PIL import Image
    rng = np.random.default_rng(11)
    seq = tmp_path / "sequences" / "09" / "image_2"
    seq.mkdir(parents=True)
    base = rng.uniform(0, 255, (60, 200, 3))
    base = np.kron(base, np.ones((8, 8, 1)))                      # 480 x 1600, smooth-ish
    for i in range(n):
        im = np.clip(base[40 + i:40 + i + 376, 10 * i:10 * i + 1241] + rng.normal(0, 5, (376, 1241, 3)), 0, 255).astype(np.uint8)
        Image.fromarray(im).save(seq / ("%06d.png" % i))
    (tmp_path / "poses").mkdir()
    poses = np.tile(np.eye(4)[:3], (n, 1, 1))
    poses[:, :, 3] = np.cumsum(rng.normal(0, 1, (n, 3)), 0)
    np.savetxt(tmp_path / "poses" / "09.txt", poses.reshape(n, 12), fmt="%.6e")
    pose = models.PoseResNet(18, False)
    pose.load_state_dict(det_weights(pose.state_dict()))
    torch.save({"epoch": 1, "state_dict": pose.state_dict()}, tmp_path / "pose.tar")
    return pose, sorted(seq.iterdir())


def test_test_pose_end_to_end(tmp_path, capsys):
    import test_pose
    from inverse_warp import pose_vec2mat
    from oracle import evaluation as E
    from oracle import nets as ON
    from scsfm import inference_io as io
    from scsfm.infer import Predictor
    pose, files = _pose_fixture(tmp_path)
    preds, errs = test_pose.main(["--dataset-dir", str(tmp_path), "--output-dir", str(tmp_path / "out"), "--batch-size", "3",
                                  str(tmp_path / "pose.tar")])
    out = capsys.readouterr().out
    assert "9 snippets to test" in out and "Results" in out
    saved = np.load(tmp_path / "out" / "predictions.npy")
    assert saved.shape == (9, 5, 3, 4) and saved.dtype == np.float64 and (saved[5:] == 0).all() and (errs[5:] == 0).all()
    np.testing.assert_array_equal(saved, preds)
    mean = errs.mean(0)
    assert "mean \t {:10.4f}, {:10.4f}".format(*mean) in out            # the zero rows are part of the mean
    # the deduplicated batched path against per-snippet batch-1 calls (the reference's call pattern)
    frames = [io.load_frame(str(f), 256, 832) for f in files]
    net = pose.to(DEV).set_conv_mode("tf32x3").eval()
    pred = Predictor(net)
    with torch.no_grad():
        for j in range(5):
            mats = [pose_vec2mat(pred(io.network_input(frames[a][None]), io.network_input(frames[a + 1][None]))).cpu().numpy()[0]
                    for a in range(j, j + 4)]
            np.testing.assert_allclose(preds[j], io.integrate(np.stack(mats)).reshape(5, 3, 4), rtol=0, atol=1e-6)
    # ATE / RE against the oracle network (fp64) fed the same decoded frames, through the reference's per-snippet loop
    ref = ON.PoseResNet(18).double().to(DEV)
    ref.load_state_dict({k: v.double() for k, v in det_weights(ON.PoseResNet(18).state_dict()).items()})
    ref.eval()
    x = torch.stack([io.network_input(f[None])[0] for f in frames]).double()
    gt = io.read_poses(str(tmp_path / "poses" / "09.txt"))
    with torch.no_grad():
        trajs, want = E.evaluate_pose_sequence(x, gt, ref)
    np.testing.assert_allclose(errs[:5], want, rtol=1e-4, atol=0)
    assert np.abs(preds[:5] - trajs).max() <= 1e-4 * np.abs(trajs).max()         # tf32x3 network against fp64, composed
