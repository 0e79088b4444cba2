"""CPU-side checks of the offline evaluation (eval_depth.py, test_pose.py): the numpy oracle against the reference's own
results (tests/golden/eval.npz, written by make_golden_eval.py), the oracle's resize against cv2, the host logic and flags of
both scripts, and the argument checks of scsfm_eval_depth (no launch on an error)."""
import ctypes
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "eval.npz")
CASES = ("kitti32", "kitti64", "nyu32", "nyu64")
REF_ORDER = {"kitti": ("abs_rel", "sq_rel", "rmse", "rmse_log", "a1", "a2", "a3"), "nyu": ("abs_rel", "log10", "rmse", "a1", "a2", "a3")}


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def case_inputs(golden, name):
    preds = golden[name + "_pred"]
    gts = [golden[name + "_gt%d" % k] for k in range(preds.shape[0])]
    return preds, gts, name[:-2]


def _threshold(pred, gt, dataset, ratio):
    """The oracle's per-pixel threshold max(gt/pred, pred/gt) of one image (for the a1-a3 tie rule)."""
    from oracle import evaluation as E
    H, W = gt.shape
    p = 1 / (E.resize_linear(1 / (pred + 1e-6), H, W) + 1e-6)
    m = E.mask_of(gt, dataset)
    v = np.clip(p[m] * ratio, E.MIN_DEPTH, E.MAX_DEPTH[dataset])
    return np.maximum(gt[m] / v, v / gt[m])


@pytest.mark.parametrize("name", CASES)
def test_oracle_depth_matches_the_reference(golden, name):
    from oracle import evaluation as E
    preds, gts, dataset = case_inputs(golden, name)
    rows, keep = E.eval_depth(preds, gts, dataset)
    ref = golden[name + "_errors"]
    assert keep == [i for i in range(len(preds)) if i != 2]             # image 2 is the skip marker
    assert rows.shape[0] == ref.shape[0] and (rows[:, 0] == ref[:, 0]).all()
    np.testing.assert_allclose(rows[:, 3], golden[name + "_ratios"], rtol=1e-12, atol=0)
    for j, col in enumerate(REF_ORDER[dataset]):
        got, want = rows[:, E.COLUMNS.index(col)], ref[:, 1 + j]
        if col in ("rmse_log", "log10"):
            np.testing.assert_allclose(got, want, rtol=1e-6, atol=0)     # logs of float32 ground truth in float32
        elif col in ("a1", "a2", "a3"):
            # equal, unless a pixel's threshold lies within 1e-12 of 1.25^k (cv2 and the restated resize differ by ~1e-13)
            k = int(col[1])
            for r, (g, w) in enumerate(zip(got, want)):
                if g != w:
                    th = _threshold(preds[keep[r]], gts[keep[r]], dataset, rows[r, 3])
                    near = np.sum(np.abs(th - 1.25 ** k) <= 1e-12 * 1.25 ** k)
                    assert abs(g - w) * rows[r, 0] <= near + 0.5, (name, col, r, g, w)
        else:
            np.testing.assert_allclose(got, want, rtol=1e-12, atol=0)
    # predictions beyond both clamp bounds after scaling, ground truth at float32(1e-3) / just below the maximum
    i0 = keep[0]
    p = 1 / (E.resize_linear(1 / (preds[i0] + 1e-6), *gts[i0].shape) + 1e-6)[E.mask_of(gts[i0], dataset)] * rows[0, 3]
    assert (p < E.MIN_DEPTH).any() and (p > E.MAX_DEPTH[dataset]).any()


def test_golden_cases_cover_odd_and_even_mask_sizes_in_both_dtypes(golden):
    for dt in ("32", "64"):
        n = np.concatenate([golden[c + "_errors"][:, 0] for c in CASES if c.endswith(dt)])
        assert {int(v) % 2 for v in n} == {0, 1}, dt


@pytest.mark.parametrize("name", CASES)
def test_script_report_reproduces_the_reference_output(golden, name):
    import eval_depth
    from oracle import evaluation as E
    preds, gts, dataset = case_inputs(golden, name)
    rows, _ = E.eval_depth(preds, gts, dataset)
    lines, ratios = eval_depth.report(rows, dataset)
    assert golden[name + "_stdout"].item() == "==> Evaluating depth result...\n" + "\n".join(lines) + "\n"
    import io
    buf = io.BytesIO()
    np.savetxt(buf, ratios, fmt='%.4f')
    assert buf.getvalue().decode() == golden[name + "_ratio_file"].item()


@pytest.mark.parametrize("shapes", [((256, 832), (375, 1242)), ((256, 832), (370, 1226)), ((256, 320), (480, 640))])
def test_oracle_resize_matches_cv2(shapes):
    cv2 = pytest.importorskip("cv2")
    from oracle import evaluation as E
    (h, w), (H, W) = shapes
    src = 1 / (np.random.default_rng(0).uniform(0.5, 80, (h, w)) + 1e-6)
    ref = cv2.resize(src, (W, H))
    got = E.resize_linear(src, H, W)
    assert np.max(np.abs(got - ref) / np.abs(ref)) <= 1e-12


def test_pose_host_logic_matches_the_reference(golden, tmp_path):
    from scsfm import inference_io as io
    snippets = golden["pose_snippets"]
    comp, pred, errs = golden["pose_compensated"], golden["pose_pred"], golden["pose_errors"]
    for seq in sorted({int(s) for s in snippets[:, 0]}):
        gt = golden["pose_gt_%02d" % seq]
        np.savetxt(tmp_path / "p.txt", gt.reshape(-1, 12), fmt="%.12e")
        np.testing.assert_array_equal(io.read_poses(str(tmp_path / "p.txt")), gt)
        rows = np.where(snippets[:, 0] == seq)[0]
        np.testing.assert_array_equal(io.snippet_indices(len(gt)), snippets[rows, 1:])
        for r in rows:
            np.testing.assert_array_equal(io.compensated_poses(gt, snippets[r, 1:]), comp[r])
            np.testing.assert_array_equal(np.array(io.pose_error(comp[r], pred[r])), errs[r])
    assert io.snippet_indices(3).shape == (0, 5) and io.snippet_indices(5).tolist() == [[0, 1, 2, 3, 4]]


def _pose_tree(root, lengths):
    from PIL import Image
    g = np.random.default_rng(3)
    for name, n in lengths.items():
        d = root / "sequences" / name / "image_2"
        d.mkdir(parents=True)
        for i in range(n):
            Image.fromarray(g.integers(0, 256, (4, 6, 3), dtype=np.uint8)).save(d / ("%06d.png" % i))
        (d / "ignored.jpg").write_bytes(b"")
        (root / "poses").mkdir(exist_ok=True)
        poses = np.tile(np.eye(4)[:3], (n, 1, 1))
        poses[:, :, 3] = g.normal(0, 1, (n, 3))
        np.savetxt(root / "poses" / (name + ".txt"), poses.reshape(n, 12))


def test_test_pose_sequence_order_and_zero_rows(tmp_path, capsys):
    import test_pose
    from scsfm import inference_io as io
    _pose_tree(tmp_path, {"10": 6, "09": 8, "11": 3, "20": 7})
    assert io.kitti_sequences(str(tmp_path), ["1*", "09"]) == ["09", "10", "11"]       # sorted, not set order
    seen = []

    def pair_mats(frames):
        seen.append(len(frames))
        m = np.tile(np.eye(4, dtype=np.float32)[:3], (len(frames) - 1, 1, 1))
        m[:, :, 3] = np.arange(1, len(frames))[:, None]
        return m

    preds, errs = test_pose.evaluate(str(tmp_path), ["1*", "09"], pair_mats, lambda f: np.zeros((4, 6, 3), np.uint8))
    assert seen == [8, 6]                               # each sequence's frames once (11 has no snippet), in sorted order
    assert "17 snippets to test" in capsys.readouterr().out
    n_snip = (8 - 4) + (6 - 4)
    assert preds.shape == (17, 5, 3, 4) and errs.shape == (17, 2) and errs.dtype == np.float32
    assert (preds[n_snip:] == 0).all() and (errs[n_snip:] == 0).all() and (preds[:n_snip, 0] == np.eye(4)[:3]).all()
    # snippet 1 of sequence 09 takes pairs 1..4: translations 2..5 composed
    np.testing.assert_allclose(preds[1, :, :, 3], -np.cumsum([[0, 0, 0], [2, 2, 2], [3, 3, 3], [4, 4, 4], [5, 5, 5]], 0))


def _defaults(parser, required):
    return vars(parser.parse_args(required))


def test_script_flags_keep_the_reference_defaults():
    import eval_depth
    import test_pose
    ed = _defaults(eval_depth.parser, ["--dataset", "kitti", "--pred_depth", "p.npy", "--gt_depth", "gt"])
    assert ed == dict(dataset="kitti", pred_depth="p.npy", gt_depth="gt", vis_dir=None, img_dir=None, ratio_name=None)
    for bad in (["--dataset", "cityscapes", "--pred_depth", "p", "--gt_depth", "g"], ["--dataset", "nyu", "--pred_depth", "p"]):
        with pytest.raises(SystemExit):
            eval_depth.parser.parse_args(bad)
    tp = _defaults(test_pose.parser, ["p.tar"])
    assert tp == dict(pretrained_posenet="p.tar", img_height=256, img_width=832, no_resize=False, min_depth=1e-3, max_depth=80,
                      dataset_dir=None, sequence_length=5, sequences=["09"], output_dir=None, img_exts=["png", "jpg", "bmp"],
                      rotation_mode="euler", conv_mode="tf32x3", batch_size=1)
    with pytest.raises(SystemExit):
        test_pose.parser.parse_args([])                  # the checkpoint is positional and required


def test_eval_depth_refuses_vis_dir_and_missing_ground_truth(tmp_path, capsys):
    import eval_depth
    from scsfm import lib
    n0 = lib.launch_count()
    np.save(tmp_path / "pred.npy", np.ones((3, 8, 8)))
    (tmp_path / "gt").mkdir()
    for k in range(2):
        np.save(tmp_path / "gt" / ("%d.npy" % k), np.ones((10, 10), np.float32))
    base = ["--dataset", "kitti", "--pred_depth", str(tmp_path / "pred.npy"), "--gt_depth", str(tmp_path / "gt")]
    with pytest.raises(SystemExit):
        eval_depth.main(base + ["--vis_dir", str(tmp_path / "vis")])
    err = capsys.readouterr().err
    assert "--vis_dir is not supported" in err and not (tmp_path / "vis").exists()
    with pytest.raises(SystemExit):
        eval_depth.main(base)
    err = capsys.readouterr().err
    assert "3 predictions" in err and "only 2 ground-truth depth maps" in err
    from scsfm import loss_ops
    with pytest.raises(ValueError, match="only 2 ground-truth"):
        loss_ops.eval_depth(np.ones((3, 8, 8)), [np.ones((10, 10), np.float32)] * 2, "kitti")
    with pytest.raises(TypeError, match="float64"):
        loss_ops.eval_depth(np.ones((3, 8, 8), np.float32), [np.ones((10, 10), np.float32)] * 3, "kitti")
    assert lib.launch_count() == n0


def test_eval_depth_kernel_rejects_bad_arguments_without_a_launch():
    from scsfm import lib
    L = lib.load()
    n0 = lib.launch_count()
    E = lib.EvalDepthImage
    P = ctypes.c_void_p(256)

    def call(imgs, n=None, min_d=1e-3, max_d=80.0, ws=1 << 20, h=8, w=8, gt_elems=10000, ptr=P, dtype=0):
        arr = (E * len(imgs))(*imgs)
        return L.scsfm_eval_depth(ptr, len(imgs) if n is None else n, h, w, P, dtype, gt_elems, arr, min_d, max_d, P, ws, P, None)

    good = E(0, 20, 30, 8, 20, 1, 29)
    assert L.scsfm_eval_depth_workspace_bytes((E * 1)(good), 1) == 256 + 12 * 28 * 16
    for kw, msg in ((dict(ptr=None), b"null"), (dict(n=0), b"non-positive"), (dict(h=0), b"non-positive"),
                    (dict(min_d=80.0), b"min_depth"), (dict(dtype=2), b"gt_dtype"), (dict(ws=100), b"workspace"),
                    (dict(gt_elems=599), b"outside the ground-truth")):
        assert call([good], **kw) == -1 and msg in L.scsfm_last_error(), kw
    for bad in (E(0, 20, 30, 8, 21, 1, 29), E(0, 20, 30, 8, 20, -1, 29), E(0, 20, 30, 9, 8, 1, 29), E(0, 0, 30, 0, 0, 0, 0)):
        assert call([good, bad]) == -1 and b"image 1" in L.scsfm_last_error()
    assert lib.launch_count() == n0
