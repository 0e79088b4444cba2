"""Writes tests/golden/eval.npz: inputs and results of the UNMODIFIED reference evaluations on small synthetic data.

    python tests/golden/make_golden_eval.py /path/to/SC-SfMLearner-Release

Depth: the reference's eval_depth.py is imported with sys.argv pointing at synthetic prediction / ground-truth files (the import
runs its main once), then DepthEvalEigen().main() runs again for every case with the module's `args` replaced.  Its module-level
compute_depth_errors is wrapped to record each image's tuple and mask size, and a profile hook reads the `ratios` array of
evaluate_depth when it returns.  Printed lines and the --ratio_name file are recorded too.  cv2 and tqdm are the real
packages; path.py, matplotlib and imageio are the stand-ins under baseline/stubs.

Pose: read_scene_data / test_framework_KITTI (kitti_eval/pose_evaluation_utils.py) on a synthetic sequences/ + poses/ tree
give the snippet indices and the compensated ground truth; test_pose.py's compute_pose_error scores random trajectories.
"""
import contextlib
import io
import os
import sys
import tempfile
import types

import numpy as np

sys.dont_write_bytecode = True
HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
REF = os.path.abspath(sys.argv[1])
sys.path[:0] = [os.path.join(REPO, "baseline", "stubs"), REF]

# (name, dataset, gt dtype, prediction size, ground-truth sizes, seed)
KITTI_SIZES = [(75, 248), (74, 245), (75, 247), (75, 248), (74, 245), (75, 247)]
CASES = [("kitti32", "kitti", np.float32, (24, 80), KITTI_SIZES, 1),
         ("kitti64", "kitti", np.float64, (24, 80), KITTI_SIZES[::-1], 2),
         ("nyu32", "nyu", np.float32, (16, 20), [(30, 40)] * 4, 3),
         ("nyu64", "nyu", np.float64, (16, 20), [(30, 40)] * 3, 4)]


def make_case(dataset, dtype, hw, sizes, seed):
    """Predictions (float64, smooth with outlier blocks beyond both clamp bounds after scaling; image 2 is the skip marker -1)
    and ground truths (KITTI: ~5 % dense, with values at float32(1e-3), just below 80 and at 80; NYU: dense, some above 10)."""
    g = np.random.default_rng(seed)
    h, w = hw
    preds = np.exp(g.normal(2.0, 0.4, (len(sizes), h, w)))
    preds[:, h // 2:h // 2 + 4, w // 8:w // 8 + 10] *= 1e-5     # inside the KITTI crop
    preds[:, -6:-2, w // 2:w // 2 + 10] *= 1e5
    preds[2] = -1.0
    gts = []
    for k, (H, W) in enumerate(sizes):
        if dataset == "kitti":
            gt = np.where(g.random((H, W)) < 0.05 + 0.01 * k, g.uniform(0.5, 90, (H, W)), 0).astype(dtype)
            gt[H - 8, W // 3:W // 3 + 4] = np.float32(1e-3)
            gt[H - 7, W // 3:W // 3 + 4] = np.nextafter(np.float32(80), np.float32(0)) if dtype == np.float32 else np.nextafter(80, 0)
            gt[H - 6, W // 3:W // 3 + 4] = 80
        else:
            gt = g.uniform(0.2, 11, (H, W)).astype(dtype)
            gt[:2] = 0
            if k == 1:
                gt[:, :1] = 0                      # another count parity
        gts.append(gt)
    return preds, gts


def depth_golden(out, tmp):
    # the reference's eval_depth.py needs a valid command line at import time: its main() runs once there
    preds, gts = make_case(*CASES[0][1:])
    os.makedirs(os.path.join(tmp, "boot"), exist_ok=True)
    np.save(os.path.join(tmp, "boot", "pred.npy"), preds)
    for k, gt in enumerate(gts):
        np.save(os.path.join(tmp, "boot", "gt_%03d.npy" % k), gt)
    sys.argv = ["eval_depth.py", "--dataset", "kitti", "--pred_depth", os.path.join(tmp, "boot", "pred.npy"), "--gt_depth",
                os.path.join(tmp, "boot")]
    with contextlib.redirect_stdout(io.StringIO()):
        import eval_depth as E          # noqa: E402  (the reference's)
    orig = E.compute_depth_errors
    for name, dataset, dtype, hw, sizes, seed in CASES:
        preds, gts = make_case(dataset, dtype, hw, sizes, seed)
        d = os.path.join(tmp, name)
        os.makedirs(d)
        np.save(os.path.join(d, "pred.npy"), preds)
        if dataset == "kitti":
            for k, gt in enumerate(gts):
                np.save(os.path.join(d, "gt_%03d.npy" % k), gt)
            gt_arg = d
        else:
            gt_arg = os.path.join(d, "gt.npy")
            np.save(gt_arg, np.stack(gts))
        ratio_file = os.path.join(d, "ratios.txt")
        E.args = E.parser.parse_args(["--dataset", dataset, "--pred_depth", os.path.join(d, "pred.npy"), "--gt_depth", gt_arg,
                                      "--ratio_name", ratio_file])
        rec, ratios = [], {}

        def wrapped(gt, pred):
            r = orig(gt, pred)
            rec.append((gt.size,) + tuple(float(v) for v in r))
            return r

        def hook(frame, event, arg):
            if event == "return" and frame.f_code.co_name == "evaluate_depth":
                ratios["r"] = np.array(frame.f_locals["ratios"], np.float64)

        E.compute_depth_errors = wrapped
        buf = io.StringIO()
        sys.setprofile(hook)
        try:
            with contextlib.redirect_stdout(buf):
                E.DepthEvalEigen().main()
        finally:
            sys.setprofile(None)
            E.compute_depth_errors = orig
        p = name + "_"
        out[p + "pred"] = preds
        for k, gt in enumerate(gts):
            out[p + "gt%d" % k] = gt
        out[p + "errors"] = np.array(rec, np.float64)           # [n, then the tuple in the reference's order]
        out[p + "ratios"] = ratios["r"]
        out[p + "stdout"] = np.array(buf.getvalue())
        out[p + "ratio_file"] = np.array(open(ratio_file).read())
        print(name, "n =", [int(r[0]) for r in rec], "ratios", ratios["r"])


def _rot(g):
    a = g.normal(0, 0.2, 3)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    th = np.linalg.norm(a)
    return np.eye(3) + np.sin(th) / th * K + (1 - np.cos(th)) / th ** 2 * K @ K


def pose_golden(out, tmp):
    from PIL import Image
    sys.modules["skimage"] = types.ModuleType("skimage")
    sys.modules["skimage.transform"] = types.SimpleNamespace(resize=None)
    sys.argv = ["test_pose.py", "weights.tar"]
    import test_pose as TP                                       # noqa: E402  (the reference's)
    from kitti_eval import pose_evaluation_utils as PU           # noqa: E402
    g = np.random.default_rng(7)
    root = os.path.join(tmp, "odometry")
    lengths = {"09": 9, "10": 6, "11": 3, "20": 7}
    for name, n in lengths.items():
        d = os.path.join(root, "sequences", name, "image_2")
        os.makedirs(d)
        for i in range(n):
            Image.fromarray(g.integers(0, 256, (4, 6, 3), dtype=np.uint8)).save(os.path.join(d, "%06d.png" % i))
        os.makedirs(os.path.join(root, "poses"), exist_ok=True)
        poses = np.stack([np.hstack([_rot(g), g.normal(0, 5, (3, 1))]) for _ in range(n)])
        np.savetxt(os.path.join(root, "poses", name + ".txt"), poses.reshape(n, 12), fmt="%.12e")
        out["pose_gt_" + name] = np.genfromtxt(os.path.join(root, "poses", name + ".txt")).reshape(n, 3, 4)   # as read back
    patterns = ["09", "1*"]
    with contextlib.redirect_stdout(io.StringIO()):
        fw = PU.test_framework_KITTI(root, patterns, 5)
    names = [os.path.basename(os.path.dirname(os.path.dirname(f[0]))) for f in fw.img_files]
    out["pose_patterns"] = np.array(patterns)
    out["pose_len"] = np.array(len(fw))
    snips, comp, preds, errs = [], [], [], []
    it = iter(fw)
    for name, idx_all in zip(names, fw.sample_indices):
        for idx in idx_all:
            sample = next(it)
            snips.append([int(name)] + [int(i) for i in idx])
            comp.append(sample["poses"])
            pred = np.stack([np.hstack([_rot(g), g.normal(0, 1, (3, 1))]) for _ in range(5)])
            pred[0] = np.eye(4)[:3]
            preds.append(pred)
            errs.append(TP.compute_pose_error(sample["poses"], pred))
    out["pose_snippets"] = np.array(snips)                      # [sequence, 5 frame indices]
    out["pose_compensated"] = np.array(comp)
    out["pose_pred"] = np.array(preds)
    out["pose_errors"] = np.array(errs, np.float64)
    print("pose: sequences", names, "snippets", len(snips), "len(framework)", len(fw))


def main():
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        depth_golden(out, tmp)
        pose_golden(out, tmp)
    path = os.path.join(HERE, "eval.npz")
    np.savez_compressed(path, **out)
    print("wrote eval.npz", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
