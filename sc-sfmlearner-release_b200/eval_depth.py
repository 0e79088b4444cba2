"""Median-scaled depth evaluation of test_disp.py's predictions (the reference's eval_depth.py: same flags, the same printed
lines and the --ratio_name file).  Per image, the prediction's inverse is resized to the ground truth's size, masked,
median-scaled, clamped and scored on the device by scsfm_eval_depth (scsfm.loss_ops.eval_depth), in fp64 and with numpy's
medians; the ratio statistics and the mean over the images are computed here on the host, as the reference does.

KITTI ground truth is every *.npy of the --gt_depth directory in sorted order (one [H,W] map each, of any size); NYU is one
[N,H,W] .npy.  A prediction whose mean is -1 is skipped.  --vis_dir (visualisation with matplotlib's magma colour map) is not
supported and is refused before any work; --img_dir is only used by it."""
import argparse
import glob
import os

import numpy as np

parser = argparse.ArgumentParser(description="NYUv2 Depth options")
parser.add_argument("--dataset", required=True, help="kitti or nyu", choices=['nyu', 'kitti'], type=str)
parser.add_argument("--pred_depth", required=True, help="depth predictions npy", type=str)
parser.add_argument("--gt_depth", required=True, help="gt depth nyu for nyu or folder for kitti", type=str)
parser.add_argument("--vis_dir", help="result directory for saving visualization", type=str)
parser.add_argument("--img_dir", help="image directory for reading image", type=str)
parser.add_argument("--ratio_name", help="names for saving ratios", type=str)

NAMES = {"kitti": ("abs_rel", "sq_rel", "rmse", "rmse_log", "a1", "a2", "a3"), "nyu": ("abs_rel", "log10", "rmse", "a1", "a2", "a3")}


class _NpyFiles:
    """The KITTI ground-truth files, loaded when a chunk needs them."""

    def __init__(self, files):
        self.files = files

    def __len__(self):
        return len(self.files)

    def __getitem__(self, i):
        return np.load(self.files[i])


def report(rows, dataset):
    """The reference's printed lines from the per-image rows (scsfm.loss_ops.EVAL_COLUMNS): ratios, then the mean errors."""
    from scsfm.loss_ops import EVAL_COLUMNS
    ratios = rows[:, EVAL_COLUMNS.index("ratio")]
    med = np.median(ratios)
    errors = np.ascontiguousarray(rows[:, [EVAL_COLUMNS.index(c) for c in NAMES[dataset]]])
    mean_errors = errors.mean(0)
    n = len(NAMES[dataset])
    return [" Scaling ratios | med: {:0.3f} | std: {:0.3f}".format(med, np.std(ratios / med)),
            " Scaling ratios | mean: {:0.3f} +- std: {:0.3f}".format(np.mean(ratios), np.std(ratios)),
            "\n  " + ("{:>8} | " * n).format(*NAMES[dataset]),
            ("&{: 8.3f}  " * n).format(*mean_errors.tolist()) + "\\\\"], ratios


def main(argv=None):
    args = parser.parse_args(argv)
    if args.vis_dir:
        parser.error("--vis_dir is not supported: the visualisation needs matplotlib's magma colour map; run without it")
    pred_depths = np.load(args.pred_depth)
    if args.dataset == 'nyu':
        gt_depths = np.load(args.gt_depth)
    else:
        gt_depths = _NpyFiles(sorted(glob.glob(os.path.join(args.gt_depth, "*.npy"))))
    if len(gt_depths) < pred_depths.shape[0]:
        parser.error("%d predictions in %s but only %d ground-truth depth maps in %s" %
                     (pred_depths.shape[0], args.pred_depth, len(gt_depths), args.gt_depth))
    from scsfm.loss_ops import eval_depth

    print("==> Evaluating depth result...")
    keep = [i for i in range(pred_depths.shape[0]) if pred_depths[i].mean() != -1]
    rows = eval_depth(pred_depths, gt_depths, args.dataset, indices=keep)
    lines, ratios = report(rows, args.dataset)
    print(lines[0])
    print(lines[1])
    if args.ratio_name:
        np.savetxt(args.ratio_name, ratios, fmt='%.4f')
    print(lines[2])
    print(lines[3])
    return rows


if __name__ == '__main__':
    main()
