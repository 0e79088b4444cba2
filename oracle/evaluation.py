"""Oracle: the reference's offline evaluations restated in numpy -- eval_depth.py (DepthEvalEigen.evaluate_depth with median
scaling, compute_depth_errors; eval_depth.py:32-56,159-227) and test_pose.py's per-snippet network loop (test_pose.py:50-83).

TEST INFRASTRUCTURE -- see oracle/__init__.py.  cv2.resize is restated as the separable fp64-weight bilinear resize
(`resize_linear`), which agrees with cv2 on float64 input to ~1e-13 relative; everything else is numpy with numpy's own dtype
behaviour (a float32 ground truth is masked, median-ed and log-ed in float32).
"""
import numpy as np

MIN_DEPTH = 1e-3
MAX_DEPTH = {"kitti": 80.0, "nyu": 10.0}
COLUMNS = ("n", "med_gt", "med_pred", "ratio", "abs_rel", "sq_rel", "rmse", "rmse_log", "log10", "a1", "a2", "a3")
REPORT = {"kitti": ("abs_rel", "sq_rel", "rmse", "rmse_log", "a1", "a2", "a3"), "nyu": ("abs_rel", "log10", "rmse", "a1", "a2", "a3")}


# --- depth -------------------------------------------------------------------------------------------------------------
def _taps(n_out, n_in):
    """One axis of cv2 INTER_LINEAR: source indices i0, i1 and fp64 weights w0, w1 of every output index."""
    f = (np.arange(n_out) + 0.5) * (n_in / n_out) - 0.5
    i = np.floor(f).astype(np.int64)
    a = f - i
    a = np.where(i < 0, 0.0, a)
    i = np.where(i < 0, 0, i)
    hi = i >= n_in - 1
    a = np.where(hi, 0.0, a)
    i = np.where(hi, n_in - 1, i)
    return i, np.minimum(i + 1, n_in - 1), 1 - a, a


def resize_linear(src, H, W):
    """cv2.resize(src, (W, H)) of a float64 map (INTER_LINEAR: half-pixel centres, edge clamp): horizontal pass, then vertical."""
    h, w = src.shape
    y0, y1, b0, b1 = _taps(H, h)
    x0, x1, a0, a1 = _taps(W, w)
    rows = src[:, x0] * a0 + src[:, x1] * a1
    return rows[y0] * b0[:, None] + rows[y1] * b1[:, None]


def eigen_crop(H, W):
    return np.array([0.40810811 * H, 0.99189189 * H, 0.03594771 * W, 0.96405229 * W]).astype(np.int32)


def mask_of(gt, dataset):
    """min_depth < gt < max_depth (numpy compares a float32 array with a Python float in float32), inside the KITTI crop."""
    mask = np.logical_and(gt > MIN_DEPTH, gt < MAX_DEPTH[dataset])
    if dataset == "kitti":
        c = eigen_crop(*gt.shape)
        crop = np.zeros(gt.shape, bool)
        crop[c[0]:c[1], c[2]:c[3]] = True
        mask &= crop
    return mask


def depth_metrics(gt, pred):
    """compute_depth_errors: {abs_rel, sq_rel, rmse, rmse_log, log10, a1, a2, a3} of the masked values."""
    thresh = np.maximum(gt / pred, pred / gt)
    return dict(abs_rel=np.mean(np.abs(gt - pred) / gt), sq_rel=np.mean(((gt - pred) ** 2) / gt),
                rmse=np.sqrt(((gt - pred) ** 2).mean()), rmse_log=np.sqrt(((np.log(gt) - np.log(pred)) ** 2).mean()),
                log10=np.mean(np.abs(np.log10(gt) - np.log10(pred))), a1=(thresh < 1.25).mean(), a2=(thresh < 1.25 ** 2).mean(),
                a3=(thresh < 1.25 ** 3).mean())


def eval_depth_image(pred, gt, dataset, resize=resize_linear):
    """One image of evaluate_depth: row of COLUMNS (NaN everywhere but n for an empty mask)."""
    H, W = gt.shape
    pred_depth = 1 / (resize(1 / (pred + 1e-6), H, W) + 1e-6)
    mask = mask_of(gt, dataset)
    val_pred, val_gt = pred_depth[mask], gt[mask]
    n = val_gt.size
    if n == 0:
        return np.array([0.0] + [np.nan] * (len(COLUMNS) - 1))
    med_gt, med_pred = np.median(val_gt), np.median(val_pred)
    ratio = med_gt / med_pred
    val_pred = val_pred * ratio
    val_pred[val_pred < MIN_DEPTH] = MIN_DEPTH
    val_pred[val_pred > MAX_DEPTH[dataset]] = MAX_DEPTH[dataset]
    m = depth_metrics(val_gt, val_pred)
    return np.array([n, med_gt, med_pred, ratio] + [m[c] for c in COLUMNS[4:]], np.float64)


def eval_depth(preds, gts, dataset, resize=resize_linear):
    """Rows of COLUMNS for the images whose prediction is not the skip marker (mean == -1), and their indices."""
    keep = [i for i in range(preds.shape[0]) if preds[i].mean() != -1]
    rows = [eval_depth_image(preds[i], gts[i], dataset, resize) for i in keep]
    return np.array(rows).reshape(len(keep), len(COLUMNS)), keep


def summary(rows, dataset):
    """The reference's report from the per-image rows: ratio statistics and the mean of the reported metrics."""
    ratios = rows[:, COLUMNS.index("ratio")]
    med = np.median(ratios)
    errors = np.ascontiguousarray(rows[:, [COLUMNS.index(c) for c in REPORT[dataset]]])
    return dict(ratios=ratios, med=med, std_rel=np.std(ratios / med), mean=np.mean(ratios), std=np.std(ratios),
                mean_errors=errors.mean(0))


# --- pose --------------------------------------------------------------------------------------------------------------
# The float64 host logic (snippets, compensation, composition, compute_pose_error) is the product's, scsfm.inference_io, which
# tests/test_eval_scripts_cpu.py checks against the reference's own functions; the oracle adds the reference's per-snippet loop.
def evaluate_pose_sequence(frames, gt_poses, pose_net):
    """The reference's per-snippet loop on one sequence: frames [N,3,H,W] normalised float32 torch tensors, gt_poses [N,3,4];
    pose_net(img1, img2) -> [1,6] (euler).  Every pair of every snippet runs through the network, at batch 1.
    Returns the snippet trajectories [n_snippets,5,3,4] and (ATE, RE) [n_snippets,2]."""
    from scsfm import inference_io as io
    from .geometry import pose_to_matrix
    trajs, errs = [], []
    for idx in io.snippet_indices(len(frames)):
        mats = [pose_to_matrix(pose_net(frames[a:a + 1], frames[a + 1:a + 2]))[0].detach().cpu().numpy().astype(np.float32)
                for a in idx[:-1]]
        traj = io.integrate(np.stack(mats)).reshape(-1, 3, 4)
        trajs.append(traj)
        errs.append(io.pose_error(io.compensated_poses(gt_poses, idx), traj))
    return np.array(trajs).reshape(-1, 5, 3, 4), np.array(errs, np.float64).reshape(-1, 2)
