"""torch.autograd wrappers over the fused loss kernels of libscsfm (csrc/warp_loss.cu, csrc/smooth.cu).

Each Function makes ONE forward launch and ONE backward launch for all pair-directions /
images of a training sample; no host synchronisation happens anywhere (the 10000-pixel
threshold of mean_on_mask is resolved on the device).
"""
import ctypes

import torch

from . import lib as L


_NO_IMAGE_GRAD = ("%s: gradients with respect to the IMAGES are not implemented (the training path never needs them: the reference "
                  "back-propagates into depths and poses only); detach the image tensors or use the reference's PyTorch code")


def _shift_of(full, part, what):
    s = 0
    while (part << s) < full:
        s += 1
    if (part << s) != full:
        raise ValueError("%s: depth size %d is not image size %d divided by a power of two" % (what, part, full))
    return s


def _flags(with_ssim, with_mask, with_auto_mask):
    # the reference compares the int flags with `== True` (loss_functions.py:103,107,111): only 1 enables
    return ((L.WITH_SSIM if with_ssim == True else 0) | (L.WITH_MASK if with_mask == True else 0) |  # noqa: E712
            (L.WITH_AUTO_MASK if with_auto_mask == True else 0))  # noqa: E712


def _padding(padding_mode):
    if padding_mode == "zeros":
        return L.PAD_ZEROS
    if padding_mode == "border":
        return L.PAD_BORDER
    raise ValueError("padding_mode must be 'zeros' or 'border', got %r" % (padding_mode,))


class PhotoGeoLoss(torch.autograd.Function):
    """compute_photo_and_geometry_loss (reference loss_functions.py:50-92) as one fused op.

    apply(cfg, tgt_img, intrinsics, *ref_imgs, *tgt_depth[s], *ref_depths[i][s], *poses, *poses_inv)
    with cfg = (n_ref, n_scales, flags, padding, bidir[, sums_allreduce, world]); bidir=False evaluates only the
    tgt<-ref direction (compute_pairwise_loss).  sums_allreduce (data-parallel "exact global masks" option): callable
    that sums a float64 device tensor over the ranks in place -- the masked sums of every pair-direction are reduced
    before mean_on_mask, so the loss and its 10000-pixel threshold are those of the GLOBAL batch (what the reference
    computes after its DataParallel gather).  Returns (photo_loss, geometry_loss).
    """

    @staticmethod
    def _jobs(cfg, tgt_img, ref_imgs, tgt_depth, ref_depths, poses, poses_inv, grads=None):
        n_ref, n_scales, bidir = cfg[0], cfg[1], cfg[4]
        H, W = tgt_img.shape[-2:]
        jobs = []
        for i in range(n_ref):
            for s in range(n_scales):
                td, rd = tgt_depth[s], ref_depths[i][s]
                ts = _shift_of(H, td.shape[-2], "tgt_depth")
                rs = _shift_of(H, rd.shape[-2], "ref_depth")
                if (td.shape[-1] << ts) != W or (rd.shape[-1] << rs) != W:
                    raise ValueError("depth width does not match the image width")
                g = grads or {}
                jobs.append(L.PairJob(L.ptr(tgt_img), L.ptr(ref_imgs[i]), L.ptr(td), L.ptr(rd), L.ptr(poses[i]),
                                      L.ptr(g.get(("td", s))), L.ptr(g.get(("rd", i, s))), L.ptr(g.get(("p", i))),
                                      ts, rs))
                if not bidir:
                    continue
                jobs.append(L.PairJob(L.ptr(ref_imgs[i]), L.ptr(tgt_img), L.ptr(rd), L.ptr(td), L.ptr(poses_inv[i]),
                                      L.ptr(g.get(("rd", i, s))), L.ptr(g.get(("td", s))), L.ptr(g.get(("pi", i))),
                                      rs, ts))
        return jobs

    @staticmethod
    def _split(cfg, tensors):
        n_ref, n_scales = cfg[0], cfg[1]
        it = iter(tensors)
        ref_imgs = [next(it) for _ in range(n_ref)]
        tgt_depth = [next(it) for _ in range(n_scales)]
        ref_depths = [[next(it) for _ in range(n_scales)] for _ in range(n_ref)]
        poses = [next(it) for _ in range(n_ref)]
        poses_inv = [next(it) for _ in range(n_ref)]
        return ref_imgs, tgt_depth, ref_depths, poses, poses_inv

    @staticmethod
    def forward(ctx, cfg, tgt_img, intrinsics, *tensors):
        lib = L.load()
        n_ref, n_scales, flags, padding = cfg[:4]
        if ctx.needs_input_grad[1] or any(ctx.needs_input_grad[3:3 + n_ref]):
            raise NotImplementedError(_NO_IMAGE_GRAD % "photometric / geometry loss")
        sums_allreduce, world = (cfg[5], cfg[6]) if len(cfg) > 5 and cfg[5] is not None else (None, 1)
        tgt_img = L.dev_f32(tgt_img, "tgt_img")
        intrinsics = L.dev_f32(intrinsics, "intrinsics")
        tensors = [L.dev_f32(t, "loss input") for t in tensors]
        ref_imgs, tgt_depth, ref_depths, poses, poses_inv = PhotoGeoLoss._split(cfg, tensors)
        B, _, H, W = tgt_img.shape
        jobs = PhotoGeoLoss._jobs(cfg, tgt_img, ref_imgs, tgt_depth, ref_depths, poses, poses_inv)
        out = torch.zeros(2, device=tgt_img.device, dtype=torch.float32)
        part = torch.empty(2, device=tgt_img.device, dtype=torch.float32)
        stats = []
        for c0 in range(0, len(jobs), L.MAX_JOBS):
            chunk = jobs[c0:c0 + L.MAX_JOBS]
            st = torch.empty(lib.scsfm_pairwise_stats_bytes(len(chunk), B) // 8, device=tgt_img.device,
                             dtype=torch.float64)
            arr = (L.PairJob * len(chunk))(*chunk)
            defer = 0x100 if sums_allreduce is not None else 0          # SCSFM_DEFER_FINALIZE
            L.launch(lib.scsfm_pairwise_fwd, "scsfm_pairwise_fwd", "pair_fwd", 2, 32.0 * len(chunk) * B * H * W, arr, len(chunk),
                     L.ptr(intrinsics), B, H, W, flags | defer, padding, L.ptr(st), L.ptr(part), None, L.stream())
            if sums_allreduce is not None:
                sums_allreduce(st[:lib.scsfm_pairwise_sums_count(len(chunk))])
                lib.scsfm_pairwise_finalize.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p]
                L.launch(lib.scsfm_pairwise_finalize, "scsfm_pairwise_finalize", "pair_fwd", 1, 0.0, L.ptr(st), len(chunk), float(world),
                         L.ptr(part), L.stream())
            out = out + part if len(jobs) > L.MAX_JOBS else part
            stats.append(st)
        ctx.cfg = cfg
        ctx.stats = stats
        ctx.save_for_backward(tgt_img, intrinsics, *tensors)
        return out[0], out[1]

    @staticmethod
    def backward(ctx, g_photo, g_geo):
        lib = L.load()
        cfg = ctx.cfg
        n_ref, n_scales, flags, padding = cfg[:4]
        tgt_img, intrinsics, *tensors = ctx.saved_tensors
        ref_imgs, tgt_depth, ref_depths, poses, poses_inv = PhotoGeoLoss._split(cfg, tensors)
        B, _, H, W = tgt_img.shape
        need = ctx.needs_input_grad[3:]
        grads = {}
        order = ([None] * n_ref + [("td", s) for s in range(n_scales)] +
                 [("rd", i, s) for i in range(n_ref) for s in range(n_scales)] +
                 [("p", i) for i in range(n_ref)] + [("pi", i) for i in range(n_ref)])
        for key, t, nd in zip(order, tensors, need):
            if key is not None and nd:
                grads[key] = torch.zeros_like(t)
        gout = torch.stack([g_photo, g_geo]).to(torch.float32).contiguous()
        jobs = PhotoGeoLoss._jobs(cfg, tgt_img, ref_imgs, tgt_depth, ref_depths, poses, poses_inv, grads)
        # learned intrinsics: d(loss)/dK from the d(K [R|t]) sums each chunk's backward leaves in its stats, added chunk by chunk
        g_K = torch.zeros(B, 3, 3, device=tgt_img.device, dtype=torch.float32) if ctx.needs_input_grad[2] else None
        for k, c0 in enumerate(range(0, len(jobs), L.MAX_JOBS)):
            chunk = jobs[c0:c0 + L.MAX_JOBS]
            arr = (L.PairJob * len(chunk))(*chunk)
            L.launch(lib.scsfm_pairwise_bwd, "scsfm_pairwise_bwd", "pair_bwd", 2, 44.0 * len(chunk) * B * H * W, arr, len(chunk),
                     L.ptr(intrinsics), B, H, W, flags, padding, L.ptr(ctx.stats[k]), L.ptr(gout), L.stream())
            if g_K is not None:
                L.launch(lib.scsfm_pairwise_intrinsics_grad, "scsfm_pairwise_intrinsics_grad", "pair_bwd", 1, 0.0, arr, len(chunk),
                         L.ptr(intrinsics), B, L.ptr(ctx.stats[k]), L.ptr(g_K), L.stream())
        return (None, None, g_K) + tuple(grads.get(k) if k is not None else None for k in order)


def photo_and_geometry_loss(tgt_img, ref_imgs, intrinsics, tgt_depth, ref_depths, poses, poses_inv, max_scales,
                            with_ssim, with_mask, with_auto_mask, padding_mode, sums_allreduce=None, world=1):
    n_scales = min(len(tgt_depth), max_scales)
    n_ref = min(len(ref_imgs), len(ref_depths), len(poses), len(poses_inv))   # zip() semantics of the reference
    cfg = (n_ref, n_scales, _flags(with_ssim, with_mask, with_auto_mask), _padding(padding_mode), True, sums_allreduce, world)
    if n_ref == 0 or n_scales == 0:
        return 0, 0
    flat = (list(ref_imgs[:n_ref]) + list(tgt_depth[:n_scales]) +
            [rd[s] for rd in ref_depths[:n_ref] for s in range(n_scales)] + list(poses[:n_ref]) +
            list(poses_inv[:n_ref]))
    return PhotoGeoLoss.apply(cfg, tgt_img, intrinsics, *flat)


def pairwise_loss(tgt_img, ref_img, tgt_depth, ref_depth, pose, intrinsic, with_ssim, with_mask, with_auto_mask,
                  padding_mode):
    """compute_pairwise_loss (reference loss_functions.py:95-119): one direction only."""
    cfg = (1, 1, _flags(with_ssim, with_mask, with_auto_mask), _padding(padding_mode), False)
    return PhotoGeoLoss.apply(cfg, tgt_img, intrinsic, ref_img, tgt_depth, ref_depth, pose, pose)


def pairwise_maps(tgt_img, ref_img, tgt_depth, ref_depth, pose, intrinsic, with_ssim, with_mask, with_auto_mask,
                  padding_mode):
    """Per-pixel maps of one pair-direction (diagnostics / parity tests); no autograd."""
    lib = L.load()
    args = [L.dev_f32(t, "input") for t in (tgt_img, ref_img, tgt_depth, ref_depth, pose, intrinsic)]
    tgt_img, ref_img, tgt_depth, ref_depth, pose, intrinsic = args
    B, _, H, W = tgt_img.shape
    dev = tgt_img.device
    names3, names1 = ("warped", "diff_img"), ("valid", "proj_depth", "comp_depth", "mask", "diff_depth")
    out = {n: torch.empty(B, 3, H, W, device=dev) for n in names3}
    out.update({n: torch.empty(B, 1, H, W, device=dev) for n in names1})
    maps = L.PairMaps(**{n: L.ptr(t) for n, t in out.items()})
    ts = _shift_of(H, tgt_depth.shape[-2], "tgt_depth")
    rs = _shift_of(H, ref_depth.shape[-2], "ref_depth")
    job = (L.PairJob * 1)(L.PairJob(L.ptr(tgt_img), L.ptr(ref_img), L.ptr(tgt_depth), L.ptr(ref_depth), L.ptr(pose),
                                    None, None, None, ts, rs))
    st = torch.empty(lib.scsfm_pairwise_stats_bytes(1, B) // 8, device=dev, dtype=torch.float64)
    loss = torch.empty(2, device=dev)
    L.check(lib.scsfm_pairwise_fwd(job, 1, L.ptr(intrinsic), B, H, W, _flags(with_ssim, with_mask, with_auto_mask),
                                   _padding(padding_mode), L.ptr(st), L.ptr(loss), ctypes.byref(maps), L.stream()),
            "scsfm_pairwise_fwd")
    out["photo"], out["geo"] = loss[0], loss[1]
    return out


class SmoothLoss(torch.autograd.Function):
    """compute_smooth_loss (reference loss_functions.py:132-159): apply(n, depth0, img0, depth1, img1, ...)."""

    @staticmethod
    def forward(ctx, n, *tensors):
        lib = L.load()
        if any(ctx.needs_input_grad[2::2]):
            raise NotImplementedError(_NO_IMAGE_GRAD % "smoothness loss")
        tensors = [L.dev_f32(t, "smooth input") for t in tensors]
        B, _, H, W = tensors[0].shape
        for d, im in zip(tensors[0::2], tensors[1::2]):
            if tuple(d.shape) != (B, 1, H, W) or tuple(im.shape) != (B, 3, H, W):
                raise ValueError("smooth loss: depth must be [B,1,H,W] and image [B,3,H,W] of the same size")
        jobs = (L.SmoothJob * n)(*[L.SmoothJob(L.ptr(tensors[2 * i]), L.ptr(tensors[2 * i + 1]), None)
                                   for i in range(n)])
        st = torch.empty(lib.scsfm_smooth_stats_bytes(n, B) // 8, device=tensors[0].device, dtype=torch.float64)
        out = torch.empty(1, device=tensors[0].device, dtype=torch.float32)
        L.launch(lib.scsfm_smooth_fwd, "scsfm_smooth_fwd", "smooth_fwd", 3, 16.0 * n * B * H * W, jobs, n, B, H, W, L.ptr(st), L.ptr(out),
                 L.stream())
        ctx.n, ctx.stats = n, st
        ctx.save_for_backward(*tensors)
        return out[0]

    @staticmethod
    def backward(ctx, g):
        lib = L.load()
        tensors = ctx.saved_tensors
        n = ctx.n
        B, _, H, W = tensors[0].shape
        need = ctx.needs_input_grad[1:]
        grads = [torch.zeros_like(tensors[2 * i]) if need[2 * i] else None for i in range(n)]
        jobs = (L.SmoothJob * n)(*[L.SmoothJob(L.ptr(tensors[2 * i]), L.ptr(tensors[2 * i + 1]), L.ptr(grads[i]))
                                   for i in range(n)])
        gout = g.reshape(1).to(torch.float32).contiguous()
        L.launch(lib.scsfm_smooth_bwd, "scsfm_smooth_bwd", "smooth_bwd", 1, 20.0 * n * B * H * W, jobs, n, B, H, W, L.ptr(ctx.stats),
                 L.ptr(gout), L.stream())
        out = [None]
        for i in range(n):
            out += [grads[i], None]
        return tuple(out)


def smooth_loss(tgt_depth, tgt_img, ref_depths, ref_imgs):
    pairs = [tgt_depth[0], tgt_img]
    for rd, ri in zip(ref_depths, ref_imgs):
        pairs += [rd[0], ri]
    return SmoothLoss.apply(len(pairs) // 2, *pairs)


class InverseWarp2(torch.autograd.Function):
    """inverse_warp2 (reference inverse_warp.py:230-269) with a hand-written backward."""

    @staticmethod
    def forward(ctx, img, depth, ref_depth, pose, intrinsics, padding):
        lib = L.load()
        if ctx.needs_input_grad[0]:
            raise NotImplementedError(_NO_IMAGE_GRAD % "inverse_warp2")
        img, depth, ref_depth, pose, intrinsics = [L.dev_f32(t, "inverse_warp2 input")
                                                   for t in (img, depth, ref_depth, pose, intrinsics)]
        B, _, H, W = img.shape
        warped = torch.empty_like(img)
        valid, proj, comp = (torch.empty_like(depth) for _ in range(3))
        L.check(lib.scsfm_inverse_warp2_fwd(L.ptr(img), L.ptr(depth), L.ptr(ref_depth), L.ptr(pose), L.ptr(intrinsics),
                                            B, H, W, padding, L.ptr(warped), L.ptr(valid), L.ptr(proj), L.ptr(comp),
                                            L.stream()), "scsfm_inverse_warp2_fwd")
        ctx.padding = padding
        ctx.save_for_backward(img, depth, ref_depth, pose, intrinsics)
        ctx.mark_non_differentiable(valid)
        return warped, valid, proj, comp

    @staticmethod
    def backward(ctx, g_warped, g_valid, g_proj, g_comp):
        lib = L.load()
        img, depth, ref_depth, pose, intrinsics = ctx.saved_tensors
        B, _, H, W = img.shape
        g_depth = torch.zeros_like(depth)
        g_ref = torch.zeros_like(ref_depth)
        g_pose = torch.zeros_like(pose)
        scratch = torch.empty(B * 12, device=img.device, dtype=torch.float64)
        c = lambda t: None if t is None else t.contiguous().to(torch.float32)  # noqa: E731
        g_warped, g_proj, g_comp = c(g_warped), c(g_proj), c(g_comp)
        L.check(lib.scsfm_inverse_warp2_bwd(L.ptr(img), L.ptr(depth), L.ptr(ref_depth), L.ptr(pose), L.ptr(intrinsics),
                                            B, H, W, ctx.padding, L.ptr(g_warped), L.ptr(g_proj), L.ptr(g_comp),
                                            L.ptr(g_depth), L.ptr(g_ref), L.ptr(g_pose), L.ptr(scratch), L.stream()),
                "scsfm_inverse_warp2_bwd")
        g_K = None
        if ctx.needs_input_grad[4]:
            g_K = torch.zeros(B, 3, 3, device=img.device, dtype=torch.float32)
            L.check(lib.scsfm_inverse_warp2_intrinsics_grad(L.ptr(pose), L.ptr(intrinsics), B, L.ptr(scratch), L.ptr(g_K),
                                                            L.stream()), "scsfm_inverse_warp2_intrinsics_grad")
        return None, g_depth, g_ref, g_pose, g_K, None


def pose_vec2mat(vec, rotation_mode="euler"):
    lib = L.load()
    if rotation_mode not in ("euler", "quat"):
        raise ValueError("rotation_mode must be 'euler' or 'quat'")
    vec = L.dev_f32(vec, "vec")
    out = torch.empty(vec.shape[0], 3, 4, device=vec.device, dtype=torch.float32)
    L.check(lib.scsfm_pose_vec2mat(L.ptr(vec), vec.shape[0], 0 if rotation_mode == "euler" else 1, L.ptr(out),
                                   L.stream()), "scsfm_pose_vec2mat")
    return out


def compute_errors(gt, pred, y1, y2, x1, x2, max_depth):
    """Per-image validation metrics [B,8] = {abs_diff, abs_rel, sq_rel, a1, a2, a3, median(gt), median(pred)} (scsfm_compute_errors)."""
    gt, pred = L.dev_f32(gt, "gt"), L.dev_f32(pred, "pred")
    if gt.dim() != 3 or gt.shape != pred.shape:
        raise ValueError("compute_errors expects gt and pred of shape [B,H,W], got %s and %s" % (tuple(gt.shape), tuple(pred.shape)))
    B, H, W = gt.shape
    lib = L.load()
    lib.scsfm_compute_errors.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                         ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p,
                                         ctypes.c_void_p]
    out = torch.empty(B, 8, device=gt.device, dtype=torch.float32)
    work = torch.empty(3 * B, device=gt.device, dtype=torch.float32)
    L.launch(lib.scsfm_compute_errors, "scsfm_compute_errors", "eval", 2, 5 * 8.0 * gt.numel(), L.ptr(gt), L.ptr(pred), B, H, W, y1, y2, x1, x2,
             max_depth, L.ptr(work), L.ptr(out), L.stream())
    return out


# --- offline evaluation (reference eval_depth.py) ------------------------------------------------------------------------
EVAL_COLUMNS = ("n", "med_gt", "med_pred", "ratio", "abs_rel", "sq_rel", "rmse", "rmse_log", "log10", "a1", "a2", "a3")
EVAL_MIN_DEPTH = 1e-3
EVAL_MAX_DEPTH = {"kitti": 80.0, "nyu": 10.0}
EVAL_CHUNK = 64          # images per launch: bounds the device memory of a call (KITTI-sized, float32 ground truth: ~0.5 GB)


def eigen_crop(H, W):
    """The reference's KITTI crop of an H x W ground truth (eval_depth.py:186-187): rows [y1,y2) x columns [x1,x2)."""
    import numpy as np
    return tuple(int(v) for v in np.array([0.40810811 * H, 0.99189189 * H, 0.03594771 * W, 0.96405229 * W]).astype(np.int32))


class _Staging:
    """Pinned host buffers reused from chunk to chunk (grown when a chunk needs more)."""

    def __init__(self):
        self.bufs = {}

    def get(self, name, n, dtype):
        b = self.bufs.get(name)
        if b is None or b.numel() < n or b.dtype != dtype:
            b = self.bufs[name] = torch.empty(max(n, 1), dtype=dtype, pin_memory=True)
        return b[:n]


def eval_depth(pred, gt_list, dataset, indices=None, chunk=EVAL_CHUNK):
    """Per-image results of the reference's median-scaled depth evaluation (eval_depth.py:159-227) on the device
    (scsfm_eval_depth): float64 numpy [len(indices), 12] with the columns EVAL_COLUMNS.

    pred: float64 [N,h,w] (test_disp.py's predictions.npy; a memory map is fine); gt_list: N or more float32 or float64
    [H,W] ground truths, of any sizes (a sequence or an array; ground truths past the N-th are ignored); dataset 'kitti'
    (depth range (1e-3, 80), Eigen crop) or 'nyu' ((1e-3, 10), whole image); indices: the images to evaluate (default all).
    The images go to the device `chunk` at a time; the results do not depend on the chunk size."""
    import numpy as np
    if dataset not in EVAL_MAX_DEPTH:
        raise ValueError("dataset must be 'kitti' or 'nyu', got %r" % (dataset,))
    if getattr(pred, "ndim", None) != 3 or pred.dtype != np.float64:
        raise TypeError("predictions must be a float64 array [N,h,w] (test_disp.py's predictions.npy), got %s %s" %
                        (getattr(pred, "dtype", type(pred)), getattr(pred, "shape", "")))
    N, h, w = pred.shape
    if len(gt_list) < N:
        raise ValueError("%d predictions but only %d ground-truth depth maps" % (N, len(gt_list)))
    idx = list(range(N)) if indices is None else [int(i) for i in indices]
    if any(i < 0 or i >= N for i in idx):
        raise IndexError("image index outside the %d predictions" % N)
    if chunk < 1:
        raise ValueError("chunk must be positive")
    lib = L.load()
    dev = torch.device("cuda")
    stage = _Staging()
    max_depth = EVAL_MAX_DEPTH[dataset]
    out = np.empty((len(idx), len(EVAL_COLUMNS)), np.float64)
    for c0 in range(0, len(idx), chunk):
        sel = idx[c0:c0 + chunk]
        gts = [np.asarray(gt_list[i]) for i in sel]
        dtypes = {g.dtype for g in gts}
        if not dtypes <= {np.dtype(np.float32), np.dtype(np.float64)} or len(dtypes) != 1 or any(g.ndim != 2 for g in gts):
            raise TypeError("ground-truth depth maps must be 2-D and all float32 or all float64, got %s" %
                            sorted({(str(g.dtype), g.ndim) for g in gts}))
        f64 = gts[0].dtype == np.float64
        descs = (L.EvalDepthImage * len(sel))()
        off = 0
        for k, g in enumerate(gts):
            H, W = g.shape
            y1, y2, x1, x2 = eigen_crop(H, W) if dataset == "kitti" else (0, H, 0, W)
            descs[k] = L.EvalDepthImage(off, H, W, y1, y2, x1, x2)
            off += g.size
        host_gt = stage.get("gt", off, torch.float64 if f64 else torch.float32)
        flat = host_gt.numpy()
        o = 0
        for g in gts:
            flat[o:o + g.size] = g.reshape(-1)
            o += g.size
        host_pred = stage.get("pred", len(sel) * h * w, torch.float64)
        hp = host_pred.numpy().reshape(len(sel), h, w)
        for k, i in enumerate(sel):
            hp[k] = pred[i]
        d_gt = host_gt.to(dev, non_blocking=True)
        d_pred = host_pred.to(dev, non_blocking=True)
        ws_bytes = lib.scsfm_eval_depth_workspace_bytes(descs, len(sel))
        ws = torch.empty((ws_bytes + 15) // 16, 2, dtype=torch.float64, device=dev)
        res = torch.empty(len(sel), len(EVAL_COLUMNS), dtype=torch.float64, device=dev)
        L.launch(lib.scsfm_eval_depth, "scsfm_eval_depth", "eval", 1, 4.0 * off + 8.0 * len(sel) * h * w, L.ptr(d_pred), len(sel), h, w,
                 L.ptr(d_gt), 1 if f64 else 0, off, descs, EVAL_MIN_DEPTH, max_depth, L.ptr(ws), ws.numel() * 8, L.ptr(res), L.stream())
        out[c0:c0 + len(sel)] = res.cpu().numpy()         # also the point after which the pinned buffers may be refilled
    return out
