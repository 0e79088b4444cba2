"""One optimisation step of the reference training loop (reference train.py:259-282, 426-444) on one
H100, and its data-parallel form: one process per GPU, each rank runs the complete step on its shard of
the batch, the two gradient arenas are all-reduced (NCCL over NVLink) as soon as the backward of the
owning network has finished, then every rank applies the identical fused Adam update.

Fine-tuning: parameters may be frozen (requires_grad False) and BatchNorm modules put in eval mode, per module, before the
first step (or before capture()); the step then skips their gradients and updates, and capture() refuses a later change.

Self-calibration: Trainer(..., camera=LearnedCamera(...)) owns a learned camera as it owns the networks.  Each step then takes the
batch's augmentation records (scsfm.camera.records, GpuAugment(..., return_records=True)) in place of intrinsics, builds every
sample's K from theta, back-propagates into theta, all-reduces d(loss)/dtheta with the arenas (data parallel) and updates theta
with its own Adam after the networks' -- all of it inside the captured step too.

A bank of cameras (LearnedCamera.bank, theta [C,4]: one camera per calibration or per scene) also takes each sample's camera
index, step(..., aug=records, camera_index=idx).  theta's Adam is dense over [C,4], as torch.optim.Adam on one [C,4] parameter:
a camera that no sample has used yet has zero moments and does not move; a camera used earlier and absent from the current batch
moves by its momentum.
"""
import torch
import torch.distributed as dist

import loss_functions as LF

from . import nnops as O
from .camera import _check as _check_camera_inputs, _check_theta
from .exchange import GradExchange
from .nets import ArenaAdam, check_image_size


def _check_sizes(tgt_img, ref_imgs):
    """The losses compare each disparity with its image pixel by pixel: refuse a size whose disparity is not the image's, or
    that DispResNet does not take, before PoseResNet is launched on the side stream."""
    for img in [tgt_img] + list(ref_imgs):
        check_image_size(img.shape[-2], img.shape[-1], training_step=True)


def compute_depth(disp_net, tgt_img, ref_imgs):
    """train.py:426-434 -- depth = 1/disparity for the target and every reference.  The 1 + len(ref_imgs) network
    calls run as one stacked launch sequence (BatchNorm statistics and running-stat updates stay per call)."""
    outs = disp_net.forward_multi([tgt_img] + list(ref_imgs))
    depths = [[1 / d for d in o] for o in outs]
    return depths[0], depths[1:]


def compute_pose_with_inv(pose_net, tgt_img, ref_imgs):
    """train.py:437-444 -- the reference's call order is (tgt,ref0), (ref0,tgt), (tgt,ref1), (ref1,tgt), ..."""
    pairs = []
    for r in ref_imgs:
        pairs += [(tgt_img, r), (r, tgt_img)]
    out = pose_net.forward_multi(pairs)
    return out[0::2], out[1::2]


class Trainer:
    """Holds the two networks, the fused Adam, (optionally) the data-parallel gradient exchange and (optionally) a learned camera:
    camera = scsfm.camera.LearnedCamera on the networks' device (one camera, or a bank of C), updated by Adam with learning rate
    camera_lr (the networks' betas and eps, no weight decay)."""

    def __init__(self, disp_net, pose_net, lr=1e-4, betas=(0.9, 0.999), weight_decay=0.0, num_scales=1, with_ssim=1,
                 with_mask=1, with_auto_mask=0, padding_mode="zeros", w1=1.0, w2=0.1, w3=0.5, distributed=None, conv_mode=None,
                 exact_global_masks=False, overlap_nets=True, overlap_wgrad=True, camera=None, camera_lr=0.1):
        self.disp_net, self.pose_net = disp_net, pose_net
        if conv_mode is not None:           # "fp32" | "tf32" | "tf32x3" (nnops.MODES); None keeps each network's own setting
            disp_net.set_conv_mode(conv_mode)
            pose_net.set_conv_mode(conv_mode)
        self.optimizer = ArenaAdam([disp_net, pose_net], lr=lr, betas=betas, weight_decay=weight_decay)
        for n in (disp_net, pose_net):
            n.trust_adam_mirror = True      # this loop changes parameters only through ArenaAdam (which writes the TF32 mirror)
        self.cfg = dict(num_scales=num_scales, with_ssim=with_ssim, with_mask=with_mask, with_auto_mask=with_auto_mask,
                        padding_mode=padding_mode)
        self.w = (w1, w2, w3)
        self.distributed = dist.is_initialized() if distributed is None else distributed
        self.world = dist.get_world_size() if self.distributed else 1
        self.exchange = None
        # data parallel only.  False (default): standard DDP semantics -- every rank is the reference at batch B/N and the
        # gradients are averaged.  True: the masked sums of mean_on_mask (loss_functions.py:123-129) are all-reduced (one
        # tiny SUM of 8 doubles per pair-direction) before the losses are formed, so the photometric / geometry losses, their
        # 10000-pixel thresholds and therefore the gradients are those of the GLOBAL batch -- exactly what the reference's
        # nn.DataParallel computes on the gathered outputs (per-GPU BatchNorm, global loss; train.py:168-169).
        self.exact_global_masks = bool(exact_global_masks)
        self.overlap_nets = bool(overlap_nets)
        self._side = None
        if overlap_wgrad:
            # weight gradients on their own stream per network (nnops.ConvCtx.wgrad_stream)
            for net in (disp_net, pose_net):
                net.ctx.wgrad_stream = torch.cuda.Stream()
        self._graph = None
        self.launches_per_step = None
        self.camera, self.camera_lr = camera, camera_lr
        if camera is not None:
            th = camera.theta
            _check_theta(th)
            # theta's Adam state: exp_avg, exp_avg_sq and the step counter, on the device (capturable, like ArenaAdam's)
            self._cam_state = (torch.zeros_like(th.data), torch.zeros_like(th.data), torch.zeros(1, device=th.device, dtype=torch.int32))
        if self.distributed:
            self.exchange = GradExchange(self.world, torch.cuda.Stream())
            for net in (disp_net, pose_net):
                net.ensure_arena()
                # fires when the last pending backward of the network has been enqueued: its gradient arena is
                # averaged on the side stream while the rest of the backward pass keeps running
                net.grads_ready_callback = lambda n: self.exchange.allreduce_async(n.flat_grads())
            arenas = [disp_net.flat_params(), pose_net.flat_params()] + ([camera.theta.data] if camera is not None else [])
            self.exchange.broadcast_params(arenas)   # identical replicas

    def losses(self, tgt_img, ref_imgs, intrinsics):
        if self.overlap_nets:
            # the two networks are independent until the losses: PoseResNet runs on a side stream next to DispResNet (autograd
            # replays each network's backward on the stream of its forward).  Their big layers fill the GPU on their own; the
            # gain is in the deep 8x26 / 16x52 layers, whose 40..100 CTAs leave a third of the SMs idle.  Fork / join through
            # events (capturable in a CUDA graph); tensors made on the side stream are first used on the main stream after
            # the join and released only after the whole step has been enqueued.
            main = torch.cuda.current_stream()
            if self._side is None:
                self._side = torch.cuda.Stream()
            fork = torch.cuda.Event()
            fork.record(main)
            with torch.cuda.stream(self._side):
                self._side.wait_event(fork)
                poses, poses_inv = compute_pose_with_inv(self.pose_net, tgt_img, ref_imgs)
            tgt_depth, ref_depths = compute_depth(self.disp_net, tgt_img, ref_imgs)
            main.wait_stream(self._side)
        else:
            tgt_depth, ref_depths = compute_depth(self.disp_net, tgt_img, ref_imgs)
            poses, poses_inv = compute_pose_with_inv(self.pose_net, tgt_img, ref_imgs)
        c = self.cfg
        if self.exchange is not None and self.exact_global_masks:
            from . import loss_ops
            photo, geo = loss_ops.photo_and_geometry_loss(tgt_img, ref_imgs, intrinsics, tgt_depth, ref_depths, poses, poses_inv,
                                                          c["num_scales"], c["with_ssim"], c["with_mask"], c["with_auto_mask"],
                                                          c["padding_mode"], self.exchange.allreduce_sums, self.world)
        else:
            photo, geo = LF.compute_photo_and_geometry_loss(tgt_img, ref_imgs, intrinsics, tgt_depth, ref_depths, poses,
                                                            poses_inv, c["num_scales"], c["with_ssim"], c["with_mask"],
                                                            c["with_auto_mask"], c["padding_mode"])
        smooth = LF.compute_smooth_loss(tgt_depth, tgt_img, ref_depths, ref_imgs)
        w1, w2, w3 = self.w
        return w1 * photo + w2 * smooth + w3 * geo, photo, smooth, geo

    def step(self, tgt_img, ref_imgs, intrinsics=None, aug=None, camera_index=None):
        """train.py:259-282 without a single host synchronisation; returns device scalars
        (loss, photo, smooth, geometry).  After `capture()` the step is one CUDA-graph replay.

        Intrinsics that require a gradient (a learned / self-calibrated K) get it in an eager single-GPU step, accumulated
        into their .grad as in the reference loop; updating them is left to the caller's own optimizer.
        With a camera the step takes `aug`, the batch's augmentation records, and no intrinsics: K is built from the camera; a bank
        of cameras also takes `camera_index`, each sample's camera (int32 or int64 [B] on the GPU).
        The images' H and W are multiples of 32, at least 64 (nets.check_image_size): else ValueError before any launch."""
        _check_sizes(tgt_img, ref_imgs)
        intrinsics = self._camera_inputs(tgt_img, intrinsics, aug, camera_index)
        self._check_intrinsics(intrinsics)
        if self._graph is not None:
            if self._flag_patterns() != self._captured_flags:
                raise RuntimeError("the requires_grad / train-eval pattern of the networks changed after capture(): the captured "
                                   "step computes the old one (drop_graph() and capture() again)")
            given = dict(tgt_img=tgt_img, intrinsics=intrinsics, aug=aug, camera_index=camera_index)
            for name, dst in self._static.items():
                if name == "ref_imgs":
                    for d, src in zip(dst, ref_imgs):
                        d.copy_(src, non_blocking=True)
                else:
                    dst.copy_(given[name], non_blocking=True)
            self._graph.replay()
            return tuple(self._static_out.unbind(0))
        return self._eager_step(tgt_img, ref_imgs, intrinsics, aug, camera_index)

    def capture(self, tgt_img, ref_imgs, intrinsics=None, allow_distributed=False, aug=None, camera_index=None):
        """Record the whole step (7 network calls forward + backward, losses, Adam) into one CUDA graph: ~2500
        kernel launches become a single graph launch.  One eager warm-up step runs first (lazy allocations,
        Adam state) and is undone, so capturing does not advance training.  Single-GPU path.  With a camera, `aug` takes the
        place of intrinsics (as in step()); the records (and a bank's camera index) become static buffers and the camera's theta and
        Adam state are undone too."""
        from . import lib as L
        _check_sizes(tgt_img, ref_imgs)
        if self.exchange is not None and not allow_distributed:
            raise RuntimeError("graph capture of the data-parallel step is opt-in (allow_distributed=True): capturing the NCCL "
                               "all-reduce on the side stream has not been validated on this pod yet")
        intrinsics = self._camera_inputs(tgt_img, intrinsics, aug, camera_index)
        self._check_intrinsics(intrinsics, capturing=True)
        # the static inputs, by _eager_step's keyword: the images, and K or the records (and a bank's camera index)
        self._static = dict(tgt_img=tgt_img.clone(), ref_imgs=[r.clone() for r in ref_imgs])
        for name, t in (("intrinsics", intrinsics), ("aug", aug), ("camera_index", camera_index)):
            if t is not None:
                self._static[name] = t.to(torch.int32, copy=True) if name == "camera_index" else t.clone()
        snap = self.optimizer.snapshot()
        cam_snap = self._camera_snapshot()
        prof = dict(L.PROF)
        L.PROF.update(enabled=False)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            self._eager_step(**self._static)
        torch.cuda.current_stream().wait_stream(side)
        self.optimizer.restore(snap)
        self._camera_restore(cam_snap)
        # restore() changed the parameters: bring the TF32 operand mirrors up to date NOW, so that the captured step contains
        # no rounding pass (during replays the Adam kernel at the end of step k writes the mirror for step k+1)
        for n in self.optimizer.nets:
            n.refresh_operand_weights()
        # the warm-up step left the persistent flipped-weight buffers and their job tables in place: the capture below
        # records one batched refresh per network instead of one flip per layer
        before = L.launch_count()
        graph = torch.cuda.CUDAGraph()
        # with the gradient exchange the capture also records the NCCL all-reduces issued on the side stream (joined through
        # events); NCCL's watchdog thread may touch CUDA meanwhile, hence the thread-local capture mode
        mode = "thread_local" if self.exchange is not None else "global"
        with torch.cuda.graph(graph, capture_error_mode=mode):
            self._static_out = torch.stack(self._eager_step(**self._static))
        self.launches_per_step = L.launch_count() - before
        self._graph = graph
        self._captured_flags = self._flag_patterns()
        L.PROF.update(prof)

    def _camera_inputs(self, tgt_img, intrinsics, aug, camera_index):
        """The intrinsics argument of a step: the caller's K without a camera; None with one, whose records (and a bank's camera
        index) are checked here against the batch."""
        if self.camera is None:
            if aug is not None or camera_index is not None:
                raise TypeError("augmentation records and a camera index are the inputs of a Trainer with a camera (Trainer(..., "
                                "camera=LearnedCamera(...))); this Trainer has no camera")
            if intrinsics is None:
                raise TypeError("intrinsics are required (or give the Trainer a camera and pass augmentation records)")
            return intrinsics
        if intrinsics is not None:
            raise ValueError("this Trainer owns a learned camera, which builds every sample's K from the augmentation records: "
                             "pass aug=records and no intrinsics")
        if aug is None:
            raise TypeError("a Trainer with a camera needs the batch's augmentation records (aug=scsfm.camera.records(...), "
                            "or GpuAugment(..., return_records=True))")
        _check_camera_inputs(self.camera.theta, aug, camera_index, tgt_img.shape[0])
        return None

    def _camera_snapshot(self):
        if self.camera is None:
            return None
        return [t.clone() for t in (self.camera.theta.data,) + self._cam_state]

    def _camera_restore(self, snap):
        if snap is not None:
            for t, t0 in zip((self.camera.theta.data,) + self._cam_state, snap):
                t.copy_(t0)

    def camera_state_dict(self):
        """theta's Adam state: {'step', 'exp_avg', 'exp_avg_sq'}."""
        m, v, step = self._cam_state
        return {"step": int(step.item()), "exp_avg": m, "exp_avg_sq": v}

    def state_dict(self):
        """CPU copies of everything training continues from: both networks' state_dict() (parameters, BatchNorm running
        statistics, num_batches_tracked), the ArenaAdam state and, with a camera, its state_dict() and Adam state."""
        cpu = lambda t: t.detach().contiguous().cpu()  # noqa: E731
        opt = self.optimizer.state_dict()
        sd = {"disp_net": {k: cpu(v) for k, v in self.disp_net.state_dict().items()},
              "pose_net": {k: cpu(v) for k, v in self.pose_net.state_dict().items()},
              "optimizer": {"step": opt["step"], "exp_avg": [cpu(t) for t in opt["exp_avg"]],
                            "exp_avg_sq": [cpu(t) for t in opt["exp_avg_sq"]]}}
        if self.camera is not None:
            sd["camera"] = {k: cpu(v) for k, v in self.camera.state_dict().items()}
            sd["camera_optimizer"] = {k: v if k == "step" else cpu(v) for k, v in self.camera_state_dict().items()}
        return sd

    def load_state_dict(self, sd):
        """Load what state_dict() returns, in place, before or after capture(): a captured step and the gradient exchange keep
        working on the same tensors.  A camera in `sd` but not in this Trainer, or the reverse, or a different number of cameras
        raises ValueError.  Data parallel: every rank loads the same state, and rank 0's parameters are broadcast once more."""
        has = "camera" in sd
        if has != (self.camera is not None):
            raise ValueError("the training state %s a learned camera and this Trainer %s" % (("holds", "has none") if has else
                                                                                              ("holds no", "has one")))
        if has and tuple(sd["camera"]["theta"].shape) != tuple(self.camera.theta.shape):
            raise ValueError("the training state's camera theta is %s, this Trainer's %s: a different number of cameras"
                             % (tuple(sd["camera"]["theta"].shape), tuple(self.camera.theta.shape)))
        self.optimizer.load_state_dict(sd["optimizer"])          # (packs the arenas first: the networks load into them)
        self.disp_net.load_state_dict(sd["disp_net"])
        self.pose_net.load_state_dict(sd["pose_net"])
        if has:
            self.camera.load_state_dict(sd["camera"])
            m, v, step = self._cam_state
            m.copy_(sd["camera_optimizer"]["exp_avg"])
            v.copy_(sd["camera_optimizer"]["exp_avg_sq"])
            step.fill_(int(sd["camera_optimizer"]["step"]))
        if self.exchange is not None:
            self.exchange.broadcast_params([self.disp_net.flat_params(), self.pose_net.flat_params()] +
                                           ([self.camera.theta.data] if has else []))
        # the operand mirror: during replays only the Adam kernel writes it and no network call runs Python, so it is brought
        # up to date here from the loaded arena (as capture() does after undoing the warm-up step)
        for n in self.optimizer.nets:
            n._tf32_version = None
            n.refresh_operand_weights()

    def _check_intrinsics(self, intrinsics, capturing=False):
        """Learned intrinsics are supported by the eager single-GPU step only; elsewhere their gradient would be lost."""
        if intrinsics is None or not (torch.is_grad_enabled() and intrinsics.requires_grad):
            return
        if capturing or self._graph is not None:
            raise RuntimeError("intrinsics that require a gradient cannot go through a captured step: the graph works on a "
                               "static copy of K, so its gradient would never reach the caller's tensor (drop_graph() and "
                               "step eagerly, or pass intrinsics.detach())")
        if self.exchange is not None:
            raise RuntimeError("intrinsics that require a gradient are not supported by the data-parallel step: only the two "
                               "networks' gradients are all-reduced, so the per-rank gradients of K would silently diverge "
                               "(pass intrinsics.detach())")

    def _flag_patterns(self):
        """What a captured step depends on beyond its inputs: which parameters are frozen and which modules are in eval mode."""
        return self.disp_net.flag_pattern(), self.pose_net.flag_pattern()

    def drop_graph(self):
        """Forget a captured graph: later steps run eagerly."""
        self._graph = None
        self.launches_per_step = None

    def _eager_step(self, tgt_img, ref_imgs, intrinsics=None, aug=None, camera_index=None):
        cam = self.camera
        if cam is not None:
            cam.theta.grad = None
            # scsfm_camera_build_indexed; its backward adds d(loss)/dtheta (scsfm_camera_grad_indexed)
            intrinsics = cam(aug, camera_index)
        loss, photo, smooth, geo = self.losses(tgt_img, ref_imgs, intrinsics)
        self.optimizer.zero_grad()
        loss.backward()
        if self.exchange is not None:
            n = 2
            if cam is not None:
                n = 3                                # d(loss)/dtheta is averaged like the arenas, after them
                if cam.theta.grad is None:
                    cam.theta.grad = torch.zeros_like(cam.theta)
                self.exchange.allreduce_async(cam.theta.grad)
            # every network must have handed its gradient arena to the exchange (a forward whose backward never ran would
            # leave the replicas silently diverging)
            if self.exchange.pending() != n:
                raise RuntimeError("data-parallel step: %d of %d gradient all-reduces were issued" % (self.exchange.pending(), n))
            self.exchange.wait()
        self.optimizer.step()
        if cam is not None:
            self._camera_adam()
        return loss.detach(), photo.detach(), smooth.detach(), geo.detach()

    def _camera_adam(self):
        th = self.camera.theta
        m, v, step = self._cam_state
        if th.grad is None:                          # (a loss that does not depend on K)
            th.grad = torch.zeros_like(th)
        step += 1
        O.adam_step(th.data, th.grad, m, v, self.camera_lr, self.optimizer.betas[0], self.optimizer.betas[1], self.optimizer.eps, 0.0,
                    0, step)
