"""Shared helpers of the learned-camera tests: the build restated in numpy and in torch, seeded augmentation records, the
Trainer with one camera or a bank, the fp64 oracle's camera gradient, a synthetic plane rendered for every augmented camera, and
the Trainer checks that one camera (tests/test_camera_gpu.py) and a bank of two (tests/test_camera_groups_gpu.py) share:
cameras = 1 or 2."""
import os
import random
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from helpers import free_port, rel_l2

DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def kernel_build(theta, rec):
    """scsfm_camera_build_indexed restated in numpy for one record and one camera: float32 subtractions for the flip and the
    crop, float64 products rounded to float32 for the zoom (csrc/camera.cu)."""
    xs, ys, flip, ox, oy, in_w = rec
    f32, f64 = np.float32, np.float64
    fx, fy, cx, cy = (f32(v) for v in theta)
    if flip != 0.0:
        cx = f32(f32(in_w) - cx)
    K = np.zeros((3, 3), np.float32)
    K[0, 0] = f32(f64(fx) * f64(xs))
    K[0, 2] = f32(f32(f64(cx) * f64(xs)) - f32(ox))
    K[1, 1] = f32(f64(fy) * f64(ys))
    K[1, 2] = f32(f32(f64(cy) * f64(ys)) - f32(oy))
    K[2, 2] = 1.0
    return K


def indexed_build(thetas, rec, idx):
    """kernel_build of camera idx of thetas, nine NaNs for an index out of range."""
    if not 0 <= idx < len(thetas):
        return np.full((3, 3), np.nan, np.float32)
    return kernel_build(thetas[idx], rec)


def bank_build(thetas, rec, idx):
    """K_b = aug_b(thetas[idx_b]) restated in torch (differentiable; the dtype of thetas [C,4]); one camera theta [4] is
    bank_build(theta[None], rec, zeros)."""
    rec = rec.to(thetas.device, thetas.dtype)
    xs, ys, flip, ox, oy, in_w = rec.unbind(1)
    fx, fy, cx, cy = thetas[idx.long().to(thetas.device)].unbind(1)
    cxb = torch.where(flip != 0, in_w - cx, cx)
    zero, one = torch.zeros_like(xs), torch.ones_like(xs)
    return torch.stack([torch.stack([fx * xs, zero, cxb * xs - ox], 1), torch.stack([zero, fy * ys, cy * ys - oy], 1),
                        torch.stack([zero, zero, one], 1)], 1)


def seeded_records(seed, B, H, W):
    from scsfm.augment import Draw
    from scsfm.camera import record_rows
    random.seed(seed)
    np.random.seed(seed)
    rows = record_rows([Draw.random(H, W) for _ in range(B)], W)
    return torch.from_numpy(rows)


def theta_of(K):
    return torch.tensor([K[0, 0], K[1, 1], K[0, 2], K[1, 2]], dtype=torch.float32)


def make_nets():
    import models
    from golden_util import det_weights
    d, p = models.DispResNet(18, False), models.PoseResNet(18, False)
    for n in (d, p):
        n.load_state_dict(det_weights(n.state_dict()))
    return d.to(DEV).train(), p.to(DEV).train()


def make_trainer(mode="fp32", theta=None, **kw):
    """theta: one camera [4], a bank [C,4], or None (no camera)."""
    from scsfm.camera import LearnedCamera
    from scsfm.trainer import Trainer
    d, p = make_nets()
    cam = None
    if theta is not None:
        theta = torch.as_tensor(theta, dtype=torch.float32)
        cam = (LearnedCamera(*theta.tolist()) if theta.dim() == 1 else LearnedCamera.bank(theta)).to(DEV)
    kw.setdefault("distributed", False)
    return Trainer(d, p, lr=1e-4, with_auto_mask=0, conv_mode=mode, camera=cam, **kw)


def oracle_theta_grads(th0, idx, tgt, refs, rec):
    """dtheta of one step of oracle.step.train_step with K_b = aug_b(th0[idx_b]) (th0 [C,4]), in fp64 and fp32 on the CPU and
    in stock PyTorch fp32 on the GPU (TF32 off): {'64', '32', '32gpu'}."""
    from golden_util import det_weights
    from oracle import nets as N
    from oracle import step as OS
    want = {}
    tf32 = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        for key, dt, dev in (("64", torch.float64, "cpu"), ("32", torch.float32, "cpu"), ("32gpu", torch.float32, DEV)):
            d, p = N.DispResNet(18).to(dt).to(dev), N.PoseResNet(18).to(dt).to(dev)
            for n in (d, p):
                n.load_state_dict({k: v.to(dt) for k, v in det_weights(n.state_dict()).items()})
                n.train()
            th = th0.to(dev, dt, copy=True).requires_grad_(True)
            OS.train_step(d, p, OS.make_optimizer(d, p, lr=1e-4), tgt.to(dev, dt), [r.to(dev, dt) for r in refs],
                          bank_build(th, rec, idx), num_scales=1, with_ssim=1, with_mask=1, with_auto_mask=0)
            want[key] = th.grad.cpu()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    return want


def render_plane(theta, rec, H, W, Z0, t, seed):
    """A textured fronto-parallel plane Z = Z0 (target camera coordinates) seen by the target camera and by a reference camera
    at P_ref = P_tgt + t_b (t: fp64 [B,3], one translation per sample), both with the sample's augmented intrinsics
    K_b = aug_b(theta); the texture is a seeded sum of sinusoids of the plane's metric coordinates, evaluated exactly (fp64) at
    every pixel of both views.  Returns tgt, ref [B,3,H,W] float32, the two constant depth maps and the pose vectors
    target->reference and back."""
    B = rec.shape[0]
    K = bank_build(torch.as_tensor(theta, dtype=torch.float64)[None], rec, torch.zeros(B, dtype=torch.long)).to(DEV)
    g = torch.Generator().manual_seed(seed)
    n = 12
    lam = 1.0 + 2.0 * torch.rand(B, 3, n, 2, generator=g, dtype=torch.float64)          # wavelengths 1..3 m: 20..60 px at Z0
    ang = 2 * np.pi * torch.rand(B, 3, n, generator=g, dtype=torch.float64)
    kx = (2 * np.pi / lam[..., 0] * torch.cos(ang)).to(DEV)
    ky = (2 * np.pi / lam[..., 1] * torch.sin(ang)).to(DEV)
    ph = (2 * np.pi * torch.rand(B, 3, n, generator=g, dtype=torch.float64)).to(DEV)
    v, u = torch.meshgrid(torch.arange(H, dtype=torch.float64, device=DEV), torch.arange(W, dtype=torch.float64, device=DEV),
                          indexing="ij")
    fx, fy, cx, cy = (K[:, 0, 0, None, None], K[:, 1, 1, None, None], K[:, 0, 2, None, None], K[:, 1, 2, None, None])

    def tex(X, Y):                       # X, Y [B,H,W] -> [B,3,H,W]
        arg = kx[..., None, None] * X[:, None, None] + ky[..., None, None] * Y[:, None, None] + ph[..., None, None]
        return (0.9 * torch.cos(arg).mean(2)).float()
    tgt = tex((u - cx) * Z0 / fx, (v - cy) * Z0 / fy)
    tx, ty, tz = (t[:, i, None, None].to(DEV) for i in range(3))
    Zr = Z0 + tz
    ref = tex((u - cx) * Zr / fx - tx, (v - cy) * Zr / fy - ty)
    pose = torch.cat([t, torch.zeros(B, 3, dtype=torch.float64)], 1).float().to(DEV)
    ref_depth = Zr.float().expand(B, H, W)[:, None].contiguous()
    return tgt, ref, torch.full((B, 1, H, W), Z0, device=DEV), ref_depth, pose, -pose


# ---- Trainer checks of one camera (cameras = 1) and of a bank of two (cameras = 2) ------------------------------------------
def eager_step_vs_oracle(cameras):
    """theta.grad of an eager step against oracle.step.train_step in fp64 with K_b built from theta (a bank: K_b =
    aug_b(theta[idx_b])); yardstick and bound of test_trainer_eager_step_gives_the_oracle_intrinsics_gradient (4x the larger fp32
    error + 1e-3)."""
    from scsfm import synth
    B, H, W = 2, 96, 160
    tgt, refs, K = synth.triplet(5, B, H, W)
    rec = seeded_records(11, B, H, W)
    th0 = theta_of(K[0]) * torch.tensor([1.05, 0.97, 1.0, 1.0]) + torch.tensor([0.0, 0.0, 2.0, -1.5])
    if cameras == 1:
        idx, ix = torch.zeros(B, dtype=torch.int32), {}
    else:
        th0 = torch.stack([th0, theta_of(K[0]) * torch.tensor([0.95, 1.02, 1.0, 1.0]) + torch.tensor([0.0, 0.0, -3.0, 1.0])])
        idx = torch.tensor([1, 0], dtype=torch.int32)
        ix = {"camera_index": idx.to(DEV)}
    tr = make_trainer("fp32", theta=th0)
    tr.step(tgt.to(DEV), [r.to(DEV) for r in refs], aug=rec.to(DEV), **ix)
    mine = tr.camera.theta.grad.cpu().reshape(-1, 4)
    assert not torch.equal(tr.camera.theta.detach().cpu(), th0)           # Adam moved theta
    want = oracle_theta_grads(th0.reshape(-1, 4), idx, tgt, refs, rec)
    errs = {k: rel_l2(g, want["64"]) for k, g in (("mine", mine), ("32", want["32"]), ("32gpu", want["32gpu"]))}
    print("%d camera(s) dtheta rel_l2 vs fp64: mine %.3g | fp32 CPU oracle %.3g | stock PyTorch fp32 on this GPU %.3g" %
          (cameras, errs["mine"], errs["32"], errs["32gpu"]))
    assert errs["mine"] < 4 * max(errs["32"], errs["32gpu"]) + 1e-3


def captured_steps_track_eager(cameras):
    """Captured steps with a camera (or a bank of two with mixed indices) against the same eager steps (theta, losses,
    parameters) within the tolerances of test_cuda_graph_replay_matches_eager_steps; capture() leaves theta and its Adam state
    bitwise unchanged.  The first step, from identical states, gives the eager camera gradient and update; every replay applies
    Adam to the gradient it computed.  A captured bank step has the launches of a captured single-camera step."""
    from scsfm import synth
    B, H, W = 2, 96, 160
    tgt, refs, K = synth.triplet(2, B, H, W)
    th0 = theta_of(K[0]) * 1.1
    ixs = [{}] * 4
    if cameras == 2:
        th0 = torch.stack([th0, theta_of(K[0]) * 0.93])
        ixs = [{"camera_index": torch.tensor(ix, dtype=torch.int64, device=DEV)} for ix in ([0, 1], [1, 1], [1, 0], [0, 0])]
    eager, graphed = make_trainer("tf32x3", theta=th0), make_trainer("tf32x3", theta=th0)
    batches = [(tgt.to(DEV), [r.to(DEV) for r in refs], seeded_records(20 + i, B, H, W).to(DEV), ixs[i]) for i in range(4)]
    before = [t.clone() for t in (graphed.camera.theta.detach(),) + graphed._cam_state]
    graphed.capture(batches[0][0], batches[0][1], aug=batches[0][2], **batches[0][3])
    torch.cuda.synchronize()
    for a, b in zip(before, (graphed.camera.theta.detach(),) + graphed._cam_state):
        assert torch.equal(a, b)
    assert graphed.optimizer.step_count == 0
    if cameras == 2:
        single = make_trainer("tf32x3", theta=th0[0])
        single.capture(batches[0][0], batches[0][1], aug=batches[0][2])
        print("captured launches per step: bank %d, one camera %d" % (graphed.launches_per_step, single.launches_per_step))
        assert graphed.launches_per_step == single.launches_per_step
    lr = eager.camera_lr
    grads = {"eager": [], "captured": []}
    for it, (t, r, rec, ix) in enumerate(batches[1:]):
        a = [float(v) for v in eager.step(t, r, aug=rec, **ix)]
        b = [float(v) for v in graphed.step(t, r, aug=rec, **ix)]
        np.testing.assert_allclose(b, a, rtol=2e-4 if it == 0 else 5e-3)
        # the camera gradient the graph computes (theta.grad is the graph's own buffer); the first step starts from identical
        # states, so it and its update are those of the eager step (measured on an H100: the same bits)
        g_e, g_g = eager.camera.theta.grad.cpu(), graphed.camera.theta.grad.cpu()
        print("step %d dtheta: eager %s captured %s rel %.2e" % (it, g_e.tolist(), g_g.tolist(), rel_l2(g_g, g_e)))
        if it == 0:
            assert rel_l2(g_g, g_e) < 1e-4
            assert float((graphed.camera.theta - eager.camera.theta).abs().max()) < 1e-4
        grads["eager"].append(g_e)
        grads["captured"].append(g_g)
    torch.cuda.synchronize()
    # each run's theta is torch.optim.Adam (fp64) applied to that run's own gradients: the update happens in the graph, every replay
    for name, th in (("eager", eager.camera.theta), ("captured", graphed.camera.theta)):
        ref = th0.double().clone().requires_grad_(True)
        opt = torch.optim.Adam([ref], lr=lr, betas=(0.9, 0.999), eps=1e-8)
        for g in grads[name]:
            ref.grad = g.double()
            opt.step()
        assert float((th.detach().cpu().double() - ref.detach()).abs().max()) < 1e-4, (name, th, ref)
    assert graphed.camera_state_dict()["step"] == 3 and eager.camera_state_dict()["step"] == 3
    th_e, th_g = eager.camera.theta.detach().cpu(), graphed.camera.theta.detach().cpu()
    print("theta after 3 steps: eager", th_e.tolist(), "captured", th_g.tolist(), "start", th0.tolist())
    assert float((th_e - th0).abs().min()) > 0                              # every parameter moved
    # Later steps: theta and the networks' parameters against the bound of test_cuda_graph_replay_matches_eager_steps, 3 steps x
    # 2 lr (+ fp32 rounding of the 100-pixel values).  Adam normalises each component's step, so a component whose gradient is at
    # the level of the fp32 atomics noise of the networks' backward (fx here: K enters the warp through K t, and a freshly
    # initialised PoseResNet gives near-zero translations) can step either way in the two runs, whatever its size; the gradients
    # of the next step then follow the two different theta.
    assert float((th_g - th_e).abs().max()) <= 3 * 2 * lr + 1e-4
    assert float((graphed.disp_net.flat_params() - eager.disp_net.flat_params()).abs().max()) <= 6.1e-4


def trainer_argument_errors(cameras):
    """The Trainer refuses malformed camera inputs (K with a camera, no or float32 records, a missing, wrong-shaped or CPU
    camera index, an index for one camera or for no camera) before any launch."""
    from scsfm import synth
    tgt, refs, K = synth.triplet(6, 2, 64, 128)
    c = lambda x: x.to(DEV)  # noqa: E731
    rec = seeded_records(1, 2, 64, 128).to(DEV)
    ix = torch.zeros(2, dtype=torch.int32, device=DEV)
    tr = make_trainer("fp32", theta=theta_of(K[0]) if cameras == 1 else torch.stack([theta_of(K[0])] * 2))
    index = {} if cameras == 1 else {"camera_index": ix}
    with pytest.raises(ValueError, match="owns a learned camera"):
        tr.step(c(tgt), [c(r) for r in refs], c(K), **index)
    with pytest.raises(TypeError, match="records"):
        tr.step(c(tgt), [c(r) for r in refs], **index)
    with pytest.raises(TypeError, match="float64"):
        tr.step(c(tgt), [c(r) for r in refs], aug=torch.zeros(2, 6, device=DEV), **index)
    if cameras == 1:
        with pytest.raises(TypeError, match="one camera"):
            tr.step(c(tgt), [c(r) for r in refs], aug=rec, camera_index=ix)
    else:
        with pytest.raises(TypeError, match="bank of 2 cameras needs"):
            tr.step(c(tgt), [c(r) for r in refs], aug=rec)
        with pytest.raises(TypeError, match="int32 or int64 CUDA"):
            tr.step(c(tgt), [c(r) for r in refs], aug=rec, camera_index=ix.cpu())
        with pytest.raises(TypeError, match="int32 or int64 CUDA"):
            tr.step(c(tgt), [c(r) for r in refs], aug=rec, camera_index=ix[:1])
        with pytest.raises(TypeError, match="bank of 2 cameras needs"):
            tr.capture(c(tgt), [c(r) for r in refs], aug=rec)
    plain = make_trainer("fp32")
    with pytest.raises(TypeError, match="camera"):
        plain.step(c(tgt), [c(r) for r in refs], c(K), aug=torch.zeros(2, 6, dtype=torch.float64, device=DEV))
    with pytest.raises(TypeError, match="no camera"):
        plain.step(c(tgt), [c(r) for r in refs], c(K), camera_index=ix)


def world_of_one(cameras):
    """A data-parallel Trainer in an in-process NCCL world of 1 gives the single-GPU dtheta and theta."""
    import torch.distributed as dist
    from scsfm import synth
    B, H, W = 2, 96, 160
    tgt, refs, K = synth.triplet(8, B, H, W)
    rec = seeded_records(3, B, H, W).to(DEV)
    args = (tgt.to(DEV), [r.to(DEV) for r in refs])
    th0 = theta_of(K[0]) * 0.9
    ix = {}
    if cameras == 2:
        th0 = torch.stack([th0, theta_of(K[0]) * 1.1])
        ix = {"camera_index": torch.tensor([1, 0], dtype=torch.int32, device=DEV)}
    single = make_trainer("tf32x3", theta=th0)
    single.step(*args, aug=rec, **ix)
    with tempfile.TemporaryDirectory() as tmp:
        dist.init_process_group("nccl", init_method="file://" + os.path.join(tmp, "rendezvous"), rank=0, world_size=1,
                                device_id=torch.device(DEV, torch.cuda.current_device()))
        try:
            ddp = make_trainer("tf32x3", distributed=True, theta=th0)
            ddp.step(*args, aug=rec, **ix)
            torch.cuda.synchronize()
            assert ddp.exchange.pending() == 0
            print("world 1 dtheta", ddp.camera.theta.grad.tolist(), "single", single.camera.theta.grad.tolist())
            assert rel_l2(ddp.camera.theta.grad.cpu(), single.camera.theta.grad.cpu()) < 1e-5
            assert rel_l2(ddp.camera.theta.detach().cpu(), single.camera.theta.detach().cpu()) < 1e-5
            assert float((ddp.camera.theta - single.camera.theta).abs().max()) < 1e-4
        finally:
            dist.destroy_process_group()


def two_gpu_check(cameras):
    """tests/camera_ddp_check.py --cameras <cameras> under torchrun on two GPUs prints its OK lines."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(free_port()), os.path.join(ROOT, "tests", "camera_ddp_check.py"), "--cameras", str(cameras)]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=1500)
    print(out.stdout[-4000:])
    assert out.returncode == 0, out.stderr[-4000:]
    for mode in ("eager", "graph"):
        assert "CAMERA_DDP_OK %s" % mode in out.stdout
