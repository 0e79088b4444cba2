"""The learned camera on the GPU: the build kernel against GpuAugment's K (bit for bit), its gradient against fp64 autograd, the
Trainer that owns a camera (eager against the fp64 oracle, captured against eager, argument errors, data parallel at world size 1
and on two GPUs: the checks of tests/camera_helpers.py with cameras = 1), the Trainer without a camera unchanged, and
self-calibration of all four intrinsics on a synthetic scene with a captured step."""
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

from camera_helpers import (DEV, bank_build, captured_steps_track_eager, eager_step_vs_oracle, make_trainer, render_plane,
                            seeded_records, theta_of, trainer_argument_errors, two_gpu_check, world_of_one)
from helpers import rel_l2

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("kind,H,W", [("kitti", 256, 832), ("nyu", 256, 320)])
@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_build_equals_gpu_augment_bit_for_bit(kind, H, W, seed):
    from scsfm import camera, synth
    from scsfm.augment import GpuAugment
    B = 16
    random.seed(seed)
    np.random.seed(seed)
    K = synth.intrinsics(B, H, W, kind)
    frames = torch.randint(0, 256, (1, B, H, W, 3), dtype=torch.uint8)
    aug = GpuAugment(train=True)
    imgs0, K0 = aug(frames, K)
    random.seed(seed)
    np.random.seed(seed)
    imgs, K_out, rec = aug(frames, K, return_records=True)
    assert torch.equal(imgs[0], imgs0[0]) and torch.equal(K_out, K0)       # the opt-in third output changes nothing else
    assert rec.dtype == torch.float64 and tuple(rec.shape) == (B, camera.AUG_DOUBLES) and rec.is_cuda
    assert {float(f) for f in rec[:, 2].cpu()} == {0.0, 1.0}
    got = camera.build(theta_of(K[0]).to(DEV), rec)
    assert got.view(torch.int32).equal(K_out.view(torch.int32)), (got - K_out).abs().max()
    # the identity draw gives theta itself
    ident = camera.build(theta_of(K[0]).to(DEV), camera.identity_records(B, W))
    assert ident.cpu().view(torch.int32).equal(K.view(torch.int32))


@pytest.mark.parametrize("B", [1, 5, 300])
def test_grad_matches_fp64_autograd_and_is_deterministic(B):
    from scsfm import camera
    rec = seeded_records(B, B, 256, 832)
    gen = torch.Generator().manual_seed(B)
    dK = torch.randn(B, 3, 3, generator=gen)
    th64 = torch.tensor([483.4, 492.6, 408.3, 118.0], dtype=torch.float64, requires_grad=True)
    (bank_build(th64[None], rec, torch.zeros(B, dtype=torch.long)) * dK.double()).sum().backward()
    runs = []
    for _ in range(2):
        d = torch.full((4,), 0.25, device=DEV)                             # the entry ADDS into dtheta
        camera.grad(rec.to(DEV), dK.to(DEV), d)
        runs.append(d.cpu())
    assert torch.equal(runs[0], runs[1])
    assert rel_l2(runs[0] - 0.25, th64.grad) < 1e-6, (runs[0] - 0.25, th64.grad)
    # through autograd: the LearnedCamera's K, any loss of it, theta.grad
    cam = camera.LearnedCamera(483.4, 492.6, 408.3, 118.0, 256, 832).to(DEV)
    (cam(rec.to(DEV)) * dK.to(DEV)).sum().backward()
    assert rel_l2(cam.theta.grad.cpu(), th64.grad) < 1e-6


def test_eager_camera_step_gives_the_oracle_theta_gradient():
    eager_step_vs_oracle(1)


def test_captured_camera_steps_track_eager_steps():
    captured_steps_track_eager(1)


def test_no_camera_step_is_unchanged_and_the_camera_path_adds_four_launches():
    """Without a camera: the step launches what it launched before the feature (eager = captured) and the K argument is used as
    given.  With a camera whose theta is the dataset's K and identity records, K_b is that K bit for bit, so the losses are the
    same bits; the camera path adds exactly build + intrinsics gradient + camera gradient + theta's Adam."""
    from scsfm import lib as L
    from scsfm import synth
    B, H, W = 2, 96, 160
    tgt, refs, K = synth.triplet(4, B, H, W)
    args = (tgt.to(DEV), [r.to(DEV) for r in refs])
    from scsfm.camera import identity_records
    runs = {}
    for name, th in (("plain", None), ("camera", theta_of(K[0]))):
        tr = make_trainer("tf32x3", th)
        inp = dict(intrinsics=K.to(DEV)) if th is None else dict(aug=identity_records(B, W))
        torch.cuda.synchronize()
        n0 = L.launch_count()
        out = torch.stack(tr.step(*args, **inp))
        torch.cuda.synchronize()
        eager_launches = L.launch_count() - n0
        tr.capture(*args, **inp)
        runs[name] = (eager_launches, tr.launches_per_step, out.cpu())
        with pytest.raises((TypeError, ValueError)):
            tr.step(*args, intrinsics=K.to(DEV), aug=identity_records(B, W))       # K and records together: refused
    print("launches per step (eager, captured): without a camera %s, with one %s" % (runs["plain"][:2], runs["camera"][:2]))
    assert runs["camera"][0] == runs["plain"][0] + 4 and runs["camera"][1] == runs["plain"][1] + 4
    assert torch.equal(runs["camera"][2], runs["plain"][2])


def test_trainer_camera_argument_errors():
    trainer_argument_errors(1)


def test_data_parallel_world_of_one_gives_the_single_gpu_theta():
    world_of_one(1)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_data_parallel_camera_on_two_gpus():
    two_gpu_check(1)


# ---- self-calibration on a synthetic scene -------------------------------------------------------------------------------------
def test_captured_self_calibration_recovers_the_camera():
    """The camera path alone in a captured step (K_b from theta, photometric + geometry loss, theta's gradient, Adam at the
    default --intrinsics-lr 0.1), on a plane at Z0 = 10 m rendered exactly for every augmented camera, each sample with its own
    translation with x, y and z parts: from fx, fy 20 % and cx, cy 10 px off, fx and fy end within 1 % and cx, cy within 1 px.

    With a pure translation t, K enters the warp only through K t: the shift of a sample is (fx tx + cx tz, fy ty + cy tz) / (Z + tz),
    so it takes translations with different x : z and y : z ratios to separate the focal length from the principal point.

    Why not exactly: the warp samples the source image at x * W / (W - 1) - 0.5 instead of x (the reference normalises by W - 1
    and grid_sample does not align corners), a stretch that no camera reproduces.  Least squares over pixels centred on
    (W - 1) / 2 puts the optimum at fx* (1 - 1/W), fy* (1 - 1/H) -- 0.31 % / 0.52 % here, the same quirk that biased fx by 0.53 %
    at W = 128 in test_self_calibration_recovers_the_focal_length -- and at cx* - cx*/W + (offset_x/W + (W - 1)/(2W)) / x_scale
    (mirrored under the flip), i.e. within 0.2 px of cx* for the crops and zooms of RandomScaleCrop (the same for cy).  The 1 px
    bound leaves room for the non-uniform pixel weights of the SSIM loss and the validity mask."""
    from scsfm import nnops as O
    from scsfm.camera import LearnedCamera
    import loss_functions as LF
    B, H, W, Z0 = 4, 192, 320, 10.0
    true = np.array([200.0, 190.0, 163.0, 93.0])
    data = []
    g = torch.Generator().manual_seed(9)
    for i in range(12):
        rec = seeded_records(100 + i, B, H, W)
        t = (torch.rand(B, 3, generator=g, dtype=torch.float64) * 2 - 1) * torch.tensor([0.6, 0.4, 1.0], dtype=torch.float64)
        data.append((rec.to(DEV),) + render_plane(true, rec, H, W, Z0, t, seed=i))
    cam = LearnedCamera(true[0] * 0.8, true[1] * 1.2, true[2] + 10, true[3] - 10, H, W).to(DEV)
    m, v, step = torch.zeros(4, device=DEV), torch.zeros(4, device=DEV), torch.zeros(1, dtype=torch.int32, device=DEV)
    static = [x.clone() for x in data[0]]

    def one_step():
        rec, tgt, ref, dt, dr, pose, pose_inv = static
        cam.theta.grad = None
        p, q = LF.compute_photo_and_geometry_loss(tgt, [ref], cam(rec), [dt], [[dr]], [pose], [pose_inv], 1, 1, 0, 0, "zeros")
        (p + 0.5 * q).backward()
        step.add_(1)
        O.adam_step(cam.theta.data, cam.theta.grad, m, v, 0.1, 0.9, 0.999, 1e-8, 0.0, 0, step)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        one_step()                                     # warm-up (autograd's lazy state), then undone
    torch.cuda.current_stream().wait_stream(side)
    cam.theta.data.copy_(torch.tensor([true[0] * 0.8, true[1] * 1.2, true[2] + 10, true[3] - 10], dtype=torch.float32))
    m.zero_(); v.zero_(); step.zero_()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        one_step()
    hist = []
    for it in range(1500):
        for dst, src in zip(static, data[it % len(data)]):
            dst.copy_(src, non_blocking=True)
        graph.replay()
        if it % 100 == 99:
            hist.append(cam.theta.detach().cpu().double().numpy().copy())
    th = hist[-1]
    print("self-calibration (captured): theta %s, true %s, rel %s" % (np.round(th, 3), true, np.round(th / true - 1, 5)))
    print("history fx fy:", [tuple(np.round(h[:2], 2)) for h in hist])
    assert abs(th[0] / true[0] - 1) < 0.01 and abs(th[1] / true[1] - 1) < 0.01
    assert abs(th[2] - true[2]) < 1.0 and abs(th[3] - true[3]) < 1.0


def test_train_entry_learns_intrinsics_with_the_captured_step(tmp_path):
    """train.py synthetic --gpu-augment 1 --learn-intrinsics 1: an epoch with the captured step, camera printed and saved."""
    pkg = os.path.join(ROOT, "sc-sfmlearner-release_b200")
    cmd = [sys.executable, os.path.join(pkg, "train.py"), "synthetic", "--name", "calib", "--gpu-augment", "1", "--learn-intrinsics",
           "1", "--epochs", "1", "--epoch-size", "4", "-b", "2", "--synthetic-size", "128", "256", "--print-freq", "2"]
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([pkg, ROOT]))
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=str(tmp_path), env=env)
    print(out.stdout[-3000:])
    assert out.returncode == 0, out.stderr[-4000:]
    assert "learned camera fx" in out.stdout
    run = os.path.join(str(tmp_path), "checkpoints", "calib")
    stamp = os.listdir(run)[0]
    files = sorted(os.listdir(os.path.join(run, stamp)))
    assert "camera_checkpoint.pth.tar" in files and "dispnet_checkpoint.pth.tar" in files and "exp_pose_checkpoint.pth.tar" in files
    ck = torch.load(os.path.join(run, stamp, "camera_checkpoint.pth.tar"))
    assert ck["epoch"] == 1 and sorted(ck["state_dict"]) == ["height", "theta", "width"]
    assert int(ck["state_dict"]["height"]) == 128 and int(ck["state_dict"]["width"]) == 256
    from scsfm import synth
    K = synth.intrinsics(1, 128, 256)[0]
    th = ck["state_dict"]["theta"]
    assert not torch.equal(th, theta_of(K)) and float((th - theta_of(K)).abs().max()) < 4 * 0.1 + 1e-3      # 4 Adam steps at lr 0.1
