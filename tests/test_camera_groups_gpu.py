"""A bank of learned cameras on the GPU: the indexed build against GpuAugment's K (bit for bit), one camera through the bank against
the single-camera path (bit for bit), the per-camera gradient against fp64 autograd, the Trainer with a bank (a bank of one against
one camera, dense Adam against torch.optim.Adam, and with two cameras the checks of tests/camera_helpers.py that one camera runs
too: eager against the fp64 oracle, captured against eager, argument errors, data parallel at world size 1 and on two GPUs),
self-calibration of two cameras at once, and train.py --camera-groups calibration on a dataset on disk."""
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
PKG = os.path.join(ROOT, "sc-sfmlearner-release_b200")


def three_cameras(K):
    """Three distinct cameras derived from one dataset K [3,3] (float32)."""
    return [K, K * torch.tensor([[1.1, 1, 0.9], [1, 0.95, 1.05], [1, 1, 1]]), K * torch.tensor([[0.8, 1, 1.02], [1, 1.2, 0.97], [1, 1, 1]])]


@pytest.mark.parametrize("kind,H,W", [("kitti", 256, 832), ("nyu", 256, 320)])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_indexed_build_equals_gpu_augment_bit_for_bit(kind, H, W, seed):
    from scsfm import camera, synth
    from scsfm.augment import GpuAugment
    B = 16
    Ks = three_cameras(synth.intrinsics(1, H, W, kind)[0])
    idx = torch.from_numpy(np.random.RandomState(seed).randint(0, 3, B)).to(torch.int32)
    K = torch.stack([Ks[int(c)] for c in idx])                              # every sample's own dataset K
    random.seed(seed)
    np.random.seed(seed)
    frames = torch.randint(0, 256, (1, B, H, W, 3), dtype=torch.uint8)
    _, K_aug, rec = GpuAugment(train=True)(frames, K, return_records=True)
    thetas = torch.stack([theta_of(k) for k in Ks]).to(DEV)
    for ix in (idx.to(DEV), idx.to(DEV).long()):
        got = camera.build(thetas, rec, ix)
        assert got.view(torch.int32).equal(K_aug.view(torch.int32)), (got - K_aug).abs().max()


def test_one_camera_bank_is_the_single_camera_path_bit_for_bit():
    from scsfm import camera
    B, H, W = 300, 256, 832
    rec = seeded_records(3, B, H, W).to(DEV)
    th = torch.tensor([483.4, 492.6, 408.3, 118.0], device=DEV)
    zeros = torch.zeros(B, dtype=torch.int32, device=DEV)
    assert camera.build(th[None], rec, zeros).view(torch.int32).equal(camera.build(th, rec).view(torch.int32))
    dK = torch.randn(B, 3, 3, generator=torch.Generator().manual_seed(1)).to(DEV)
    a, b = torch.full((4,), 0.25, device=DEV), torch.full((1, 4), 0.25, device=DEV)
    camera.grad(rec, dK, a)
    camera.grad(rec, dK, b, zeros)
    assert torch.equal(a, b[0])


@pytest.mark.parametrize("B", [1, 5, 300])
@pytest.mark.parametrize("C", [1, 3, 40])
def test_bank_grad_matches_fp64_autograd_per_camera(B, C):
    from scsfm import camera
    rec = seeded_records(B + C, B, 256, 832)
    gen = torch.Generator().manual_seed(B * 100 + C)
    idx = torch.randint(0, C, (B,), generator=gen, dtype=torch.int32)
    dK = torch.randn(B, 3, 3, generator=gen)
    th64 = (torch.tensor([483.4, 492.6, 408.3, 118.0], dtype=torch.float64) * (1 + 0.1 * torch.rand(C, 4, generator=gen,
                                                                                                      dtype=torch.float64)))
    th64.requires_grad_(True)
    (bank_build(th64, rec, idx) * dK.double()).sum().backward()
    runs = []
    for _ in range(2):
        d = torch.full((C, 4), 0.25, device=DEV)                            # the entry ADDS into dtheta
        camera.grad(rec.to(DEV), dK.to(DEV), d, idx.to(DEV))
        runs.append(d.cpu())
    assert torch.equal(runs[0], runs[1])                                    # deterministic: the same bits
    used = set(idx.tolist())
    for c in range(C):
        if c in used:
            assert rel_l2(runs[0][c] - 0.25, th64.grad[c]) < 1e-6, (c, runs[0][c] - 0.25, th64.grad[c])
        else:
            assert torch.equal(runs[0][c], torch.full((4,), 0.25))         # an unused camera: nothing added
    # through autograd: the bank's K, any loss of it, theta.grad (unused rows exact zeros)
    cam = camera.LearnedCamera.bank(th64.detach().float(), 256, 832).to(DEV)
    (cam(rec.to(DEV), idx.to(DEV).long()) * dK.to(DEV)).sum().backward()
    g = cam.theta.grad.cpu()
    for c in range(C):
        if c in used:
            assert rel_l2(g[c], th64.grad[c]) < 1e-6
        else:
            assert torch.equal(g[c], torch.zeros(4))


def test_out_of_range_index_gives_a_nan_k_and_no_gradient():
    from scsfm import camera
    B, C = 6, 3
    rec = seeded_records(4, B, 256, 832).to(DEV)
    th = torch.tensor([[483.4, 492.6, 408.3, 118.0]] * C, device=DEV) * torch.tensor([[1.0], [1.1], [0.9]], device=DEV)
    idx = torch.tensor([0, 3, 1, -1, 2, 1 << 30], dtype=torch.int32, device=DEV)
    K = camera.build(th, rec, idx).cpu()
    bad = [1, 3, 5]
    assert torch.isnan(K[bad]).all()
    good = [0, 2, 4]
    assert not torch.isnan(K[good]).any()
    assert K[good].view(torch.int32).equal(camera.build(th, rec[good], idx[good]).cpu().view(torch.int32))
    dK = torch.randn(B, 3, 3, generator=torch.Generator().manual_seed(2)).to(DEV)
    d_all, d_good = torch.zeros(C, 4, device=DEV), torch.zeros(C, 4, device=DEV)
    camera.grad(rec, dK, d_all, idx)
    camera.grad(rec[good], dK[good], d_good, idx[good])
    assert torch.equal(d_all, d_good)


def test_bank_argument_errors():
    from scsfm.camera import LearnedCamera
    rec = seeded_records(0, 2, 64, 128).to(DEV)
    bank = LearnedCamera.bank(torch.tensor([[100.0, 100, 60, 30]] * 2), 64, 128).to(DEV)
    one = LearnedCamera(100.0, 100, 60, 30, 64, 128).to(DEV)
    with pytest.raises(TypeError, match="camera index of every sample"):
        bank(rec)
    with pytest.raises(TypeError, match="for a bank"):
        one(rec, torch.zeros(2, dtype=torch.int32, device=DEV))
    with pytest.raises(TypeError, match="int32 or int64"):
        bank(rec, torch.zeros(2, dtype=torch.float32, device=DEV))
    with pytest.raises(TypeError, match="int32 or int64"):
        bank(rec, torch.zeros(3, dtype=torch.int32, device=DEV))
    with pytest.raises(RuntimeError, match="device"):
        bank(rec, torch.zeros(2, dtype=torch.int32))


# ---- the Trainer with a bank --------------------------------------------------------------------------------------------------
def test_one_camera_bank_trainer_is_todays_trainer():
    """Two eager steps and a capture: the bank of one camera with every index 0 against LearnedCamera(theta).  The launches are
    the same at every step, and the first step, from identical states, gives the same loss bits and theta.  After it the two
    Trainers' networks differ by the fp32 atomics of their weight gradients (as any two Trainers do), so the later steps are held
    to the tolerances of test_captured_camera_steps_track_eager_steps; the camera arithmetic itself is compared bit for bit in
    test_one_camera_bank_is_the_single_camera_path_bit_for_bit."""
    from scsfm import lib as L
    from scsfm import synth
    B, H, W = 2, 96, 160
    tgt, refs, K = synth.triplet(4, B, H, W)
    th0 = theta_of(K[0]) * 1.05
    batches = [(tgt.to(DEV), [r.to(DEV) for r in refs], seeded_records(40 + i, B, H, W).to(DEV)) for i in range(3)]
    zeros = torch.zeros(B, dtype=torch.int32, device=DEV)
    runs = {}
    for name in ("single", "bank"):
        tr = make_trainer("tf32x3", theta=th0 if name == "single" else th0[None])
        ix = {} if name == "single" else {"camera_index": zeros}
        out, thetas, launches = [], [], []
        for t, r, rec in batches[:2]:
            torch.cuda.synchronize()
            n0 = L.launch_count()
            out.append(torch.stack(tr.step(t, r, aug=rec, **ix)).cpu())
            torch.cuda.synchronize()
            launches.append(L.launch_count() - n0)
            thetas.append(tr.camera.theta.detach().cpu().reshape(4))
        tr.capture(batches[2][0], batches[2][1], aug=batches[2][2], **ix)
        launches.append(tr.launches_per_step)
        out.append(torch.stack(tr.step(batches[2][0], batches[2][1], aug=batches[2][2], **ix)).cpu())
        torch.cuda.synchronize()
        thetas.append(tr.camera.theta.detach().cpu().reshape(4))
        runs[name] = (out, thetas, launches)
    print("launches (eager, eager, captured): single %s bank %s" % (runs["single"][2], runs["bank"][2]))
    for i in range(3):
        print("step %d loss single %s bank %s | theta single %s bank %s" % (i, runs["single"][0][i].tolist(), runs["bank"][0][i].tolist(),
                                                                           runs["single"][1][i].tolist(), runs["bank"][1][i].tolist()))
    assert runs["bank"][2] == runs["single"][2]
    assert torch.equal(runs["bank"][0][0], runs["single"][0][0]) and torch.equal(runs["bank"][1][0], runs["single"][1][0])
    for i in (1, 2):
        np.testing.assert_allclose(runs["bank"][0][i].numpy(), runs["single"][0][i].numpy(), rtol=5e-3)
        assert float((runs["bank"][1][i] - runs["single"][1][i]).abs().max()) <= 3 * 2 * 0.1 + 1e-4


def test_eager_bank_step_gives_the_oracle_theta_gradient():
    eager_step_vs_oracle(2)


def test_bank_adam_is_dense_torch_adam():
    """Three eager steps with C = 3: camera 1 appears only in the first step (then moves by its momentum alone), camera 2 never
    (it keeps theta and zero moments, bit for bit).  theta against torch.optim.Adam on one [3,4] parameter fed the kernel's own
    dtheta, within the bound of test_adam_vs_torch_optim_fp64."""
    from scsfm import synth
    B, H, W = 2, 96, 160
    tgt, refs, K = synth.triplet(6, B, H, W)
    th0 = torch.stack([theta_of(K[0]) * s for s in (1.05, 0.95, 1.1)])
    tr = make_trainer("fp32", theta=th0)
    idxs = [[0, 1], [0, 0], [0, 0]]
    grads = []
    for i, ix in enumerate(idxs):
        tr.step(tgt.to(DEV), [r.to(DEV) for r in refs], aug=seeded_records(60 + i, B, H, W).to(DEV),
                camera_index=torch.tensor(ix, dtype=torch.int32, device=DEV))
        grads.append(tr.camera.theta.grad.detach().cpu().clone())
    torch.cuda.synchronize()
    assert torch.equal(grads[1][1], torch.zeros(4)) and torch.equal(grads[2][1], torch.zeros(4))
    assert float(grads[0][1].abs().max()) > 0
    ref = th0.double().clone().requires_grad_(True)
    opt = torch.optim.Adam([ref], lr=tr.camera_lr, betas=(0.9, 0.999), eps=1e-8)
    for g in grads:
        ref.grad = g.double()
        opt.step()
    th = tr.camera.theta.detach().cpu()
    print("theta after 3 steps", th.tolist(), "torch.optim.Adam", ref.detach().tolist())
    # per step, test_adam_vs_torch_optim_fp64's bound: 1e-5 of the update (at most lr) plus the fp32 rounding of the parameter
    bound = 3 * (1e-5 * tr.camera_lr + 2.0 ** -24 * ref.detach().abs())
    assert bool(((th.double() - ref.detach()).abs() <= bound).all()), (th.double() - ref.detach()).abs()
    assert not torch.equal(th[1], th0[1]) and float((th[1] - th0[1]).abs().min()) > 0          # momentum moved camera 1
    st = tr.camera_state_dict()
    assert st["step"] == 3
    assert torch.equal(th[2], th0[2])
    assert torch.equal(st["exp_avg"][2].cpu(), torch.zeros(4)) and torch.equal(st["exp_avg_sq"][2].cpu(), torch.zeros(4))


def test_captured_bank_steps_track_eager_steps():
    captured_steps_track_eager(2)


def test_trainer_bank_argument_errors():
    trainer_argument_errors(2)


def test_data_parallel_world_of_one_gives_the_single_gpu_bank():
    world_of_one(2)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_data_parallel_bank_on_two_gpus():
    two_gpu_check(2)


# ---- self-calibration of two cameras ------------------------------------------------------------------------------------------
def test_captured_self_calibration_recovers_two_cameras():
    """test_captured_self_calibration_recovers_the_camera with two cameras of different true intrinsics in mixed batches, both
    starting from one common guess (camera 0's fx, fy 20 % and cx, cy 10 px off; camera 1 further), at --intrinsics-lr 0.1:
    each camera ends within 1 % in fx, fy and 1 px in cx, cy (the bounds, and the W - 1 sampling quirk, of that test)."""
    from scsfm import nnops as O
    from scsfm.camera import LearnedCamera
    import loss_functions as LF
    B, H, W, Z0 = 4, 192, 320, 10.0
    true = np.array([[200.0, 190.0, 163.0, 93.0], [240.0, 200.0, 150.0, 100.0]])
    guess = [true[0, 0] * 0.8, true[0, 1] * 1.2, true[0, 2] + 10, true[0, 3] - 10]
    data = []
    g = torch.Generator().manual_seed(9)
    for i in range(12):
        rec = seeded_records(100 + i, B, H, W)
        t = (torch.rand(B, 3, generator=g, dtype=torch.float64) * 2 - 1) * torch.tensor([0.6, 0.4, 1.0], dtype=torch.float64)
        idx = torch.randperm(B, generator=g) % 2                     # two samples of each camera, mixed
        parts = [render_plane(true[int(idx[b])], rec[b:b + 1], H, W, Z0, t[b:b + 1], seed=100 * i + b) for b in range(B)]
        data.append((rec.to(DEV), idx.to(torch.int32).to(DEV)) + tuple(torch.cat(x, 0) for x in zip(*parts)))
    cam = LearnedCamera.bank(torch.tensor([guess, guess]), H, W).to(DEV)
    m, v, step = torch.zeros(2, 4, device=DEV), torch.zeros(2, 4, device=DEV), torch.zeros(1, dtype=torch.int32, device=DEV)
    static = [x.clone() for x in data[0]]

    def one_step():
        rec, idx, tgt, ref, dt, dr, pose, pose_inv = static
        cam.theta.grad = None
        p, q = LF.compute_photo_and_geometry_loss(tgt, [ref], cam(rec, idx), [dt], [[dr]], [pose], [pose_inv], 1, 1, 0, 0, "zeros")
        (p + 0.5 * q).backward()
        step.add_(1)
        O.adam_step(cam.theta.data, cam.theta.grad, m, v, 0.1, 0.9, 0.999, 1e-8, 0.0, 0, step)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        one_step()                                     # warm-up (autograd's lazy state), then undone
    torch.cuda.current_stream().wait_stream(side)
    cam.theta.data.copy_(torch.tensor([guess, guess], dtype=torch.float32))
    m.zero_(); v.zero_(); step.zero_()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        one_step()
    hist = []
    for it in range(3000):
        for dst, src in zip(static, data[it % len(data)]):
            dst.copy_(src, non_blocking=True)
        graph.replay()
        if it % 250 == 249:
            hist.append(cam.theta.detach().cpu().double().numpy().copy())
    th = hist[-1]
    print("two-camera self-calibration (captured): theta %s, true %s, rel %s" % (np.round(th, 3).tolist(), true.tolist(),
                                                                                 np.round(th / true - 1, 5).tolist()))
    print("history:", [np.round(h, 2).tolist() for h in hist])
    for c in range(2):
        assert abs(th[c, 0] / true[c, 0] - 1) < 0.01 and abs(th[c, 1] / true[c, 1] - 1) < 0.01, c
        assert abs(th[c, 2] - true[c, 2]) < 1.0 and abs(th[c, 3] - true[c, 3]) < 1.0, c


# ---- train.py end to end ------------------------------------------------------------------------------------------------------
def test_train_entry_learns_one_camera_per_calibration(tmp_path):
    """train.py on a JPEG tree with 3 training scenes and 2 calibrations (plus a validation scene of the first), the reference's
    loader classes, --learn-intrinsics 1 --camera-groups calibration: an epoch with the captured step and validation, one printed
    line per camera, and a camera checkpoint with theta [2,4] and two group labels."""
    from helpers import make_disk_dataset, reference_loader_env
    env = reference_loader_env()
    if env is None:
        pytest.skip("the original project's modules are not installed (oracle/_ref/, made by __graft_entry__.build())")
    data = make_disk_dataset(str(tmp_path / "data"), scenes=("a", "b", "c", "v"))
    K2 = np.array([[0.62 * 160, 0, 0.5 * 160], [0, 2.0 * 128, 0.45 * 128], [0, 0, 1]])
    np.savetxt(os.path.join(data, "b", "cam.txt"), K2)
    env["PYTHONPATH"] = os.pathsep.join([env["PYTHONPATH"], ROOT])
    cmd = [sys.executable, os.path.join(PKG, "train.py"), data, "--name", "groups", "--learn-intrinsics", "1", "--camera-groups",
           "calibration", "--epochs", "1", "--epoch-size", "3", "-b", "2", "-j", "0", "--print-freq", "1"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=str(tmp_path), env=env)
    print(out.stdout[-3000:])
    assert out.returncode == 0, out.stderr[-4000:]
    assert "learning 2 cameras" in out.stdout
    assert "validation: 3 samples use their training group's learned camera, 0 keep their dataset K" in out.stdout
    lines = [ln for ln in out.stdout.splitlines() if ln.startswith(" * epoch 0 camera ")]
    assert len(lines) == 2 and "a/cam.txt" in lines[0] and "b/cam.txt" in lines[1], lines
    run = os.path.join(str(tmp_path), "checkpoints", "groups")
    stamp = os.listdir(run)[0]
    ck = torch.load(os.path.join(run, stamp, "camera_checkpoint.pth.tar"))
    assert ck["epoch"] == 1 and sorted(ck["state_dict"]) == ["height", "theta", "width"]
    assert ck["groups"] == ["a/cam.txt", "b/cam.txt"]
    th = ck["state_dict"]["theta"]
    assert tuple(th.shape) == (2, 4)
    K1 = np.genfromtxt(os.path.join(data, "a", "cam.txt")).astype(np.float32)
    start = torch.tensor([[K[0, 0], K[1, 1], K[0, 2], K[1, 2]] for K in (K1, K2.astype(np.float32))])
    assert not torch.equal(th, start) and float((th - start).abs().max()) < 3 * 0.1 + 1e-3       # 3 Adam steps at lr 0.1
    assert int(ck["state_dict"]["height"]) == 128 and int(ck["state_dict"]["width"]) == 160
