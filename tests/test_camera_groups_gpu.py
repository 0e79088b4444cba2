"""A bank of learned cameras on the GPU: the indexed build against GpuAugment's K (bit for bit), one camera through the bank against
the single-camera path (bit for bit), the per-camera gradient against fp64 autograd, the Trainer with a bank (eager against the
fp64 oracle, dense Adam against torch.optim.Adam, captured against eager, launch counts, data parallel at world size 1 and on two
GPUs), self-calibration of two cameras at once, and train.py --camera-groups calibration on a dataset on disk."""
import os
import random
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from helpers import rel_l2
from test_camera_gpu import _free_port, _nets, render_plane, seeded_records, theta_of, torch_build

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "sc-sfmlearner-release_b200")


def bank_build(thetas, rec, idx):
    """K_b = aug_b(thetas[idx_b]) restated in torch (differentiable; the dtype of thetas)."""
    rec = rec.to(thetas.device, thetas.dtype)
    xs, ys, flip, ox, oy, in_w = rec.unbind(1)
    fx, fy, cx, cy = thetas[idx.long().to(thetas.device)].unbind(1)
    cxb = torch.where(flip != 0, in_w - cx, cx)
    zero, one = torch.zeros_like(xs), torch.ones_like(xs)
    return torch.stack([torch.stack([fx * xs, zero, cxb * xs - ox], 1), torch.stack([zero, fy * ys, cy * ys - oy], 1),
                        torch.stack([zero, zero, one], 1)], 1)


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
def _trainer(mode="fp32", theta=None, bank=None, **kw):
    """theta: one camera [4]; bank: thetas [C,4]."""
    from scsfm.camera import LearnedCamera
    from scsfm.trainer import Trainer
    d, p = _nets()
    cam = None
    if theta is not None:
        cam = LearnedCamera(*[float(v) for v in theta]).to(DEV)
    elif bank is not None:
        cam = LearnedCamera.bank(torch.as_tensor(bank, dtype=torch.float32)).to(DEV)
    kw.setdefault("distributed", False)
    return Trainer(d, p, lr=1e-4, with_auto_mask=0, conv_mode=mode, camera=cam, **kw)


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
        tr = _trainer("tf32x3", theta=th0) if name == "single" else _trainer("tf32x3", bank=th0[None])
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
    """dtheta [2,4] of an eager step against oracle.step.train_step in fp64 with K_b = aug_b(theta[idx_b]); the bound of
    test_eager_camera_step_gives_the_oracle_theta_gradient (4x the larger fp32 error + 1e-3)."""
    from golden_util import det_weights
    from oracle import nets as N
    from oracle import step as OS
    from scsfm import synth
    B, H, W = 2, 96, 160
    tgt, refs, K = synth.triplet(5, B, H, W)
    rec = seeded_records(11, B, H, W)
    idx = torch.tensor([1, 0], dtype=torch.int32)
    th0 = torch.stack([theta_of(K[0]) * torch.tensor([1.05, 0.97, 1.0, 1.0]) + torch.tensor([0.0, 0.0, 2.0, -1.5]),
                       theta_of(K[0]) * torch.tensor([0.95, 1.02, 1.0, 1.0]) + torch.tensor([0.0, 0.0, -3.0, 1.0])])
    tr = _trainer("fp32", bank=th0)
    tr.step(tgt.to(DEV), [r.to(DEV) for r in refs], aug=rec.to(DEV), camera_index=idx.to(DEV))
    mine = tr.camera.theta.grad.cpu()
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
    errs = {k: rel_l2(g, want["64"]) for k, g in (("mine", mine), ("32", want["32"]), ("32gpu", want["32gpu"]))}
    print("bank dtheta rel_l2 vs fp64: mine %.3g | fp32 CPU oracle %.3g | stock PyTorch fp32 on this GPU %.3g" %
          (errs["mine"], errs["32"], errs["32gpu"]))
    assert errs["mine"] < 4 * max(errs["32"], errs["32gpu"]) + 1e-3


def test_bank_adam_is_dense_torch_adam():
    """Three eager steps with C = 3: camera 1 appears only in the first step (then moves by its momentum alone), camera 2 never
    (it keeps theta and zero moments, bit for bit).  theta against torch.optim.Adam on one [3,4] parameter fed the kernel's own
    dtheta, within the bound of test_adam_vs_torch_optim_fp64."""
    from scsfm import synth
    B, H, W = 2, 96, 160
    tgt, refs, K = synth.triplet(6, B, H, W)
    th0 = torch.stack([theta_of(K[0]) * s for s in (1.05, 0.95, 1.1)])
    tr = _trainer("fp32", bank=th0)
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
    """As test_captured_camera_steps_track_eager_steps with a bank of two cameras and mixed indices; capture() leaves theta and its
    Adam state bitwise unchanged, and a captured bank step has the launches of a captured single-camera step."""
    from scsfm import synth
    B, H, W = 2, 96, 160
    tgt, refs, K = synth.triplet(2, B, H, W)
    th0 = torch.stack([theta_of(K[0]) * 1.1, theta_of(K[0]) * 0.93])
    eager, graphed = _trainer("tf32x3", bank=th0), _trainer("tf32x3", bank=th0)
    ixs = [[0, 1], [1, 1], [1, 0], [0, 0]]
    batches = [(tgt.to(DEV), [r.to(DEV) for r in refs], seeded_records(20 + i, B, H, W).to(DEV),
                torch.tensor(ix, dtype=torch.int64, device=DEV)) for i, ix in enumerate(ixs)]
    before = [t.clone() for t in (graphed.camera.theta.detach(),) + graphed._cam_state]
    graphed.capture(batches[0][0], batches[0][1], aug=batches[0][2], camera_index=batches[0][3])
    torch.cuda.synchronize()
    for a, b in zip(before, (graphed.camera.theta.detach(),) + graphed._cam_state):
        assert torch.equal(a, b)
    single = _trainer("tf32x3", theta=th0[0])
    single.capture(batches[0][0], batches[0][1], aug=batches[0][2])
    print("captured launches per step: bank %d, one camera %d" % (graphed.launches_per_step, single.launches_per_step))
    assert graphed.launches_per_step == single.launches_per_step
    lr = eager.camera_lr
    grads = {"eager": [], "captured": []}
    for it, (t, r, rec, ix) in enumerate(batches[1:]):
        a = [float(v) for v in eager.step(t, r, aug=rec, camera_index=ix)]
        b = [float(v) for v in graphed.step(t, r, aug=rec, camera_index=ix)]
        np.testing.assert_allclose(b, a, rtol=2e-4 if it == 0 else 5e-3)
        g_e, g_g = eager.camera.theta.grad.cpu(), graphed.camera.theta.grad.cpu()
        print("step %d dtheta: eager %s captured %s rel %.2e" % (it, g_e.tolist(), g_g.tolist(), rel_l2(g_g, g_e)))
        if it == 0:
            assert rel_l2(g_g, g_e) < 1e-4
            assert float((graphed.camera.theta - eager.camera.theta).abs().max()) < 1e-4
        grads["eager"].append(g_e)
        grads["captured"].append(g_g)
    torch.cuda.synchronize()
    for name, th in (("eager", eager.camera.theta), ("captured", graphed.camera.theta)):
        ref = th0.double().clone().requires_grad_(True)
        opt = torch.optim.Adam([ref], lr=lr, betas=(0.9, 0.999), eps=1e-8)
        for g in grads[name]:
            ref.grad = g.double()
            opt.step()
        assert float((th.detach().cpu().double() - ref.detach()).abs().max()) < 1e-4, (name, th, ref)
    assert graphed.camera_state_dict()["step"] == 3
    th_e, th_g = eager.camera.theta.detach().cpu(), graphed.camera.theta.detach().cpu()
    assert float((th_g - th_e).abs().max()) <= 3 * 2 * lr + 1e-4
    assert float((graphed.disp_net.flat_params() - eager.disp_net.flat_params()).abs().max()) <= 6.1e-4


def test_trainer_bank_argument_errors():
    from scsfm import synth
    tgt, refs, K = synth.triplet(6, 2, 64, 128)
    c = lambda x: x.to(DEV)  # noqa: E731
    rec = seeded_records(1, 2, 64, 128).to(DEV)
    ix = torch.zeros(2, dtype=torch.int32, device=DEV)
    bank = _trainer("fp32", bank=torch.stack([theta_of(K[0])] * 2))
    with pytest.raises(TypeError, match="bank of 2 cameras needs"):
        bank.step(c(tgt), [c(r) for r in refs], aug=rec)
    with pytest.raises(TypeError, match="int32 or int64 CUDA"):
        bank.step(c(tgt), [c(r) for r in refs], aug=rec, camera_index=ix.cpu())
    with pytest.raises(TypeError, match="int32 or int64 CUDA"):
        bank.step(c(tgt), [c(r) for r in refs], aug=rec, camera_index=ix[:1])
    with pytest.raises(TypeError, match="bank of 2 cameras needs"):
        bank.capture(c(tgt), [c(r) for r in refs], aug=rec)
    one = _trainer("fp32", theta=theta_of(K[0]))
    with pytest.raises(TypeError, match="one camera"):
        one.step(c(tgt), [c(r) for r in refs], aug=rec, camera_index=ix)
    plain = _trainer("fp32")
    with pytest.raises(TypeError, match="no camera"):
        plain.step(c(tgt), [c(r) for r in refs], c(K), camera_index=ix)


def test_data_parallel_world_of_one_gives_the_single_gpu_bank():
    import torch.distributed as dist
    from scsfm import synth
    B, H, W = 2, 96, 160
    tgt, refs, K = synth.triplet(8, B, H, W)
    rec = seeded_records(3, B, H, W).to(DEV)
    ix = torch.tensor([1, 0], dtype=torch.int32, device=DEV)
    args = (tgt.to(DEV), [r.to(DEV) for r in refs])
    th0 = torch.stack([theta_of(K[0]) * 0.9, theta_of(K[0]) * 1.1])
    single = _trainer("tf32x3", bank=th0)
    single.step(*args, aug=rec, camera_index=ix)
    with tempfile.TemporaryDirectory() as tmp:
        dist.init_process_group("nccl", init_method="file://" + os.path.join(tmp, "rendezvous"), rank=0, world_size=1,
                                device_id=torch.device(DEV, torch.cuda.current_device()))
        try:
            ddp = _trainer("tf32x3", bank=th0, distributed=True)
            ddp.step(*args, aug=rec, camera_index=ix)
            torch.cuda.synchronize()
            assert ddp.exchange.pending() == 0
            print("world 1 dtheta", ddp.camera.theta.grad.tolist(), "single", single.camera.theta.grad.tolist())
            assert rel_l2(ddp.camera.theta.grad.cpu(), single.camera.theta.grad.cpu()) < 1e-5
            assert rel_l2(ddp.camera.theta.detach().cpu(), single.camera.theta.detach().cpu()) < 1e-5
        finally:
            dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_data_parallel_bank_on_two_gpus():
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), os.path.join(ROOT, "tests", "camera_groups_ddp_check.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=1500)
    print(out.stdout[-4000:])
    assert out.returncode == 0, out.stderr[-4000:]
    for mode in ("eager", "graph"):
        assert "CAMERA_GROUPS_DDP_OK %s" % mode in out.stdout


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
