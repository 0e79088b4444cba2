"""Gradients with respect to the camera intrinsics (learned / self-calibrated K) through the fused loss and inverse_warp2, on
the GPU, against the fp64 oracle.  Yardstick, as for the pose gradients in test_warp_loss_gpu.py: the L2 error against fp64 is
at most 3x that of an independent fp32 evaluation (the reference's own, or the fp32 oracle's) plus 2e-4."""
import os
import tempfile

import numpy as np
import pytest
import torch

from helpers import SUB, frac_within, golden_loss_inputs, rel_l2
from test_intrinsics_grad_cpu import golden_k, iw2_upstream, oracle_iw2_dK, oracle_loss_dK  # noqa: F401  (golden_k: fixture)

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _api():
    import inverse_warp
    import loss_functions
    return inverse_warp, loss_functions


def _yardstick(mine, ref32, ref64):
    return rel_l2(mine, ref64) < 3 * rel_l2(ref32, ref64) + 2e-4


def _cuda_inputs(d, requires_grad=True):
    c = lambda x: x.to(DEV)  # noqa: E731
    leaf = lambda x: c(x).requires_grad_(requires_grad)  # noqa: E731
    return (c(d["tgt_img"]), [c(x) for x in d["ref_imgs"]], leaf(d["intrinsics"]), [leaf(x) for x in d["tgt_depth"]],
            [[leaf(x) for x in r] for r in d["ref_depths"]], [leaf(x) for x in d["poses"]], [leaf(x) for x in d["poses_inv"]])


def _oracle_dK(d, n_scales, flags, pm, dtype):
    from oracle import losses as OL
    K = d["intrinsics"].to(dtype, copy=True).requires_grad_(True)
    cv = lambda x: x.to(dtype)  # noqa: E731
    p, q = OL.compute_photo_and_geometry_loss(cv(d["tgt_img"]), [cv(x) for x in d["ref_imgs"]], K, [cv(x) for x in d["tgt_depth"]],
                                              [[cv(x) for x in r] for r in d["ref_depths"]], [cv(x) for x in d["poses"]],
                                              [cv(x) for x in d["poses_inv"]], n_scales, *flags, pm)
    (p + 0.5 * q).backward()
    return K.grad


@pytest.mark.parametrize("pm", ["zeros", "border"])
@pytest.mark.parametrize("flags", [(1, 1, 0), (1, 1, 1)])
def test_loss_intrinsics_gradient_vs_reference_and_fp64_oracle(golden_warp, golden_k, pm, flags):  # noqa: F811
    """The golden loss inputs (2 references, 2 scales): dK within the reference's yardstick, and the depth and pose gradients of
    the same call still within the bounds of test_gradients_vs_reference_and_fp64_oracle."""
    from oracle import losses as OL
    _, lf = _api()
    g = golden_warp
    tag = f"{pm}_g{flags[0]}{flags[1]}{flags[2]}"
    tgt, refs, K, td, rd, ps, pi = golden_loss_inputs(g, device=DEV, requires_grad=True)
    K.requires_grad_(True)
    p, q = lf.compute_photo_and_geometry_loss(tgt, refs, K, td, rd, ps, pi, 2, *flags, pm)
    s = lf.compute_smooth_loss(td, tgt, rd, refs)
    (p + 0.5 * q + 0.1 * s).backward()
    k64 = oracle_loss_dK(g, pm, flags)
    k32 = golden_k[f"{pm}_loss_K{flags[0]}{flags[1]}{flags[2]}"]
    print(pm, flags, "dK rel_l2 vs fp64: mine %.3g, reference fp32 %.3g" % (rel_l2(K.grad, k64), rel_l2(k32, k64)))
    assert _yardstick(K.grad, k32, k64)
    o = golden_loss_inputs(g, torch.float64, requires_grad=True)
    po, qo = OL.compute_photo_and_geometry_loss(o[0], o[1], o[2], o[3], o[4], o[5], o[6], 2, *flags, pm)
    (po + 0.5 * qo + 0.1 * OL.compute_smooth_loss(o[3], o[0], o[4], o[1])).backward()
    for sidx in range(2):
        for mine, ref32, ref64 in [(td[sidx], g[f"{tag}_tgt_depth_s{sidx}"], o[3][sidx])] + \
                                  [(rd[i][sidx], g[f"{tag}_ref_depth{i}_s{sidx}"], o[4][i][sidx]) for i in range(2)]:
            assert frac_within(mine.grad[SUB], ref32, 1e-4) > 0.995
            assert rel_l2(mine.grad[SUB], ref64.grad[SUB]) < 3 * rel_l2(ref32, ref64.grad[SUB]) + 1e-4
    for i in range(2):
        assert _yardstick(ps[i].grad, g[f"{tag}_pose{i}"], o[5][i].grad)
        assert _yardstick(pi[i].grad, g[f"{tag}_pose_inv{i}"], o[6][i].grad)


@pytest.mark.parametrize("pm", ["zeros", "border"])
def test_inverse_warp2_intrinsics_gradient_vs_reference(golden_warp, golden_k, pm):  # noqa: F811
    iw, _ = _api()
    tgt, refs, K, td, rd, ps, pi = golden_loss_inputs(golden_warp, device=DEV)
    K.requires_grad_(True)
    B, _, H, W = tgt.shape
    ups = [u.to(DEV) for u in iw2_upstream(golden_k, B, H, W)]
    w, v, pd, cd = iw.inverse_warp2(refs[0], td[0], rd[0][0], ps[0], K, pm)
    ((w * ups[0]).sum() + (pd * ups[1]).sum() + (cd * ups[2]).sum()).backward()
    k64 = oracle_iw2_dK(golden_warp, golden_k, pm)
    assert _yardstick(K.grad, golden_k[f"{pm}_iw2_K"], k64), (rel_l2(K.grad, k64), rel_l2(golden_k[f"{pm}_iw2_K"], k64))


@pytest.mark.parametrize("shape", [(1, 50, 70), (3, 33, 97)])
@pytest.mark.parametrize("pm", ["zeros", "border"])
def test_inverse_warp2_ragged_sizes_vs_fp64_oracle(shape, pm):
    """Sizes that are not multiples of the block; random upstream gradients on warped image, projected and computed depth."""
    import scsfm.synth as synth
    from oracle import geometry as OG
    iw, _ = _api()
    B, H, W = shape
    d = synth.loss_inputs(5, B, H, W, n_ref=1, n_scales=1)
    pose = d["poses"][0] * 4
    gen = torch.Generator().manual_seed(2)
    ups = [torch.randn(B, c, H, W, generator=gen) for c in (3, 1, 1)]
    Kc = d["intrinsics"].to(DEV).requires_grad_(True)
    w, _, pd, cd = iw.inverse_warp2(d["ref_imgs"][0].to(DEV), d["tgt_depth"][0].to(DEV), d["ref_depths"][0][0].to(DEV), pose.to(DEV),
                                    Kc, pm)
    ((w * ups[0].to(DEV)).sum() + (pd * ups[1].to(DEV)).sum() + (cd * ups[2].to(DEV)).sum()).backward()
    want = {}
    for dt in (torch.float32, torch.float64):
        K = d["intrinsics"].to(dt, copy=True).requires_grad_(True)
        w2, _, pd2, cd2 = OG.inverse_warp2(d["ref_imgs"][0].to(dt), d["tgt_depth"][0].to(dt), d["ref_depths"][0][0].to(dt),
                                           pose.to(dt), K, pm)
        ((w2 * ups[0].to(dt)).sum() + (pd2 * ups[1].to(dt)).sum() + (cd2 * ups[2].to(dt)).sum()).backward()
        want[dt] = K.grad
    assert _yardstick(Kc.grad, want[torch.float32], want[torch.float64]), (rel_l2(Kc.grad, want[torch.float64]),
                                                                          rel_l2(want[torch.float32], want[torch.float64]))


def test_pairwise_loss_intrinsics_gradient_vs_fp64_oracle(golden_warp):
    """compute_pairwise_loss: one direction, one job."""
    from oracle import losses as OL
    _, lf = _api()
    tgt, refs, K, td, rd, ps, pi = golden_loss_inputs(golden_warp, device=DEV)
    K.requires_grad_(True)
    p, q = lf.compute_pairwise_loss(tgt, refs[1], td[0], rd[1][0], ps[1], K, 1, 1, 1, "zeros")
    (p + 0.5 * q).backward()
    want = {}
    for dt in (torch.float32, torch.float64):
        o = golden_loss_inputs(golden_warp, dt)
        Ko = o[2].clone().requires_grad_(True)
        po, qo = OL.compute_pairwise_loss(o[0], o[1][1], o[3][0], o[4][1][0], o[5][1], Ko, 1, 1, 1, "zeros")
        (po + 0.5 * qo).backward()
        want[dt] = Ko.grad
    assert _yardstick(K.grad, want[torch.float32], want[torch.float64]), (rel_l2(K.grad, want[torch.float64]),
                                                                         rel_l2(want[torch.float32], want[torch.float64]))


def test_two_chunks_of_jobs_accumulate():
    """4 references x 4 scales x 2 directions = 32 pair-directions: two MAX_JOBS chunks, one extra launch each."""
    import scsfm.synth as synth
    from scsfm import lib as L
    _, lf = _api()
    d = synth.loss_inputs(9, 2, 64, 128, n_ref=4, n_scales=4)
    tgt, refs, K, td, rd, ps, pi = _cuda_inputs(d)
    p, q = lf.compute_photo_and_geometry_loss(tgt, refs, K, td, rd, ps, pi, 4, 1, 1, 0, "zeros")
    assert 2 * 4 * 4 == 2 * L.MAX_JOBS
    torch.cuda.synchronize()
    n0 = L.launch_count()
    (p + 0.5 * q).backward()
    torch.cuda.synchronize()
    assert L.launch_count() - n0 == 2 * 3          # per chunk: loss backward, pose gradient, intrinsics gradient
    k32 = _oracle_dK(d, 4, (1, 1, 0), "zeros", torch.float32)
    k64 = _oracle_dK(d, 4, (1, 1, 0), "zeros", torch.float64)
    assert _yardstick(K.grad, k32, k64), (rel_l2(K.grad, k64), rel_l2(k32, k64))


def test_shared_parameter_gets_the_sum_over_the_batch(golden_warp):
    """One [3,3] parameter expanded to the batch gets the sum of the per-sample gradients."""
    _, lf = _api()
    tgt, refs, K, td, rd, ps, pi = golden_loss_inputs(golden_warp, device=DEV)
    B = tgt.shape[0]
    per = K[:1].clone().expand(B, 3, 3).contiguous().requires_grad_(True)     # the same K for every sample, per-sample leaf
    p, q = lf.compute_photo_and_geometry_loss(tgt, refs, per, td, rd, ps, pi, 2, 1, 1, 1, "border")
    (p + 0.5 * q).backward()
    shared = torch.nn.Parameter(K[0].clone())
    p2, q2 = lf.compute_photo_and_geometry_loss(tgt, refs, shared.expand(B, 3, 3), td, rd, ps, pi, 2, 1, 1, 1, "border")
    (p2 + 0.5 * q2).backward()
    assert shared.grad.shape == (3, 3)
    assert rel_l2(shared.grad, per.grad.sum(0)) < 1e-6


def test_deferred_finalize_equals_the_plain_path(golden_warp):
    """The exact-global data-parallel path (sums all-reduced between forward and finalize) at world size 1: the backward scales
    carry the loss scale, so dK equals the plain path's."""
    from scsfm import loss_ops
    out = []
    for allreduce in (None, lambda t: None):
        tgt, refs, K, td, rd, ps, pi = golden_loss_inputs(golden_warp, device=DEV)
        K.requires_grad_(True)
        p, q = loss_ops.photo_and_geometry_loss(tgt, refs, K, td, rd, ps, pi, 2, 1, 1, 1, "zeros", sums_allreduce=allreduce, world=1)
        (p + 0.5 * q).backward()
        out.append(K.grad)
    assert rel_l2(out[1], out[0]) < 1e-6


def test_launches_and_outputs_without_and_with_intrinsics_gradient(golden_warp):
    """K without a gradient: the backward launches exactly what it launched before the feature (loss backward + pose gradient per
    chunk) and the outputs do not depend on whether K asks for a gradient.  K with a gradient: one more launch per chunk."""
    from scsfm import lib as L
    _, lf = _api()
    runs = []
    for k_grad in (False, True):
        tgt, refs, K, td, rd, ps, pi = golden_loss_inputs(golden_warp, device=DEV, n_scales=1, requires_grad=True)
        K.requires_grad_(k_grad)
        p, q = lf.compute_photo_and_geometry_loss(tgt, refs, K, td, rd, ps, pi, 1, 1, 1, 0, "zeros")
        torch.cuda.synchronize()
        n0 = L.launch_count()
        (p + 0.5 * q).backward()
        torch.cuda.synchronize()
        runs.append(dict(launches=L.launch_count() - n0, loss=torch.stack([p, q]).detach(), K=K.grad,
                         poses=[x.grad for x in ps + pi], depths=[x.grad for x in td + [r[0] for r in rd]]))
    off, on = runs
    assert off["K"] is None and on["K"] is not None
    assert off["launches"] == 2 and on["launches"] == 3
    assert torch.equal(off["loss"], on["loss"])
    for a, b in zip(off["poses"], on["poses"]):
        assert torch.equal(a, b)
    for a, b in zip(off["depths"], on["depths"]):      # scattered with fp32 atomics: summation order only
        assert rel_l2(b, a) < 1e-6


def _nets(mode="fp32"):
    import models
    from golden_util import det_weights
    d, p = models.DispResNet(18, False), models.PoseResNet(18, False)
    for n in (d, p):
        n.load_state_dict(det_weights(n.state_dict()))
    return d, p


def test_trainer_eager_step_gives_the_oracle_intrinsics_gradient():
    """A learned K in the eager single-GPU step: K.grad against the fp64 oracle's train_step, with the fp32 oracle as yardstick."""
    from golden_util import det_weights
    from oracle import nets as N
    from oracle import step as OS
    from scsfm import synth
    from scsfm.trainer import Trainer
    B, H, W = 2, 96, 160
    tgt, refs, K = synth.triplet(5, B, H, W)
    disp, pose = _nets()
    tr = Trainer(disp.to(DEV).train(), pose.to(DEV).train(), lr=1e-4, with_auto_mask=0, distributed=False, conv_mode="fp32")
    Kc = K.to(DEV).requires_grad_(True)
    tr.step(tgt.to(DEV), [r.to(DEV) for r in refs], Kc)
    want = {}
    # fp64 oracle; fp32 oracle on the CPU; fp32 oracle through stock PyTorch / cuDNN on this GPU with TF32 off
    tf32 = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        for key, dt, dev in (("64", torch.float64, "cpu"), ("32", torch.float32, "cpu"), ("32gpu", torch.float32, DEV)):
            d, p = N.DispResNet(18).to(dt).to(dev), N.PoseResNet(18).to(dt).to(dev)
            for n in (d, p):
                n.load_state_dict({k: v.to(dt) for k, v in det_weights(n.state_dict()).items()})
                n.train()
            Ko = K.to(dev, dt, copy=True).requires_grad_(True)
            OS.train_step(d, p, OS.make_optimizer(d, p, lr=1e-4), tgt.to(dev, dt), [r.to(dev, dt) for r in refs], Ko, num_scales=1,
                          with_ssim=1, with_mask=1, with_auto_mask=0)
            want[key] = Ko.grad.cpu()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    errs = {k: rel_l2(g, want["64"]) for k, g in (("mine", Kc.grad), ("32", want["32"]), ("32gpu", want["32gpu"]))}
    print("trainer dK rel_l2 vs fp64: mine %.3g | fp32 CPU oracle %.3g | stock PyTorch fp32 on this GPU %.3g" %
          (errs["mine"], errs["32"], errs["32gpu"]))
    # bound of test_two_training_steps_match_the_oracle (worst case): 4x the larger error of two independent fp32 evaluations +
    # 1e-3.  Measured on an H100: 8.8e-3 against 2.1e-3 / 2.3e-3.  A freshly initialised PoseResNet gives near-identity poses,
    # where the two terms of the closed form cancel most (DESIGN section 2.2); the golden cases above meet 3x + 2e-4.
    assert errs["mine"] < 4 * max(errs["32"], errs["32gpu"]) + 1e-3


def test_trainer_refuses_learned_intrinsics_in_a_captured_step():
    from scsfm import synth
    from scsfm.trainer import Trainer
    tgt, refs, K = synth.triplet(6, 1, 64, 128)
    c = lambda x: x.to(DEV)  # noqa: E731
    disp, pose = _nets()
    tr = Trainer(disp.to(DEV).train(), pose.to(DEV).train(), lr=1e-4, distributed=False)
    Kg = c(K).requires_grad_(True)
    with pytest.raises(RuntimeError, match="captured step"):
        tr.capture(c(tgt), [c(r) for r in refs], Kg)
    assert tr._graph is None
    tr.capture(c(tgt), [c(r) for r in refs], c(K))
    with pytest.raises(RuntimeError, match="captured step"):
        tr.step(c(tgt), [c(r) for r in refs], Kg)
    assert Kg.grad is None
    tr.step(c(tgt), [c(r) for r in refs], c(K))          # a plain K still replays
    with torch.no_grad():
        tr.step(c(tgt), [c(r) for r in refs], Kg)        # no gradient is asked for under no_grad
    torch.cuda.synchronize()


def test_data_parallel_trainer_refuses_learned_intrinsics():
    import torch.distributed as dist
    from scsfm import synth
    from scsfm.trainer import Trainer
    tgt, refs, K = synth.triplet(6, 1, 64, 128)
    c = lambda x: x.to(DEV)  # noqa: E731
    with tempfile.TemporaryDirectory() as tmp:
        dist.init_process_group("nccl", init_method="file://" + os.path.join(tmp, "rendezvous"), rank=0, world_size=1,
                                device_id=torch.device(DEV, torch.cuda.current_device()))
        try:
            disp, pose = _nets()
            tr = Trainer(disp.to(DEV).train(), pose.to(DEV).train(), lr=1e-4, distributed=True)
            Kg = c(K).requires_grad_(True)
            with pytest.raises(RuntimeError, match="data-parallel"):
                tr.step(c(tgt), [c(r) for r in refs], Kg)
            assert Kg.grad is None
        finally:
            dist.destroy_process_group()


def _plane_scene(fx_true, B=2, H=64, W=128, Z0=10.0, tx=0.8, seed=0):
    """A textured fronto-parallel plane at depth Z0 seen by two cameras a sideways translation tx apart: the target view is the
    reference view shifted by fx * tx / Z0 pixels.  The texture is a seeded sum of sinusoids evaluated exactly at both views."""
    g = torch.Generator().manual_seed(seed)
    n = 12
    kx = (2 * np.pi) / (14 + 34 * torch.rand(B, 3, n, generator=g, dtype=torch.float64))
    ky = (2 * np.pi) / (14 + 34 * torch.rand(B, 3, n, generator=g, dtype=torch.float64))
    ph = 2 * np.pi * torch.rand(B, 3, n, generator=g, dtype=torch.float64)
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")

    def render(shift):
        arg = kx[..., None, None] * (xs + shift) + ky[..., None, None] * ys + ph[..., None, None]
        return (torch.cos(arg).mean(2) * 0.9).float()        # [B,3,H,W]
    shift = fx_true * tx / Z0
    ref = render(0.0)
    tgt = render(shift)                                        # tgt(u) = ref(u + shift): the plane moved left in the target
    depth = torch.full((B, 1, H, W), Z0)
    pose = torch.tensor([[tx, 0, 0, 0, 0, 0]], dtype=torch.float32).repeat(B, 1)
    return tgt, ref, depth, pose


def test_self_calibration_recovers_the_focal_length():
    """Adam on fx alone, starting 20 % off, with the photometric loss of a synthetic plane scene: fx ends within 1 % of the truth."""
    _, lf = _api()
    fx_true, H, W = 100.0, 64, 128
    tgt, ref, depth, pose = (x.to(DEV) for x in _plane_scene(fx_true, H=H, W=W))
    B = tgt.shape[0]
    fx = torch.nn.Parameter(torch.tensor(0.8 * fx_true, device=DEV))
    opt = torch.optim.Adam([fx], lr=0.5)
    first = None
    for it in range(300):
        zero, one = torch.zeros((), device=DEV), torch.ones((), device=DEV)
        K = torch.stack([torch.stack([fx, zero, zero + (W - 1) / 2]), torch.stack([zero, one * fx_true, zero + (H - 1) / 2]),
                         torch.stack([zero, zero, one])]).expand(B, 3, 3)
        p, _ = lf.compute_photo_and_geometry_loss(tgt, [ref], K, [depth], [[depth]], [pose], [-pose], 1, 1, 0, 0, "zeros")
        opt.zero_grad()
        p.backward()
        opt.step()
        err = abs(float(fx) - fx_true) / fx_true
        if first is None and err < 0.01:
            first = it + 1
        elif first is not None and err >= 0.01:
            first = None
    print("self-calibration: fx %.3f (true %.1f), within 1%% from step %s on" % (float(fx), fx_true, first))
    assert abs(float(fx) - fx_true) < 0.01 * fx_true
    assert first is not None
