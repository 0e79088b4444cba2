"""Whole optimisation step (train.py:259-282): CUDA path vs the oracle's train_step on identical
weights and inputs.  Needs a GPU."""
import numpy as np
import pytest
import torch

from golden_util import det_weights
from helpers import rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.mark.parametrize("mode", ["fp32", "tf32x3"])
def test_two_training_steps_match_the_oracle(mode):
    """Both 1e-4 parity modes: exact CUDA-core convolutions and split-accumulate tensor-core convolutions."""
    import models
    from oracle import nets as N
    from oracle import step as OS
    from scsfm import synth
    from scsfm.trainer import Trainer
    B, H, W = 2, 96, 160
    tgt, refs, K = synth.triplet(5, B, H, W)
    disp, pose = models.DispResNet(18, False), models.PoseResNet(18, False)
    odisp, opose = N.DispResNet(18), N.PoseResNet(18)
    for a, b in ((disp, odisp), (pose, opose)):
        sd = det_weights(b.state_dict())
        a.load_state_dict(sd)
        b.load_state_dict(sd)
    disp, pose = disp.to(DEV).train(), pose.to(DEV).train()
    odisp.train(); opose.train()
    tr = Trainer(disp, pose, lr=1e-4, with_auto_mask=0, distributed=False, conv_mode=mode)
    opt = OS.make_optimizer(odisp, opose, lr=1e-4)
    c = lambda x: x.to(DEV)  # noqa: E731
    for it in range(2):
        got = tr.step(c(tgt), [c(r) for r in refs], c(K))
        # gradients of this step (before they are zeroed by the next one) for the comparison below
        g_disp = {k: p.grad.clone() for k, p in disp.named_parameters()}
        want = OS.train_step(odisp, opose, opt, tgt, refs, K, num_scales=1, with_ssim=1, with_mask=1, with_auto_mask=0)
        print("step %d  cuda %s  oracle %s" % (it, [round(float(v), 6) for v in got], [round(float(v), 6) for v in want]))
        # step 0: identical weights -> fp32 noise only.  step 1: Adam has moved every weight by ~lr with a sign that is
        # noise-determined wherever the gradient is ~0, so the two trajectories legitimately drift (~1e-3)
        np.testing.assert_allclose([float(v) for v in got], [float(v) for v in want], rtol=3e-4 if it == 0 else 5e-3, atol=1e-6)
        if it == 0:
            # yardstick: the fp32 oracle's own gradient error against an fp64 run of the same step (kink pixels of the
            # photometric / consistency terms differ between ANY two evaluations, SURVEY.md section 7)
            d64, p64 = N.DispResNet(18).double(), N.PoseResNet(18).double()
            for net64 in (d64, p64):
                net64.load_state_dict({k: v.double() for k, v in det_weights(net64.state_dict()).items()})
                net64.train()
            OS.train_step(d64, p64, OS.make_optimizer(d64, p64, lr=1e-4), tgt.double(), [r.double() for r in refs], K.double(),
                          num_scales=1, with_ssim=1, with_mask=1, with_auto_mask=0)
            g64 = {k: p.grad for k, p in d64.named_parameters() if p.grad is not None}
            g32 = {k: p.grad for k, p in odisp.named_parameters() if p.grad is not None}
            for k, p in odisp.named_parameters():
                if p.grad is None:
                    assert float(g_disp[k].abs().max()) == 0.0
            # second independent fp32 evaluation: the oracle step through stock PyTorch / cuDNN on this GPU with TF32 off
            torch.backends.cudnn.allow_tf32 = False
            torch.backends.cuda.matmul.allow_tf32 = False
            dg, pg = N.DispResNet(18).to(DEV), N.PoseResNet(18).to(DEV)
            for netg in (dg, pg):
                netg.load_state_dict({k: v.to(DEV) for k, v in det_weights(netg.state_dict()).items()})
                netg.train()
            OS.train_step(dg, pg, OS.make_optimizer(dg, pg, lr=1e-4), c(tgt), [c(r) for r in refs], c(K),
                          num_scales=1, with_ssim=1, with_mask=1, with_auto_mask=0)
            ggpu = {k: p.grad for k, p in dg.named_parameters() if p.grad is not None}
            mine = sorted(rel_l2(g_disp[k], g64[k]) for k in g64)
            ref = sorted(rel_l2(g32[k], g64[k]) for k in g64)
            refg = sorted(rel_l2(ggpu[k], g64[k]) for k in g64)
            print("DispResNet parameter-gradient rel-L2 vs fp64 oracle after a full step [%s]: CUDA median %.2e worst %.2e | fp32 CPU oracle "
                  "median %.2e worst %.2e | stock PyTorch/cuDNN fp32 on this GPU median %.2e worst %.2e"
                  % (mode, mine[len(mine) // 2], mine[-1], ref[len(ref) // 2], ref[-1], refg[len(refg) // 2], refg[-1]))
            # yardstick: the larger error of the two independent fp32 evaluations (a single ReLU / validity decision flipping on a
            # ~0 value moves every upstream gradient at once, so one evaluation alone is a noisy yardstick)
            ymed, yworst = max(ref[len(ref) // 2], refg[len(refg) // 2]), max(ref[-1], refg[-1])
            assert mine[len(mine) // 2] < 4 * ymed + 1e-4 and mine[-1] < 4 * yworst + 1e-3
    # parameters after two Adam updates: elementwise bounded by 2 * lr (Adam's step bound), nearly all identical
    osd = odisp.state_dict()
    for k, v in disp.state_dict().items():
        if v.dtype == torch.float32 and "running" not in k:
            assert float((v.cpu() - osd[k]).abs().max()) <= 4.1e-4, k


_FULL = {}
# benchmarked shapes: BASELINE config 2 (KITTI 256x832, 2 refs, 4 frames per GPU) and config 5 (NYU 256x320, `--folder-type pair`:
# ONE reference frame, 8 frames per GPU)
FULL_SHAPES = {"kitti": (4, 256, 832, 2, "kitti"), "nyu": (8, 256, 320, 1, "nyu")}


def _full_size_oracle(shape="kitti"):
    """One oracle step (fp32 and fp64 on the CPU, fp32 through stock PyTorch on the GPU) on a BENCHMARKED configuration, ssim +
    mask + auto-mask.  Computed once per test session (~1 minute)."""
    if shape not in _FULL:
        from oracle import nets as N
        from oracle import step as OS
        from scsfm import synth
        B, H, W, n_ref, kind = FULL_SHAPES[shape]
        tgt, refs, K = synth.triplet(1234, B, H, W, n_ref, kind)
        out = {"inputs": (tgt, refs, K)}
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        for name, dt, dev in (("f32", torch.float32, "cpu"), ("f64", torch.float64, "cpu"), ("f32gpu", torch.float32, DEV)):
            d, p = N.DispResNet(18).to(dt).to(dev), N.PoseResNet(18).to(dt).to(dev)
            for net in (d, p):
                net.load_state_dict({k: v.to(dt).to(dev) for k, v in det_weights(net.state_dict()).items()})
                net.train()
            losses = OS.train_step(d, p, OS.make_optimizer(d, p, lr=1e-4), tgt.to(dt).to(dev), [r.to(dt).to(dev) for r in refs],
                                   K.to(dt).to(dev), num_scales=1, with_ssim=1, with_mask=1, with_auto_mask=1)
            out[name] = ([float(v) for v in losses],
                         {"disp." + k: q.grad.clone().cpu() for k, q in d.named_parameters() if q.grad is not None} |
                         {"pose." + k: q.grad.clone().cpu() for k, q in p.named_parameters() if q.grad is not None})
        _FULL[shape] = out
    return _FULL[shape]


@pytest.mark.parametrize("mode,shape", [("tf32x3", "kitti"), ("tf32", "kitti"), ("fp32", "kitti"), ("tf32x3", "nyu")])
def test_full_size_benchmarked_step_vs_oracle(mode, shape):
    """The step bench.py times (B=4, 256x832, auto-mask on) against the oracle, in every convolution mode: the four
    scalar losses and EVERY parameter gradient of both networks.  Yardstick for the gradients = the fp32 CPU oracle's own
    error against the fp64 oracle (kink pixels and ReLU gates flip between any two evaluations).  tf32x3 and fp32 are the
    parity modes (bound: 3x the larger error of two independent fp32 evaluations -- the CPU oracle and stock PyTorch / cuDNN with
    TF32 off on this GPU); tf32 (single product, cuDNN's default arithmetic) is only
    required to stay within 1e-2 on the losses and is reported."""
    import models
    from scsfm.trainer import Trainer
    o = _full_size_oracle(shape)
    tgt, refs, K = o["inputs"]
    disp, pose = models.DispResNet(18, False), models.PoseResNet(18, False)
    for net in (disp, pose):
        net.load_state_dict(det_weights(net.state_dict()))
    tr = Trainer(disp.to(DEV).train(), pose.to(DEV).train(), lr=1e-4, with_auto_mask=1, distributed=False, conv_mode=mode)
    got = [float(v) for v in tr.step(tgt.to(DEV), [r.to(DEV) for r in refs], K.to(DEV))]
    grads = {"disp." + k: q.grad for k, q in disp.named_parameters()} | {"pose." + k: q.grad for k, q in pose.named_parameters()}
    want64, g64 = o["f64"]
    want32, g32 = o["f32"]
    _, g32gpu = o["f32gpu"]
    mine = sorted((rel_l2(grads[k], g64[k]), k) for k in g64)
    ref = sorted(rel_l2(g32[k], g64[k]) for k in g64)
    refg = sorted(rel_l2(g32gpu[k], g64[k]) for k in g64)
    med, worst = mine[len(mine) // 2][0], mine[-1]
    rmed, rworst = max(ref[len(ref) // 2], refg[len(refg) // 2]), max(ref[-1], refg[-1])
    print("full-size step [%s %s]: losses %s (fp64 oracle %s) | parameter-gradient rel-L2 vs fp64 oracle: median %.2e worst %.2e (%s) | "
          "fp32 CPU oracle's own: median %.2e worst %.2e | stock PyTorch/cuDNN fp32 on this GPU: median %.2e worst %.2e"
          % (shape, mode, [round(v, 6) for v in got], [round(v, 6) for v in want64], med, worst[0], worst[1], ref[len(ref) // 2], ref[-1],
             refg[len(refg) // 2], refg[-1]))
    if mode == "tf32":
        np.testing.assert_allclose(got, want64, rtol=1e-2, atol=1e-5)
        return
    np.testing.assert_allclose(got, want64, rtol=1e-4, atol=1e-6)        # north_star: scalar losses within 1e-4
    assert med < 3 * rmed + 1e-4 and worst[0] < 3 * rworst + 1e-3


def test_step_issues_no_host_synchronisation():
    """The whole step must be stream-ordered (no .item(), no blocking copies): run it under
    torch.cuda.set_sync_debug_mode('error')."""
    import models
    from scsfm import synth
    from scsfm.trainer import Trainer
    tgt, refs, K = synth.triplet(1, 1, 64, 96)
    tr = Trainer(models.DispResNet(18, False).to(DEV).train(), models.PoseResNet(18, False).to(DEV).train(),
                 distributed=False)
    args = (tgt.to(DEV), [r.to(DEV) for r in refs], K.to(DEV))
    tr.step(*args)          # warm-up: allocations, arena packing
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        tr.step(*args)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


def test_cuda_graph_replay_matches_eager_steps():
    """Trainer.capture(): the whole step as one CUDA graph.  Three replayed steps must track three eager steps
    (same weights, same data) and capturing itself must not advance training."""
    import models
    from scsfm import synth
    from scsfm.trainer import Trainer
    tgt, refs, K = synth.triplet(2, 2, 96, 160)
    args = (tgt.to(DEV), [r.to(DEV) for r in refs], K.to(DEV))

    def make():
        d, p = models.DispResNet(18, False), models.PoseResNet(18, False)
        d.load_state_dict(det_weights(d.state_dict())); p.load_state_dict(det_weights(p.state_dict()))
        return Trainer(d.to(DEV).train(), p.to(DEV).train(), lr=1e-4, with_auto_mask=0, distributed=False)
    eager, graphed = make(), make()
    w0 = graphed.disp_net.flat_params().clone()
    graphed.capture(*args)
    torch.cuda.synchronize()
    assert torch.equal(graphed.disp_net.flat_params(), w0)          # warm-up step undone
    assert graphed.optimizer.step_count == 0
    assert graphed.launches_per_step > 300
    for it in range(3):
        a = [float(v) for v in eager.step(*args)]
        b = [float(v) for v in graphed.step(*args)]
        np.testing.assert_allclose(b, a, rtol=2e-4 if it == 0 else 5e-3)
    assert graphed.optimizer.step_count == 3
    assert float((graphed.disp_net.flat_params() - eager.disp_net.flat_params()).abs().max()) <= 6.1e-4   # 3 steps x 2 lr


@pytest.mark.parametrize("mode", ["tf32", "tf32x3"])
def test_tf32_operand_mirror_and_batched_flips_stay_exact(mode):
    """Tensor-core mode shortcuts of the training loop: ArenaAdam writes the operand mirror of the parameters itself (TF32-
    rounded copy / low parts; no extra pass per network call) and all flipped data-gradient weights of a network are
    refreshed by ONE batched launch.  Both must be bit-identical to the plain per-tensor kernels, eagerly and under
    CUDA-graph replay."""
    import math
    import models
    from scsfm import nnops as O
    from scsfm import synth
    from scsfm.trainer import Trainer
    tgt, refs, K = synth.triplet(3, 2, 96, 160)
    args = (tgt.to(DEV), [r.to(DEV) for r in refs], K.to(DEV))

    def make():
        d, p = models.DispResNet(18, False), models.PoseResNet(18, False)
        d.load_state_dict(det_weights(d.state_dict())); p.load_state_dict(det_weights(p.state_dict()))
        return Trainer(d.to(DEV).train(), p.to(DEV).train(), lr=1e-4, with_auto_mask=1, distributed=False, conv_mode=mode)

    def mirror_in_sync(net):
        want = torch.empty_like(net._flat)
        (O.split_tf32 if mode == "tf32x3" else O.round_tf32)(net._flat, want)
        return torch.equal(net._flat_tf32, want)

    if True:
        tr = make()
        for _ in range(3):                      # steps 2 and 3 run on the shortcuts
            losses = tr.step(*args)
        assert all(math.isfinite(float(v)) for v in losses)
        nets = (tr.disp_net, tr.pose_net)
        for net in nets:
            assert net.trust_adam_mirror and net._tf32_version == net._versions()
            assert mirror_in_sync(net)
            net.refresh_operand_weights()       # batched flip refresh from the (current) mirror
        seen = 0
        for net in nets:
            cached = {k: v[1].clone() for k, v in net.ctx._flips.items()}
            assert len(cached) > 10
            src = net._flat if mode == "tf32x3" else net._flat_tf32      # arena the flips are derived from
            lo = src.data_ptr()
            fresh = O.ConvCtx(mode)
            for key, got in cached.items():
                ptr, shape, stride, pad, operand = key
                assert lo <= ptr < lo + 4 * src.numel()
                off = (ptr - lo) // 4
                w = src[off:off + math.prod(shape)].view(shape)
                assert w.data_ptr() == ptr
                assert torch.equal(fresh.flipped_weights(w, stride, pad, operand), got), key
                seen += 1
        assert seen > 40
        # the same loop as one CUDA graph per step
        gr = make()
        gr.capture(*args)
        for _ in range(2):
            gr.step(*args)
        torch.cuda.synchronize()
        for net in (gr.disp_net, gr.pose_net):
            assert mirror_in_sync(net)
        # a parameter change the optimizer did not make must be noticed (torch version counters)
        with torch.no_grad():
            next(iter(gr.disp_net.parameters())).mul_(1.5)
        assert gr.disp_net._tf32_version != gr.disp_net._versions()


@pytest.mark.parametrize("wgrad", [False, True])
@pytest.mark.parametrize("graph", [False, True])
def test_overlapped_networks_reproduce_the_serial_step(graph, wgrad):
    """Trainer(overlap_nets=True): PoseResNet on a side stream next to DispResNet (forward and, through autograd's stream
    tracking, backward).  Same kernels on the same data: losses, gradients and updated parameters must match the serial step to
    atomics-order noise, eagerly and as a captured CUDA graph (fork / join inside the graph)."""
    import models
    from scsfm import synth
    from scsfm.trainer import Trainer
    tgt, refs, K = synth.triplet(9, 2, 128, 160)
    args = (tgt.to(DEV), [r.to(DEV) for r in refs], K.to(DEV))

    def make(overlap):
        d, p = models.DispResNet(18, False), models.PoseResNet(18, False)
        d.load_state_dict(det_weights(d.state_dict())); p.load_state_dict(det_weights(p.state_dict()))
        return Trainer(d.to(DEV).train(), p.to(DEV).train(), lr=1e-4, with_auto_mask=1, distributed=False, conv_mode="tf32x3",
                       overlap_nets=overlap, overlap_wgrad=overlap and wgrad)
    a, b = make(False), make(True)
    if graph:
        b.capture(*args)
    for it in range(3):
        la = [float(v) for v in a.step(*args)]
        lb = [float(v) for v in b.step(*args)]
        np.testing.assert_allclose(lb, la, rtol=1e-5 if it == 0 else 5e-3, atol=1e-7)
        if it == 0 and not graph:
            for na, nb in ((a.disp_net, b.disp_net), (a.pose_net, b.pose_net)):
                assert rel_l2(nb.flat_grads(), na.flat_grads()) < 1e-4
    torch.cuda.synchronize()
    assert float((b.disp_net.flat_params() - a.disp_net.flat_params()).abs().max()) <= 6.1e-4
    assert float((b.pose_net.flat_params() - a.pose_net.flat_params()).abs().max()) <= 6.1e-4
