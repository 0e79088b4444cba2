"""Fine-tuning on the GPU: partially frozen networks and per-module BatchNorm.eval() against the fp64 oracle (plain nn.Modules
with the same freezing and eval() calls), the launches the backward cut saves, the masked Adam against torch.optim.Adam, and
Trainer steps with frozen parts.  Needs a GPU."""
import numpy as np
import pytest
import torch
import torch.nn as nn

from golden_util import det_image, det_weights
from helpers import rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda"


# ----- freezing patterns, applied identically to the oracle and to the CUDA networks ---------------------------------------------
def _bns(net):
    return [m for m in net.modules() if isinstance(m, nn.BatchNorm2d)]


def _frozen_bias_weight(kind):
    return "decoder.decoder.4.conv.conv.weight" if kind == "disp" else "decoder.net.1.weight"


def apply_pattern(net, kind, pattern):
    """net in train mode, then the pattern's requires_grad_(False) / eval() calls (module names are the reference's)."""
    net.train()
    if pattern == "encoder_frozen_eval":
        net.encoder.requires_grad_(False)
        net.encoder.eval()
    elif pattern == "decoder_frozen":
        net.decoder.requires_grad_(False)
    elif pattern == "stem_layer1_frozen":
        t = net.encoder.encoder
        for m in (t.conv1, t.bn1, t.layer1):
            m.requires_grad_(False)
    elif pattern == "bn_eval":
        for m in _bns(net):
            m.eval()
    elif pattern == "bn_affine_frozen":
        for m in _bns(net):
            m.requires_grad_(False)
    elif pattern == "decoder_weight_frozen":
        dict(net.named_parameters())[_frozen_bias_weight(kind)].requires_grad_(False)
    else:
        raise ValueError(pattern)
    return net


PATTERNS = ["encoder_frozen_eval", "decoder_frozen", "stem_layer1_frozen", "bn_eval", "bn_affine_frozen", "decoder_weight_frozen"]


def _images(B=2, H=64, W=96):
    return det_image("img1", B, H, W), det_image("img2", B, H, W)


def _state(kind, layers, imgs):
    """Deterministic weights and running statistics that normalise the test images (eval-mode layers with untouched statistics
    would leave their activations unnormalised): the batch statistics of one fp64 train-mode oracle pass."""
    import models
    from oracle import nets as N
    sd = det_weights((models.DispResNet(layers, False) if kind == "disp" else models.PoseResNet(layers, False)).state_dict())
    ref = (N.DispResNet(layers) if kind == "disp" else N.PoseResNet(layers)).double()
    ref.load_state_dict({k: v.double() if v.is_floating_point() else v for k, v in sd.items()})
    for m in _bns(ref):
        m.momentum = None
        m.reset_running_stats()
    ref.train()
    with torch.no_grad():
        ref(*[i.double() for i in imgs[:1 if kind == "disp" else 2]])
    sd.update({k: v.float() for k, v in ref.state_dict().items() if "running" in k})
    return sd


def _loss(kind, out):
    if kind == "disp":
        outs = out if isinstance(out, (list, tuple)) else [out]
        return sum(((1.0 / o) * (i + 1)).mean() for i, o in enumerate(outs))
    return (out * torch.arange(1, 7, dtype=out.dtype, device=out.device)).sum() * 100


def _run(net, kind, imgs, dtype, dev):
    xs = [i.detach().clone().to(dtype).to(dev) for i in imgs[:1 if kind == "disp" else 2]]
    out = net(*xs)
    _loss(kind, out).backward()
    outs = out if isinstance(out, (list, tuple)) else [out]
    return ([o.detach() for o in outs], {k: p.grad for k, p in net.named_parameters()},
            {k: b.detach().clone() for k, b in net.named_buffers()})


def _run_oracle(kind, layers, sd, imgs, pattern, dtype, dev="cpu"):
    from oracle import nets as N
    ref = (N.DispResNet(layers) if kind == "disp" else N.PoseResNet(layers)).to(dtype).to(dev)
    ref.load_state_dict({k: v.to(dtype).to(dev) if v.is_floating_point() else v.to(dev) for k, v in sd.items()})
    return _run(apply_pattern(ref, kind, pattern), kind, imgs, dtype, dev)


def _run_mine(kind, layers, sd, imgs, pattern, mode):
    import models
    net = models.DispResNet(layers, False) if kind == "disp" else models.PoseResNet(layers, False)
    net.load_state_dict(sd)
    net = net.to(DEV).set_conv_mode(mode)
    return _run(apply_pattern(net, kind, pattern), kind, imgs, torch.float32, DEV)


CASES = [(k, 18, m, p) for k in ("disp", "pose") for m in ("fp32", "tf32x3") for p in PATTERNS]
CASES += [(k, 50, "tf32x3", p) for k in ("disp", "pose") for p in ("encoder_frozen_eval", "stem_layer1_frozen")]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "%s%d_%s_%s" % c)
def test_partially_frozen_network_vs_oracle(case):
    """Outputs, every trainable gradient, None exactly for the frozen parameters, running statistics and num_batches_tracked
    against the fp64 oracle with the same freezing; the yardstick of test_nets_gpu.py (4x the larger error of the fp32 CPU
    oracle and of cuDNN fp32 on this GPU)."""
    kind, layers, mode, pattern = case
    imgs = _images()
    sd = _state(kind, layers, imgs)
    o_mine, g_mine, b_mine = _run_mine(kind, layers, sd, imgs, pattern, mode)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    o64, g64, b64 = _run_oracle(kind, layers, sd, imgs, pattern, torch.float64)
    o32, g32, b32 = _run_oracle(kind, layers, sd, imgs, pattern, torch.float32)
    o32g, g32g, b32g = _run_oracle(kind, layers, sd, imgs, pattern, torch.float32, DEV)
    # outputs
    assert len(o_mine) == len(o64)
    for k, (a, r) in enumerate(zip(o_mine, o64)):
        yard = max(rel_l2(o32[k], r), rel_l2(o32g[k], r))
        assert rel_l2(a, r) < 4 * yard + 1e-5, ("output", k, rel_l2(a, r), yard)
    # frozen parameters: grad None, as for the oracle's; trainable ones the oracle never reaches (the fc head): zero
    mine_none = {k for k, g in g_mine.items() if g is None}
    oracle_none = {k for k, g in g64.items() if g is None}
    unreached = {k for k in oracle_none if dict(_named(kind, layers, pattern))[k]}     # trainable but unused by the oracle
    assert mine_none == oracle_none - unreached, (sorted(mine_none ^ (oracle_none - unreached))[:5])
    for k in unreached:
        assert float(g_mine[k].abs().max()) == 0.0, k
    # trainable gradients with the yardstick
    keys = sorted(k for k, g in g64.items() if g is not None)
    assert keys
    errs = sorted((rel_l2(g_mine[k], g64[k]), k) for k in keys)
    errs_cpu = sorted(rel_l2(g32[k], g64[k]) for k in keys)
    errs_gpu = sorted(rel_l2(g32g[k], g64[k]) for k in keys)
    med, worst = errs[len(errs) // 2][0], errs[-1]
    yard_med = max(errs_cpu[len(errs_cpu) // 2], errs_gpu[len(errs_gpu) // 2])
    yard_worst = max(errs_cpu[-1], errs_gpu[-1])
    print(case, "rel-L2 vs fp64: median %.2e worst %.2e (%s); yardstick median %.2e worst %.2e" % (med, worst[0], worst[1], yard_med,
                                                                                                  yard_worst))
    assert med < 4 * yard_med + 1e-4 and worst[0] < 4 * yard_worst + 3e-3
    # BatchNorm buffers: train-mode modules updated like the oracle's, eval-mode ones bitwise unchanged
    import models
    net = models.DispResNet(layers, False) if kind == "disp" else models.PoseResNet(layers, False)
    apply_pattern(net, kind, pattern)
    eval_prefixes = [n + "." for n, m in net.named_modules() if isinstance(m, nn.BatchNorm2d) and not m.training]
    for k, v in b64.items():
        got = b_mine[k].cpu()
        if any(k.startswith(p) for p in eval_prefixes):
            assert torch.equal(got, sd[k]), k
        elif k.endswith("num_batches_tracked"):
            assert int(got) == int(v), k
        else:
            yard = max(rel_l2(b32[k], v), rel_l2(b32g[k], v))
            assert rel_l2(got, v) < 4 * yard + 1e-6, (k, rel_l2(got, v), yard)


def _named(kind, layers, pattern):
    """(name, requires_grad) of the CUDA network's parameters under `pattern`."""
    import models
    net = models.DispResNet(layers, False) if kind == "disp" else models.PoseResNet(layers, False)
    return [(k, p.requires_grad) for k, p in apply_pattern(net, kind, pattern).named_parameters()]


# ----- what the cut saves ----------------------------------------------------------------------------------------------------------
def _events(fn):
    """(library launches, profiled launch families) of fn()."""
    from scsfm import lib as L
    torch.cuda.synchronize()
    L.PROF["enabled"], L.PROF["events"] = True, []
    n0 = L.launch_count()
    out = fn()
    n1 = L.launch_count()
    fams = [e[0] for e in L.PROF["events"]]
    L.PROF["enabled"], L.PROF["events"] = False, []
    torch.cuda.synchronize()
    return n1 - n0, fams, out


ENCODER_ONLY = ("bn_apply", "bn_bwd", "pool", "stem_dgrad", "layout")


@pytest.mark.parametrize("mode", ["fp32", "tf32x3"])
def test_frozen_eval_encoder_issues_no_encoder_backward(mode):
    import models
    from scsfm import nets as N
    imgs = _images()
    sd = _state("disp", 18, imgs)
    net = models.DispResNet(18, False)
    net.load_state_dict(sd)
    net = net.to(DEV).set_conv_mode(mode).train()
    n_dec_convs = sum(isinstance(m, N.ConvParams) for m in net.decoder.modules()) - 4          # minus the 4 disparity heads
    n_enc_convs = sum(isinstance(m, N.ConvParams) for m in net.encoder.modules())
    n_enc_bns = len(_bns(net))

    def step(x):
        """(outputs, forward launches, forward families, backward launches, backward families)"""
        nf, ff, out = _events(lambda: net(x))
        nb, fb, _ = _events(_loss("disp", out).backward)
        return out, nf, ff, nb, fb
    x = imgs[0].to(DEV)
    step(x)                                    # first call: operand caches
    out_all, nf_all, ff_all, nb_all, fb_all = step(x)
    assert fb_all.count("bn_bwd") == n_enc_bns and "stem_dgrad" not in fb_all
    assert sum(f.startswith("conv_wgrad") for f in fb_all) == n_dec_convs + n_enc_convs
    net.encoder.requires_grad_(False)
    net.encoder.eval()
    net.zero_grad()
    step(x)
    out, nf, ff, nb, fb = step(x)
    # forward: the encoder runs the fused eval forward (no bn_apply, one batched coefficient launch) ...
    assert "bn_apply" not in ff and ff.count("bn_prepare") == 1
    # ... and the backward nothing of the encoder: no BatchNorm, pooling or stem launches, only the decoder's weight gradients
    assert not any(f in ENCODER_ONLY for f in fb), fb
    assert sum(f.startswith("conv_wgrad") for f in fb) == n_dec_convs
    assert fb.count("head_wgrad") == fb_all.count("head_wgrad") == 4
    assert nb < nb_all and nf < nf_all
    # the features the fused encoder forward hands the decoder are bitwise what the recording forward gives: the same call with
    # the image needing a gradient records the encoder (and runs its data gradients, not its weight gradients)
    xg = imgs[0].to(DEV).requires_grad_(True)
    out_g, _, _, _, fb_g = step(xg)
    for a, b in zip(out, out_g):
        assert torch.equal(a, b)
    assert xg.grad is not None and float(xg.grad.abs().max()) > 0
    assert fb_g.count("bn_bwd") == n_enc_bns and fb_g.count("stem_dgrad") == 1
    assert sum(f.startswith("conv_wgrad") for f in fb_g) == n_dec_convs
    assert sum(f.startswith("conv_dgrad") for f in fb_g) == sum(f.startswith("conv_dgrad") for f in fb_all)
    for k, p in net.named_parameters():
        assert (p.grad is None) == k.startswith("encoder"), k


def test_frozen_pose_network_keeps_no_record_and_issues_no_backward():
    import models
    imgs = _images()
    net = models.PoseResNet(18, False)
    net.load_state_dict(_state("pose", 18, imgs))
    net = net.to(DEV).set_conv_mode("tf32x3").train()
    net.requires_grad_(False)
    nbt0 = {k: int(b) for k, b in net.named_buffers() if k.endswith("num_batches_tracked")}
    a, b = imgs[0].to(DEV), imgs[1].to(DEV)
    out = net(a, b)
    n, _, _ = _events(lambda: _loss("pose", out).backward())
    assert n == 0
    # train-mode BatchNorm still counts the batch and updates its statistics, as the reference's does
    for k, v in net.named_buffers():
        if k.endswith("num_batches_tracked"):
            assert int(v) == nbt0[k] + 1


# ----- masked Adam ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("wd", [0.0, 0.01])
def test_masked_adam_vs_torch_optim(wd):
    """Three steps on an arena of four tensors against torch.optim.Adam in fp64; tensor 1 is frozen after step 1 (grad None for
    torch): its value and moments stay bitwise, the others within the bound of test_adam_vs_torch_optim_fp64."""
    from scsfm import nnops as O
    f32 = lambda x: float(np.float32(x))   # noqa: E731
    lr, b1, b2, eps, wdf = f32(1e-3), f32(0.9), f32(0.999), f32(1e-8), f32(wd)
    g = torch.Generator().manual_seed(11)
    sizes = [1000, 333, 64, 70_001]
    offs = np.cumsum([0] + [O.aligned64(n) for n in sizes])
    n = int(offs[-1])
    p0 = torch.zeros(n)
    for i, s in enumerate(sizes):
        p0[offs[i]:offs[i] + s] = 0.05 * torch.randn(s, generator=g)
    ts = [p0[offs[i]:offs[i] + s].double().clone().requires_grad_(True) for i, s in enumerate(sizes)]
    opt = torch.optim.Adam(ts, lr=lr, betas=(b1, b2), eps=eps, weight_decay=wdf, foreach=False)
    p, m, v = p0.to(DEV), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    pu, mu, vu = p.clone(), m.clone(), v.clone()            # the unmasked kernel on the same data while all are trainable
    step_dev = torch.zeros(1, dtype=torch.int32, device=DEV)
    frozen_after = {1: [1]}
    trainable = [True] * 4
    for step in range(1, 4):
        gr = torch.zeros(n)
        for i, s in enumerate(sizes):
            gr[offs[i]:offs[i] + s] = torch.randn(s, generator=g) * (1e-3 if i == 2 else 1.0)
        for i, t in enumerate(ts):
            t.grad = gr[offs[i]:offs[i] + sizes[i]].double() if trainable[i] else None
        before64 = [t.detach().clone() for t in ts]
        m_prev = [opt.state[t]["exp_avg"].clone() if opt.state[t] else torch.zeros(sizes[i], dtype=torch.float64)
                  for i, t in enumerate(ts)]
        opt.step()
        before = p.double().cpu()
        m_before, v_before = m.cpu(), v.cpu()
        mask = O.chunk_mask(sizes, trainable, DEV)
        step_dev.fill_(step)
        O.adam_step_masked(p, gr.to(DEV), m, v, mask, lr, b1, b2, eps, wdf, 0, step_dev)
        if all(trainable):
            O.adam_step(pu, gr.to(DEV), mu, vu, lr, b1, b2, eps, wdf, 0, step_dev)
            assert torch.equal(p, pu) and torch.equal(m, mu) and torch.equal(v, vu)       # bitwise the unmasked kernel
        after, m_after, v_after = p.double().cpu(), m.cpu(), v.cpu()
        for i, t in enumerate(ts):
            sl = slice(int(offs[i]), int(offs[i + 1]))           # the tensor and its padding
            if not trainable[i]:
                assert torch.equal(after[sl], before[sl]) and torch.equal(m_after[sl], m_before[sl]) and \
                    torch.equal(v_after[sl], v_before[sl]), i
                continue
            s = slice(int(offs[i]), int(offs[i]) + sizes[i])
            got, want = after[s] - before[s], t.detach() - before64[i]
            g_eff = t.grad + wdf * before64[i]
            den = opt.state[t]["exp_avg_sq"].sqrt() / (1 - b2 ** step) ** 0.5 + eps
            size = lr / (1 - b1 ** step) * (b1 * m_prev[i].abs() + (1 - b1) * g_eff.abs()) / den
            assert bool(((got - want).abs() <= 1e-5 * size + 2.0 ** -24 * after[s].abs()).all()), (step, i)
        for i in frozen_after.get(step, []):
            trainable[i] = False


# ----- Trainer with frozen parts -------------------------------------------------------------------------------------------------
def _finetune_trainer(sd_disp, sd_pose, mode="tf32x3"):
    import models
    from scsfm.trainer import Trainer
    d, p = models.DispResNet(18, False), models.PoseResNet(18, False)
    d.load_state_dict(sd_disp)
    p.load_state_dict(sd_pose)
    d, p = d.to(DEV).train(), p.to(DEV).train()
    d.encoder.requires_grad_(False)
    d.encoder.eval()
    p.requires_grad_(False)
    return Trainer(d, p, lr=1e-4, with_auto_mask=0, distributed=False, conv_mode=mode)


def test_trainer_with_frozen_parts():
    import models
    from oracle import nets as N
    from oracle import step as OS
    from scsfm import synth
    tgt, refs, K = synth.triplet(4, 2, 128, 160)
    args = (tgt.to(DEV), [r.to(DEV) for r in refs], K.to(DEV))
    imgs = (tgt, refs[0])
    sd_disp = _state("disp", 18, imgs)
    sd_pose = det_weights(models.PoseResNet(18, False).state_dict())
    eager, graphed = _finetune_trainer(sd_disp, sd_pose), _finetune_trainer(sd_disp, sd_pose)
    enc0 = {k: p.detach().clone() for k, p in eager.disp_net.named_parameters() if k.startswith("encoder")}
    pose0 = eager.pose_net.flat_params().clone()
    # one step against the oracle's train_step with the same freezing (torch.optim.Adam over all parameters, as train.py builds
    # it: the frozen ones have grad None and are skipped)
    od, op = N.DispResNet(18), N.PoseResNet(18)
    od.load_state_dict(sd_disp)
    op.load_state_dict(sd_pose)
    od.train(); op.train()
    od.encoder.requires_grad_(False); od.encoder.eval(); op.requires_grad_(False)
    opt = OS.make_optimizer(od, op, lr=1e-4)
    want = [float(v) for v in OS.train_step(od, op, opt, tgt, refs, K, num_scales=1, with_ssim=1, with_mask=1, with_auto_mask=0)]
    got = [float(v) for v in eager.step(*args)]
    np.testing.assert_allclose(got, want, rtol=3e-4, atol=1e-6)
    for k, p in eager.disp_net.named_parameters():
        assert (p.grad is None) == k.startswith("encoder"), k
    for k, p in eager.pose_net.named_parameters():
        assert p.grad is None, k
    # the decoder moved like the oracle's (first Adam step: ~lr per weight), running statistics and counters like the oracle's
    ref_sd = od.state_dict()
    for k, v in eager.disp_net.state_dict().items():
        if k.startswith("decoder"):
            assert float((v.cpu() - ref_sd[k]).abs().max()) <= 2.1e-4, k
        elif "running" in k or "num_batches" in k:
            assert torch.equal(v.cpu(), ref_sd[k]), k            # eval-mode encoder: untouched
    pose_sd = op.state_dict()
    for k, v in eager.pose_net.state_dict().items():
        if "num_batches" in k:
            assert int(v) == int(pose_sd[k]), k           # the frozen network's BatchNorms are in train mode: they count
    # the captured step tracks the eager one, as in test_cuda_graph_replay_matches_eager_steps (the fp32 atomics of the
    # weight gradients and losses are not bitwise repeatable; Adam turns their noise into sign flips of size lr)
    graphed.step(*args)                   # the same first step, eagerly
    graphed.capture(*args)
    assert graphed.launches_per_step > 100
    for it in range(3):
        a = [float(v) for v in eager.step(*args)]
        b = [float(v) for v in graphed.step(*args)]
        np.testing.assert_allclose(b, a, rtol=5e-3)
    assert float((graphed.disp_net.flat_params() - eager.disp_net.flat_params()).abs().max()) <= 8.1e-4   # 4 steps x 2 lr
    # frozen parameters are bitwise unchanged after four steps, eager and replayed
    for tr in (eager, graphed):
        assert tr.optimizer.step_count == 4
        for k, p in tr.disp_net.named_parameters():
            if k in enc0:
                assert torch.equal(p.detach(), enc0[k]), k
        assert torch.equal(tr.pose_net.flat_params(), pose0)
    # a pattern change after capture() is refused instead of replaying the stale graph
    graphed.disp_net.decoder.up(0, 0).weight.requires_grad_(False)
    with pytest.raises(RuntimeError, match="capture"):
        graphed.step(*args)
    graphed.disp_net.decoder.up(0, 0).weight.requires_grad_(True)
    graphed.disp_net.encoder.encoder.bn1.train()
    with pytest.raises(RuntimeError, match="capture"):
        graphed.step(*args)
