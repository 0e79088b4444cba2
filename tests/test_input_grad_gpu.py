"""Gradients of the input images and the eval-mode backward of DispResNet / PoseResNet (the autograd contract of the reference's
nn.Modules): the stem input-gradient kernel and the frozen-statistics BatchNorm backward against fp64, then whole networks
against the fp64 oracle in both modes, partial image gradients, forward_multi, frozen networks and a learnable module in front
of a network.  Needs a GPU."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from golden_util import det_image, det_weights
from helpers import rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda"
BN_EPS = 1e-5


def _ops():
    from scsfm import nnops
    return nnops


def _close(a, ref, tol, what):
    a = torch.as_tensor(a, dtype=torch.float64).cpu()
    ref = torch.as_tensor(ref, dtype=torch.float64).cpu()
    err = float((a - ref).abs().max()) / (float(ref.abs().max()) + 1e-30)
    assert err <= tol and rel_l2(a, ref) <= tol, "%s: max err %.2e, rel-L2 %.2e (bound %.0e)" % (what, err, rel_l2(a, ref), tol)


# ----- stem input gradient ------------------------------------------------------------------------------------------------------
STEM_CASES = [(3, 4, 256, 832), (6, 4, 256, 832), (3, 2, 256, 320), (6, 2, 256, 320), (3, 2, 65, 97), (6, 1, 65, 97), (6, 3, 6, 5)]


@pytest.mark.parametrize("case", STEM_CASES, ids=lambda c: "Cin%d_B%d_%dx%d" % c)
def test_stem_input_gradient_vs_fp64(case):
    O = _ops()
    Cin, N, H, W = case
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    g = torch.Generator().manual_seed(Cin * 1000 + H + W)
    dy = torch.randn(N, 64, Ho, Wo, generator=g).float()
    w = (torch.randn(64, Cin, 7, 7, generator=g) / (Cin * 49) ** 0.5).float()
    ref = torch.nn.grad.conv2d_input((N, Cin, H, W), w.double(), dy.double(), stride=2, padding=3)
    dy_nhwc = dy.permute(0, 2, 3, 1).contiguous().to(DEV)
    w_khwc = w.permute(0, 2, 3, 1).contiguous().to(DEV)
    need = (True,) if Cin == 3 else (True, True)
    outs = O.stem_dgrad(dy_nhwc, w_khwc, H, W, need)
    for k, o in enumerate(outs):
        assert o.shape == (N, 3, H, W)
        assert rel_l2(o, ref[:, 3 * k:3 * k + 3]) <= 1e-6, (k, rel_l2(o, ref[:, 3 * k:3 * k + 3]))
    # no atomics: bitwise the same on a second call
    again = O.stem_dgrad(dy_nhwc, w_khwc, H, W, need)
    for a, b in zip(outs, again):
        assert torch.equal(a, b)
    # the composition it replaces: the CUDA-core data gradient (NHWC) and a layout change
    din = O.ConvCtx("fp32").conv_dgrad(dy_nhwc, w_khwc, (N, H, W, Cin), 2, 3)
    comp = O.nhwc_to_nchw(din)
    for k, o in enumerate(outs):
        assert rel_l2(o, comp[:, 3 * k:3 * k + 3]) <= 1e-6
    if Cin == 6:
        # one image only: the other output is not written
        only2 = O.stem_dgrad(dy_nhwc, w_khwc, H, W, (False, True))
        assert only2[0] is None and torch.equal(only2[1], outs[1])


# ----- frozen-statistics BatchNorm backward -------------------------------------------------------------------------------------
FROZEN_BN_CASES = [
    # C, groups, rows per group, relu, residual (dres wanted), TF32 rounding, low part
    (64, 1, 700, 1, 0, 0, 0),
    (64, 3, 130, 1, 1, 0, 1),
    (128, 2, 96, 0, 1, 0, 0),
    (256, 1, 333, 1, 1, 1, 0),
    (512, 4, 24, 1, 0, 0, 1),
    (1024, 2, 40, 1, 1, 0, 0),
    (2048, 3, 12, 1, 1, 0, 1),
]


@pytest.mark.parametrize("case", FROZEN_BN_CASES, ids=lambda c: "C%d_G%d_R%d_relu%d_res%d_rnd%d_lo%d" % c)
def test_frozen_batchnorm_backward_vs_fp64(case):
    O = _ops()
    C, G, R, relu, residual, rnd, with_lo = case
    g = torch.Generator().manual_seed(C + 7 * G + R)
    rows = G * R
    y = (torch.randn(rows, C, generator=g) * (0.5 + torch.rand(C, generator=g)) + torch.randn(C, generator=g)).float()
    res = torch.randn(rows, C, generator=g).float() if residual else None
    gamma = (1 + 0.2 * torch.randn(C, generator=g)).float()
    beta = (0.2 * torch.randn(C, generator=g)).float()
    rm, rv = (0.3 * torch.randn(C, generator=g)).float(), (0.5 + torch.rand(C, generator=g)).float()
    dz = torch.randn(rows, C, generator=g).float()
    dg0, db0 = torch.randn(C, generator=g).float(), torch.randn(C, generator=g).float()

    y64 = y.double().requires_grad_(True)
    gm64, bt64 = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    pre = F.batch_norm(y64, rm.double(), rv.double(), gm64, bt64, False, 0.1, BN_EPS)
    if residual:
        pre = pre + res.double()
    yc, gc, bc = y.to(DEV), gamma.to(DEV), beta.to(DEV)
    flags = (1 if relu else 0) | (O.ROUND_TF32 if rnd else 0)
    z, saved = O.bn_apply(yc, None, gc, bc, rm.to(DEV), rv.to(DEV), 0.1, BN_EPS, res.to(DEV) if residual else None, flags, G)
    gate = z.cpu() > 0 if relu else torch.ones(rows, C, dtype=torch.bool)
    pre.backward(torch.where(gate, dz.double(), 0.0))
    dgc, dbc = dg0.to(DEV), db0.to(DEV)
    dzc = dz.to(DEV)
    dy, dres = O.bn_backward(dzc, z, yc, saved, dgc, dbc, flags | O.BN_FROZEN, bool(residual), G, bool(with_lo))
    if rnd:
        # the same call without rounding: the rounded dy is within TF32 rounding of it
        dy_plain, _ = O.bn_backward(dz.to(DEV), z, yc, saved, None, None, (flags & ~O.ROUND_TF32) | O.BN_FROZEN, False, G)
        _close(dy_plain, y64.grad, 1e-5, "dy")
        _close(dy, y64.grad, 1e-3, "dy (TF32)")
    else:
        _close(dy, y64.grad, 1e-5, "dy")
    _close(dgc - dg0.to(DEV), gm64.grad, 1e-5, "dgamma")
    _close(dbc - db0.to(DEV), bt64.grad, 1e-5, "dbeta")
    if residual:
        assert torch.equal(dres.cpu(), torch.where(gate, dz, 0.0))
    if with_lo:
        from scsfm import nnops
        lo = nnops.split_tf32(dy.clone())
        assert torch.equal(dy._scsfm_lo, lo)
    # without parameter gradients (frozen network): the same dy, bitwise, from the single pass alone
    dy2, _ = O.bn_backward(dz.to(DEV), z, yc, saved, None, None, flags | O.BN_FROZEN, False, G)
    assert torch.equal(dy2, dy)


# ----- whole networks against the fp64 oracle -----------------------------------------------------------------------------------
def _build(kind, layers, mode="fp32"):
    import models
    net = models.DispResNet(layers, False) if kind == "disp" else models.PoseResNet(layers, False)
    net.load_state_dict(det_weights(net.state_dict()))
    return net.to(DEV).set_conv_mode(mode)


def _images(B=2, H=64, W=96):
    return det_image("img1", B, H, W), det_image("img2", B, H, W)


def _running_stats(kind, layers, imgs):
    """Running statistics that normalise the test images (an eval-mode network with untouched statistics would leave its
    activations unnormalised): the batch statistics of one fp64 train-mode oracle pass, accumulated with momentum None."""
    from oracle import nets as N
    ref = (N.DispResNet(layers) if kind == "disp" else N.PoseResNet(layers)).double()
    ref.load_state_dict({k: v.double() for k, v in det_weights(ref.state_dict()).items()})
    for m in ref.modules():
        if isinstance(m, nn.BatchNorm2d):
            m.momentum = None
            m.reset_running_stats()
    ref.train()
    with torch.no_grad():
        ref(*[i.double() for i in imgs[:1 if kind == "disp" else 2]])
    return {k: v.float() for k, v in ref.state_dict().items() if "running" in k}


def _state(kind, layers, imgs, training):
    import models
    sd = det_weights((models.DispResNet(layers, False) if kind == "disp" else models.PoseResNet(layers, False)).state_dict())
    if not training:
        sd.update(_running_stats(kind, layers, imgs))
    return sd


def _loss(kind, out):
    if kind == "disp":
        outs = out if isinstance(out, (list, tuple)) else [out]
        return sum(((1.0 / o) * (i + 1)).mean() for i, o in enumerate(outs))
    return (out * torch.arange(1, 7, dtype=out.dtype, device=out.device)).sum() * 100


def _run_oracle(kind, layers, sd, imgs, training, dtype, dev="cpu"):
    from oracle import nets as N
    ref = (N.DispResNet(layers) if kind == "disp" else N.PoseResNet(layers)).to(dtype).to(dev)
    ref.load_state_dict({k: v.to(dtype).to(dev) if v.is_floating_point() else v for k, v in sd.items()})
    ref.train(training)
    xs = [i.detach().clone().to(dtype).to(dev).requires_grad_(True) for i in imgs[:1 if kind == "disp" else 2]]
    _loss(kind, ref(*xs)).backward()
    grads = {k: p.grad for k, p in ref.named_parameters() if p.grad is not None}
    for n, x in enumerate(xs):
        grads["input%d" % (n + 1)] = x.grad
    return grads


def _run_mine(kind, layers, sd, imgs, training, mode):
    import models
    net = models.DispResNet(layers, False) if kind == "disp" else models.PoseResNet(layers, False)
    net.load_state_dict(sd)
    net = net.to(DEV).set_conv_mode(mode)
    net.train(training)
    xs = [i.detach().clone().to(DEV).requires_grad_(True) for i in imgs[:1 if kind == "disp" else 2]]
    _loss(kind, net(*xs)).backward()
    grads = {k: p.grad for k, p in net.named_parameters()}
    for n, x in enumerate(xs):
        assert x.grad is not None and x.grad.shape == x.shape
        grads["input%d" % (n + 1)] = x.grad
    return grads


@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("mode", ["fp32", "tf32x3"])
@pytest.mark.parametrize("layers", [18, 50])
@pytest.mark.parametrize("kind", ["disp", "pose"])
def test_network_input_and_parameter_gradients_vs_oracle(kind, layers, mode, training):
    """Every parameter gradient and the gradient of every input image against the fp64 oracle run in the same mode, with the
    yardstick of test_nets_gpu.py: no worse than 4x the larger error of the fp32 CPU oracle and of stock PyTorch / cuDNN fp32."""
    imgs = _images()
    sd = _state(kind, layers, imgs, training)
    mine = _run_mine(kind, layers, sd, imgs, training, mode)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    g64 = _run_oracle(kind, layers, sd, imgs, training, torch.float64)
    g32 = _run_oracle(kind, layers, sd, imgs, training, torch.float32)
    g32gpu = _run_oracle(kind, layers, sd, imgs, training, torch.float32, DEV)
    errs = sorted((rel_l2(mine[k], gr), k) for k, gr in g64.items())
    errs_cpu = sorted(rel_l2(g32[k], gr) for k, gr in g64.items())
    errs_gpu = sorted(rel_l2(g32gpu[k], gr) for k, gr in g64.items())
    med, worst = errs[len(errs) // 2][0], errs[-1]
    yard_med = max(errs_cpu[len(errs_cpu) // 2], errs_gpu[len(errs_gpu) // 2])
    yard_worst = max(errs_cpu[-1], errs_gpu[-1])
    inputs = {k: e for e, k in errs if k.startswith("input")}
    print(kind, layers, mode, "train" if training else "eval", "rel-L2 vs fp64: median %.2e worst %.2e (%s), inputs %s; fp32 CPU oracle "
          "median %.2e worst %.2e; cuDNN fp32 median %.2e worst %.2e" % (med, worst[0], worst[1], inputs, errs_cpu[len(errs_cpu) // 2],
                                                                      errs_cpu[-1], errs_gpu[len(errs_gpu) // 2], errs_gpu[-1]))
    assert med < 4 * yard_med + 1e-4 and worst[0] < 4 * yard_worst + 3e-3
    for k, e in inputs.items():
        yard = max(rel_l2(g32[k], g64[k]), rel_l2(g32gpu[k], g64[k]))
        assert e < 4 * yard + 1e-4, (k, e, yard)


def test_disp_net_tf32_mode_input_gradient_vs_oracle():
    """Single-product TF32 mode, eval mode: no worse than 3x stock PyTorch / cuDNN TF32 (the bound of
    test_disp_net_tf32_mode_vs_oracle), input gradient included."""
    imgs = _images()
    sd = _state("disp", 18, imgs, False)
    mine = _run_mine("disp", 18, sd, imgs, False, "tf32")
    g64 = _run_oracle("disp", 18, sd, imgs, False, torch.float64)
    torch.backends.cudnn.allow_tf32 = True
    stock = _run_oracle("disp", 18, sd, imgs, False, torch.float32, DEV)
    torch.backends.cudnn.allow_tf32 = False
    errs = sorted(rel_l2(mine[k], gr) for k, gr in g64.items())
    errs_stock = sorted(rel_l2(stock[k], gr) for k, gr in g64.items())
    med, med_stock = errs[len(errs) // 2], errs_stock[len(errs_stock) // 2]
    e_in, e_in_stock = rel_l2(mine["input1"], g64["input1"]), rel_l2(stock["input1"], g64["input1"])
    print("tf32 eval: median %.2e worst %.2e input %.2e | cuDNN TF32: median %.2e worst %.2e input %.2e"
          % (med, errs[-1], e_in, med_stock, errs_stock[-1], e_in_stock))
    assert med < 3 * med_stock + 1e-3 and errs[-1] < 3 * errs_stock[-1] + 1e-2
    assert e_in < 3 * e_in_stock + 1e-3


# ----- partial image gradients, forward_multi -----------------------------------------------------------------------------------
def test_pose_only_second_image_requires_grad():
    imgs = _images()
    sd = _state("pose", 18, imgs, False)
    import models
    net = models.PoseResNet(18, False)
    net.load_state_dict(sd)
    net = net.to(DEV).eval()
    a1, a2 = imgs[0].to(DEV).requires_grad_(True), imgs[1].to(DEV).requires_grad_(True)
    _loss("pose", net(a1, a2)).backward()
    b1, b2 = imgs[0].to(DEV), imgs[1].to(DEV).requires_grad_(True)
    net.zero_grad()
    _loss("pose", net(b1, b2)).backward()
    assert b1.grad is None
    assert rel_l2(b2.grad, a2.grad) < 1e-6
    g64 = _run_oracle("pose", 18, sd, imgs, False, torch.float64)
    assert rel_l2(b2.grad, g64["input2"]) < 1e-3


@pytest.mark.parametrize("kind", ["disp", "pose"])
def test_forward_multi_input_gradients_equal_separate_calls(kind):
    imgs = [det_image(n, 2, 64, 96).to(DEV) for n in ("img1", "img2", "img3")]
    a, b = _build(kind, 18), _build(kind, 18)
    a.train(); b.train()
    if kind == "disp":
        xa = [x.clone().requires_grad_(True) for x in imgs]
        xb = [x.clone().requires_grad_(True) for x in imgs]
        la = sum(_loss(kind, a(x)) * (i + 1) for i, x in enumerate(xa))
        lb = sum(_loss(kind, o) * (i + 1) for i, o in enumerate(b.forward_multi(xb)))
    else:
        xa = [(imgs[i].clone().requires_grad_(True), imgs[(i + 1) % 3].clone().requires_grad_(True)) for i in range(3)]
        xb = [(x.detach().clone().requires_grad_(True), y.detach().clone().requires_grad_(True)) for x, y in xa]
        la = sum(_loss(kind, a(x, y)) * (i + 1) for i, (x, y) in enumerate(xa))
        lb = sum(_loss(kind, o) * (i + 1) for i, o in enumerate(b.forward_multi(xb)))
        xa = [t for p in xa for t in p]
        xb = [t for p in xb for t in p]
    la.backward(); lb.backward()
    for u, v in zip(xa, xb):
        assert u.grad is not None and v.grad is not None
        assert rel_l2(v.grad, u.grad) < 1e-4


# ----- frozen networks, launch accounting -----------------------------------------------------------------------------------------
def _backward_events(net, kind, xs):
    """(library launches, profiled launch families) of one backward."""
    from scsfm import lib as L
    out = net(*xs)
    loss = _loss(kind, out)
    torch.cuda.synchronize()
    L.PROF["enabled"], L.PROF["events"] = True, []
    n0 = L.launch_count()
    loss.backward()
    n1 = L.launch_count()
    fams = [e[0] for e in L.PROF["events"]]
    L.PROF["enabled"], L.PROF["events"] = False, []
    torch.cuda.synchronize()
    return n1 - n0, fams


@pytest.mark.parametrize("mode", ["fp32", "tf32x3"])
@pytest.mark.parametrize("kind", ["disp", "pose"])
def test_frozen_network_runs_data_gradients_only(kind, mode):
    imgs = _images()
    sd = _state(kind, 18, imgs, False)
    import models
    net = models.DispResNet(18, False) if kind == "disp" else models.PoseResNet(18, False)
    net.load_state_dict(sd)
    net = net.to(DEV).set_conv_mode(mode).eval()
    n_img = 1 if kind == "disp" else 2
    _backward_events(net, kind, [i.to(DEV).requires_grad_(True) for i in imgs[:n_img]])     # first call: operand caches
    xa = [i.to(DEV).requires_grad_(True) for i in imgs[:n_img]]
    n_full, fams_full = _backward_events(net, kind, xa)
    net.requires_grad_(False)
    sentinel = torch.randn(net.flat_grads().shape, generator=torch.Generator().manual_seed(5)).to(DEV)
    net.flat_grads().copy_(sentinel)
    xb = [i.to(DEV).requires_grad_(True) for i in imgs[:n_img]]
    n_frozen, fams_frozen = _backward_events(net, kind, xb)
    for u, v in zip(xa, xb):
        assert rel_l2(v.grad, u.grad) < 1e-6
    assert torch.equal(net.flat_grads(), sentinel)              # the gradient arena is untouched
    assert any(f.startswith("conv_wgrad") for f in fams_full) and ("head_wgrad" in fams_full) == (kind == "disp")
    assert not any(f.startswith("conv_wgrad") or f in ("head_wgrad", "weight_round") for f in fams_frozen)
    # BatchNorm: one kernel per layer (the single frozen pass) instead of two (plus the parameter-gradient kernel)
    n_bn = fams_frozen.count("bn_bwd")
    assert n_bn == fams_full.count("bn_bwd") > 0
    assert n_frozen < n_full - n_bn
    # nothing at all to compute: no image and no parameter wants a gradient
    xc = [i.to(DEV) for i in imgs[:n_img]]
    n_none, _ = _backward_events(net, kind, xc)
    assert n_none == 0


@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("kind", ["disp", "pose"])
def test_image_gradients_cost_exactly_the_stem_gradient_launches(kind, training):
    imgs = _images()
    net = _build(kind, 18, "tf32x3").train(training)
    n_img = 1 if kind == "disp" else 2
    _backward_events(net, kind, [i.to(DEV) for i in imgs[:n_img]])     # first call: operand caches
    n_off, fams_off = _backward_events(net, kind, [i.to(DEV) for i in imgs[:n_img]])
    n_on, fams_on = _backward_events(net, kind, [i.to(DEV).requires_grad_(True) for i in imgs[:n_img]])
    assert "stem_dgrad" not in fams_off and fams_on.count("stem_dgrad") == 1
    assert n_on - n_off == 1
    # only one of PoseResNet's images: still one launch
    if kind == "pose":
        n_one, _ = _backward_events(net, kind, [imgs[0].to(DEV), imgs[1].to(DEV).requires_grad_(True)])
        assert n_one - n_off == 1


# ----- a learnable module in front of a network -----------------------------------------------------------------------------------
class _Affine(nn.Module):
    """Per-channel affine input normaliser."""

    def __init__(self):
        super().__init__()
        self.scale = nn.Parameter(torch.tensor([1.1, 0.9, 1.05]))
        self.shift = nn.Parameter(torch.tensor([0.05, -0.1, 0.02]))

    def forward(self, x):
        return x * self.scale.view(1, 3, 1, 1) + self.shift.view(1, 3, 1, 1)


def test_learnable_module_in_front_of_the_network_gets_its_gradient():
    from oracle import nets as N
    imgs = _images()
    sd = _state("disp", 18, imgs, False)

    def run(dtype, dev, mine):
        import models
        aff = _Affine().to(dtype).to(dev)
        if mine:
            net = models.DispResNet(18, False)
            net.load_state_dict(sd)
            net = net.to(dev)
        else:
            net = N.DispResNet(18).to(dtype).to(dev)
            net.load_state_dict({k: v.to(dtype).to(dev) if v.is_floating_point() else v for k, v in sd.items()})
        net.eval()
        _loss("disp", net(aff(imgs[0].to(dtype).to(dev)))).backward()
        return torch.cat([aff.scale.grad, aff.shift.grad])

    got = run(torch.float32, DEV, True)
    ref64 = run(torch.float64, "cpu", False)
    ref32 = run(torch.float32, "cpu", False)
    assert float(got.abs().max()) > 0
    assert rel_l2(got, ref64) < 4 * rel_l2(ref32, ref64) + 1e-5, (rel_l2(got, ref64), rel_l2(ref32, ref64))
