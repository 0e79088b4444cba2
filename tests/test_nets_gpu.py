"""Parity of the network kernels (conv fwd/dgrad/wgrad, BN, pool, decoder ops) and of the whole
DispResNet / PoseResNet forward+backward against the oracle and the reference vectors.  Needs a GPU.

fp32 CUDA-core mode ("fp32"): same arithmetic class as the CPU reference -> tolerances are fp32 noise.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from golden_util import det_image, det_weights
from helpers import rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _ops():
    from scsfm import nnops
    return nnops


CONV_CASES = [
    # B, H, W, Cin, Cout, k, stride, pad, pad_mode(0 zero/1 reflect), act, bias
    (2, 20, 28, 3, 64, 7, 2, 3, 0, 0, False),     # stem
    (2, 20, 28, 6, 64, 7, 2, 3, 0, 0, False),     # pose stem
    (2, 12, 20, 64, 64, 3, 1, 1, 0, 0, False),    # layer1
    (2, 12, 20, 64, 128, 3, 2, 1, 0, 0, False),   # layer2.0.conv1
    (2, 12, 20, 64, 128, 1, 2, 0, 0, 0, False),   # downsample
    (1, 9, 13, 32, 16, 3, 1, 1, 1, 2, True),      # decoder reflect + ELU, Cout 16
    (1, 10, 14, 96, 32, 3, 1, 1, 1, 2, True),     # decoder, Cout 32
    (2, 10, 14, 16, 1, 3, 1, 1, 1, 3, True),      # dispconv + sigmoid
    (2, 4, 6, 256, 6, 1, 1, 0, 0, 0, True),       # pose head
    (2, 4, 6, 512, 256, 1, 1, 0, 0, 1, True),     # pose squeeze + ReLU
    (1, 7, 9, 256, 64, 1, 1, 0, 0, 0, False),     # bottleneck 1x1
]


def _ref_conv(x, w, b, stride, pad, pad_mode, act):
    if pad_mode == 1:
        x = F.pad(x, (pad, pad, pad, pad), mode="reflect")
        pad = 0
    y = F.conv2d(x, w, b, stride, pad)
    if act == 1:
        y = F.relu(y)
    elif act == 2:
        y = F.elu(y)
    elif act == 3:
        y = 10 * torch.sigmoid(y) + 0.01
    return y


@pytest.mark.parametrize("case", CONV_CASES)
def test_conv_fwd_dgrad_wgrad_vs_torch_fp64(case):
    O = _ops()
    B, H, W, Cin, Cout, k, stride, pad, pad_mode, act, bias = case
    g = torch.Generator().manual_seed(7)
    x = torch.randn(B, Cin, H, W, generator=g, dtype=torch.float64, requires_grad=True)
    w = (torch.randn(Cout, Cin, k, k, generator=g, dtype=torch.float64) / (Cin * k * k) ** 0.5).requires_grad_(True)
    b = torch.randn(Cout, generator=g, dtype=torch.float64).requires_grad_(True) if bias else None
    pre = _ref_conv(x, w, b, stride, pad, pad_mode, 0)
    y = _ref_conv(x, w, b, stride, pad, pad_mode, act)
    dpre = torch.randn(pre.shape, generator=g, dtype=torch.float64)
    pre.backward(dpre)

    xc = x.detach().float().permute(0, 2, 3, 1).contiguous().to(DEV)
    wc = w.detach().float().permute(0, 2, 3, 1).contiguous().to(DEV)
    bc = b.detach().float().to(DEV) if bias else None
    sums = torch.zeros(O.BN_SLOTS * Cout * 2, device=DEV, dtype=torch.float64)
    cx = O.ConvCtx("fp32")
    yc = cx.conv_fwd(xc, wc, bc, stride, pad, pad_mode, act, sums, 1)
    assert rel_l2(yc.permute(0, 3, 1, 2), y.detach()) < 2e-6
    s = sums.view(O.BN_SLOTS, Cout, 2).sum(0).cpu()
    np.testing.assert_allclose(s[:, 0], y.detach().sum((0, 2, 3)), rtol=1e-4, atol=1e-3)
    np.testing.assert_allclose(s[:, 1], (y.detach() ** 2).sum((0, 2, 3)), rtol=1e-4, atol=1e-3)

    dc = dpre.float().permute(0, 2, 3, 1).contiguous().to(DEV)
    dw = torch.zeros_like(wc)
    db = torch.zeros(Cout, device=DEV) if bias else None
    cx.conv_wgrad(xc, dc, dw, db, stride, pad, pad_mode)
    assert rel_l2(dw.permute(0, 3, 1, 2), w.grad) < 2e-6
    if bias:
        assert rel_l2(db, b.grad) < 1e-5
    if pad_mode == 0:
        add = torch.randn(B, H, W, Cin, generator=g).to(DEV)
        dx = cx.conv_dgrad(dc, wc, xc.shape, stride, pad, add)
        assert rel_l2((dx - add).permute(0, 3, 1, 2), x.grad) < 2e-6
    else:
        dpad = cx.conv_dgrad(dc, wc, xc.shape, stride, pad, None, padded_input=True)
        dx = torch.zeros_like(xc)
        O.fold_plain(dpad, dx, None, O.ACT_NONE, accumulate=False)
        assert rel_l2(dx.permute(0, 3, 1, 2), x.grad) < 2e-6


def test_bn_pool_upcat_ops_vs_torch():
    O = _ops()
    g = torch.Generator().manual_seed(3)
    B, H, W, C = 3, 10, 14, 32
    y = torch.randn(B, C, H, W, generator=g, dtype=torch.float64, requires_grad=True)
    res = torch.randn(B, C, H, W, generator=g, dtype=torch.float64, requires_grad=True)
    gamma = (1 + 0.1 * torch.randn(C, generator=g, dtype=torch.float64)).requires_grad_(True)
    beta = (0.1 * torch.randn(C, generator=g, dtype=torch.float64)).requires_grad_(True)
    rm, rv = torch.zeros(C, dtype=torch.float64), torch.ones(C, dtype=torch.float64)
    z = F.relu(F.batch_norm(y, rm, rv, gamma, beta, True, 0.1, 1e-5) + res)
    dz = torch.randn(z.shape, generator=g, dtype=torch.float64)
    z.backward(dz)
    nh = lambda t: t.detach().float().permute(0, 2, 3, 1).contiguous().to(DEV)  # noqa: E731
    yc, rc = nh(y), nh(res)
    sums = torch.zeros(O.BN_SLOTS, C, 2, device=DEV, dtype=torch.float64)
    sums[3] = torch.stack([yc.double().sum((0, 1, 2)), (yc.double() ** 2).sum((0, 1, 2))], 1)
    gm, bt = gamma.detach().float().to(DEV), beta.detach().float().to(DEV)
    rmc, rvc = torch.zeros(C, device=DEV), torch.ones(C, device=DEV)
    zc, saved = O.bn_apply(yc, sums, gm, bt, rmc, rvc, 0.1, 1e-5, rc, 1, 1, True)
    assert rel_l2(zc.permute(0, 3, 1, 2), z.detach()) < 2e-6
    assert torch.equal(zc._scsfm_lo, O.split_tf32(zc))           # low part produced with the tensor itself (split-accumulate mode)
    hi = (zc.view(torch.int32) & -8192).view(torch.float32)      # what kind::tf32 reads: the upper 19 bits
    assert float((hi.double() + zc._scsfm_lo.double() - zc.double()).abs().max()) <= 2.0 ** -20 * float(zc.abs().max())
    assert rel_l2(rmc, rm) < 1e-5 and rel_l2(rvc, rv) < 1e-5
    dgm, dbt = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
    dzc = nh(dz)
    dy, dres = O.bn_backward(dzc, zc, yc, saved, dgm, dbt, True, True, 1, True)
    assert torch.equal(dy._scsfm_lo, O.split_tf32(dy))
    assert rel_l2(dy.permute(0, 3, 1, 2), y.grad) < 1e-5
    assert rel_l2(dres.permute(0, 3, 1, 2), res.grad) < 1e-6
    assert rel_l2(dgm, gamma.grad) < 1e-5 and rel_l2(dbt, beta.grad) < 1e-5
    # eval mode uses the running statistics
    ze, _ = O.bn_apply(yc, None, gm, bt, rmc, rvc, 0.1, 1e-5, None, 0)
    want = F.batch_norm(y.detach(), rm, rv, gamma.detach(), beta.detach(), False, 0.1, 1e-5)
    assert rel_l2(ze.permute(0, 3, 1, 2), want) < 2e-6

    # max-pool 3x3/2 pad 1 (odd sizes too)
    for (h, w) in ((10, 14), (9, 13)):
        x = torch.randn(2, 8, h, w, generator=g, dtype=torch.float64, requires_grad=True)
        p = F.max_pool2d(x, 3, 2, 1)
        dp = torch.randn(p.shape, generator=g, dtype=torch.float64)
        p.backward(dp)
        xc = nh(x)
        pc, idx = O.maxpool_fwd(xc)
        assert rel_l2(pc.permute(0, 3, 1, 2), p.detach()) < 1e-6
        dx = torch.ones_like(xc)
        O.maxpool_bwd(nh(dp), idx, xc.shape, dx, True)
        assert rel_l2((dx - 1).permute(0, 3, 1, 2), x.grad) < 1e-6

    # upsample + concat, forward and (through a reflect-pad conv's padded gradient) backward
    lo = torch.randn(2, 8, 5, 7, generator=g, dtype=torch.float64, requires_grad=True)
    sk = torch.randn(2, 12, 10, 14, generator=g, dtype=torch.float64, requires_grad=True)
    a = F.elu(lo)
    cat = torch.cat([F.interpolate(a, scale_factor=2, mode="nearest"), sk], 1)
    padded = F.pad(cat, (1, 1, 1, 1), mode="reflect")
    dpad = torch.randn(padded.shape, generator=g, dtype=torch.float64)
    padded.backward(dpad)
    ac = nh(a)
    catc = O.upcat_fwd(ac, nh(sk))
    assert rel_l2(catc.permute(0, 3, 1, 2), cat.detach()) < 1e-6
    d_lo, d_sk = O.fold_upcat(nh(dpad), 8, ac, O.ACT_ELU)
    assert rel_l2(d_lo.permute(0, 3, 1, 2), lo.grad) < 1e-6
    assert rel_l2(d_sk.permute(0, 3, 1, 2), sk.grad) < 1e-6


def _build(kind, layers, mode="fp32"):
    import models
    net = models.DispResNet(layers, False) if kind == "disp" else models.PoseResNet(layers, False)
    net.load_state_dict(det_weights(net.state_dict()))
    return net.to(DEV).set_conv_mode(mode)


@pytest.mark.parametrize("mode", ["fp32", "tf32x3"])
@pytest.mark.parametrize("layers", [18, 50])
@pytest.mark.parametrize("kind", ["disp", "pose"])
def test_networks_vs_reference_vectors_and_oracle(golden_nets, layers, kind, mode):
    """Train-mode forward, backward (every parameter gradient), BN running stats and eval-mode forward, in both 1e-4
    parity modes: exact CUDA-core convolutions ("fp32") and split-accumulate tensor-core convolutions ("tf32x3")."""
    from oracle import nets as N
    g = golden_nets
    tag = f"{kind}{layers}"
    net = _build(kind, layers, mode)
    sd = net.state_dict()
    assert list(sd.keys()) == list(g[f"{tag}_keys"])
    net.train()
    img1, img2 = det_image("img1", 2, 64, 96), det_image("img2", 2, 64, 96)
    if kind == "disp":
        outs = net(img1.to(DEV))
        assert isinstance(outs, list) and len(outs) == 4
        loss = sum(((1.0 / o) * (i + 1)).mean() for i, o in enumerate(outs))
        for s, o in enumerate(outs):
            assert rel_l2(o.detach(), g[f"{tag}_out_s{s}"]) < 1e-4
            np.testing.assert_allclose(o.detach().cpu().numpy(), g[f"{tag}_out_s{s}"], rtol=2e-3, atol=5e-5)
    else:
        o = net(img1.to(DEV), img2.to(DEV))
        loss = (o * torch.arange(1, 7, dtype=o.dtype, device=DEV)).sum() * 100
        np.testing.assert_allclose(o.detach().cpu().numpy(), g[f"{tag}_out"], rtol=1e-3, atol=2e-7)
    loss.backward()
    np.testing.assert_allclose(float(loss.detach()), g[f"{tag}_loss"][0], rtol=2e-4)
    grads = {k: p.grad for k, p in net.named_parameters()}
    names = list(g[f"{tag}_grad_names"])
    norms = np.array([float(grads[k].double().norm()) for k in names])
    np.testing.assert_allclose(norms, g[f"{tag}_grad_norms"], rtol=2e-2, atol=1e-8)
    # parameters the reference leaves without gradient (fc head) stay exactly zero here
    for k, v in grads.items():
        if k not in names:
            assert float(v.abs().max()) == 0.0, k
    # element-wise gradients against the fp64 oracle run on the same weights; the yardstick is the error the
    # fp32 CPU oracle itself makes against fp64 (deep nets with tiny BatchNorm populations amplify fp32 noise)
    def oracle_grads(dtype, dev="cpu"):
        ref = (N.DispResNet(layers) if kind == "disp" else N.PoseResNet(layers)).to(dtype).to(dev)
        ref.load_state_dict({k: v.to(dtype).to(dev) for k, v in det_weights(ref.state_dict()).items()})
        ref.train()
        if kind == "disp":
            ro = ref(img1.to(dtype).to(dev))
            rl = sum(((1.0 / o) * (i + 1)).mean() for i, o in enumerate(ro))
        else:
            ro = ref(img1.to(dtype).to(dev), img2.to(dtype).to(dev))
            rl = (ro * torch.arange(1, 7, dtype=ro.dtype, device=dev)).sum() * 100
        rl.backward()
        return {k: p.grad for k, p in ref.named_parameters() if p.grad is not None}
    # Yardstick = what INDEPENDENT fp32 evaluations of the same network do against fp64: the CPU oracle and stock PyTorch / cuDNN on
    # this GPU with TF32 off.  These deliberately ill-conditioned test networks (random weights, BatchNorm over 12 samples at the
    # deepest stage) amplify fp32 rounding by 1e2..1e4 and a single ReLU / max-pool decision that flips on a ~0 activation moves
    # every upstream gradient at once: the round-1 "ResNet-50 drift" (1.5e-3 vs 1.5e-4) was exactly that -- tools/diag_grad_error.py
    # shows the CPU oracle itself at 4.4e-3 on another run.  Hence two yardsticks, no per-depth slack.
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    g64, g32, g32gpu = oracle_grads(torch.float64), oracle_grads(torch.float32), oracle_grads(torch.float32, DEV)
    errs = sorted((rel_l2(grads[k], gr), k) for k, gr in g64.items())
    errs_cpu = sorted(rel_l2(g32[k], gr) for k, gr in g64.items())
    errs_gpu = sorted(rel_l2(g32gpu[k], gr) for k, gr in g64.items())
    med, worst = errs[len(errs) // 2][0], errs[-1]
    yard_med = max(errs_cpu[len(errs_cpu) // 2], errs_gpu[len(errs_gpu) // 2])
    yard_worst = max(errs_cpu[-1], errs_gpu[-1])
    print(tag, mode, "per-parameter gradient rel-L2 vs fp64 oracle: median %.2e worst %.2e (%s); fp32 CPU oracle: median %.2e worst %.2e; "
          "stock PyTorch/cuDNN fp32 on this GPU: median %.2e worst %.2e"
          % (med, worst[0], worst[1], errs_cpu[len(errs_cpu) // 2], errs_cpu[-1], errs_gpu[len(errs_gpu) // 2], errs_gpu[-1]))
    # (worst: a BatchNorm scale whose gradient nearly cancels, e.g. layer2.1.bn2.weight of the 18-layer net, carries a few 1e-3 of
    # relative error in any evaluation whose rounding differs)
    assert med < 4 * yard_med + 1e-4 and worst[0] < 4 * yard_worst + 3e-3
    sd2 = net.state_dict()
    rn = np.array([float(sd2[k].double().norm()) for k in g[f"{tag}_running_names"]])
    np.testing.assert_allclose(rn, g[f"{tag}_running_norms"], rtol=1e-4)
    net.eval()
    with torch.no_grad():
        e = net(img1.to(DEV)) if kind == "disp" else net(img1.to(DEV), img2.to(DEV))
    assert torch.is_tensor(e)
    assert rel_l2(e, g[f"{tag}_eval_out"]) < 1e-4
    np.testing.assert_allclose(e.cpu().numpy(), g[f"{tag}_eval_out"], rtol=2e-3, atol=5e-5)


def test_state_dict_roundtrip_and_gradient_accumulation():
    import models
    net = models.DispResNet(18, False).to(DEV)
    sd = {k: v.clone() for k, v in net.state_dict().items()}
    net2 = models.DispResNet(18, False).to(DEV)
    net2.load_state_dict(sd)
    x = det_image("img1", 1, 64, 96).to(DEV)
    net.train(); net2.train()
    a, b = net(x)[0], net2(x)[0]
    assert rel_l2(a, b) < 1e-6          # BatchNorm sums use atomics: bitwise equality is not guaranteed
    # two backward passes accumulate; zero_grad resets
    (a.mean()).backward()
    g1 = net.flat_grads().clone()
    (net(x)[0].mean()).backward()
    assert rel_l2(net.flat_grads(), 2 * g1) < 1e-4
    net.zero_grad()
    assert float(net.flat_grads().abs().max()) == 0.0
    # a torch optimizer that drops gradients (set_to_none) is handled too
    opt = torch.optim.Adam(net.parameters(), lr=1e-4)
    opt.zero_grad(set_to_none=True)
    (net(x)[0].mean()).backward()
    assert rel_l2(net.flat_grads(), g1) < 1e-4
    assert all(p.grad is not None for p in net.parameters())
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        models.PoseResNet(18, False)(x.cpu(), x.cpu())


def test_arena_adam_matches_torch_adam():
    from oracle import nets as N
    from scsfm.nets import ArenaAdam
    import models
    net = models.PoseResNet(18, False)
    net.load_state_dict(det_weights(net.state_dict()))
    net = net.to(DEV)
    ref = N.PoseResNet(18)
    ref.load_state_dict(det_weights(ref.state_dict()))
    ref = ref.to(DEV)
    opt = ArenaAdam([net], lr=1e-3)
    ropt = torch.optim.Adam(ref.parameters(), lr=1e-3)
    x1, x2 = det_image("img1", 2, 64, 96).to(DEV), det_image("img2", 2, 64, 96).to(DEV)
    net.train(); ref.train()
    torch.backends.cudnn.allow_tf32 = False
    for _ in range(3):
        opt.zero_grad()
        (net(x1, x2).sum() * 100).backward()
        opt.step()
        ropt.zero_grad()
        (ref(x1, x2).sum() * 100).backward()
        ropt.step()
    rsd = ref.state_dict()
    for k, v in net.state_dict().items():
        if v.dtype == torch.float32 and "fc." not in k:
            assert rel_l2(v, rsd[k]) < 1e-2, k


TC_CASES = [
    # B, H, W, Cin, Cout, k, stride, pad, pad_mode, act, bias
    (2, 24, 40, 64, 64, 3, 1, 1, 0, 0, False),     # BN=64, K=576 (18 k-blocks, > pipeline depth)
    (2, 24, 40, 64, 128, 3, 2, 1, 0, 0, False),    # stride 2
    (2, 24, 40, 64, 128, 1, 2, 0, 0, 0, False),    # 1x1 stride 2, K=64
    (1, 30, 50, 32, 16, 3, 1, 1, 1, 2, True),      # reflect, ELU, Cout 16, ragged M
    (1, 30, 50, 16, 16, 3, 1, 1, 1, 2, True),      # Cin 16: k-blocks straddle taps, K=144 (ragged K)
    (1, 20, 36, 96, 32, 3, 1, 1, 1, 2, True),      # Cin 96 (cat 32+64)
    (4, 8, 26, 512, 256, 3, 1, 1, 1, 2, True),     # deep: K=4608 (144 k-blocks)
    (2, 16, 28, 128, 256, 3, 1, 1, 0, 0, False),   # BN 64/128 dispatch
    (2, 9, 13, 256, 64, 1, 1, 0, 0, 0, False),     # bottleneck 1x1
    (2, 9, 13, 64, 256, 1, 1, 0, 0, 1, True),      # 1x1 expand + ReLU + bias
    (4, 64, 104, 64, 128, 3, 1, 1, 0, 0, False),   # large M -> 128-wide N tile (3-stage pipeline)
    (3, 64, 104, 128, 256, 1, 1, 0, 0, 0, False),  # 128-wide tile, two N tiles
    (2, 25, 41, 64, 128, 3, 2, 1, 0, 0, False),    # stride 2 on odd sizes (parity classes of unequal size)
    (2, 16, 52, 256, 512, 1, 2, 0, 0, 0, False),   # 1x1 stride 2: three parity classes have no taps
]


# ScsfmConv.tune words (nnops.tune): the heuristic, the cp.async gather kernel alone (+ the cp.async weight-gradient
# kernel), and two forced tilings of the persistent TMA kernel (128 / 256-pixel tiles -- the latter over 64-channel Cout
# tiles on the wider layers; 8- / 16-pixel-wide tiles; forcing also sends small reflection-padded layers through the
# zero-padded TMA pass + border-ring pass), the second one with the weight-gradient selector value 2, which selects the
# tensor-core weight-gradient kernel (the id keeps its historical name "wgradtma")
TMA_CONFIGS = {"auto": dict(), "gather": dict(no_tma=1, wgrad=1), "tma-128px-tw8": dict(mt=1, tw_log2=3),
               "tma-256px-tw16-wgradtma": dict(mt=2, tw_log2=4, wgrad=2)}


@pytest.mark.parametrize("mode", ["tf32", "tf32x3"])
@pytest.mark.parametrize("tma", sorted(TMA_CONFIGS))
@pytest.mark.parametrize("case", TC_CASES)
def test_tcgen05_conv_fwd_and_dgrad_vs_fp64(case, tma, mode):
    """Tensor-core (wgmma) kernels against fp64 on the operands they read.  "tf32": operands rounded to nearest TF32 by their
    producers, one product (exact in fp32), fp32 accumulation.  "tf32x3": raw fp32 operands + their low parts, three products
    into short accumulation chains: bound 1e-5 (north_star: 1e-4).  tf32 adds a whole K loop into one wgmma accumulator, which
    adds with truncation: bound 5e-5 (worst on an H100: 7.8e-6, at K = 4608)."""
    O = _ops()
    cx = O.ConvCtx(mode)
    cx.tune = O.tune(**TMA_CONFIGS[tma])
    x3 = mode == "tf32x3"
    tol = 1e-5 if x3 else 5e-5
    B, H, W, Cin, Cout, k, stride, pad, pad_mode, act, bias = case
    g = torch.Generator().manual_seed(11)
    x0 = torch.randn(B, Cin, H, W, generator=g, dtype=torch.float64)
    w0 = torch.randn(Cout, Cin, k, k, generator=g, dtype=torch.float64) / (Cin * k * k) ** 0.5
    b0 = torch.randn(Cout, generator=g, dtype=torch.float64) if bias else None
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    dpre = torch.randn(B, Cout, Ho, Wo, generator=g, dtype=torch.float64)
    xc = x0.float().permute(0, 2, 3, 1).contiguous().to(DEV)
    wc = w0.float().permute(0, 2, 3, 1).contiguous().to(DEV)
    bc = b0.float().to(DEV) if bias else None
    dc = dpre.float().permute(0, 2, 3, 1).contiguous().to(DEV)
    w_lo = None
    if x3:
        w_lo = O.split_tf32(wc)
    else:
        # the single-product kernels expect operands already rounded to TF32 by their producers (SCSFM_ROUND_TF32)
        for tns in (xc, wc, dc):
            O.round_tf32(tns, tns)
    # the fp64 reference from exactly these operands
    x = xc.double().permute(0, 3, 1, 2).cpu().requires_grad_(True)
    w = wc.double().permute(0, 3, 1, 2).cpu().requires_grad_(True)
    b = bc.double().cpu().requires_grad_(True) if bias else None
    pre = _ref_conv(x, w, b, stride, pad, pad_mode, 0)
    y = _ref_conv(x, w, b, stride, pad, pad_mode, act)
    pre.backward(dc.double().permute(0, 3, 1, 2).cpu())
    assert cx._use_tc("fwd", Cin, Cout, k, stride)
    sums = torch.zeros(O.BN_SLOTS * Cout * 2, device=DEV, dtype=torch.float64)
    yc = cx.conv_fwd(xc, wc, bc, stride, pad, pad_mode, act, sums, 1, w_lo)
    assert rel_l2(yc.permute(0, 3, 1, 2), y.detach()) < tol
    s = sums.view(O.BN_SLOTS, Cout, 2).sum(0).cpu()
    np.testing.assert_allclose(s[:, 0], yc.double().sum((0, 1, 2)).cpu(), rtol=1e-5, atol=1e-3)
    np.testing.assert_allclose(s[:, 1], (yc.double() ** 2).sum((0, 1, 2)).cpu(), rtol=1e-5, atol=1e-3)
    assert cx._use_tc("wgrad", Cin, Cout, k, stride)
    dw = torch.zeros_like(wc)
    db = torch.zeros(Cout, device=DEV) if bias else None
    cx.conv_wgrad(xc, dc, dw, db, stride, pad, pad_mode)
    assert rel_l2(dw.permute(0, 3, 1, 2), w.grad) < tol
    if bias:
        assert rel_l2(db, b.grad) < tol
    assert cx._use_tc("dgrad", Cin, Cout, k, stride)       # stride 2 runs as four parity-class sub-convolutions
    if pad_mode == 0:
        add = torch.randn(B, H, W, Cin, generator=g).to(DEV)
        dx = cx.conv_dgrad(dc, wc, xc.shape, stride, pad, add)
        assert rel_l2((dx.double() - add.double()).permute(0, 3, 1, 2), x.grad) < 2 * tol
    else:
        dpad = cx.conv_dgrad(dc, wc, xc.shape, stride, pad, None, padded_input=True)
        dx = torch.zeros_like(xc)
        O.fold_plain(dpad, dx, None, O.ACT_NONE, accumulate=False)
        assert rel_l2(dx.permute(0, 3, 1, 2), x.grad) < 2 * tol


THIN_CASES = [
    # B, H, W, Cin, pad_mode: 3x3 stride-1 pad-1 layers with 16 output channels (conv_wgrad_thin.cu)
    (2, 11, 37, 16, 1),      # partial tiles in both directions, reflection
    (2, 11, 37, 16, 0),      # zero padding
    (1, 3, 3, 16, 1),        # smallest plane reflection padding allows
    (4, 64, 320, 16, 1),     # 320 tiles: more than one tile per CTA (double-buffered staging)
    (2, 9, 21, 32, 1),       # Cin 32: 16-pixel-wide tiles
    (2, 16, 16, 32, 0),
    (3, 64, 208, 32, 1),     # 312 tiles: more than two per CTA
]


@pytest.mark.parametrize("mode", ["fp32", "tf32x3"])
@pytest.mark.parametrize("case", THIN_CASES)
def test_thin_layer_wgrad_kernel_vs_fp64(case, mode):
    """The fp32-FMA weight-gradient kernel of the 16-output-channel decoder layers (forced through the tune word, and what
    both modes pick on their own) against autograd in fp64: exact products, short fp32 chains -> 2e-6."""
    O = _ops()
    B, H, W, Cin, pad_mode = case
    Cout = 16
    g = torch.Generator().manual_seed(5)
    x = torch.randn(B, Cin, H, W, generator=g, dtype=torch.float64)
    w = torch.zeros(Cout, Cin, 3, 3, dtype=torch.float64, requires_grad=True)
    b = torch.zeros(Cout, dtype=torch.float64, requires_grad=True)
    dpre = torch.randn(B, Cout, H, W, generator=g, dtype=torch.float64)
    _ref_conv(x, w, b, 1, 1, pad_mode, 0).backward(dpre)
    xc = x.float().permute(0, 2, 3, 1).contiguous().to(DEV)
    dc = dpre.float().permute(0, 2, 3, 1).contiguous().to(DEV)
    for forced in (3, 0):
        cx = O.ConvCtx(mode)
        cx.tune = O.tune(wgrad=forced)
        dw = torch.zeros(Cout, 3, 3, Cin, device=DEV)
        db = torch.zeros(Cout, device=DEV)
        cx.conv_wgrad(xc, dc, dw, db, 1, 1, pad_mode)
        assert rel_l2(dw.permute(0, 3, 1, 2), w.grad) < 2e-6, forced
        assert rel_l2(db, b.grad) < 1e-5
        # it accumulates: a second call doubles the gradient
        cx.conv_wgrad(xc, dc, dw, None, 1, 1, pad_mode)
        assert rel_l2(dw.permute(0, 3, 1, 2), 2 * w.grad) < 2e-6


def test_disp_net_tf32_mode_vs_oracle(golden_nets):
    """Whole DispResNet-18 forward/backward with the single-product TF32 tensor-core kernels (the arithmetic the
    reference gets from cuDNN on a GPU by default; NOT the parity mode, which is tf32x3 above): outputs within 1e-2, every
    parameter gradient no worse than 3x stock PyTorch/cuDNN-TF32 against the fp64 oracle."""
    from oracle import nets as N
    if True:
        net = _build("disp", 18, "tf32")
        net.train()
        img1 = det_image("img1", 2, 64, 96)
        outs = net(img1.to(DEV))
        loss = sum(((1.0 / o) * (i + 1)).mean() for i, o in enumerate(outs))
        loss.backward()
        for s, o in enumerate(outs):
            assert rel_l2(o.detach(), golden_nets[f"disp18_out_s{s}"]) < 1e-2
        ref = N.DispResNet(18).double()
        ref.load_state_dict({k: v.double() for k, v in det_weights(ref.state_dict()).items()})
        ref.train()
        ro = ref(img1.double())
        sum(((1.0 / o) * (i + 1)).mean() for i, o in enumerate(ro)).backward()
        grads = {k: p.grad for k, p in net.named_parameters()}
        errs = sorted(rel_l2(grads[k], p.grad) for k, p in ref.named_parameters() if p.grad is not None)
        # yardstick: the same network in stock PyTorch on this GPU with cuDNN's TF32 convolutions (the reference's own
        # default arithmetic on a GPU), against the same fp64 oracle
        torch.backends.cudnn.allow_tf32 = True
        stock = N.DispResNet(18).to(DEV)
        stock.load_state_dict({k: v.to(DEV) for k, v in det_weights(stock.state_dict()).items()})
        stock.train()
        so = stock(img1.to(DEV))
        sum(((1.0 / o) * (i + 1)).mean() for i, o in enumerate(so)).backward()
        sg = {k: p.grad for k, p in stock.named_parameters()}
        errs_stock = sorted(rel_l2(sg[k], p.grad) for k, p in ref.named_parameters() if p.grad is not None)
        med, med_stock = errs[len(errs) // 2], errs_stock[len(errs_stock) // 2]
        print("tf32 mode: per-parameter gradient rel-L2 vs fp64 oracle: median %.2e worst %.2e | stock PyTorch/cuDNN TF32: median %.2e worst %.2e"
              % (med, errs[-1], med_stock, errs_stock[-1]))
        assert med < 3 * med_stock + 1e-3 and errs[-1] < 3 * errs_stock[-1] + 1e-2


@pytest.mark.parametrize("mode", ["fp32", "tf32", "tf32x3"])
def test_forward_multi_equals_separate_calls(mode):
    """Stacking the 3 DispResNet / 4 PoseResNet calls of a training step into one launch sequence must not change
    anything: per-call BatchNorm statistics, running-stat updates in call order, outputs, parameter gradients."""
    if True:
        imgs = [det_image(n, 2, 64, 96).to(DEV) for n in ("img1", "img2", "img3")]
        tol = 1e-5 if mode == "fp32" else 2e-5     # identical kernels and inputs; only atomics order differs
        for kind in ("disp", "pose"):
            a, b = _build(kind, 18, mode), _build(kind, 18, mode)
            a.train(); b.train()
            if kind == "disp":
                outs_a = [a(x) for x in imgs]
                outs_b = b.forward_multi(imgs)
                la = sum((1 / o[0]).mean() * (i + 1) for i, o in enumerate(outs_a))
                lb = sum((1 / o[0]).mean() * (i + 1) for i, o in enumerate(outs_b))
                for oa, ob in zip(outs_a, outs_b):
                    for s in range(4):
                        assert rel_l2(ob[s], oa[s]) < tol
            else:
                pairs = [(imgs[0], imgs[1]), (imgs[1], imgs[0]), (imgs[0], imgs[2]), (imgs[2], imgs[0])]
                outs_a = [a(x, y) for x, y in pairs]
                outs_b = b.forward_multi(pairs)
                wts = torch.arange(1, 7, device=DEV, dtype=torch.float32)
                la = sum((o * wts).sum() * (i + 1) for i, o in enumerate(outs_a)) * 100
                lb = sum((o * wts).sum() * (i + 1) for i, o in enumerate(outs_b)) * 100
                for oa, ob in zip(outs_a, outs_b):
                    assert rel_l2(ob, oa) < 10 * tol
            la.backward(); lb.backward()
            assert rel_l2(b.flat_grads(), a.flat_grads()) < (1e-4 if mode == "fp32" else 1e-3)
            sa, sb = a.state_dict(), b.state_dict()
            for k in sa:
                if "running" in k:
                    assert rel_l2(sb[k], sa[k]) < 1e-5, k
                if "num_batches_tracked" in k:
                    assert int(sa[k]) == int(sb[k]) == (3 if kind == "disp" else 4)


@pytest.mark.parametrize("mode", ["fp32", "tf32", "tf32x3"])
@pytest.mark.parametrize("shape", [(6, 4, 6, 64, 3), (6, 8, 12, 64, 3), (8, 16, 24, 128, 4), (3, 5, 7, 32, 3),
                                   (10, 8, 26, 64, 5), (16, 4, 13, 512, 8)])
def test_fused_batchnorm_sums_per_group(mode, shape):
    """Per-group BatchNorm partial sums out of the conv epilogue when several calls are stacked: groups whose
    row ranges straddle the 128-row (tensor-core) / 64-row (CUDA-core) tiles.  G=5 and G=8 are the DispResNet and PoseResNet
    group counts of a five-frame sequence (--sequence-length 5)."""
    O = _ops()
    B, H, W, C, G = shape
    cx = O.ConvCtx(mode)
    if True:
        g = torch.Generator().manual_seed(5)
        x = torch.randn(B, H, W, C, generator=g).to(DEV)
        w = (torch.randn(C, 3, 3, C, generator=g) / (9 * C) ** 0.5).to(DEV)
        sums = torch.zeros(O.BN_SLOTS * G * C * 2, device=DEV, dtype=torch.float64)
        y = cx.conv_fwd(x, w, None, 1, 1, O.PAD_ZERO, O.ACT_NONE, sums, G, O.split_tf32(w) if cx.split else None)
        got = sums.view(O.BN_SLOTS, G, C, 2).sum(0)
        yg = y.double().view(G, -1, C)
        np.testing.assert_allclose(got[..., 0].cpu(), yg.sum(1).cpu(), rtol=1e-5, atol=1e-4)
        np.testing.assert_allclose(got[..., 1].cpu(), (yg ** 2).sum(1).cpu(), rtol=1e-5, atol=1e-4)
