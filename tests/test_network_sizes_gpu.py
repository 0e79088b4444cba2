"""The networks at every image size and batch the scripts accept, against fp64, and the sizes refused before any launch.

Accepted DispResNet sizes other than multiples of 32 (H, W = 31 mod 32: 255x831, 95x127) run the stem on odd planes, stride-2
convolutions of odd inputs, max-pool on odd planes and a disparity one pixel larger than the image; PoseResNet takes any size and
runs odd planes at every level on raw KITTI frames (375x1242 -> 188x621 -> 94x311 -> 47x156 -> 24x78 -> 12x39).

Whole-network comparisons use the yardstick of test_nets_gpu.py: the relative L2 error that independent fp32 evaluations of the
same network make against fp64 -- the fp32 CPU oracle and stock PyTorch / cuDNN fp32 with TF32 off -- times 4, plus a floor.
Plain tf32 rounds every operand to 10 mantissa bits and is not an fp32 evaluation, so its bound is measured (TF32_EVAL).
Needs a GPU."""
import os

import numpy as np
import pytest
import torch

from golden_util import det_image, det_weights
from helpers import rel_l2
from test_infer_gpu import _bits_equal, _nontrivial_bn_state

pytestmark = pytest.mark.gpu
DEV = "cuda"

REFUSED = [(250, 832), (256, 830), (375, 1242), (30, 64)]
ODD_DISP = [(255, 831), (95, 127)]
RAW_KITTI = [(375, 1242), (370, 1226), (374, 1238), (376, 1241)]
# plain tf32 eval forwards against fp64, relative L2 of the output: about 3x the worst measured on an H100 80GB HBM3 (700 W),
# DispResNet-50 at 255x831 6.1e-3 (ResNet-18 1.3e-3), PoseResNet-50 at the raw KITTI sizes 6.1e-4 (ResNet-18 3.9e-4)
TF32_EVAL = {"disp": 2e-2, "pose": 2e-3}


@pytest.fixture(scope="module", autouse=True)
def _no_tf32_in_torch():
    """The cuDNN yardstick is fp32: TF32 off for torch's own convolutions while this module runs."""
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def _weights(kind, layers):
    import models
    net = models.DispResNet(layers, False) if kind == "disp" else models.PoseResNet(layers, False)
    net.load_state_dict(det_weights(net.state_dict()))
    _nontrivial_bn_state(net)
    return net.state_dict()


def _net(kind, layers, mode, sd=None):
    import models
    net = models.DispResNet(layers, False) if kind == "disp" else models.PoseResNet(layers, False)
    net.load_state_dict(sd if sd is not None else _weights(kind, layers))
    return net.to(DEV).set_conv_mode(mode)


def _oracle(kind, layers, sd, dtype, dev):
    from oracle import nets as ON
    ref = ON.DispResNet(layers) if kind == "disp" else ON.PoseResNet(layers)
    ref.load_state_dict({k: v.to(dtype) for k, v in sd.items()})
    return ref.to(dtype).to(dev)


YARD = (("fp64", torch.float64, DEV), ("cpu fp32", torch.float32, "cpu"), ("cudnn fp32", torch.float32, DEV))
_EVAL_CACHE = {}


def _oracle_eval(kind, layers, size, B):
    """{"fp64" | "cpu fp32" | "cudnn fp32": the oracle's eval output} on the seeded inputs of (kind, layers, size), batch B (eval
    mode: every image on its own, so B = 1 is the first image of B = 3)."""
    key = (kind, layers, size)
    if key not in _EVAL_CACHE:
        sd = _weights(kind, layers)
        H, W = size
        inputs = [det_image("%s%d" % (kind, i), 3, H, W) for i in range(1 if kind == "disp" else 2)]
        outs = {}
        for name, dtype, dev in YARD:
            ref = _oracle(kind, layers, sd, dtype, dev).eval()
            with torch.no_grad():
                outs[name] = ref(*[x.to(dtype).to(dev) for x in inputs]).double().cpu()
            del ref
        _EVAL_CACHE.clear()
        _EVAL_CACHE[key] = (sd, inputs, outs)
    sd, inputs, outs = _EVAL_CACHE[key]
    return sd, [x[:B] for x in inputs], {k: v[:B] for k, v in outs.items()}


def _check_eval(kind, layers, size, B, mode):
    from scsfm.infer import Predictor
    sd, inputs, want = _oracle_eval(kind, layers, size, B)
    net = _net(kind, layers, mode, sd).eval()
    got = Predictor(net)(*[x.to(DEV) for x in inputs]).double().cpu()
    err = rel_l2(got, want["fp64"])
    yard = max(rel_l2(want["cpu fp32"], want["fp64"]), rel_l2(want["cudnn fp32"], want["fp64"]))
    bound = TF32_EVAL[kind] if mode == "tf32" else 4 * yard + 1e-5
    print("%s%d %s B=%d %dx%d eval vs fp64: rel-L2 %.2e (fp32 yardstick %.2e, bound %.2e)" % (kind, layers, mode, B, *size, err,
                                                                                              yard, bound))
    assert err < bound
    return got


# --- refusals -----------------------------------------------------------------------------------------------------------
def test_disp_resnet_and_predictor_refuse_before_any_launch():
    """DispResNet eval, train and forward_multi, and the Predictor, refuse each size with ValueError and no launch; afterwards the
    same network computes bitwise what a fresh one does (eval forward, direct and through a Predictor) and the same train-mode
    forward and backward (up to the order of the BatchNorm batch-sum atomics)."""
    from scsfm import lib
    from scsfm.infer import Predictor
    sd = _weights("disp", 18)
    net, fresh = _net("disp", 18, "tf32x3", sd), _net("disp", 18, "tf32x3", sd)
    ok = det_image("ok", 2, 64, 96).to(DEV)
    pred = Predictor(net.eval())
    with torch.no_grad():
        pred(ok)
    n0 = lib.launch_count()
    for H, W in REFUSED:
        x = torch.zeros(1, 3, H, W, device=DEV)
        for training in (False, True):
            net.train(training)
            for grad in (False, True):
                with torch.set_grad_enabled(grad):
                    with pytest.raises(ValueError, match="image size %dx%d" % (H, W)):
                        net(x.clone().requires_grad_(grad))
                    with pytest.raises(ValueError, match="image size %dx%d" % (H, W)):
                        net.forward_multi([ok[:1], x])
        net.eval()
        with pytest.raises(ValueError, match="image size %dx%d" % (H, W)):
            pred(x)
        assert pred.num_graphs == 1
    assert lib.launch_count() == n0 and net._pending == 0
    with torch.no_grad():
        fresh.eval()
        assert _bits_equal(net(ok), fresh(ok)) and _bits_equal(pred(ok), fresh(ok))
    outs = []
    for n in (net, fresh):
        n.train()
        n.zero_grad()
        o = n(ok)
        sum(((1.0 / d) * (i + 1)).mean() for i, d in enumerate(o)).backward()
        outs.append((o[0].detach(), n.flat_grads().clone()))
    assert rel_l2(outs[0][0], outs[1][0]) < 1e-6 and rel_l2(outs[0][1], outs[1][1]) < 1e-5


def test_trainer_refuses_before_any_launch():
    """Trainer.step and Trainer.capture refuse the four sizes DispResNet refuses and 255x831 (accepted by DispResNet, but its
    disparity is 256x832) with ValueError before anything runs: no launch, no pending network call, no graph, the whole training
    state bit-identical to a fresh Trainer's; the next valid step computes what the fresh Trainer's does."""
    import models
    from scsfm import lib, synth
    from scsfm.trainer import Trainer
    from test_resume_gpu import assert_identical

    def make():
        d, p = models.DispResNet(18, False), models.PoseResNet(18, False)
        d.load_state_dict(_weights("disp", 18))
        p.load_state_dict(det_weights(p.state_dict()))
        return Trainer(d.to(DEV).train(), p.to(DEV).train(), lr=1e-4, with_auto_mask=1, distributed=False, conv_mode="tf32x3")
    tr, fresh = make(), make()
    tgt, refs, K = synth.triplet(3, 2, 64, 96)
    tgt, refs, K = tgt.to(DEV), [r.to(DEV) for r in refs], K.to(DEV)
    n0 = lib.launch_count()
    for H, W in REFUSED + [(255, 831)]:
        bad = torch.zeros(2, 3, H, W, device=DEV)
        for args in ((bad, [bad, bad]), (tgt, [refs[0], bad])) if (H, W) == (255, 831) else ((bad, [bad, bad]),):
            with pytest.raises(ValueError, match="image size %dx%d" % (H, W)):
                tr.step(*args, K)
            with pytest.raises(ValueError, match="image size %dx%d" % (H, W)):
                tr.capture(*args, K)
    assert lib.launch_count() == n0 and tr._graph is None
    assert tr.disp_net._pending == 0 and tr.pose_net._pending == 0
    assert_identical(tr.state_dict(), fresh.state_dict())
    a = torch.stack(tr.step(tgt, refs, K)).cpu()
    b = torch.stack(fresh.step(tgt, refs, K)).cpu()
    # (the pose gradient of the loss is reduced with fp32 atomics: one step is not bitwise repeatable)
    assert rel_l2(a, b) < 1e-5 and rel_l2(tr.disp_net.flat_params(), fresh.disp_net.flat_params()) < 1e-6


# --- accepted odd DispResNet sizes -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["fp32", "tf32x3", "tf32"])
@pytest.mark.parametrize("size", ODD_DISP)
@pytest.mark.parametrize("layers", [18, 50])
def test_disp_eval_at_odd_sizes_vs_fp64(layers, size, mode):
    """Predictor eval forward at B = 1 (the scripts' default): a [1,1,2 ceil(H/2),2 ceil(W/2)] disparity within the yardstick."""
    got = _check_eval("disp", layers, size, 1, mode)
    H, W = size
    assert got.shape == (1, 1, 2 * ((H + 1) // 2), 2 * ((W + 1) // 2))


def _train_grads(kind, net_or_ref, imgs, dtype, dev):
    """Train-mode forward and backward with test_nets_gpu.py's losses; {parameter name | "input k": gradient} and the outputs."""
    xs = [x.detach().to(dtype).to(dev).clone().requires_grad_(True) for x in imgs]
    net_or_ref.zero_grad()
    if kind == "disp":
        outs = net_or_ref(*xs)
        loss = sum(((1.0 / o) * (i + 1)).mean() for i, o in enumerate(outs))
    else:
        outs = [net_or_ref(*xs)]
        loss = (outs[0] * torch.arange(1, 7, dtype=outs[0].dtype, device=dev)).sum() * 100
    loss.backward()
    grads = {k: p.grad.double().cpu() for k, p in net_or_ref.named_parameters() if p.grad is not None}
    grads.update({"input %d" % i: x.grad.double().cpu() for i, x in enumerate(xs)})
    return grads, [o.detach().double().cpu() for o in outs]


# Train-mode inputs and the fp64 gradient's continuity.  These random-weight test networks have ReLU / max-pool decisions
# within fp32 rounding of a tie: there a perturbation of the image by 1e-6 relative moves the fp64 oracle's OWN gradients
# by up to 2e-2 in every encoder layer below the decision (DispResNet-18, 96x128, image "img1": 5e-3..9e-3 from the stem to
# layer3.0, 1e-5 in layer4 and the decoder), and any fp32 evaluation, this library or cuDNN, lands on one side or the
# other.  The "jump" of an input is the largest relative change of an fp64 gradient tensor under three such perturbations:
# 1e-5..2e-5 where the gradient is continuous, 3e-4..5e-2 across a decision.  Each case takes, of the candidate images, the
# one with the smallest jump.  Where it is continuous (jump <= STABLE) the yardstick is the fp32 evaluations alone, and the
# small cases must find such an input (strict).  Where every candidate jumps (every DispResNet-50 case, DispResNet-18 at
# 255x831, PoseResNet at 375x1242: many more decisions), the perturbed fp64 evaluations join the yardstick as further
# evaluations of the same network within fp32 noise.
CANDIDATES = ["train%d" % i for i in range(8)]
STABLE = 1e-4


def _least_jump_inputs(kind, layers, sd, B, H, W):
    """(name, inputs, fp64 (gradients, outputs), jump, fp64 gradients at each perturbation) of the candidate with the smallest
    jump; stops at the first continuous one."""
    ref = _oracle(kind, layers, sd, torch.float64, DEV).train()
    best, jumps = None, []
    for name in CANDIDATES:
        imgs = [det_image("%s%s%d" % (name, kind, i), B, H, W) for i in range(1 if kind == "disp" else 2)]
        g64 = _train_grads(kind, ref, imgs, torch.float64, DEV)
        moved, jump = [], 0.0
        for seed in range(3):
            g = torch.Generator().manual_seed(seed)
            xs = [x.double() * (1 + 1e-6 * torch.randn(x.shape, generator=g, dtype=torch.float64)) for x in imgs]
            moved.append(_train_grads(kind, ref, xs, torch.float64, DEV)[0])
            jump = max(jump, max(rel_l2(moved[-1][k], v) for k, v in g64[0].items()))
        jumps.append("%s %.1e" % (name, jump))
        if best is None or jump < best[3]:
            best = (name, imgs, g64, jump, moved)
        if jump <= STABLE:
            break
    print("%s%d %dx%d candidate jumps: %s" % (kind, layers, H, W, ", ".join(jumps)))
    return best


def _check_train(kind, layers, size, B, modes, strict=False):
    """Every parameter gradient and the input gradients (the stem's weight and data gradients on odd inputs, max-pool backward on
    odd planes) against fp64, median and worst relative L2 per tensor against the yardstick (test_nets_gpu.py; see above)."""
    import models
    net0 = models.DispResNet(layers, False) if kind == "disp" else models.PoseResNet(layers, False)
    sd = det_weights(net0.state_dict())
    H, W = size
    name, imgs, (g64, o64), jump, moved = _least_jump_inputs(kind, layers, sd, B, H, W)
    assert jump <= STABLE or not strict, "no candidate input with a continuous fp64 gradient (smallest jump %.1e)" % jump
    ref = {}
    for yname, dtype, dev in YARD[1:]:
        r = _oracle(kind, layers, sd, dtype, dev).train()
        ref[yname] = _train_grads(kind, r, imgs, dtype, dev)
        del r
    others = [ref[n][0] for n in ("cpu fp32", "cudnn fp32")] + (moved if jump > STABLE else [])
    yard = [sorted(rel_l2(gr[k], g) for k, g in g64.items()) for gr in others]
    yard_med, yard_worst = max(y[len(y) // 2] for y in yard), max(y[-1] for y in yard)
    yard_out = max(rel_l2(ref[n][1][0], o64[0]) for n in ("cpu fp32", "cudnn fp32"))
    for mode in modes:
        net = _net(kind, layers, mode, sd).train()
        grads, outs = _train_grads(kind, net, imgs, torch.float32, DEV)
        if kind == "disp":
            assert [tuple(o.shape) for o in outs] == [(B, 1, 2 * ((H + 1) // 2) >> s, 2 * ((W + 1) // 2) >> s) for s in range(4)]
        # the parameters the reference leaves without a gradient (the unused fc head) keep an exactly zero one here
        assert set(g64) <= set(grads) and all(float(grads[k].abs().max()) == 0 for k in set(grads) - set(g64))
        errs = sorted((rel_l2(grads[k], g), k) for k, g in g64.items())
        med, worst = errs[len(errs) // 2][0], errs[-1]
        inp = max(rel_l2(grads[k], g64[k]) for k in g64 if k.startswith("input"))
        out = rel_l2(outs[0], o64[0])
        print("%s%d %s B=%d %dx%d train vs fp64 (input %s, jump %.1e): output %.2e (yardstick %.2e); gradient rel-L2 "
              "median %.2e worst %.2e (%s), input %.2e; yardstick median %.2e worst %.2e"
              % (kind, layers, mode, B, H, W, name, jump, out, yard_out, med, worst[0], worst[1], inp, yard_med, yard_worst))
        assert out < 4 * yard_out + 1e-5
        assert med < 4 * yard_med + 1e-4 and worst[0] < 4 * yard_worst + 3e-3
        del net


@pytest.mark.parametrize("size", ODD_DISP + [(96, 128)])
@pytest.mark.parametrize("layers", [18, 50])
def test_disp_train_at_odd_sizes_vs_fp64(layers, size):
    """255x831 and 95x127, and 96x128, a training size whose encoder planes are those of 95x127."""
    _check_train("disp", layers, size, 2, ("fp32", "tf32x3"), strict=layers == 18 and size != (255, 831))


def test_gradient_jump_at_a_near_tie_is_the_networks_own():
    """The evidence for the input choice above, kept as a test: at DispResNet-18, 96x128, image "img1", the fp64 oracle's gradients
    jump under a 1e-6 relative perturbation of the image, below a decision in the encoder (stem through layer3.0) and not in the
    decoder.  (This library's fp32 gradients there land on the perturbed side: printed, not asserted, since which side an fp32
    evaluation lands on is not part of its contract.)"""
    import models
    sd = det_weights(models.DispResNet(18, False).state_dict())
    imgs = [det_image("img1", 2, 96, 128)]
    ref = _oracle("disp", 18, sd, torch.float64, DEV).train()
    g64 = _train_grads("disp", ref, imgs, torch.float64, DEV)[0]
    g = torch.Generator().manual_seed(1)
    moved = [imgs[0].double() * (1 + 1e-6 * torch.randn(imgs[0].shape, generator=g, dtype=torch.float64))]
    gp = _train_grads("disp", ref, moved, torch.float64, DEV)[0]
    ours = _train_grads("disp", _net("disp", 18, "fp32", sd).train(), imgs, torch.float32, DEV)[0]

    def worst(gr, prefix):
        return max(rel_l2(gr[k], g64[k]) for k in g64 if k.startswith(prefix))
    for who, gr in (("fp64 perturbed", gp), ("ours", ours)):
        enc, l4, dec = worst(gr, "encoder.encoder.conv1"), worst(gr, "encoder.encoder.layer4"), worst(gr, "decoder")
        print("%s vs fp64 at 96x128 img1: stem %.1e, layer4 %.1e, decoder %.1e" % (who, enc, l4, dec))
        if who == "fp64 perturbed":
            assert enc > 1e-3 and l4 < 1e-4 and dec < 1e-4


# --- PoseResNet on raw KITTI frames ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("size", RAW_KITTI)
@pytest.mark.parametrize("layers", [18, 50])
def test_pose_eval_at_raw_kitti_sizes_vs_fp64(layers, size, B):
    for mode in ("fp32", "tf32x3", "tf32"):
        got = _check_eval("pose", layers, size, B, mode)
        assert got.shape == (B, 6)


@pytest.mark.parametrize("size", [(375, 1242), (75, 109)])
def test_pose_train_at_odd_sizes_vs_fp64(size):
    """A raw KITTI frame, and 75x109 (38x55 -> 19x28 -> 10x14 -> 5x7 -> 3x4: odd planes at most levels), small enough for a
    continuous fp64 gradient."""
    _check_train("pose", 18, size, 2, ("fp32", "tf32x3"), strict=size == (75, 109))


# --- more shapes than graphs ----------------------------------------------------------------------------------------------
def test_predictor_cycles_more_shapes_than_graphs():
    """run_inference.py --no-resize on mixed sizes: six accepted shapes twice through Predictor(max_graphs=4).  LRU eviction
    recaptures every shape each time round (12 captures), at most 4 graphs are kept, every output is bitwise net(x)."""
    from scsfm.infer import Predictor
    net = _net("disp", 18, "tf32x3").eval()
    pred = Predictor(net, max_graphs=4)
    shapes = [(1, 256, 832), (1, 255, 831), (2, 95, 127), (1, 64, 64), (1, 63, 95), (3, 128, 160)]
    for rnd in range(2):
        for i, (B, H, W) in enumerate(shapes):
            x = det_image("cyc%d" % i, B, H, W).to(DEV)
            got = pred(x)
            assert pred.num_graphs <= 4
            with torch.no_grad():
                assert _bits_equal(got, net(x)), (B, H, W)
            assert got.shape == (B, 1, 2 * ((H + 1) // 2), 2 * ((W + 1) // 2))
    assert pred.captures == 12 and pred.num_graphs == 4


# --- run_inference.py --no-resize -----------------------------------------------------------------------------------------
def test_run_inference_no_resize_mixed_sizes(tmp_path):
    """A folder with a 256x832 and a 255x831 frame: the saved images are those of per-image Predictor calls; with a 375x1242 frame
    added the script raises the size error (the reference's torch.cat fails there too)."""
    import run_inference
    from PIL import Image
    from scsfm import inference_io as io
    from scsfm.infer import Predictor
    rng = np.random.default_rng(3)
    d = tmp_path / "imgs"
    d.mkdir()
    for name, (H, W) in (("a", (256, 832)), ("b", (255, 831))):
        Image.fromarray(rng.integers(0, 256, (H, W, 3)).astype(np.uint8)).save(d / (name + ".png"))
    sd = _weights("disp", 18)
    torch.save({"epoch": 1, "state_dict": sd}, tmp_path / "disp.pth.tar")
    argv = ["--output-disp", "--output-depth", "--no-resize", "--pretrained", str(tmp_path / "disp.pth.tar"), "--dataset-dir",
            str(d), "--output-dir", str(tmp_path / "out"), "--resnet-layers", "18", "--batch-size", "2"]
    run_inference.main(argv)
    pred = Predictor(_net("disp", 18, "tf32x3", sd).eval())
    for name in ("a", "b"):
        fr = io.load_frame(str(d / (name + ".png")), 256, 832, False)
        out = pred(io.network_input(fr[None]))[0].cpu().numpy()[0]
        assert out.shape == (256, 832)
        for suffix, want in (("disp", io.colorize(out, out.max(), "bone")), ("depth", io.colorize(1 / out, 10, "rainbow"))):
            saved = np.asarray(Image.open(tmp_path / "out" / ("%s_%s.png" % (name, suffix))))
            assert np.array_equal(saved, (255 * want).astype(np.uint8)), (name, suffix)
    Image.fromarray(rng.integers(0, 256, (375, 1242, 3)).astype(np.uint8)).save(d / "c.png")
    with pytest.raises(ValueError, match="image size 375x1242"):
        run_inference.main(argv)
    assert sorted(os.listdir(tmp_path / "out")) == ["a_depth.png", "a_disp.png", "b_depth.png", "b_disp.png"]
