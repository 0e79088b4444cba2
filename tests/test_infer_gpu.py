"""Eval-mode inference: BatchNorm fused into the convolution epilogues, the no-record eval forward of the networks and the
graph-captured Predictor.  The fused paths repeat bn_apply's arithmetic after the same convolution main loops, so every
comparison with the recording eval path is bitwise.  Needs a GPU."""
import os

import numpy as np
import pytest
import torch

from golden_util import det_image, det_weights
from helpers import rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _O():
    from scsfm import nnops
    return nnops


class _BN:
    """Non-trivial eval-mode BatchNorm state of C channels."""

    def __init__(self, C, seed):
        g = torch.Generator().manual_seed(seed)
        self.weight = (1 + 0.3 * torch.randn(C, generator=g)).to(DEV)
        self.bias = (0.2 * torch.randn(C, generator=g)).to(DEV)
        self.running_mean = (0.3 * torch.randn(C, generator=g)).to(DEV)
        self.running_var = (0.5 + 1.5 * torch.rand(C, generator=g)).to(DEV)


def _nontrivial_bn_state(net, seed=5):
    from scsfm import nets as N
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in net.modules():
            if isinstance(m, N.BNParams):
                C = m.weight.numel()
                m.weight.copy_(1 + 0.3 * torch.randn(C, generator=g))
                m.bias.copy_(0.2 * torch.randn(C, generator=g))
                m.running_mean.copy_(0.3 * torch.randn(C, generator=g))
                m.running_var.copy_(0.5 + 1.5 * torch.rand(C, generator=g))


def _bits_equal(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


# B, H, W, Cin, Cout, k, stride, pad, pad_mode, mode, tune kwargs
KCASES = [
    # persistent TMA kernel: 3x3 / 1x1 stride 1, 128- and 256-pixel tiles, weight tiles of 16..128 rows, partial tiles
    (2, 19, 37, 64, 64, 3, 1, 1, 0, "tf32x3", dict(mt=1, bn=64)),
    (2, 19, 37, 64, 64, 3, 1, 1, 0, "tf32", dict(mt=2, bn=64)),
    (1, 21, 29, 32, 16, 3, 1, 1, 0, "tf32x3", dict(mt=2, bn=16)),
    (1, 21, 29, 32, 32, 3, 1, 1, 0, "tf32", dict(mt=1, bn=32)),
    (2, 11, 27, 128, 256, 3, 1, 1, 0, "tf32x3", dict(mt=1, bn=128)),
    (2, 13, 23, 256, 128, 1, 1, 0, 0, "tf32", dict(mt=1, bn=128)),
    (1, 13, 23, 64, 256, 1, 1, 0, 0, "tf32x3", {}),
    (2, 16, 52, 256, 64, 1, 1, 0, 0, "tf32x3", dict(mt=2)),
    # cp.async gather kernel: stride 2 (STACK in split mode for Cout <= 64), the padded 7x7 stems, STACK off
    (2, 20, 36, 64, 128, 3, 2, 1, 0, "tf32x3", {}),
    (2, 20, 36, 64, 64, 3, 2, 1, 0, "tf32x3", {}),
    (2, 20, 36, 64, 64, 3, 2, 1, 0, "tf32", {}),
    (2, 20, 36, 64, 256, 1, 2, 0, 0, "tf32x3", {}),
    (2, 34, 50, 4, 64, 7, 2, 3, 0, "tf32x3", {}),
    (2, 34, 50, 8, 64, 7, 2, 3, 0, "tf32", {}),
    (1, 34, 50, 8, 64, 7, 2, 3, 0, "tf32x3", dict(no_tma=1)),
    # the reflection border ring (TMA interior with zero padding + the gather kernel's border view), and gather-only reflection
    (1, 18, 30, 32, 32, 3, 1, 1, 1, "tf32x3", dict(mt=1)),
    (2, 18, 30, 64, 128, 3, 1, 1, 1, "tf32", dict(mt=1)),
    (1, 18, 30, 32, 16, 3, 1, 1, 1, "tf32x3", {}),
    # CUDA-core kernel (fp32 mode), every tile shape and the 3-channel stem
    (2, 17, 25, 64, 64, 3, 1, 1, 0, "fp32", {}),
    (2, 17, 25, 64, 32, 3, 2, 1, 0, "fp32", {}),
    (2, 17, 25, 32, 16, 1, 1, 0, 0, "fp32", {}),
    (2, 34, 50, 3, 64, 7, 2, 3, 0, "fp32", {}),
]
EPI = [(False, False, False), (True, True, False), (False, True, True), (True, False, True)]      # (residual, ReLU, ROUND_TF32)


@pytest.mark.parametrize("case", KCASES)
def test_conv_fused_bn_equals_conv_then_bn_apply(case):
    O = _O()
    B, H, W, Cin, Cout, k, stride, pad, pad_mode, mode, knobs = case
    g = torch.Generator().manual_seed(B * 1000 + H * 10 + Cin + Cout + k)
    x = torch.randn(B, H, W, Cin, generator=g).to(DEV)
    w = (torch.randn(Cout, k, k, Cin, generator=g) / (k * k * Cin) ** 0.5).to(DEV)
    cx = O.ConvCtx(mode)
    cx.tune = O.tune(**knobs)
    w_lo = O.split_tf32(w) if cx.split else None
    bn = _BN(Cout, Cout + k)
    tab = O.BnEvalTable([bn], 1e-5)
    tab.prepare()
    sc, sh = tab.coeffs[0]
    for res_on, relu, rnd in EPI:
        y = cx.conv_fwd(x, w, None, stride, pad, pad_mode, O.ACT_NONE, None, 1, w_lo)
        res = torch.randn(y.shape, generator=g).to(DEV) if res_on else None
        flags = (1 if relu else 0) | (O.ROUND_TF32 if rnd else 0)
        z, saved = O.bn_apply(y, None, bn.weight, bn.bias, bn.running_mean, bn.running_var, 0.1, 1e-5, res, flags, 1, with_lo=True)
        act = (O.ACT_RELU if relu else O.ACT_NONE) | (O.ROUND_TF32 if rnd else 0)
        zf = cx.conv_fwd(x, w, None, stride, pad, pad_mode, act, None, 1, w_lo, bn_scale=sc, bn_shift=sh, addend=res, with_lo=True)
        torch.cuda.synchronize()
        assert _bits_equal(sc, saved[0, :, 0]) and _bits_equal(sh, saved[0, :, 1])      # one per-channel expression
        assert _bits_equal(zf, z), (case, res_on, relu, rnd, float((zf - z).abs().max()))
        assert _bits_equal(zf._scsfm_lo, z._scsfm_lo)
        assert _bits_equal(zf._scsfm_lo, O.split_tf32(zf))
    # (the eval BatchNorm changed the values: the comparison is not trivially between two plain convolutions)
    assert float((zf - cx.conv_fwd(x, w, None, stride, pad, pad_mode, act, None, 1, w_lo)).abs().max()) > 0


def test_fused_bn_refuses_bias_and_batch_sums():
    O = _O()
    x = torch.randn(1, 8, 8, 16, device=DEV)
    w = torch.randn(32, 3, 3, 16, device=DEV)
    bn = _BN(32, 1)
    tab = O.BnEvalTable([bn], 1e-5)
    sc, sh = tab.coeffs[0]
    bias = torch.zeros(32, device=DEV)
    sums = torch.zeros(O.BN_SLOTS * 32 * 2, device=DEV, dtype=torch.float64)
    for mode in ("fp32", "tf32"):
        cx = O.ConvCtx(mode)
        with pytest.raises(ValueError, match="excludes bias"):
            cx.conv_fwd(x, w, bias, 1, 1, bn_scale=sc, bn_shift=sh)
        with pytest.raises(ValueError, match="excludes bias"):
            cx.conv_fwd(x, w, None, 1, 1, bn_sums=sums, bn_scale=sc, bn_shift=sh)


def _build(kind, layers, mode):
    import models
    net = models.DispResNet(layers, False) if kind == "disp" else models.PoseResNet(layers, False)
    net.load_state_dict(det_weights(net.state_dict()))
    _nontrivial_bn_state(net)
    return net.to(DEV).set_conv_mode(mode).eval()


def _oracle_eval(kind, layers, net, imgs):
    from oracle import nets as ON
    ref = (ON.DispResNet(layers) if kind == "disp" else ON.PoseResNet(layers)).double().to(DEV)
    ref.load_state_dict({k: v.double() for k, v in net.state_dict().items()})
    ref.eval()
    with torch.no_grad():
        return ref(*[i.double().to(DEV) for i in imgs])


NET_CASES = ([(kind, layers, mode, 2, 64, 160) for kind in ("disp", "pose") for layers in (18, 50) for mode in ("fp32", "tf32", "tf32x3")] +
             [("disp", 18, "tf32x3", 4, 256, 832), ("pose", 18, "tf32x3", 4, 256, 832)])


@pytest.mark.parametrize("kind,layers,mode,B,H,W", NET_CASES)
def test_fused_eval_forward_equals_recording_eval(kind, layers, mode, B, H, W):
    net = _build(kind, layers, mode)
    imgs = [det_image("inf1", B, H, W)] + ([det_image("inf2", B, H, W)] if kind == "pose" else [])
    dimgs = [i.to(DEV) for i in imgs]
    with torch.enable_grad():
        rec = net(*dimgs).detach()            # eval mode with autograd on: the recording path (conv, then bn_apply)
    with torch.no_grad():
        fused = net(*dimgs)
    torch.cuda.synchronize()
    assert _bits_equal(fused, rec), (kind, layers, mode, float((fused - rec).abs().max()))
    want = _oracle_eval(kind, layers, net, imgs)
    err = rel_l2(fused, want)
    assert err < (1e-2 if mode == "tf32" else 1e-4), err
    if mode != "tf32":
        np.testing.assert_allclose(fused.cpu().numpy(), want.cpu().numpy(), rtol=2e-3, atol=5e-5)


def test_predictor_replays_track_state():
    from scsfm.infer import Predictor
    from scsfm import nets as N
    net = _build("disp", 18, "tf32x3")
    pred = Predictor(net)
    x = det_image("pred", 2, 128, 416).to(DEV)

    def eager():
        with torch.no_grad():
            return net(x).clone()

    a, b = pred(x), pred(x)
    assert _bits_equal(a, eager()) and _bits_equal(a, b) and pred.captures == 1
    assert a.shape == (2, 1, 128, 416)
    assert a.data_ptr() != pred(x).data_ptr()
    x2 = det_image("pred2", 1, 64, 192).to(DEV)
    c = pred(x2)
    assert pred.captures == 2 and c.shape == (1, 1, 64, 192)
    with torch.no_grad():
        assert _bits_equal(c, net(x2))
    # ArenaAdam step (raw-pointer writes of parameters and operand mirror)
    net.train()
    out = net(x)
    sum((1.0 / o).mean() for o in out).backward()      # training forward: moves the running statistics too
    N.ArenaAdam([net], lr=1e-3).step()
    net.eval()
    assert _bits_equal(pred(x), eager())
    # torch.optim.Adam on the parameters
    net.train()
    out = net(x)
    sum((1.0 / o).mean() for o in out).backward()
    torch.optim.Adam(net.parameters(), lr=1e-3).step()
    net.eval()
    assert _bits_equal(pred(x), eager())
    # load_state_dict
    sd = {k: v.clone() for k, v in net.state_dict().items()}
    for k in sd:
        if k.endswith("running_mean"):
            sd[k] += 0.05
    net.load_state_dict(sd)
    assert _bits_equal(pred(x), eager())
    # training-mode forward alone (running statistics move)
    net.train()
    with torch.no_grad():
        net(x)
    net.eval()
    assert _bits_equal(pred(x), eager())
    # set_conv_mode replaces the context: a new graph
    n0 = pred.captures
    net.set_conv_mode("tf32")
    y = pred(x)
    assert pred.captures == n0 + 1 and _bits_equal(y, eager())
    assert pred.num_graphs <= pred.max_graphs
    with pytest.raises(RuntimeError):
        net.train()
        pred(x)


def test_predictor_pose_and_batching():
    from scsfm.infer import Predictor
    net = _build("pose", 18, "tf32x3")
    N_ = 6
    a, b = det_image("pa", N_, 256, 832).to(DEV), det_image("pb", N_, 256, 832).to(DEV)
    pred = Predictor(net)
    batched = pred(a, b)
    assert batched.shape == (N_, 6)
    with torch.no_grad():
        assert _bits_equal(batched, net(a, b))
    single = torch.cat([pred(a[i:i + 1], b[i:i + 1]) for i in range(N_)])
    err = float(((batched - single).abs() / single.abs().clamp_min(1e-30)).max())
    print("PoseResNet18 tf32x3: %d pairs in one batch vs %d calls at B=1: bitwise equal %s, max relative difference %.3e"
          % (N_, N_, _bits_equal(batched, single), err))
    assert rel_l2(batched, single) <= 1e-6


def test_no_grad_eval_peak_memory():
    net = _build("disp", 18, "tf32x3")
    x = det_image("mem", 4, 256, 832).to(DEV)
    peaks = {}
    for name, ctx in (("recording", torch.enable_grad), ("fused", torch.no_grad)):
        with ctx():
            net(x)             # warm-up (tables, mirrors)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        with ctx():
            out = net(x)
        torch.cuda.synchronize()
        peaks[name] = torch.cuda.max_memory_allocated() - base
        del out
    ratio = peaks["fused"] / peaks["recording"]
    print("DispResNet18 tf32x3 B=4 256x832 eval peak allocation: recording %.1f MB, fused no-grad %.1f MB, ratio %.3f"
          % (peaks["recording"] / 2 ** 20, peaks["fused"] / 2 ** 20, ratio))
    assert ratio <= 0.5


# --- the inference scripts end to end ----------------------------------------------------------------------------------
def _script_fixture(tmp_path):
    """A folder of PNGs at 256x832 plus one 375x1242 frame (resized by the scripts), and checkpoints saved as train.py
    saves them ({'epoch', 'state_dict'})."""
    import models
    from PIL import Image
    rng = np.random.default_rng(1)
    seq = tmp_path / "seqs" / "05" / "image_2"
    seq.mkdir(parents=True)
    base = np.kron(rng.integers(30, 226, (30, 90, 3)), np.ones((16, 16, 1)))
    names = []
    for i in range(5):
        im = np.clip(base[:256, 3 * i:3 * i + 832] + rng.normal(0, 5, (256, 832, 3)), 0, 255).astype(np.uint8)
        Image.fromarray(im).save(seq / ("%06d.png" % i))
        names.append(seq / ("%06d.png" % i))
    Image.fromarray(base[:375, :1242].astype(np.uint8)).save(seq / "000005.png")      # base is 480 x 1440
    names.append(seq / "000005.png")
    disp, pose = models.DispResNet(18, False), models.PoseResNet(18, False)
    disp.load_state_dict(det_weights(disp.state_dict()))
    pose.load_state_dict(det_weights(pose.state_dict()))
    _nontrivial_bn_state(disp)
    _nontrivial_bn_state(pose)
    torch.save({"epoch": 1, "state_dict": disp.state_dict()}, tmp_path / "dispnet_checkpoint.pth.tar")
    torch.save({"epoch": 1, "state_dict": pose.state_dict()}, tmp_path / "exp_pose_checkpoint.pth.tar")
    return seq, names, disp, pose


def _oracle_input(path):
    from scsfm import inference_io as io
    fr = io.load_frame(str(path), 256, 832).astype(np.float64)
    return ((torch.from_numpy(fr).permute(2, 0, 1)[None] / 255 - 0.45) / 0.225)


def test_scripts_end_to_end(tmp_path, capsys):
    import test_disp
    import run_inference
    import test_vo
    from oracle import nets as ON
    seq, names, disp, pose = _script_fixture(tmp_path)
    # test_disp.py: predictions.npy = 1/disp, per image within 1e-4 of the fp64 oracle
    test_disp.main(["--pretrained-dispnet", str(tmp_path / "dispnet_checkpoint.pth.tar"), "--dataset-dir", str(seq),
                    "--output-dir", str(tmp_path / "out"), "--resnet-layers", "18", "--batch-size", "2"])
    text = capsys.readouterr().out
    assert "Avg Time: " in text and "Avg Speed: " in text and "6 files to test" in text
    preds = np.load(tmp_path / "out" / "predictions.npy")
    assert preds.shape == (6, 256, 832) and preds.dtype == np.float64
    ref = ON.DispResNet(18).double().to(DEV)
    ref.load_state_dict({k: v.double() for k, v in disp.state_dict().items()})
    ref.eval()
    with torch.no_grad():
        for j, p in enumerate(names):
            want = 1 / ref(_oracle_input(p).to(DEV))[0, 0].cpu().numpy()
            assert rel_l2(preds[j], want) < 1e-4, (j, rel_l2(preds[j], want))
    # run_inference.py: the reference's output names
    run_inference.main(["--output-disp", "--output-depth", "--pretrained", str(tmp_path / "dispnet_checkpoint.pth.tar"),
                        "--dataset-dir", str(seq), "--output-dir", str(tmp_path / "vis"), "--resnet-layers", "18"])
    got = sorted(os.listdir(tmp_path / "vis"))
    assert got == sorted(["%06d_%s.png" % (i, k) for i in range(6) for k in ("disp", "depth")])
    from PIL import Image
    assert Image.open(tmp_path / "vis" / "000000_disp.png").size == (832, 256)
    # test_vo.py: trajectory vs a numpy restatement of the reference loop driven by oracle poses
    test_vo.main(["--pretrained-posenet", str(tmp_path / "exp_pose_checkpoint.pth.tar"), "--dataset-dir", str(tmp_path / "seqs") + "/",
                  "--output-dir", str(tmp_path / "vo") + "/", "--sequence", "05", "--batch-size", "3"])
    traj = np.loadtxt(tmp_path / "vo" / "05.txt")
    assert traj.shape == (6, 12)
    oref = ON.PoseResNet(18).double().to(DEV)
    oref.load_state_dict({k: v.double() for k, v in pose.state_dict().items()})
    oref.eval()
    from oracle import geometry as OG
    g, want = np.eye(4), [np.eye(4)[:3].reshape(12)]
    with torch.no_grad():
        for i in range(5):
            vec = oref(_oracle_input(names[i]).to(DEV), _oracle_input(names[i + 1]).to(DEV)).cpu()
            m = OG.pose_to_matrix(vec, "euler")[0].numpy()
            g = g @ np.linalg.inv(np.vstack([m, [0, 0, 0, 1]]))
            want.append(g[:3].reshape(12))
    err = rel_l2(traj, np.stack(want))
    print("test_vo trajectory vs fp64 oracle poses: rel-L2 %.2e" % err)
    assert err < 1e-4
