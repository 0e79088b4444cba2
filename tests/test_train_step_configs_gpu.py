"""The whole training step (train.py:259-282) against the fp64 oracle in the configurations train.py accepts beyond the
benchmarked one: several scales (a partial set of disparity heads), the loss switches, border padding, five-frame sequences
(BatchNorm groups of 5 and 8, the loss split over two launches), other loss weights, weight decay and betas, and DispResNet-50.

Each configuration runs two eager steps on a fresh Trainer and two steps replayed from the CUDA graph of a second Trainer built
the same way.  Step 1 is compared with one oracle step: the losses, every parameter gradient, the BatchNorm state, and the
parameters the oracle leaves without a gradient.  Every step, eager or replayed, is compared with an fp64 Adam update recomputed
from the gradient the step left behind, so an update that read a partial or stale gradient shows.  Needs a GPU."""
import math

import numpy as np
import pytest
import torch

from golden_util import det_weights
from helpers import Adam64, assert_adam_change, oracle_train_step, rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda"
SEED = 2024
EPS = 1e-8          # ArenaAdam's and torch.optim.Adam's default

# train.py's defaults at 128x416 (flags = with_ssim, with_mask, with_auto_mask; weights = -p, -s, -c)
BASE = dict(disp_layers=18, pose_layers=18, mode="tf32x3", B=2, H=128, W=416, kind="kitti", n_ref=2, num_scales=1,
            flags=(1, 1, 1), padding="zeros", weights=(1.0, 0.1, 0.5), lr=1e-4, weight_decay=0.0, betas=(0.9, 0.999))
CONFIGS = {
    "scales2": dict(num_scales=2),                                               # heads 0-1 live, 2-3 unused
    "scales4": dict(num_scales=4, flags=(1, 1, 0)),                              # every head in the step
    "scales4_fp32": dict(num_scales=4, flags=(1, 1, 0), mode="fp32"),
    "seq5_scales3": dict(n_ref=4, num_scales=3),                                 # G=5 / G=8 calls, 24 pair-directions
    "pair_nyu_scales2_border": dict(B=1, H=128, W=160, kind="nyu", n_ref=1, num_scales=2, padding="border"),
    "plain": dict(flags=(0, 0, 0)),
    "mask_only_border": dict(flags=(0, 1, 0), padding="border"),
    "ssim_automask_border": dict(flags=(1, 0, 1), padding="border"),
    "no_smooth": dict(weights=(0.7, 0.0, 1.3)),
    "no_geometry_fp32": dict(weights=(1.0, 0.3, 0.0), mode="fp32"),
    "wd_betas": dict(weight_decay=1e-2, betas=(0.8, 0.99)),                      # --wd, --momentum, --beta
    "r50_scales2": dict(disp_layers=50, num_scales=2),                           # train.py --resnet-layers 50
}


@pytest.fixture(scope="module")
def tf32_off():
    """The fp32 GPU oracle is stock PyTorch / cuDNN with TF32 off; the flags are restored after the module."""
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def _step_kwargs(c):
    ssim, mask, auto = c["flags"]
    w1, w2, w3 = c["weights"]
    return dict(num_scales=c["num_scales"], with_ssim=ssim, with_mask=mask, with_auto_mask=auto, padding_mode=c["padding"],
                w1=w1, w2=w2, w3=w3)


def _trainer(c):
    import models
    from scsfm.trainer import Trainer
    disp, pose = models.DispResNet(c["disp_layers"], False), models.PoseResNet(c["pose_layers"], False)
    for net in (disp, pose):
        net.load_state_dict(det_weights(net.state_dict()))
    return Trainer(disp.to(DEV).train(), pose.to(DEV).train(), lr=c["lr"], betas=c["betas"], weight_decay=c["weight_decay"],
                   distributed=False, conv_mode=c["mode"], **_step_kwargs(c))


def _two_steps(c, args, captured):
    """Two steps of a fresh Trainer, eager or replayed from its captured graph.  Keeps the arenas before and after every step,
    the gradient arenas each step left, and after step 1 every parameter gradient and the BatchNorm buffers; counts the
    photometric / geometry loss launches of the eager steps."""
    from scsfm import lib as L
    tr = _trainer(c)
    if captured:
        tr.capture(*args)
    nets = {"disp": tr.disp_net, "pose": tr.pose_net}
    r = {"losses": [], "params": [{k: n.flat_params().clone() for k, n in nets.items()}], "grads": [], "pair_fwd": []}
    for t in range(2):
        prof = dict(L.PROF)
        if not captured:
            L.PROF.update(enabled=True, only={"pair_fwd"}, events=[])
        try:
            losses = tr.step(*args)
            r["pair_fwd"].append(len(L.PROF["events"]) if not captured else None)
        finally:
            L.PROF.update(prof)
        r["losses"].append([float(v) for v in losses])
        r["grads"].append({k: n.flat_grads().clone() for k, n in nets.items()})
        r["params"].append({k: n.flat_params().clone() for k, n in nets.items()})
        if t == 0:
            r["param_grads"] = {k + "." + name: q.grad.clone().cpu() for k, n in nets.items() for name, q in n.named_parameters()}
            r["buffers"] = {k + "." + name: b.clone().cpu() for k, n in nets.items() for name, b in n.named_buffers()}
    # where every parameter lies in its network's arena
    r["slices"] = {}
    for k, n in nets.items():
        base = n.flat_params().data_ptr()
        for name, q in n.named_parameters():
            r["slices"][k + "." + name] = (k, (q.data_ptr() - base) // 4, q.numel())
    # the parameters of each disparity head
    d = tr.disp_net
    ids = {id(q): "disp." + name for name, q in d.named_parameters()}
    r["heads"] = [[ids[id(d.decoder.disp(s).weight)], ids[id(d.decoder.disp(s).bias)]] for s in range(4)]
    return r


@pytest.fixture(scope="module", params=list(CONFIGS))
def run(request, tf32_off):
    """One configuration: its three oracle steps and the eager and captured Trainer runs (module scope: pytest runs every test
    of one configuration before building the next)."""
    from scsfm import synth
    name = request.param
    c = BASE | CONFIGS[name]
    tgt, refs, K = synth.triplet(SEED, c["B"], c["H"], c["W"], c["n_ref"], c["kind"])
    oracle = oracle_train_step(tgt, refs, K, disp_layers=c["disp_layers"], pose_layers=c["pose_layers"], lr=c["lr"],
                               betas=c["betas"], weight_decay=c["weight_decay"], gpu=DEV, **_step_kwargs(c))
    args = (tgt.to(DEV), [r.to(DEV) for r in refs], K.to(DEV))
    out = dict(name=name, cfg=c, oracle=oracle, eager=_two_steps(c, args, False), captured=_two_steps(c, args, True))
    yield out
    out.clear()
    torch.cuda.empty_cache()


def test_losses_match_fp64(run):
    """Check 1: the four losses of step 1 (the initial weights) against the fp64 oracle."""
    np.testing.assert_allclose(run["eager"]["losses"][0], run["oracle"]["f64"][0], rtol=1e-4, atol=1e-6)


def test_gradients_match_fp64(run):
    """Check 2: every parameter gradient of both networks after step 1 against fp64, per tensor by relative L2.  Yardstick:
    the larger error of two independent fp32 evaluations (the CPU oracle and stock PyTorch / cuDNN with TF32 off on this GPU)."""
    want64, g64, _ = run["oracle"]["f64"]
    g32, g32gpu = run["oracle"]["f32"][1], run["oracle"]["f32gpu"][1]
    got, grads = run["eager"]["losses"][0], run["eager"]["param_grads"]
    mine = sorted((rel_l2(grads[k], g64[k]), k) for k in g64)
    ref = sorted(rel_l2(g32[k], g64[k]) for k in g64)
    refg = sorted(rel_l2(g32gpu[k], g64[k]) for k in g64)
    med, worst = mine[len(mine) // 2][0], mine[-1]
    rmed, rworst = max(ref[len(ref) // 2], refg[len(refg) // 2]), max(ref[-1], refg[-1])
    lerr = max(abs(a - b) / max(abs(b), 1e-30) for a, b in zip(got, want64))
    print("step configuration [%s %s]: losses %s (fp64 oracle %s, worst rel error %.1e) | parameter-gradient rel-L2 vs fp64 "
          "oracle: median %.2e worst %.2e (%s) | fp32 CPU oracle's own: median %.2e worst %.2e | stock PyTorch/cuDNN fp32 on this "
          "GPU: median %.2e worst %.2e" % (run["name"], run["cfg"]["mode"], [round(v, 6) for v in got], [round(v, 6) for v in want64],
                                           lerr, med, worst[0], worst[1], ref[len(ref) // 2], ref[-1], refg[len(refg) // 2], refg[-1]))
    assert med < 3 * rmed + 1e-4 and worst[0] < 3 * rworst + 1e-3


@pytest.mark.parametrize("which", ["eager", "captured"])
def test_parameters_without_gradient(run, which):
    """Check 3: what the oracle leaves with grad None (the encoders' fc, the heads of the scales the loss does not use) has an
    arena gradient of exactly 0 in both steps.  Without weight decay it stays bit-identical; with weight decay ArenaAdam decays
    it -- its documented deviation from torch.optim.Adam, which skips grad-None parameters -- so its change is Adam applied to
    the gradient wd * p.  The heads of the scales in use have a gradient: the step reaches the head plan it is named for."""
    c, r = run["cfg"], run[which]
    g64 = run["oracle"]["f64"][1]
    unused = [k for k in r["slices"] if k not in g64]
    assert any(".fc." in k for k in unused) and all(k in r["slices"] for k in g64)
    K = c["num_scales"]
    for s, names in enumerate(r["heads"]):
        for k in names:
            if s < K:
                assert k in g64 and float(r["param_grads"][k].abs().max()) > 0, "%s: head %d has no gradient" % (k, s)
            else:
                assert k in unused, "%s: head %d is not among the oracle's unused parameters" % (k, s)
    for t in range(2):
        for k in unused:
            net, off, n = r["slices"][k]
            g = r["grads"][t][net][off:off + n]
            assert float(g.abs().max()) == 0.0, "%s step %d: %s has a gradient" % (which, t + 1, k)
            if c["weight_decay"] == 0.0:
                assert torch.equal(r["params"][t + 1][net][off:off + n], r["params"][0][net][off:off + n]), \
                    "%s step %d: %s changed" % (which, t + 1, k)
    if c["weight_decay"] == 0.0:
        return
    for net in ("disp", "pose"):
        sel = torch.cat([torch.arange(off, off + n) for k in unused for nt, off, n in [r["slices"][k]] if nt == net]).to(DEV)
        ref = Adam64(r["params"][0][net][sel], c["lr"], c["betas"], EPS, c["weight_decay"])
        for t in range(2):
            before, after, g = r["params"][t][net][sel], r["params"][t + 1][net][sel], r["grads"][t][net][sel]
            want, size = ref.step(g, before)
            assert_adam_change(after.double() - before.double(), want, size, after, g,
                               "%s %s step %d, parameters without gradient" % (which, net, t + 1))
            assert bool((after != before)[before != 0].all()), "weight decay skipped a parameter without gradient"


@pytest.mark.parametrize("which", ["eager", "captured"])
def test_batchnorm_state_after_step_1(run, which):
    """Check 4: every running_mean / running_var after step 1 against fp64 (relative L2 within 3x the larger fp32 oracle's own
    error + 1e-6), and num_batches_tracked counts every network call: 1 + n_ref DispResNet calls, 2 n_ref PoseResNet calls."""
    c, got = run["cfg"], run[which]["buffers"]
    b64, b32, b32gpu = (run["oracle"][k][2] for k in ("f64", "f32", "f32gpu"))
    calls = {"disp": 1 + c["n_ref"], "pose": 2 * c["n_ref"]}
    bad = []
    for k, want in b64.items():
        if k.endswith("num_batches_tracked"):
            assert int(got[k]) == int(want) == calls[k.split(".")[0]], (k, int(got[k]), int(want))
            continue
        err, y = rel_l2(got[k], want), max(rel_l2(b32[k], want), rel_l2(b32gpu[k], want))
        if not err <= 3 * y + 1e-6:
            bad.append("%s: rel-L2 %.2e (fp32 yardstick %.2e)" % (k, err, y))
    assert not bad, bad


@pytest.mark.parametrize("which", ["eager", "captured"])
def test_adam_used_this_steps_gradient(run, which):
    """Check 5: each step's parameter change is the fp64 Adam update (weight decay folded in, moments carried over from the
    previous step) of the gradient that step left in the arena.  An update that ran before a side-stream weight gradient or
    PoseResNet's backward was joined, or on the previous step's gradient, does not match it."""
    c, r = run["cfg"], run[which]
    for net in ("disp", "pose"):
        ref = Adam64(r["params"][0][net], c["lr"], c["betas"], EPS, c["weight_decay"])
        for t in range(2):
            before, after, g = r["params"][t][net], r["params"][t + 1][net], r["grads"][t][net]
            assert float(g.abs().max()) > 0
            want, size = ref.step(g, before)
            assert_adam_change(after.double() - before.double(), want, size, after, g, "%s %s step %d" % (which, net, t + 1))


def test_captured_step_matches_eager(run):
    """Check 6: the replayed step 1 runs the same kernels as the eager one, only the order of atomic adds differs."""
    e, g = run["eager"], run["captured"]
    np.testing.assert_allclose(g["losses"][0], e["losses"][0], rtol=2e-5)
    for net in ("disp", "pose"):
        assert rel_l2(g["grads"][0][net], e["grads"][0][net]) < 1e-4, net


def test_loss_launches_per_step(run):
    """Check 7: the photometric / geometry loss takes at most MAX_JOBS pair-directions per launch; five frames with three
    scales (2 x 4 x 3 = 24) take two launches, whose partial losses the step adds."""
    from scsfm import lib as L
    c = run["cfg"]
    want = math.ceil(2 * c["n_ref"] * c["num_scales"] / L.MAX_JOBS)
    if run["name"] == "seq5_scales3":
        assert want == 2
    assert run["eager"]["pair_fwd"] == [want, want]
