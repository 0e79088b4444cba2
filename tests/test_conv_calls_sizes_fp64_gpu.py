"""The element-by-element fp64 replay of test_conv_calls_fp64_gpu.py on the convolution calls the other accepted configurations
make: the NYU benchmark (B=8, 256x320, 1 ref) in every mode, ResNet-50 at 256x832 in fp32 and tf32, the inference scripts'
batch of one (whose fewer tiles change the tile-count decisions of conv_tc.cu against the SM count), PoseResNet on raw KITTI
frames (odd planes at every level: stride-2 convolutions of odd inputs, partial TMA tiles on both axes) and DispResNet at
255x831 (odd stem input, 2^k - 1 decoder).

The calls are recorded as there (ConvCtx entry points wrapped while the networks run) and replayed with the same operands,
kernel choices, TAU, relative-L2 bounds and checks (NaN-filled outputs, repeatability, image independence, epilogues).  The four
256x832 configurations of that file are recorded here too: a call already in them is replayed there, so each configuration
here replays only the calls first seen in it, and must contribute at least one.  Needs a GPU."""
import collections
import math
import time

import pytest
import torch

from test_conv_calls_fp64_gpu import (CHECK, CONFIGS as BASE_CONFIGS, REL_L2, TAU, VARIANTS, _Check, _label, _Operands, _Recording,
                                      _reference, _ways, kernel_key)

pytestmark = pytest.mark.gpu
DEV = "cuda"
RAW_KITTI = [(375, 1242), (370, 1226), (374, 1238), (376, 1241)]
NEW_CONFIGS = ["nyu_r18-fp32", "nyu_r18-tf32", "nyu_r18-tf32x3", "kitti_r50-fp32", "kitti_r50-tf32", "infer_b1", "raw_kitti_pose",
               "odd_disp"]


def _nets(layers, mode):
    import models
    torch.manual_seed(0)
    return (models.DispResNet(layers, False).to(DEV).set_conv_mode(mode),
            models.PoseResNet(layers, False).to(DEV).set_conv_mode(mode))


def _train_step(layers, mode, batch, H, W, n_ref, kind):
    """One eager Trainer.step with bench.py's flags, then the fused eval forward of each network."""
    from scsfm import synth
    from scsfm.trainer import Trainer
    tgt, refs, K = synth.triplet(1234, batch, H, W, n_ref, kind)
    tgt, refs, K = tgt.to(DEV), [r.to(DEV) for r in refs], K.to(DEV)
    disp, pose = _nets(layers, mode)
    tr = Trainer(disp.train(), pose.train(), lr=1e-4, num_scales=1, with_ssim=1, with_mask=1, with_auto_mask=1,
                 padding_mode="zeros", distributed=False, conv_mode=mode)
    losses = [float(v) for v in tr.step(tgt, refs, K)]
    assert all(math.isfinite(v) for v in losses), losses
    disp.eval()
    pose.eval()
    with torch.no_grad():
        disp(tgt)
        pose(tgt, refs[0])


def _eval(net, *shape, n=1):
    with torch.no_grad():
        net.eval()(*[torch.randn(*shape, device=DEV) for _ in range(n)])


def _infer_b1():
    for layers in (18, 50):
        for mode in ("fp32", "tf32", "tf32x3"):
            disp, pose = _nets(layers, mode)
            for H, W in ((256, 832), (256, 320)):
                _eval(disp, 1, 3, H, W)
                _eval(pose, 1, 3, H, W, n=2)


def _raw_kitti_pose():
    for mode in ("fp32", "tf32x3"):
        _, pose = _nets(18, mode)
        for H, W in RAW_KITTI:
            _eval(pose, 1, 3, H, W, n=2)


def _odd_disp():
    disp, _ = _nets(18, "tf32x3")
    _eval(disp, 1, 3, 255, 831)
    disp.train()
    x = torch.randn(2, 3, 255, 831, device=DEV, requires_grad=True)
    sum(((1.0 / o) * (i + 1)).mean() for i, o in enumerate(disp(x))).backward()


RECORD = {"nyu_r18-%s" % m: (lambda m=m: _train_step(18, m, 8, 256, 320, 1, "nyu")) for m in ("fp32", "tf32", "tf32x3")}
RECORD.update({"kitti_r50-%s" % m: (lambda m=m: _train_step(50, m, 2, 256, 832, 2, "kitti")) for m in ("fp32", "tf32")})
RECORD.update({"infer_b1": _infer_b1, "raw_kitti_pose": _raw_kitti_pose, "odd_disp": _odd_disp})
for cfg, layers, mode, batch in BASE_CONFIGS:
    RECORD["base " + cfg] = lambda layers=layers, mode=mode, batch=batch: _train_step(layers, mode, batch, 256, 832, 2, "kitti")


@pytest.fixture(scope="module")
def recorded():
    """{"base": the distinct calls of the four 256x832 configurations of test_conv_calls_fp64_gpu.py, config: its distinct calls}."""
    runs = {}
    for cfg, run in RECORD.items():
        calls = []
        with _Recording(calls):
            run()
            torch.cuda.synchronize()
        runs[cfg] = list(dict.fromkeys(calls))
        torch.cuda.empty_cache()
    base = set()
    for cfg in [c for c in runs if c.startswith("base ")]:
        base |= set(runs.pop(cfg))
    runs["base"] = base
    return runs


def _plan_kernels(calls):
    """The kernels scsfm_conv_plan picks for the calls (SCSFM_KERNEL_* names)."""
    from scsfm import nnops as O
    names = {O.KERNEL_SIMT: "simt", O.KERNEL_GATHER: "gather", O.KERNEL_TMA: "tma", O.KERNEL_TMA_RING: "tma+ring",
             O.KERNEL_STEM: "stem", O.KERNEL_THIN: "thin"}
    got = set()
    for c in calls:
        d = O.conv_desc(c.x if c.kind != "dgrad" else c.out, c.w, c.stride, c.pad, c.pad_mode, c.act)
        cx = O.ConvCtx(c.mode)
        cx.tune = c.tune
        cx._finish(d)
        got.add(names[cx.plan(d, {"fwd": O.PASS_FWD, "dgrad": O.PASS_DGRAD, "wgrad": O.PASS_WGRAD}[c.kind]) & 0xff])
    return sorted(got)


def test_every_configuration_makes_new_calls(recorded):
    """Each configuration here makes at least one convolution call that the 256x832 configurations do not."""
    seen = set(recorded["base"])
    for cfg in NEW_CONFIGS:
        calls = recorded[cfg]
        new = [c for c in calls if c not in recorded["base"]]
        first = [c for c in new if c not in seen]
        seen |= set(first)
        print("%s: %d distinct calls, %d not in the 256x832 configurations (%d first replayed here); plan kernels: %s"
              % (cfg, len(calls), len(new), len(first), ", ".join(_plan_kernels(calls))))
        assert new, cfg


@pytest.fixture(scope="module")
def replays(recorded):
    """Replays, per configuration, the calls first seen in it (test_conv_calls_fp64_gpu.py replays the 256x832 ones):
    {config: {"rows": [(label, way, variant, check)], "worst": [ratio, rel-L2], "seconds": wall time}}."""
    from torch.profiler import ProfilerActivity, profile
    out, seen = {}, set(recorded["base"])
    for cfg in NEW_CONFIGS:
        t1 = time.time()
        calls = [c for c in recorded[cfg] if c not in seen]
        seen |= set(calls)
        rows, worst = [], [0.0, 0.0]
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for i, c in enumerate(calls):
                for vi, variant in enumerate(VARIANTS):
                    op = _Operands(c, variant, 1000 * i + vi)
                    ref, A = _reference(c, op)
                    for way, tune in (_ways(c) if variant == "dense" else _ways(c)[:1]):
                        chk = _Check(REL_L2[c.mode][c.kind])
                        try:
                            CHECK[c.kind](c, op, ref, A, tune, chk)
                        except Exception as e:          # noqa: BLE001 -- reported with the call that raised it
                            chk.items.append(("raised %r" % e, float("inf"), None, 0))
                        rows.append((_label(c), way, variant, chk))
                        for what, ratio, rl2, _ in chk.items:
                            if what in ("out", "din", "dw"):
                                worst[0], worst[1] = max(worst[0], ratio), max(worst[1], rl2)
                    del op, ref, A
            torch.cuda.synchronize()
        torch.cuda.empty_cache()
        kernels = sorted({kernel_key(e.key) for e in prof.key_averages() if kernel_key(e.key).startswith("scsfm::conv_")})
        out[cfg] = dict(rows=rows, worst=worst, seconds=time.time() - t1, kernels=kernels, n=len(calls))
        print("%s: %d calls replayed in %.1f s, worst elementwise ratio %.3g (tau %g), worst relative L2 %.3g; kernels: %s"
              % (cfg, len(calls), out[cfg]["seconds"], worst[0], TAU, worst[1], ", ".join(kernels)), flush=True)
    return out


@pytest.mark.parametrize("cfg", NEW_CONFIGS)
def test_conv_calls_vs_fp64(replays, cfg):
    r = replays[cfg]
    assert r["rows"], cfg
    bad = []
    for label, way, variant, chk in r["rows"]:
        for what, ratio, rl2, nan in chk.failures():
            bad.append("%s | %s | %s | %s: ratio %.3g (tau %g) rel-L2 %s (bound %g) NaN %d" % (
                label, way, variant, what, ratio, TAU, "-" if rl2 is None else "%.3g" % rl2, chk.rel, nan))
    kinds = collections.Counter(label.split()[0] for label, _, _, _ in r["rows"])
    print("%s: %d replays (%s), worst elementwise ratio %.3g, worst relative L2 %.3g, %.1f s" % (
        cfg, len(r["rows"]), dict(kinds), r["worst"][0], r["worst"][1], r["seconds"]))
    assert not bad, "\n".join(bad[:40]) + ("\n... %d more" % (len(bad) - 40) if len(bad) > 40 else "")
