"""The split-mode (tf32x3) bookkeeping paths of the TMA convolution kernels, against fp64.

In tf32x3 every stage of conv_tma_kernel is an accumulation chain of its own per consumer warpgroup, and
conv_wgrad_tma_kernel runs two chains per tap and stage; how many wgmma a chain holds, and how many chains and work items
a CTA runs, depend on the layer.  The replays of test_conv_calls_fp64_gpu.py cover the shapes the training step makes;
the calls here aim at the edges instead: CTAs with one work item, with an even and an odd number of them (work counts
just above one and two waves of the SMs), partial last channel chunks (Cin 20, 36: fewer K8 slices, all-zero slices
skipped), 1x1 and 3x3 kernels at stride 1 and 2 (the stride-2 data gradient's parity classes have 1, 2 and 4 taps, the
1x1's a single one), every (Cout tile, pixel tile) instantiation of the forward kernel forced through the tune knobs, and
weight gradients whose pixel range is split over one CTA and over many.  Each is checked element by element and in
relative L2 with the bounds and checks of test_conv_calls_fp64_gpu.py (forward and data gradient bitwise repeatable,
images independent, no element unwritten), and each forward and data gradient must have run on conv_tma_kernel
(its debug counters give the work items of every CTA); together the cases launch every forward instantiation and every
split-mode weight-gradient instantiation of the TMA kernels.  Plain tf32 runs a few of
the same calls as a control (one chain per tile).  Needs a GPU.
"""
import math

import pytest
import torch

import test_conv_calls_fp64_gpu as base

pytestmark = pytest.mark.gpu
DEV = base.DEV


def _call(kind, B, H, W, Cin, Cout, k, stride, pad, mode="tf32x3", **knobs):
    """A Call of `kind` on an input of B x H x W x Cin (data gradient: that input's gradient) with a k x k kernel, and
    the tune knobs forcing its kernel choice."""
    from scsfm import nnops as O
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    x, out = ((B, H, W, Cin), (B, Ho, Wo, Cout)) if kind != "dgrad" else ((B, Ho, Wo, Cout), (B, H, W, Cin))
    c = base.Call(kind=kind, mode=mode, tune=O.tune(**knobs), x=x, w=(Cout, k, k, Cin), out=out, stride=stride, pad=pad,
                  pad_mode=0, act=0, bias=False, addend=False, bn_groups=0, bn_eval=False, with_lo=False, padded=False,
                  zero_ch=())
    return c


def _cases():
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    cases = []
    # --- forward / data gradient on conv_tma_kernel.  128-pixel tiles of 8 rows x 16 columns (mt=1, tw_log2=4) and one
    # Cout tile: B * ceil(H / 8) * ceil(W / 16) work items, one CTA per SM
    tile = dict(mt=1, tw_log2=4)
    for kind in ("fwd", "dgrad"):
        cases += [
            ("%s one work item" % kind, _call(kind, 1, 8, 16, 64, 64, 3, 1, 1, **tile)),
            ("%s SMs + 1 work items (1 or 2 per CTA)" % kind, _call(kind, 1, 8 * (nsm + 1), 16, 32, 32, 3, 1, 1, **tile)),
            ("%s 2 SMs + 1 work items (2 or 3 per CTA)" % kind, _call(kind, 1, 8 * (2 * nsm + 1), 16, 32, 32, 3, 1, 1, **tile)),
            ("%s Cin 20" % kind, _call(kind, 2, 37, 45, 20, 24, 3, 1, 1)),
            ("%s Cin 36" % kind, _call(kind, 3, 19, 21, 36, 40, 3, 1, 1)),
            ("%s Cin 36 1x1" % kind, _call(kind, 2, 19, 21, 36, 40, 1, 1, 0)),
            ("%s 1x1 s1" % kind, _call(kind, 2, 16, 52, 128, 64, 1, 1, 0)),
            ("%s 3x3 s2" % kind, _call(kind, 2, 32, 52, 64, 128, 3, 2, 1)),
            ("%s 3x3 s2 odd size, Cin 20" % kind, _call(kind, 2, 37, 45, 20, 24, 3, 2, 1)),
            ("%s 1x1 s2" % kind, _call(kind, 2, 32, 52, 64, 128, 1, 2, 0)),
        ]
    # every (BNW, MT) instantiation, forced; Cout 16 leaves the weight tile to the knob
    for bnw, mt in ((16, 1), (32, 1), (64, 1), (128, 1), (16, 2), (32, 2), (64, 2)):
        for tw in (3, 4):
            cases.append(("fwd BNW %d MT %d TW %d" % (bnw, mt, 1 << tw), _call("fwd", 2, 21, 35, 36, 16, 3, 1, 1, mt=mt, tw_log2=tw, bn=bnw)))
        cases.append(("dgrad BNW %d MT %d" % (bnw, mt), _call("dgrad", 2, 21, 35, 16, 40, 3, 2, 1, mt=mt, tw_log2=3, bn=bnw)))
    # --- weight gradient on conv_wgrad_tma_kernel: at most 8 tiles of 4 x 16 pixels -> one pixel split; large -> many
    for bn in (32, 64):
        wt = dict(wgrad=2, bn=bn)
        cases += [
            ("wgrad BN %d one split" % bn, _call("wgrad", 1, 8, 32, 64, 64, 3, 1, 1, **wt)),
            ("wgrad BN %d one split, one tile" % bn, _call("wgrad", 1, 4, 16, 20, 24, 3, 1, 1, **wt)),
            ("wgrad BN %d many splits" % bn, _call("wgrad", 2, 64, 64, 64, 64, 3, 1, 1, **wt)),
            ("wgrad BN %d Cin 36" % bn, _call("wgrad", 3, 19, 21, 36, 40, 3, 1, 1, **wt)),
            ("wgrad BN %d 1x1 s1" % bn, _call("wgrad", 2, 16, 52, 128, 64, 1, 1, 0, **wt)),
            ("wgrad BN %d 3x3 s2" % bn, _call("wgrad", 2, 37, 45, 20, 24, 3, 2, 1, **wt)),
            ("wgrad BN %d 1x1 s2" % bn, _call("wgrad", 2, 32, 52, 64, 128, 1, 2, 0, **wt)),
            ("wgrad BN %d 7x7 stem" % bn, _call("wgrad", 2, 64, 96, 4, 64, 7, 2, 3, **wt)),
        ]
    # plain tf32: the same kernels without turns
    cases += [(label + " [tf32]", c._replace(mode="tf32")) for label, c in cases
              if label in ("fwd SMs + 1 work items (1 or 2 per CTA)", "dgrad 3x3 s2", "wgrad BN 64 many splits")]
    return cases


def _tma_items(c, op):
    """Work items per CTA of conv_tma_kernel for call c (fwd / dgrad), read from its debug slot 7 (written by every CTA);
    an empty tensor if no launch of that kernel wrote it."""
    from scsfm import nnops as O
    cx = O.ConvCtx(c.mode)
    cx.tune = c.tune
    cx.debug = torch.zeros(8 * 4096, dtype=torch.int64, device=DEV)
    if c.kind == "fwd":
        cx.conv_fwd(op.a, op.w, None, c.stride, c.pad, c.pad_mode, O.ACT_NONE, None, 1, op.w_lo)
    else:
        cx.conv_dgrad(op.a, op.w, c.out, c.stride, c.pad)
    torch.cuda.synchronize()
    items = cx.debug.view(-1, 8)[:, 7]
    return items[items > 0].cpu()


@pytest.fixture(scope="module")
def results():
    """(label, call, checks, items per CTA of the TMA kernel or None) per case, and the convolution kernels launched."""
    from torch.profiler import ProfilerActivity, profile
    out = []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i, (label, c) in enumerate(_cases()):
            op = base._Operands(c, "dense", 7000 + i)
            ref, A = base._reference(c, op)
            chk = base._Check(base.REL_L2[c.mode][c.kind])
            try:
                base.CHECK[c.kind](c, op, ref, A, c.tune, chk)
            except Exception as e:          # noqa: BLE001 -- reported with the call that raised it
                chk.items.append(("raised %r" % e, float("inf"), None, 0))
            out.append((label, c, chk, _tma_items(c, op) if c.kind != "wgrad" else None))
            del op, ref, A
        torch.cuda.synchronize()
    kernels = {base.kernel_key(e.key) for e in prof.key_averages()}
    torch.cuda.empty_cache()
    return out, kernels


def test_cases_reach_their_kernels(results):
    """Every forward and data-gradient case ran on conv_tma_kernel with the work items per CTA it aims at, the forward
    cases launched every instantiation of it, and the weight-gradient cases every split-mode instantiation of the TMA
    weight-gradient kernel."""
    rows, kernels = results
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    missed = [label for label, c, _, items in rows if items is not None and items.numel() == 0]
    assert not missed, missed
    want = {"one work item": (1, 1), "SMs + 1 work items": (nsm, 2), "2 SMs + 1 work items": (nsm, 3)}
    for label, c, _, items in rows:
        for key, (ctas, most) in want.items():
            if label.split(" ", 1)[1].startswith(key):
                assert (items.numel(), int(items.max())) == (ctas, most), (label, items.numel(), int(items.max()))
    fwd = {k for k in kernels if k.startswith("scsfm::conv_tma_kernel<")}
    assert fwd == {"scsfm::conv_tma_kernel<%d, %d>" % a for a in ((16, 1), (32, 1), (64, 1), (128, 1), (16, 2), (32, 2), (64, 2))}, fwd
    wt = {"scsfm::conv_wgrad_tma_kernel<%d, true, %d, %d>" % (bn, kw, st) for bn in (32, 64) for kw, st in ((1, 1), (1, 2), (3, 1), (3, 2), (7, 2))}
    assert not wt - kernels, sorted(wt - kernels)


def test_edge_paths_vs_fp64(results):
    rows, _ = results
    bad = []
    for label, c, chk, _ in rows:
        for what, ratio, rl2, nan in chk.failures():
            bad.append("%s | %s: ratio %.3g (tau %g) rel-L2 %s (bound %g) NaN %d" % (
                label, what, ratio, base.TAU, "-" if rl2 is None else "%.3g" % rl2, chk.rel, nan))
    worst = max(it[1] for _, _, chk, _ in rows for it in chk.items if it[0] in ("out", "din", "dw"))
    print("%d calls, worst elementwise ratio %.3g (tau %g)" % (len(rows), worst, base.TAU))
    assert not bad, "\n".join(bad)
    # the forward and data-gradient checks include bitwise repeatability
    assert all(any(it[0] == "repeatable" for it in chk.items) for _, c, chk, _ in rows if c.kind != "wgrad")
    assert math.isfinite(worst)
