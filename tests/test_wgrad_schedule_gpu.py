"""The stream-K schedule and the pixel tiles of the TMA weight-gradient kernel (conv_wgrad_tma_kernel), against fp64.

The kernel's work is a flat range of (unit, pixel tile) iterations, a unit being one kernel row, 64 input channels and a
Cout tile; one wave of CTAs shares the range evenly, and a CTA adds its sums into dw at the end of every unit its range
touches.  The calls here put those ranges inside one unit, across one and two unit boundaries, on fewer iterations than
SMs and on an exact multiple of the grid; they run the 8 x 8 pixel tile where it pads less than 4 x 16 (widths 52, 104)
and, forced through the tune knob, at widths 26 and 45; 1x1 and 3x3 kernels at stride 1 and 2, both 7x7 stems and a
reflection-padded layer (its border ring on the gather kernel).  Each call is checked element by element and in relative
L2 with the bounds of test_conv_calls_fp64_gpu.py, in tf32x3 and tf32, with Cout tiles of 32 and 64.  The kernel's
debug slot 7 gives the tiles of every CTA: they must sum to the iteration count and, under stream-K, differ by at most
one.  The two tune knobs (pixel tile, split grid) must reproduce the other schedule inside the same bounds.  Needs a GPU.
"""
import math

import pytest
import torch

import test_conv_calls_fp64_gpu as base

pytestmark = pytest.mark.gpu
DEV = base.DEV


def _out_hw(H, W, k, s, pad):
    return (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1


def _tile(Ho, Wo, force=0):
    """(rows, columns) of the pixel tile: forced, or the one with the smaller padded output area (4 x 16 on a tie)."""
    if force:
        return 64 // force, force
    p416 = -(-Ho // 4) * 4 * (-(-Wo // 16) * 16)
    p88 = -(-Ho // 8) * 8 * (-(-Wo // 8) * 8)
    return (8, 8) if p88 < p416 else (4, 16)


def _schedule(B, H, W, Cin, Cout, k, s, pad, bn, nsm, wt_tile=0, wt_split_grid=0):
    """(tile, iterations T, CTAs) the launcher must choose for a call."""
    Ho, Wo = _out_hw(H, W, k, s, pad)
    th, tw = _tile(Ho, Wo, wt_tile)
    n_tiles = B * -(-Ho // th) * -(-Wo // tw)
    units = -(-Cin // 64) * k * -(-Cout // bn)
    if wt_split_grid:
        splits = max(1, min(nsm // units, (n_tiles + 7) // 8))
        per = -(-n_tiles // splits)
        return (th, tw), units * n_tiles, units * -(-n_tiles // per)
    return (th, tw), units * n_tiles, min(nsm, -(-units * n_tiles // 8))


def _shapes(nsm):
    """(label, B, H, W, Cin, Cout, k, stride, pad, reflect, knobs)."""
    return [
        # one unit (1x1, Cin <= 64, Cout <= BN): every range lies inside it
        ("inside one unit", 2, 64, 128, 64, 32, 1, 1, 0, 0, {}),
        # 3x3, 2 channel blocks: 6 or 12 units of 5 tiles, 30 or 60 iterations over 4 or 8 CTAs of 7-8
        ("across one and two unit boundaries", 1, 20, 16, 128, 64, 3, 1, 1, 0, {}),
        ("fewer iterations than SMs", 1, 8, 16, 64, 64, 3, 1, 1, 0, {}),
        # one unit, 10 * nsm tiles: exactly 10 per CTA
        ("T a multiple of the grid", nsm, 40, 16, 64, 32, 1, 1, 0, 0, {}),
        ("8x8 width 52", 2, 16, 52, 64, 64, 3, 1, 1, 0, {}),
        ("8x8 width 104", 1, 32, 104, 32, 64, 3, 1, 1, 0, {}),
        ("8x8 width 26 (forced)", 3, 8, 26, 128, 64, 3, 1, 1, 0, dict(wt_tile=8)),
        ("8x8 37x45 (forced)", 2, 37, 45, 20, 24, 3, 1, 1, 0, dict(wt_tile=8)),
        ("4x16 width 52 (forced)", 2, 16, 52, 64, 64, 3, 1, 1, 0, dict(wt_tile=16)),
        ("1x1 s1", 2, 16, 52, 128, 64, 1, 1, 0, 0, {}),
        ("1x1 s2", 2, 32, 104, 64, 128, 1, 2, 0, 0, {}),
        ("3x3 s2", 2, 37, 45, 20, 24, 3, 2, 1, 0, {}),
        ("3x3 s2 8x8", 2, 32, 104, 64, 64, 3, 2, 1, 0, {}),
        ("3x3 s2 8x8 (forced)", 2, 37, 45, 20, 24, 3, 2, 1, 0, dict(wt_tile=8)),
        ("1x1 s2 8x8 (forced)", 2, 32, 52, 64, 128, 1, 2, 0, 0, dict(wt_tile=8)),
        ("stem Cin 4", 2, 64, 96, 4, 64, 7, 2, 3, 0, {}),
        ("stem Cin 8", 2, 64, 96, 8, 64, 7, 2, 3, 0, {}),
        ("stem Cin 4 8x8 (forced)", 2, 64, 104, 4, 64, 7, 2, 3, 0, dict(wt_tile=8)),
        ("stem Cin 8 8x8", 2, 64, 104, 8, 64, 7, 2, 3, 0, {}),
        ("reflection padded", 2, 16, 52, 64, 64, 3, 1, 1, 1, {}),
        ("reflection padded 37x45", 2, 37, 45, 36, 40, 3, 1, 1, 1, {}),
        # the knobs: the split grid, and the split grid with the other tile
        ("split grid", 2, 16, 52, 128, 64, 3, 1, 1, 0, dict(wt_split_grid=1)),
        ("split grid 4x16", 2, 16, 52, 128, 64, 3, 1, 1, 0, dict(wt_split_grid=1, wt_tile=16)),
        ("split grid stem", 2, 64, 96, 4, 64, 7, 2, 3, 0, dict(wt_split_grid=1)),
    ]


def _cases():
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    from scsfm import nnops as O
    out = []
    for mode in ("tf32x3", "tf32"):
        for bn in (32, 64):
            for label, B, H, W, Cin, Cout, k, s, pad, refl, knobs in _shapes(nsm):
                Ho, Wo = _out_hw(H, W, k, s, pad)
                c = base.Call(kind="wgrad", mode=mode, tune=O.tune(wgrad=2, bn=bn, **knobs), x=(B, H, W, Cin),
                              w=(Cout, k, k, Cin), out=(B, Ho, Wo, Cout), stride=s, pad=pad, pad_mode=refl, act=0,
                              bias=False, addend=False, bn_groups=0, bn_eval=False, with_lo=False, padded=False, zero_ch=())
                out.append(("%s [%s BN %d]" % (label, mode, bn), c, _schedule(B, H, W, Cin, Cout, k, s, pad, bn, nsm, **knobs),
                            bool(knobs.get("wt_split_grid"))))
    return out


def _tiles_per_cta(c, op):
    """Tiles of every CTA of the call's TMA weight-gradient launch, from its debug slot 7."""
    from scsfm import nnops as O
    cx = O.ConvCtx(c.mode)
    cx.tune = c.tune
    cx.debug = torch.zeros(8 * 8192, dtype=torch.int64, device=DEV)
    dw = torch.zeros(c.w, device=DEV)
    cx.conv_wgrad(op.a, op.b, dw, None, c.stride, c.pad, c.pad_mode)
    cx.join_wgrad()
    torch.cuda.synchronize()
    t = cx.debug.view(-1, 8)[:, 7].cpu()
    return t[t > 0]


@pytest.fixture(scope="module")
def results():
    """(label, call, schedule, split grid, checks, tiles per CTA) per case, and the convolution kernels launched."""
    from torch.profiler import ProfilerActivity, profile
    rows = []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i, (label, c, sched, split) in enumerate(_cases()):
            op = base._Operands(c, "dense", 9100 + i)
            ref, A = base._reference(c, op)
            chk = base._Check(base.REL_L2[c.mode]["wgrad"])
            try:
                base.CHECK["wgrad"](c, op, ref, A, c.tune, chk)
            except Exception as e:          # noqa: BLE001 -- reported with the call that raised it
                chk.items.append(("raised %r" % e, float("inf"), None, 0))
            rows.append((label, c, sched, split, chk, _tiles_per_cta(c, op)))
            del op, ref, A
        torch.cuda.synchronize()
    kernels = {base.kernel_key(e.key) for e in prof.key_averages()}
    torch.cuda.empty_cache()
    return rows, kernels


def test_schedule_vs_fp64(results):
    rows, _ = results
    bad = []
    for label, c, _, _, chk, _ in rows:
        for what, ratio, rl2, nan in chk.failures():
            bad.append("%s | %s: ratio %.3g (tau %g) rel-L2 %s (bound %g) NaN %d" % (
                label, what, ratio, base.TAU, "-" if rl2 is None else "%.3g" % rl2, chk.rel, nan))
    worst = max(it[1] for _, _, _, _, chk, _ in rows for it in chk.items)
    print("%d calls, worst elementwise ratio %.3g (tau %g)" % (len(rows), worst, base.TAU))
    assert not bad, "\n".join(bad)
    assert math.isfinite(worst)


def test_tiles_per_cta(results):
    """Every CTA of the launch reports its tiles; they sum to units x tiles, over the grid the launcher must choose, and
    under stream-K two CTAs differ by at most one tile."""
    rows, _ = results
    bad = []
    for label, c, (_, T, ctas), split, _, tiles in rows:
        got = (tiles.numel(), int(tiles.sum()))
        spread = int(tiles.max() - tiles.min()) if tiles.numel() else -1
        if got != (ctas, T) or (not split and spread > 1):
            bad.append("%s: %d CTAs, %d tiles, spread %d; want %d CTAs, %d tiles" % (label, got[0], got[1], spread, ctas, T))
    assert not bad, "\n".join(bad)


def test_every_instantiation_ran(results):
    """The cases launch every TMA weight-gradient instantiation of both modes."""
    _, kernels = results
    want = {"scsfm::conv_wgrad_tma_kernel<%d, %s, %d, %d>" % (bn, sp, kw, st) for bn in (32, 64) for sp in ("true", "false")
            for kw, st in ((1, 1), (1, 2), (3, 1), (3, 2), (7, 2))}
    assert not want - kernels, sorted(want - kernels)
