"""Per-layer correctness + timing of the tensor-core convolution kernels (forward, data gradient, weight gradient) over
the layer shapes of DispResNet18 / PoseResNet18 at 256x832 (B = 12 stacked DispResNet calls).

    python tools/conv_layers.py [--mode tf32|tf32x3] [--pass fwd,dgrad,wgrad] [--tune key=val,...] [--compare key=val,...]
                                [--roles] [--only substring] [--reps N]

--tune / --compare: nnops.tune() keywords (no_tma, mt, tw_log2, bn, wgrad, wt_tile, wt_split_grid); with --compare
every layer is run in both configurations and the second is checked against the first.  The weight-gradient pass also
prints the TMA kernel's schedule: CTAs, tiles per CTA and the fill (useful pixels over the SM time of the busiest SM).  --roles prints the TMA kernel's per-role cycle counters
(ScsfmConv.debug).  The chain-drain counter (wgmma_wait of a split-accumulate chain; the weight gradient's consumer
counters too) is compiled in only by a build with NVCC_EXTRA=-DSCSFM_DRAIN_COUNTERS; --roles then also prints its share
of the consumer cycles.  Errors are relative L2 against an fp64 torch reference.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "sc-sfmlearner-release_b200"))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from scsfm import nnops as O  # noqa: E402

torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False

# name, B, H, W, Cin, Cout, k, stride, pad, reflect, launches per step in DispResNet18 (B=12) + PoseResNet18 (B=16)
LAYERS = [
    ("stem 7x7 s2", 12, 256, 832, 4, 64, 7, 2, 3, 0),
    ("pose stem 7x7 s2", 16, 256, 832, 8, 64, 7, 2, 3, 0),
    ("enc L1", 12, 64, 208, 64, 64, 3, 1, 1, 0),
    ("enc L2 s2", 12, 64, 208, 64, 128, 3, 2, 1, 0),
    ("down2 1x1 s2", 12, 64, 208, 64, 128, 1, 2, 0, 0),
    ("enc L2", 12, 32, 104, 128, 128, 3, 1, 1, 0),
    ("enc L3 s2", 12, 32, 104, 128, 256, 3, 2, 1, 0),
    ("down3 1x1 s2", 12, 32, 104, 128, 256, 1, 2, 0, 0),
    ("enc L3", 12, 16, 52, 256, 256, 3, 1, 1, 0),
    ("enc L4 s2", 12, 16, 52, 256, 512, 3, 2, 1, 0),
    ("down4 1x1 s2", 12, 16, 52, 256, 512, 1, 2, 0, 0),
    ("enc L4", 12, 8, 26, 512, 512, 3, 1, 1, 0),
    ("dec 4_0", 12, 8, 26, 512, 256, 3, 1, 1, 1),
    ("dec 4_1", 12, 16, 52, 512, 256, 3, 1, 1, 1),
    ("dec 3_0", 12, 16, 52, 256, 128, 3, 1, 1, 1),
    ("dec 3_1", 12, 32, 104, 256, 128, 3, 1, 1, 1),
    ("dec 2_0", 12, 32, 104, 128, 64, 3, 1, 1, 1),
    ("dec 2_1", 12, 64, 208, 128, 64, 3, 1, 1, 1),
    ("dec 1_0", 12, 64, 208, 64, 32, 3, 1, 1, 1),
    ("dec 1_1", 12, 128, 416, 96, 32, 3, 1, 1, 1),
    ("dec 0_0", 12, 128, 416, 32, 16, 3, 1, 1, 1),
    ("dec 0_1", 12, 256, 832, 16, 16, 3, 1, 1, 1),
    ("pose 1x1", 16, 8, 26, 512, 256, 1, 1, 0, 0),
    ("pose 3x3", 16, 8, 26, 256, 256, 3, 1, 1, 0),
    ("r50 1x1 256->64", 6, 64, 208, 256, 64, 1, 1, 0, 0),
    ("r50 1x1 64->256", 6, 64, 208, 64, 256, 1, 1, 0, 0),
    ("r50 1x1 1024->256", 6, 16, 52, 1024, 256, 1, 1, 0, 0),
    ("r50 L2 3x3 s2", 6, 64, 208, 128, 128, 3, 2, 1, 0),
    ("r50 L3 3x3 s2", 6, 32, 104, 256, 256, 3, 2, 1, 0),
    ("r50 L4 3x3 s2", 6, 16, 52, 512, 512, 3, 2, 1, 0),
    ("r50 down2 1x1 s2", 6, 64, 208, 256, 512, 1, 2, 0, 0),
    ("r50 down3 1x1 s2", 6, 32, 104, 512, 1024, 1, 2, 0, 0),
    ("r50 down4 1x1 s2", 6, 16, 52, 1024, 2048, 1, 2, 0, 0),
    ("odd zero", 2, 37, 45, 20, 24, 3, 1, 1, 0),
    ("odd refl", 3, 19, 21, 36, 40, 3, 1, 1, 1),
    ("odd s2", 2, 37, 45, 24, 20, 3, 2, 1, 0),
]


def rel(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


def timeit(fn, reps):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def parse_tune(s):
    return O.tune(**{k: int(v) for k, v in (kv.split("=") for kv in s.split(",") if kv)}) if s else 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="tf32x3", choices=["fp32", "tf32", "tf32x3"])
    ap.add_argument("--pass", dest="passes", default="fwd,dgrad,wgrad")
    ap.add_argument("--tune", default="")
    ap.add_argument("--compare", default=None)
    ap.add_argument("--roles", action="store_true")
    ap.add_argument("--only", default="")
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    passes = args.passes.split(",")
    cfgs = [("base", parse_tune(args.tune))] + ([("cmp", parse_tune(args.compare))] if args.compare is not None else [])
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    g = torch.Generator().manual_seed(0)
    bad = 0
    totals = {(c, p): 0.0 for c, _ in cfgs for p in passes}
    # the counters the TMA kernels write per CTA (slot: meaning, in cycles; consumer slots from warpgroup 0); slot 7 = tiles.
    # The weight-gradient kernel writes the consumer slots only.
    names = {0: "producer wait-empty", 1: "producer total", 2: "consumer wait-full", 3: "consumer drain", 4: "consumer total"}
    for (name, B, H, W, Cin, Cout, k, s, pad, reflect) in LAYERS:
        if args.only and args.only not in name:
            continue
        x = torch.randn(B, H, W, Cin, generator=g).cuda()
        w = (torch.randn(Cout, k, k, Cin, generator=g) / (k * k * Cin) ** 0.5).cuda()
        Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
        dout = torch.randn(B, Ho, Wo, Cout, generator=g).cuda()
        if args.mode == "tf32":
            for t in (x, w, dout):
                O.round_tf32(t, t)
        w_lo = O.split_tf32(w) if args.mode == "tf32x3" else None
        pm = O.PAD_REFLECT if reflect else O.PAD_ZERO
        # fp64 reference
        xd = x.double().permute(0, 3, 1, 2).requires_grad_(True)
        xp = F.pad(xd, (pad,) * 4, mode="reflect") if (reflect and pad) else xd
        wd = w.double().permute(0, 3, 1, 2).requires_grad_(True)
        yd = F.conv2d(xp, wd, None, s, 0 if (reflect and pad) else pad)
        yd.backward(dout.double().permute(0, 3, 1, 2))
        ref = {"fwd": yd.detach().permute(0, 2, 3, 1), "wgrad": wd.grad.permute(0, 2, 3, 1), "dgrad": xd.grad.permute(0, 2, 3, 1)}
        flops = 2.0 * B * Ho * Wo * Cout * k * k * Cin
        first = {}
        for cname, tw in cfgs:
            cx = O.ConvCtx(args.mode)
            cx.tune = tw

            def run(p):
                if p == "fwd":
                    return cx.conv_fwd(x, w, None, s, pad, pm, O.ACT_NONE, None, 1, w_lo)
                if p == "wgrad":
                    dw = torch.zeros_like(w)
                    cx.conv_wgrad(x, dout, dw, None, s, pad, pm)
                    return dw
                if reflect:
                    dpad = cx.conv_dgrad(dout, w, x.shape, s, pad, None, padded_input=True)
                    dx = torch.zeros_like(x)
                    O.fold_plain(dpad, dx, None, O.ACT_NONE, accumulate=False)
                    return dx
                return cx.conv_dgrad(dout, w, x.shape, s, pad)
            for p in passes:
                if p == "dgrad" and Cin < 16:
                    continue
                out = run(p)
                torch.cuda.synchronize()
                err = rel(out, ref[p])
                t = timeit(lambda: run(p), args.reps)
                totals[(cname, p)] += t
                tol = 2e-3 if args.mode == "tf32" else 2e-5
                msg = ""
                if cname == "base":
                    first[p] = (out, t)
                else:
                    d = rel(out, first[p][0])
                    msg = " | vs base %.1e  x%.2f" % (d, first[p][1] / t)
                    if d > tol:
                        msg += "  <-- MISMATCH"
                        bad += 1
                if err > tol:
                    msg += "  <-- ERROR vs fp64"
                    bad += 1
                print("%-18s B%-2d %3dx%-3d C%4d->%-3d k%d s%d %-5s %-5s err %.1e  %8.3f ms %7.1f TF/s%s"
                      % (name, B, H, W, Cin, Cout, k, s, p, cname, err, t, flops / t / 1e9, msg), flush=True)
                if p == "wgrad":
                    # the TMA weight gradient's schedule: tiles per CTA (debug slot 7) and the share of SM time spent on
                    # real pixels, units x B Ho Wo / 64 / SMs over the busiest SM's tile-steps
                    dbg = torch.zeros(8192 * 8, dtype=torch.int64, device="cuda")
                    cx.debug = dbg
                    run(p)
                    torch.cuda.synchronize()
                    cx.debug = None
                    tiles = dbg.view(-1, 8)[:, 7]
                    tiles = tiles[tiles > 0]
                    if tiles.numel():
                        knob = (tw >> 8) & 7                 # the Cout tile launch_conv_wgrad_tma picks
                        bn = 32 if knob == 2 or (knob != 3 and Cout <= 32) else 64
                        units = -(-Cin // 64) * k * -(-Cout // bn)
                        busiest = -(-tiles.numel() // nsm) * int(tiles.max())
                        print("      schedule: %d CTAs, tiles per CTA %d..%d, fill %.2f"
                              % (tiles.numel(), int(tiles.min()), int(tiles.max()), units * B * Ho * Wo / 64 / nsm / busiest),
                              flush=True)
                if args.roles:
                    dbg = torch.zeros(8192 * 8, dtype=torch.int64, device="cuda")
                    cx.debug = dbg
                    run(p)
                    torch.cuda.synchronize()
                    cx.debug = None
                    d_ = dbg.view(-1, 8).double()
                    d_ = d_[d_[:, 7] > 0]
                    if d_.shape[0]:
                        m = d_.mean(0)
                        print("      roles (%d CTAs, %.1f tiles/CTA): " % (d_.shape[0], m[7]) +
                              "  ".join("%s=%.0f" % (n, float(m[k])) for k, n in names.items()) +
                              "  drain share %.1f%%" % (100.0 * float(m[3]) / max(float(m[4]), 1.0)), flush=True)
    for (c, p), t in totals.items():
        print("total %-5s %-5s %.3f ms" % (c, p, t))
    print("MISMATCHES: %d" % bad)
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
