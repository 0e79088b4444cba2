"""Kernel-level timing of the fused loss kernels (CUDA events, L2 flushed between iterations).
Usage: python tools/bench_loss.py [B H W] [--intrinsics-grad]

--intrinsics-grad times the loss backward twice, with intrinsics that need no gradient and with intrinsics that do (a learned
K: one extra small launch per chunk of pair-directions), and prints both."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "sc-sfmlearner-release_b200"))
import torch  # noqa: E402

from scsfm import lib as L  # noqa: E402
from scsfm import synth  # noqa: E402
import loss_functions as lf  # noqa: E402


def run(B, H, W, k_grad=False, label=""):
    d = synth.loss_inputs(0, B, H, W, n_ref=2, n_scales=1)
    c = lambda x: x.cuda()  # noqa: E731
    tgt, refs, K = c(d["tgt_img"]), [c(x) for x in d["ref_imgs"]], c(d["intrinsics"]).requires_grad_(k_grad)
    td = [c(x).requires_grad_(True) for x in d["tgt_depth"]]
    rd = [[c(x).requires_grad_(True) for x in r] for r in d["ref_depths"]]
    ps = [c(x).requires_grad_(True) for x in d["poses"]]
    pi = [c(x).requires_grad_(True) for x in d["poses_inv"]]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
    res = {"pair_fwd": [], "pair_bwd": [], "smooth_fwd": [], "smooth_bwd": []}
    bwd_launches = None
    for it in range(13):
        flush.zero_()
        e = [ev() for _ in range(6)]
        e[0].record()
        p, q = lf.compute_photo_and_geometry_loss(tgt, refs, K, td, rd, ps, pi, 1, 1, 1, 1, "zeros")
        e[1].record()
        flush.zero_()
        e[2].record()
        s = lf.compute_smooth_loss(td, tgt, rd, refs)
        e[3].record()
        loss = p + 0.5 * q
        flush.zero_()
        e4, e5 = ev(), ev()
        n0 = L.launch_count()
        e4.record()
        loss.backward()
        e5.record()
        bwd_launches = L.launch_count() - n0
        flush.zero_()
        e6, e7 = ev(), ev()
        e6.record()
        s.backward()
        e7.record()
        torch.cuda.synchronize()
        if it >= 3:
            res["pair_fwd"].append(e[0].elapsed_time(e[1]))
            res["smooth_fwd"].append(e[2].elapsed_time(e[3]))
            res["pair_bwd"].append(e4.elapsed_time(e5))
            res["smooth_bwd"].append(e6.elapsed_time(e7))
        for t in td + [x for r in rd for x in r] + ps + pi + [K]:
            t.grad = None
    px = B * H * W
    alg = {"pair_fwd": 4 * 32 * px, "pair_bwd": 4 * 44 * px, "smooth_fwd": 3 * 16 * px, "smooth_bwd": 3 * 20 * px}
    for k, v in res.items():
        v.sort()
        med = v[len(v) // 2]
        print("%s%-11s median %.3f ms (min %.3f)  algorithmic %.1f MB -> %.0f GB/s (incl. launch/autograd overhead)"
              % (label, k, med, v[0], alg[k] / 1e6, alg[k] / med / 1e6))
    print("%spair_bwd launches %d" % (label, bwd_launches))


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    B, H, W = (int(a) for a in args[:3]) if len(args) >= 3 else (4, 256, 832)
    print("%s, power limit %s" % (torch.cuda.get_device_name(), _power_limit()))
    if "--intrinsics-grad" in sys.argv[1:]:
        run(B, H, W, False, "[K no grad]   ")
        run(B, H, W, True, "[K with grad] ")
    else:
        run(B, H, W)


def _power_limit():
    import subprocess
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=10).stdout.strip()
        return out.splitlines()[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


if __name__ == "__main__":
    main()
