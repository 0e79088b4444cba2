"""Generate tests/golden/loss_edges.npz by running the UNMODIFIED reference loss on the sharp, large-motion and behind-the-camera
inputs of loss_edge_inputs.py (the regime of tests/test_loss_backward_edges_gpu.py), so that tests/test_loss_edges_cpu.py can
pin the oracle there.

Needs a checkout of the original SC-SfMLearner project:

    python tests/golden/make_golden_loss_edges.py /path/to/SC-SfMLearner-Release

Its modules are imported read-only (bytecode writing disabled).  Per setting the file holds the input checksums, both loss
values, the gradient of photo + 0.5 * geometry with respect to every depth (every fourth row and column, SUB4) and every pose.
"""
import os
import sys

import numpy as np

sys.dont_write_bytecode = True
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "sc-sfmlearner-release_b200"))
sys.path.insert(0, HERE)

import torch  # noqa: E402

import loss_edge_inputs as E  # noqa: E402


def np32(t):
    return t.detach().to(torch.float32).cpu().numpy()


def main():
    import importlib
    torch.set_num_threads(8)
    path = os.path.abspath(sys.argv[1])
    sys.path.insert(0, path)
    iw, lf = importlib.import_module("inverse_warp"), importlib.import_module("loss_functions")
    sys.path.remove(path)
    out = {}
    for name in E.GOLDEN_SETTINGS:
        (tgt, refs, K, td, rd, ps, pi), n_scales, flags, pm = E.golden_setting(name)
        out[f"{name}_in_checksum"] = np.array(E.checksums((tgt, refs, K, td, rd, ps, pi)), np.float64)
        td = [t.clone().requires_grad_(True) for t in td]
        rd = [[t.clone().requires_grad_(True) for t in r] for r in rd]
        ps = [t.clone().requires_grad_(True) for t in ps]
        pi = [t.clone().requires_grad_(True) for t in pi]
        iw.pixel_coords = None
        p, g = lf.compute_photo_and_geometry_loss(tgt, refs, K, td, rd, ps, pi, n_scales, *flags, pm)
        (p + 0.5 * g).backward()
        out[f"{name}_loss"] = np.array([float(p.detach()), float(g.detach())], np.float32)
        for s, t in enumerate(td):
            out[f"{name}_tgt_depth_s{s}"] = np32(t.grad)[E.SUB4]
        for i, r in enumerate(rd):
            for s, t in enumerate(r):
                out[f"{name}_ref_depth{i}_s{s}"] = np32(t.grad)[E.SUB4]
        for i in range(len(ps)):
            out[f"{name}_pose{i}"] = np32(ps[i].grad)
            out[f"{name}_pose_inv{i}"] = np32(pi[i].grad)
    f = os.path.join(HERE, "loss_edges.npz")
    np.savez_compressed(f, **out)
    print(f, os.path.getsize(f) // 1024, "KiB")


if __name__ == "__main__":
    main()
