"""Generate tests/golden/intrinsics.npz by running the UNMODIFIED reference: its fp32 gradients with respect to the camera
intrinsics, which it differentiates through intrinsics.inverse() and intrinsics @ pose_mat (inverse_warp.py:253,258).

Needs a checkout of the original SC-SfMLearner project:

    python tests/golden/make_golden_intrinsics.py /path/to/SC-SfMLearner-Release

Its modules are imported read-only (bytecode writing disabled).  The inputs are those of warp_loss.npz (make_golden.py,
rebuilt by helpers.golden_loss_inputs); their checksums are stored again here so that this file can be checked on its own.
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

from make_golden import _load_reference, np32  # noqa: E402

# upstream gradients of the stand-alone inverse_warp2 case (warped [B,3,H,W], projected depth, computed depth [B,1,H,W])
IW2_UPSTREAM_SEED = 21


def iw2_upstream(B, H, W):
    g = torch.Generator().manual_seed(IW2_UPSTREAM_SEED)
    return [torch.randn(B, c, H, W, generator=g) for c in (3, 1, 1)]


def golden_intrinsics(ref, out):
    from scsfm import synth
    iw, lf = ref["inverse_warp"], ref["loss_functions"]
    B, H, W = 2, 64, 128
    d = synth.loss_inputs(7, B, H, W, n_ref=2, n_scales=2)
    poses = [p * 3 for p in d["poses"]]
    poses_inv = [p * 3 for p in d["poses_inv"]]
    out["in_checksum"] = np.array([float(x.double().abs().sum()) for x in
                                   [d["tgt_img"], *d["ref_imgs"], d["intrinsics"], *d["tgt_depth"],
                                    *[t for r in d["ref_depths"] for t in r], *poses, *poses_inv]], np.float64)
    for pm in ("zeros", "border"):
        # (1) d(1*photo + 0.5*geo)/dK, flags (1,1,0) and (1,1,1), 2 scales, 2 references
        for flags in ((1, 1, 0), (1, 1, 1)):
            iw.pixel_coords = None
            K = d["intrinsics"].clone().requires_grad_(True)
            p, g = lf.compute_photo_and_geometry_loss(d["tgt_img"], d["ref_imgs"], K, d["tgt_depth"], d["ref_depths"], poses,
                                                      poses_inv, 2, *flags, pm)
            (p + 0.5 * g).backward()
            out[f"{pm}_loss_K{flags[0]}{flags[1]}{flags[2]}"] = np32(K.grad)
        # (2) inverse_warp2 of (tgt <- ref0) at scale 0 under a seeded upstream gradient on its three differentiable outputs
        iw.pixel_coords = None
        K = d["intrinsics"].clone().requires_grad_(True)
        w, v, pd, cd = iw.inverse_warp2(d["ref_imgs"][0], d["tgt_depth"][0], d["ref_depths"][0][0], poses[0], K, pm)
        ups = iw2_upstream(B, H, W)
        out["iw2_up_checksum"] = np.array([float(u.double().abs().sum()) for u in ups], np.float64)
        out["iw2_up_seed"] = np.array([IW2_UPSTREAM_SEED], np.int64)
        ((w * ups[0]).sum() + (pd * ups[1]).sum() + (cd * ups[2]).sum()).backward()
        out[f"{pm}_iw2_K"] = np32(K.grad)


def main():
    torch.manual_seed(0)
    torch.set_num_threads(8)
    ref = _load_reference(os.path.abspath(sys.argv[1]))
    out = {}
    golden_intrinsics(ref, out)
    path = os.path.join(HERE, "intrinsics.npz")
    np.savez_compressed(path, **out)
    print("intrinsics.npz", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
