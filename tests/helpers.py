"""Shared helpers for the parity tests."""
import numpy as np
import torch


def t(a, dtype=torch.float32, device="cpu"):
    return torch.from_numpy(np.asarray(a)).to(device=device, dtype=dtype)


SUB = (Ellipsis, slice(None, None, 2), slice(None, None, 2))      # the stored maps keep every second row and column


def _warp_inputs():
    """The seeded inputs the golden vectors of warp_loss.npz were computed from (tests/golden/make_golden.py)."""
    from scsfm import synth
    d = synth.loss_inputs(7, 2, 64, 128, n_ref=2, n_scales=2)
    return (d["tgt_img"], d["ref_imgs"], d["intrinsics"], d["tgt_depth"], d["ref_depths"], [p * 3 for p in d["poses"]],
            [p * 3 for p in d["poses_inv"]])


def golden_loss_inputs(g, dtype=torch.float32, device="cpu", n_scales=2, requires_grad=False):
    """Rebuild the (tgt_img, ref_imgs, K, tgt_depth, ref_depths, poses, poses_inv) tuple behind warp_loss.npz, checked against
    the stored checksums."""
    tgt, refs, K, td, rd, ps, pi = _warp_inputs()
    flat = [tgt, *refs, K, *td, *[x for r in rd for x in r], *ps, *pi]
    np.testing.assert_allclose([float(x.double().abs().sum()) for x in flat], g["in_checksum"], rtol=1e-6)

    def conv(x, leaf=False):
        x = x.detach().to(device=device, dtype=dtype)
        return x.requires_grad_(True) if leaf and requires_grad else x
    return (conv(tgt), [conv(r) for r in refs], conv(K), [conv(x, True) for x in td[:n_scales]],
            [[conv(x, True) for x in r[:n_scales]] for r in rd], [conv(x, True) for x in ps], [conv(x, True) for x in pi])


def error_pair():
    """The synthetic ground truth / prediction pair of the compute_errors golden values."""
    g = torch.Generator().manual_seed(3)
    gt = torch.rand(2, 64, 128, generator=g) * 90
    gt[gt < 9] = 0
    pred = (gt * (1 + 0.2 * torch.randn(2, 64, 128, generator=g))).abs() * 0.37 + 0.05
    return gt, pred


def rel_l2(a, b):
    a = torch.as_tensor(a, dtype=torch.float64).cpu()
    b = torch.as_tensor(b, dtype=torch.float64).cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def frac_within(a, b, tol):
    """Fraction of elements with |a-b| <= tol * max|b|."""
    a = torch.as_tensor(a, dtype=torch.float64).cpu()
    b = torch.as_tensor(b, dtype=torch.float64).cpu()
    return float(((a - b).abs() <= tol * b.abs().max()).double().mean())


def make_disk_dataset(root, H=128, W=160, scenes=("scene_a", "scene_b", "scene_v"), frames=5, seed=0):
    """A tiny dataset in the layout the reference's SequenceFolder crawls (datasets/sequence_folders.py:13-21): root/<scene>/
    NNNNNNN.jpg + cam.txt, train.txt / val.txt listing the scene folders (the last scene is the validation scene)."""
    import os
    import numpy as np
    from PIL import Image
    g = np.random.default_rng(seed)
    os.makedirs(root, exist_ok=True)
    for s in scenes:
        d = os.path.join(root, s)
        os.makedirs(d, exist_ok=True)
        base = np.kron(g.integers(40, 216, (H // 16 + 1, W // 16 + 2, 3)).astype(np.float32), np.ones((16, 16, 1), np.float32))
        for i in range(frames):
            im = base[:H, 2 * i:2 * i + W] + g.normal(0, 6, (H, W, 3))          # a slow pan: consecutive frames overlap
            Image.fromarray(np.clip(im, 0, 255).astype(np.uint8)).save(os.path.join(d, "%07d.jpg" % i), quality=95)
        np.savetxt(os.path.join(d, "cam.txt"), np.array([[0.58 * W, 0, 0.49 * W], [0, 1.92 * H, 0.47 * H], [0, 0, 1]]))
    with open(os.path.join(root, "train.txt"), "w") as f:
        f.write("".join(s + "\n" for s in scenes[:-1]))
    with open(os.path.join(root, "val.txt"), "w") as f:
        f.write(scenes[-1] + "\n")
    return root


def reference_loader_env():
    """Environment for a subprocess in which the original project's host-side loaders (datasets/*.py, custom_transforms.py as
    installed by __graft_entry__.build() into oracle/_ref/, or $SCSFM_REFERENCE_DIR, plus the stand-ins for path / imageio under
    baseline/stubs) are importable from PYTHONPATH, as train.py expects for real datasets.  None if neither holds them."""
    import os
    from oracle import reference
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    ref, stubs = reference.installed(), os.path.join(root, "baseline", "stubs")
    if ref is None:
        return None
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([stubs, ref] + ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    env["PYTHONDONTWRITEBYTECODE"] = "1"
    return env
