"""Shared helpers for the parity tests."""
import socket

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


def oracle_train_step(tgt, refs, K, *, disp_layers=18, pose_layers=18, lr=1e-4, betas=(0.9, 0.999), weight_decay=0.0,
                      gpu="cuda", **step_cfg):
    """One step of the oracle's training loop (oracle/step.py:train_step; step_cfg = its loss switches, padding and w1..w3)
    from det_weights on the given inputs, evaluated three ways: "f32" and "f64" on the CPU, "f32gpu" through stock PyTorch /
    cuDNN on `gpu` (the caller turns cuDNN / matmul TF32 off).  Each gives (the four losses, every gradient autograd produced
    keyed "disp.*" / "pose.*" -- parameters left with grad None are absent --, the BatchNorm buffers after the step)."""
    from golden_util import det_weights
    from oracle import nets as N
    from oracle import step as OS
    assert not (torch.backends.cudnn.allow_tf32 or torch.backends.cuda.matmul.allow_tf32), "the fp32 GPU oracle needs TF32 off"
    out = {}
    for name, dt, dev in (("f32", torch.float32, "cpu"), ("f64", torch.float64, "cpu"), ("f32gpu", torch.float32, gpu)):
        d, p = N.DispResNet(disp_layers).to(dt).to(dev), N.PoseResNet(pose_layers).to(dt).to(dev)
        for net in (d, p):
            net.load_state_dict({k: v.to(dt).to(dev) for k, v in det_weights(net.state_dict()).items()})
            net.train()
        losses = OS.train_step(d, p, OS.make_optimizer(d, p, lr=lr, betas=betas, weight_decay=weight_decay), tgt.to(dt).to(dev),
                               [r.to(dt).to(dev) for r in refs], K.to(dt).to(dev), **step_cfg)
        out[name] = ([float(v) for v in losses],
                     {"disp." + k: q.grad.clone().cpu() for k, q in d.named_parameters() if q.grad is not None} |
                     {"pose." + k: q.grad.clone().cpu() for k, q in p.named_parameters() if q.grad is not None},
                     {"disp." + k: b.clone().cpu() for k, b in d.named_buffers()} |
                     {"pose." + k: b.clone().cpu() for k, b in p.named_buffers()})
    return out


class Adam64:
    """torch.optim.Adam in fp64 on one flat vector, as the reference of an fp32 Adam kernel compared per step on the parameter
    CHANGE.  The hyper-parameters are the fp32 values the kernel receives.  step(g) continues the fp64 trajectory from p0;
    step(g, before) starts the step from the parameters the kernel under test started from instead.  m and v carry over from
    step to step in fp64 either way."""

    def __init__(self, p0, lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0):
        f = lambda v: float(np.float32(v))  # noqa: E731
        self.lr, self.b1, self.b2, self.eps, self.wd = f(lr), f(betas[0]), f(betas[1]), f(eps), f(weight_decay)
        self.p = p0.detach().double().clone().requires_grad_(True)
        self.opt = torch.optim.Adam([self.p], lr=self.lr, betas=(self.b1, self.b2), eps=self.eps, weight_decay=self.wd,
                                    foreach=False)
        self.t = 0

    def step(self, grad, before=None):
        """Returns (change, size): the fp64 change of this step and the update's size, taken before m = b1 m + (1-b1) g
        cancels (where g undoes the previous steps the change itself is tiny, but the fp32 rounding of the two terms is not)."""
        self.t += 1
        with torch.no_grad():
            if before is not None:
                self.p.copy_(before.double())
            before = self.p.detach().clone()
        state = self.opt.state[self.p]
        m_prev = state["exp_avg"].clone() if state else torch.zeros_like(before)
        grad = grad.double().to(before.device)
        g_eff = grad + self.wd * before
        self.p.grad = grad
        self.opt.step()
        den = state["exp_avg_sq"].sqrt() / (1 - self.b2 ** self.t) ** 0.5 + self.eps
        size = self.lr / (1 - self.b1 ** self.t) * (self.b1 * m_prev.abs() + (1 - self.b1) * g_eff.abs()) / den
        return self.p.detach() - before, size


def assert_adam_change(got, want, size, after, grad, what=""):
    """An fp32 Adam step's parameter change `got` against the fp64 change `want`: within 1e-5 of the update's size, plus the
    rounding of the new fp32 parameter `after` (at most 2^-24 of its magnitude)."""
    got, want, size, after, grad = (torch.as_tensor(x).double() for x in (got, want, size, after, grad))
    err = (got - want).abs()
    bound = 1e-5 * size + 2.0 ** -24 * after.abs()
    worst = int(torch.argmax(err / bound.clamp_min(1e-300)))
    assert bool((err <= bound).all()), "%s: change %.9g vs fp64 %.9g at %d (g = %.3g, error %.3g of the update size)" % (
        what, float(got[worst]), float(want[worst]), worst, float(grad[worst]), float(err[worst] / size[worst]))


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


def free_port():
    """A free TCP port on 127.0.0.1 for a process group's rendezvous."""
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p
