"""Resumable training on the GPU: Trainer.state_dict() / load_state_dict() restore every bit a step depends on, in place (under a
captured graph too), and train.py --resume continues a run as if it had not stopped."""
import os
import sys

import numpy as np
import pytest
import torch

from helpers import rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda"
B, H, W = 2, 128, 416


def make(mode="tf32x3", cameras=0, frozen=False, seed=0):
    """A Trainer on freshly initialised networks (torch seed `seed`); cameras: 0 (none), 1 (theta [4]) or C (a bank [C,4]).
    frozen: DispResNet's encoder frozen and in eval mode (fine-tuning)."""
    import models
    from scsfm.camera import LearnedCamera
    from scsfm.trainer import Trainer
    torch.manual_seed(seed)
    d, p = models.DispResNet(18, False).to(DEV).train(), models.PoseResNet(18, False).to(DEV).train()
    if frozen:
        d.encoder.requires_grad_(False)
        d.encoder.eval()
    cam = None
    th = [[150.0 + 5 * c + seed, 160.0 - 3 * c, 205.0 + c, 62.0 - c] for c in range(max(cameras, 1))]
    if cameras == 1:
        cam = LearnedCamera(*th[0], H, W).to(DEV)
    elif cameras > 1:
        cam = LearnedCamera.bank(th, H, W).to(DEV)
    return Trainer(d, p, lr=1e-4, with_auto_mask=1, distributed=False, conv_mode=mode, camera=cam)


def batch(tr, seed):
    """(args, inputs) of one step of tr on the seeded batch `seed`."""
    from scsfm import synth
    from scsfm.augment import Draw
    from scsfm.camera import records
    tgt, refs, K = synth.triplet(seed, B, H, W)
    args = (tgt.to(DEV), [r.to(DEV) for r in refs])
    if tr.camera is None:
        return args, {"intrinsics": K.to(DEV)}
    draws = [Draw.given(H, W, (i + seed) % 2 == 0, 1.0 + 0.03 * i, 1.1 - 0.02 * i, i, 2 * i) for i in range(B)]
    inputs = {"aug": records(draws, W, DEV)}
    if tr.camera.theta.dim() == 2:
        inputs["camera_index"] = torch.arange(B, device=DEV, dtype=torch.int32) % tr.camera.theta.shape[0]
    return args, inputs


def run_steps(tr, seeds):
    for s in seeds:
        args, inputs = batch(tr, s)
        out = tr.step(*args, **inputs)
    torch.cuda.synchronize()
    return out


def through_file(sd, tmp_path):
    path = str(tmp_path / "state.pt")
    torch.save(sd, path)
    return torch.load(path)


def assert_identical(a, b, where="state"):
    """Two (nested) state dicts: the same keys, bit-identical tensors, equal numbers."""
    if isinstance(a, dict):
        assert list(a) == list(b), where
        for k in a:
            assert_identical(a[k], b[k], "%s.%s" % (where, k))
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), where
        for i, (x, y) in enumerate(zip(a, b)):
            assert_identical(x, y, "%s[%d]" % (where, i))
    elif isinstance(a, torch.Tensor):
        assert a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b), where
    else:
        assert a == b, where


def device_tensors(tr):
    """The tensors a captured step holds by address: the arenas, their operand mirrors, the moments, the step counters, theta and
    its Adam state, the num_batches_tracked arenas."""
    out = []
    for n in (tr.disp_net, tr.pose_net):
        m, v, _ = tr.optimizer.state[id(n)]
        out += [n._flat, n._flat_grad, n._flat_tf32, m, v] + [bn.num_batches_tracked for bn in n._bns]
    out.append(tr.optimizer._step)
    if tr.camera is not None:
        out += [tr.camera.theta] + list(tr._cam_state)
    return out


def mirror_is_exact(n, mode):
    from scsfm import nnops as O
    want = torch.empty_like(n._flat)
    (O.split_tf32 if mode == "tf32x3" else O.round_tf32)(n._flat, want)
    return torch.equal(n._flat_tf32, want)


# ---- 1. exact round trip ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["eager", "captured", "bank3", "frozen"])
def test_round_trip_is_bit_identical(case, tmp_path):
    """k = 3 steps, the state through a file into a fresh Trainer on differently initialised networks: every parameter,
    BatchNorm buffer, num_batches_tracked, Adam moment and step counter, theta and its Adam state come back bit for bit, and
    num_batches_tracked stays a view of the network's one counter arena."""
    cams = {"bank3": 3, "captured": 1}.get(case, 0)
    tr = make(cameras=cams, frozen=case == "frozen")
    if case == "captured":
        tr.capture(*batch(tr, 0)[0], **batch(tr, 0)[1])
    run_steps(tr, [1, 2, 3])
    saved = tr.state_dict()
    assert saved["optimizer"]["step"] == 3
    counts = {int(v) for k, v in saved["pose_net"].items() if k.endswith("num_batches_tracked")}
    assert len(counts) == 1 and counts.pop() > 0
    fresh = make(cameras=cams, frozen=case == "frozen", seed=1)
    fresh.optimizer._ensure_state()
    nbt = [[bn.num_batches_tracked.data_ptr() for bn in n._bns] for n in (fresh.disp_net, fresh.pose_net)]
    assert not torch.equal(fresh.disp_net.flat_params(), tr.disp_net.flat_params())
    fresh.load_state_dict(through_file(saved, tmp_path))
    assert_identical(fresh.state_dict(), saved)
    assert_identical(tr.state_dict(), saved)                      # state_dict() changes nothing
    for n, ptrs in zip((fresh.disp_net, fresh.pose_net), nbt):
        assert [bn.num_batches_tracked.data_ptr() for bn in n._bns] == ptrs
        assert all(bn.num_batches_tracked.data_ptr() == n.encoder._nbt[i].data_ptr() for i, bn in enumerate(n._bns))
        assert mirror_is_exact(n, "tf32x3")
    if cams:
        assert fresh.camera_state_dict()["step"] == 3 and tuple(fresh.camera.theta.shape) == ((4,) if cams == 1 else (cams, 4))


# ---- 2. continuation --------------------------------------------------------------------------------------------------------
def one_step(trainers, seed):
    """One step of every trainer on the same batch: (losses, [gradient arenas], [parameter changes]) per trainer."""
    before = [[n.flat_params().clone() for n in (t.disp_net, t.pose_net)] for t in trainers]
    args, inputs = batch(trainers[0], seed)
    losses = [[float(v) for v in t.step(*args, **inputs)] for t in trainers]
    torch.cuda.synchronize()
    return [(l, [n.flat_grads().clone() for n in (t.disp_net, t.pose_net)] + ([t.camera.theta.grad.clone()] if t.camera else []),
             [n.flat_params() - b for n, b in zip((t.disp_net, t.pose_net), b0)]) for t, l, b0 in zip(trainers, losses, before)]


def assert_same_step(ref, got, twin, seed):
    """One step of ref, got and twin on the same batch; got and twin hold bit-identical states.  got agrees with ref to the bounds
    of a captured step against an eager one: losses to rtol 2e-5, gradients to rel-L2 1e-4, and parameter changes to rel-L2 1e-4
    or 4x the change's own run-to-run noise (got against twin), whichever is larger: where a gradient is at the noise level, Adam
    turns its atomics-order noise into a change of full size (lr), and in tf32 that alone exceeds 1e-4."""
    (l_ref, g_ref, d_ref), (l_got, g_got, d_got), (_, _, d_twin) = one_step([ref, got, twin], seed)
    np.testing.assert_allclose(l_got, l_ref, rtol=2e-5)
    for a, b in zip(g_got, g_ref):
        assert rel_l2(a, b) < 1e-4
    for a, b, c in zip(d_got, d_ref, d_twin):
        assert float(b.abs().max()) > 0
        err, noise = rel_l2(a, b), rel_l2(a, c)
        print("parameter change: rel-L2 %.2e, run-to-run noise %.2e" % (err, noise))
        assert err < max(1e-4, 4 * noise), (err, noise)


@pytest.mark.parametrize("mode", ["tf32x3", "tf32"])
def test_restored_trainer_continues_the_run(mode, tmp_path):
    tr = make(mode, cameras=1)
    run_steps(tr, [1, 2, 3])
    sd = through_file(tr.state_dict(), tmp_path)
    fresh, twin = make(mode, cameras=1, seed=1), make(mode, cameras=1, seed=2)
    fresh.load_state_dict(sd)
    twin.load_state_dict(sd)
    assert_same_step(tr, fresh, twin, 4)
    assert fresh.optimizer.step_count == tr.optimizer.step_count == 4


# ---- 3. in place under a graph ----------------------------------------------------------------------------------------------
def test_load_under_a_captured_graph(tmp_path):
    """tf32, where a stale operand mirror (the old weights, TF32-rounded) cannot pass the continuation bounds: a Trainer that
    captured first and then loads another run's state replays that run's next step, with the same launches and addresses."""
    mode = "tf32"
    graphed = make(mode, cameras=1)
    graphed.capture(*batch(graphed, 0)[0], **batch(graphed, 0)[1])
    run_steps(graphed, [1])
    launches = graphed.launches_per_step
    ptrs = [t.data_ptr() for t in device_tensors(graphed)]
    other = make(mode, cameras=1, seed=2)
    run_steps(other, [5, 6, 7])
    sd = through_file(other.state_dict(), tmp_path)
    graphed.load_state_dict(sd)
    torch.cuda.synchronize()
    assert graphed._graph is not None and graphed.launches_per_step == launches
    assert [t.data_ptr() for t in device_tensors(graphed)] == ptrs
    for n in (graphed.disp_net, graphed.pose_net):
        assert mirror_is_exact(n, mode)
    assert_identical(graphed.state_dict(), sd)
    eager, twin = make(mode, cameras=1, seed=3), make(mode, cameras=1, seed=4)
    eager.load_state_dict(sd)
    twin.load_state_dict(sd)
    assert_same_step(eager, graphed, twin, 8)


# ---- 4. train.py end to end -------------------------------------------------------------------------------------------------
def run_train(monkeypatch, cwd, argv):
    """train.main() in this process with `argv`; returns (the augmentation draws in order, the number of captures)."""
    import train as T
    from scsfm import augment
    from scsfm.trainer import Trainer
    draws, captures = [], []
    orig_random, orig_capture = augment.Draw.random.__func__, Trainer.capture

    def record(cls, in_h, in_w):
        d = orig_random(cls, in_h, in_w)
        draws.append((d.flip, float(d.x_scaling), float(d.y_scaling), d.offset_x, d.offset_y))
        return d

    def capture(self, *a, **k):
        captures.append(1)
        return orig_capture(self, *a, **k)
    monkeypatch.chdir(cwd)
    monkeypatch.setattr(augment.Draw, "random", classmethod(record))
    monkeypatch.setattr(Trainer, "capture", capture)
    monkeypatch.setattr(sys, "argv", ["train.py"] + argv)
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    T.main()
    monkeypatch.undo()
    return draws, len(captures)


def rows(path):
    with open(path) as f:
        return f.read().splitlines()


@pytest.mark.parametrize("learn", [0, 1])
def test_train_resume_matches_the_uninterrupted_run(learn, tmp_path, monkeypatch):
    """--epochs 2 against --epochs 1 then --epochs 2 --resume DIR, on synthetic data with the GPU transforms: one run directory,
    whole epochs in the logs (rows a cut-off epoch wrote are dropped), epoch 2 in the checkpoints, the same augmentation draws
    in the resumed epoch, and the resumed process replays a captured step."""
    base = ["synthetic", "-b", str(B), "--synthetic-size", str(H), str(W), "--epoch-size", "3", "--gpu-augment", "1",
            "--learn-intrinsics", str(learn), "--print-freq", "1", "-j", "0"]
    (tmp_path / "a").mkdir()
    (tmp_path / "b").mkdir()
    full, cap_full = run_train(monkeypatch, tmp_path / "a", base + ["--name", "full", "--epochs", "2"])
    first, cap_first = run_train(monkeypatch, tmp_path / "b", base + ["--name", "cut", "--epochs", "1"])
    run_dir = tmp_path / "b" / "checkpoints" / "cut"
    assert len(os.listdir(run_dir)) == 1
    run_dir = run_dir / os.listdir(run_dir)[0]
    per_epoch = 3 * B
    assert len(full) == 2 * per_epoch and first == full[:per_epoch]
    log_full = run_dir / "progress_log_full.csv"
    with open(log_full, "a") as f:                                    # what an epoch cut off after two iterations leaves
        f.write("9.0\t9.0\t9.0\t9.0\n9.0\t9.0\t9.0\t9.0\n")
    header = rows(log_full)[0]
    resumed, cap_resumed = run_train(monkeypatch, tmp_path / "b", base + ["--name", "cut", "--epochs", "2", "--resume", str(run_dir)])
    assert resumed == full[per_epoch:]
    assert cap_full == cap_first == cap_resumed == 1
    assert len(os.listdir(tmp_path / "b" / "checkpoints" / "cut")) == 1
    lines = rows(log_full)
    assert len(lines) == 1 + 6 and lines[0] == header and not any(line.startswith("9.0") for line in lines)
    assert len(rows(run_dir / "progress_log_summary.csv")) == 1 + 2
    names = ["dispnet", "exp_pose"] + (["camera"] if learn else [])
    for name in names:
        assert torch.load(run_dir / ("%s_checkpoint.pth.tar" % name))["epoch"] == 2
    state = torch.load(run_dir / "training_state.pth.tar", weights_only=False)
    assert state["epoch"] == 2 and state["n_iter"] == 6 and state["log_rows"] == {"summary": 2, "full": 6}
    assert not os.path.exists(str(run_dir / "training_state.pth.tar.tmp"))
