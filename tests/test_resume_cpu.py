"""Host side of train.py --resume (no GPU): the random streams saved and restored per rank, the refusals of a command line that
cannot continue a run, the CSV logs cut back to whole epochs and the atomic save of the training state."""
import os
import random
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from helpers import free_port

CPU = torch.device("cpu")


def draws():
    """Values from every stream train.py's loop draws from, the augmentation's own draws included."""
    from scsfm.augment import Draw
    d = [Draw.random(128, 416) for _ in range(3)]
    return ([random.random(), float(np.random.uniform()), torch.rand(3).tolist()] +
            [(x.flip, float(x.x_scaling), float(x.y_scaling), x.offset_x, x.offset_y) for x in d])


def test_rng_round_trip():
    import train as T
    random.seed(5)
    np.random.seed(6)
    torch.manual_seed(7)
    draws()
    state = T.rng_state(CPU)
    assert state["cuda"] is None
    first = draws()
    assert draws() != first
    T.set_rng_state(state, CPU)
    assert draws() == first


def _gather_worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import train as T
    random.seed(100 + rank)
    np.random.seed(200 + rank)
    torch.manual_seed(300 + rank)
    mine = draws()
    random.seed(100 + rank)
    np.random.seed(200 + rank)
    torch.manual_seed(300 + rank)
    states = T.gather_rng_states(world, CPU)
    draws()
    ok = len(states) == world
    for r, s in enumerate(states):             # every rank's streams, in RANK order
        T.set_rng_state(s, CPU)
        ok = ok and (draws() == mine) == (r == rank)
    out[rank] = bool(ok)
    dist.destroy_process_group()


def test_gathered_rng_states_world2_gloo():
    with mp.Manager() as m:
        out = m.dict()
        mp.spawn(_gather_worker, args=(2, free_port(), out), nprocs=2, join=True)
        assert dict(out) == {0: True, 1: True}


# ---- refusals --------------------------------------------------------------------------------------------------------------
def _state(run_dir, world=1, cameras=0, **args):
    """A training state file with the fields the checks read."""
    saved = dict(resnet_layers=18, learn_intrinsics=int(cameras > 0), camera_groups="one" if cameras < 2 else "calibration")
    saved.update(args)
    trainer = {"camera": {"theta": torch.zeros(cameras, 4) if cameras > 1 else torch.zeros(4)}} if cameras else {}
    os.makedirs(run_dir, exist_ok=True)
    torch.save({"world_size": world, "args": saved, "trainer": trainer, "epoch": 1}, os.path.join(run_dir, "training_state.pth.tar"))
    return str(run_dir)


def _two_calibrations(root):
    """A dataset tree as CameraTable reads it: three training scenes, two distinct cam.txt matrices."""
    for i, scene in enumerate(("s0", "s1", "s2")):
        os.makedirs(os.path.join(root, scene))
        np.savetxt(os.path.join(root, scene, "cam.txt"), np.array([[200.0 + 10 * (i % 2), 0, 200], [0, 200, 60], [0, 0, 1]]))
    with open(os.path.join(root, "train.txt"), "w") as f:
        f.write("s0\ns1\ns2\n")
    return str(root)


def _main_refuses(monkeypatch, argv, match, world=None):
    import train as T
    monkeypatch.setattr(sys, "argv", ["train.py"] + argv + ["--name", "x"])
    if world is None:
        monkeypatch.delenv("WORLD_SIZE", raising=False)
    else:
        monkeypatch.setenv("WORLD_SIZE", str(world))
    with pytest.raises(SystemExit, match=match):
        T.main()


def test_resume_refusals(tmp_path, monkeypatch):
    run = _state(tmp_path / "run")
    _main_refuses(monkeypatch, ["synthetic", "--resume", run, "--pretrained-disp", "d.pth.tar"], "--resume.*--pretrained-disp")
    _main_refuses(monkeypatch, ["synthetic", "--resume", run, "--pretrained-pose", "p.pth.tar"], "--resume.*--pretrained-pose")
    _main_refuses(monkeypatch, ["synthetic", "--resume", str(tmp_path)], "--resume .*training_state.pth.tar")
    _main_refuses(monkeypatch, ["synthetic", "--resume", _state(tmp_path / "ddp", world=2)],
                  "--resume: the run was trained by 2 processes \\(WORLD_SIZE\\), this one has 1")
    _main_refuses(monkeypatch, ["synthetic", "--resume", run], "--resume: .*WORLD_SIZE", world=4)
    _main_refuses(monkeypatch, ["synthetic", "--resume", run, "--resnet-layers", "50"], "--resnet-layers 50, .*--resnet-layers 18")
    _main_refuses(monkeypatch, ["synthetic", "--resume", run, "--learn-intrinsics", "1", "--gpu-augment", "1"],
                  "--learn-intrinsics 1, .*--learn-intrinsics 0")
    data = _two_calibrations(tmp_path / "data")
    one = _state(tmp_path / "one", cameras=1)
    _main_refuses(monkeypatch, [data, "--resume", one, "--learn-intrinsics", "1", "--camera-groups", "calibration"],
                  "--camera-groups calibration, .*--camera-groups one")
    three = _state(tmp_path / "three", cameras=3)
    _main_refuses(monkeypatch, [data, "--resume", three, "--learn-intrinsics", "1", "--camera-groups", "calibration"],
                  "--resume: the run learned 3 cameras, the training scenes now give 2 \\(--camera-groups calibration\\)")


# ---- logs and the state file -----------------------------------------------------------------------------------------------
def test_logs_are_cut_back_to_the_saved_rows(tmp_path):
    import train as T
    path = str(tmp_path / "progress_log_full.csv")
    header = "train_loss\tphoto_loss\tsmooth_loss\tgeometry_consistency_loss\n"
    body = "".join("%d.5\t0.1\t0.2\t0.3\n" % i for i in range(5))
    with open(path, "w") as f:
        f.write(header + body)
    assert T.log_rows(path) == 5
    T.truncate_log(path, 3)
    with open(path) as f:
        assert f.read() == header + "".join(body.splitlines(True)[:3])
    assert T.log_rows(path) == 3
    T.truncate_log(path, 3)
    assert T.log_rows(path) == 3
    with pytest.raises(SystemExit, match="--resume: .* 3 data rows, fewer than the 4"):
        T.truncate_log(path, 4)


def test_state_save_is_atomic(tmp_path, monkeypatch):
    import train as T
    T.save_training_state(str(tmp_path), {"epoch": 1, "w": torch.arange(10)})
    path = tmp_path / "training_state.pth.tar"
    before = path.read_bytes()
    real_save = torch.save

    def dies_half_way(obj, f, *a, **k):
        real_save({"epoch": 2, "w": torch.arange(1000)}, f)
        f.seek(f.tell() // 2)
        f.truncate()
        raise KeyboardInterrupt("killed while saving")
    monkeypatch.setattr(torch, "save", dies_half_way)
    with pytest.raises(KeyboardInterrupt):
        T.save_training_state(str(tmp_path), {"epoch": 2, "w": torch.arange(1000)})
    monkeypatch.undo()
    assert path.read_bytes() == before
    state = torch.load(path)
    assert state["epoch"] == 1 and torch.equal(state["w"], torch.arange(10))
    assert sorted(os.listdir(tmp_path)) == ["training_state.pth.tar"]
    T.save_training_state(str(tmp_path), {"epoch": 2})
    assert torch.load(path) == {"epoch": 2}
