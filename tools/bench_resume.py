"""Cost of resumable training: the size of train.py's training_state.pth.tar and the wall time to save it (Trainer.state_dict()
plus the atomic write, as train.py does at the end of every epoch) and to load it (torch.load plus Trainer.load_state_dict, as
train.py --resume does), for bench.py's kitti_r18 and kitti_r50 networks after one captured step.

    python tools/bench_resume.py [--repeats 3] [--dir DIR]

The file goes to a temporary directory (or DIR); times are the median of the repeats, each ending in a device synchronise.  The
card's name and power limit are printed with the numbers."""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "sc-sfmlearner-release_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from bench_finetune import card  # noqa: E402

NETS = {"kitti_r18": (18, 18, 4), "kitti_r50": (50, 50, 2)}       # bench.py: DispResNet / PoseResNet layers, frames per GPU


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--dir", default=None)
    args = ap.parse_args()
    import models
    import train as T
    from scsfm import synth
    from scsfm.trainer import Trainer
    if not torch.cuda.is_available():
        raise SystemExit("bench_resume needs a GPU")
    dev = torch.device("cuda", 0)
    H, W = 256, 832
    results = {"card": card()}
    for name, (dl, pl, B) in NETS.items():
        tgt, refs, K = synth.triplet(1234, B, H, W, 2, "kitti")
        step = (tgt.to(dev), [r.to(dev) for r in refs], K.to(dev))
        tr = Trainer(models.DispResNet(dl, False).to(dev).train(), models.PoseResNet(pl, False).to(dev).train(), distributed=False,
                     conv_mode="tf32x3")
        tr.capture(*step)
        tr.step(*step)
        torch.cuda.synchronize()
        with tempfile.TemporaryDirectory(dir=args.dir) as d:
            save, load = [], []
            for _ in range(args.repeats):
                t0 = time.perf_counter()
                T.save_training_state(d, {"trainer": tr.state_dict(), "epoch": 1, "rng": T.gather_rng_states(1, dev)})
                save.append(time.perf_counter() - t0)
                t0 = time.perf_counter()
                tr.load_state_dict(torch.load(os.path.join(d, T.TRAINING_STATE), map_location="cpu", weights_only=False)["trainer"])
                torch.cuda.synchronize()
                load.append(time.perf_counter() - t0)
            size = os.path.getsize(os.path.join(d, T.TRAINING_STATE))
        n = sum(x.numel() for x in (tr.disp_net.flat_params(), tr.pose_net.flat_params()))
        results[name] = {"arena_floats": n, "file_MB": round(size / 2 ** 20, 1), "save_s": round(statistics.median(save), 3),
                         "load_s": round(statistics.median(load), 3)}
        del tr
        torch.cuda.empty_cache()
    print(json.dumps(results))


if __name__ == "__main__":
    main()
