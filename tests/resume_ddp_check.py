"""Launched by tests/test_resume_ddp_gpu.py under torchrun (2 ranks, one GPU each): train.py's main() with the command line after
`--`, on every rank.  Once the datasets are built each rank's Python and numpy streams are reseeded with a seed of its own, so
that ranks whose streams were mixed up draw differently.  Each rank then writes OUT/<tag>_rank<r>.pt: its augmentation draws in
order and its two parameter arenas at the end of the run.

    python -m torch.distributed.run --nproc-per-node 2 tests/resume_ddp_check.py OUT TAG -- synthetic --name x ...
"""
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "sc-sfmlearner-release_b200")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import train as T  # noqa: E402
from scsfm import augment  # noqa: E402
from scsfm.trainer import Trainer  # noqa: E402


def main():
    out, tag, argv = sys.argv[1], sys.argv[2], sys.argv[sys.argv.index("--") + 1:]
    rank = int(os.environ["RANK"])
    draws, trainers = [], []
    draw, make_loaders, init = augment.Draw.random.__func__, T.make_loaders, Trainer.__init__

    def recorded_draw(cls, in_h, in_w):
        d = draw(cls, in_h, in_w)
        draws.append((d.flip, float(d.x_scaling), float(d.y_scaling), d.offset_x, d.offset_y))
        return d

    def loaders(args, r, world, *a, **k):
        made = make_loaders(args, r, world, *a, **k)
        random.seed(1000 + r)
        np.random.seed(2000 + r)
        return made

    def kept_init(self, *a, **k):
        init(self, *a, **k)
        trainers.append(self)
    augment.Draw.random = classmethod(recorded_draw)
    T.make_loaders = loaders
    Trainer.__init__ = kept_init
    sys.argv = ["train.py"] + argv
    T.main()
    tr = trainers[0]
    torch.cuda.synchronize()
    torch.save({"draws": draws, "arenas": [tr.disp_net.flat_params().cpu(), tr.pose_net.flat_params().cpu()]},
               os.path.join(out, "%s_rank%d.pt" % (tag, rank)))


if __name__ == "__main__":
    main()
