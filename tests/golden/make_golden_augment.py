"""Writes tests/golden/augment.npz: inputs, random draws and outputs of the UNMODIFIED reference transform chain
(custom_transforms.py: RandomHorizontalFlip, RandomScaleCrop, ArrayToTensor, Normalize) on small seeded samples.

Needs a checkout of the original project (Pillow does the resize inside its code):
    python tests/golden/make_golden_augment.py /path/to/SC-SfMLearner-Release
The draws are recorded by replaying the reference's RNG call order (random.random(); np.random.uniform(1, 1.15, 2);
np.random.randint(scaled_h - in_h + 1); np.random.randint(scaled_w - in_w + 1)) from the same seeds.
"""
import os
import random
import sys

import numpy as np

sys.dont_write_bytecode = True
sys.path.insert(0, os.path.abspath(sys.argv[1]))
import custom_transforms as T  # noqa: E402  (the reference's)

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = [(0, 24, 40, 3), (1, 24, 40, 3), (2, 37, 53, 2), (3, 16, 64, 3), (5, 32, 48, 2), (8, 30, 30, 3)]


def main():
    out = {}
    chain = T.Compose([T.RandomHorizontalFlip(), T.RandomScaleCrop(), T.ArrayToTensor(),
                       T.Normalize(mean=[0.45, 0.45, 0.45], std=[0.225, 0.225, 0.225])])
    plain = T.Compose([T.ArrayToTensor(), T.Normalize(mean=[0.45, 0.45, 0.45], std=[0.225, 0.225, 0.225])])
    for seed, H, W, n in CASES:
        g = np.random.default_rng(100 + seed)
        # smooth-ish images (low-pass noise) so the bicubic overshoot / clipping paths are both exercised
        imgs = []
        for _ in range(n):
            a = g.integers(0, 256, (H // 4 + 2, W // 4 + 2, 3)).astype(np.float32)
            a = np.kron(a, np.ones((4, 4, 1), np.float32))[:H, :W]
            a = np.clip(a + g.normal(0, 20, a.shape), 0, 255)
            imgs.append(np.floor(a).astype(np.float32))            # integer-valued float32, like load_as_float of a JPEG
        K = np.array([[0.58 * W, 0, 0.49 * W], [0, 1.92 * H, 0.47 * H], [0, 0, 1]], np.float32)
        random.seed(seed)
        np.random.seed(seed)
        tens, K2 = chain([im.copy() for im in imgs], np.copy(K))
        # replay the draws
        random.seed(seed)
        np.random.seed(seed)
        flip = random.random() < 0.5
        xs, ys = np.random.uniform(1, 1.15, 2)
        sh, sw = int(H * ys), int(W * xs)
        oy = np.random.randint(sh - H + 1)
        ox = np.random.randint(sw - W + 1)
        p = "s%d_" % seed
        out[p + "images"] = np.stack(imgs).astype(np.uint8)
        out[p + "K"] = K
        out[p + "draws"] = np.array([float(flip), xs, ys, ox, oy], np.float64)
        out[p + "out"] = np.stack([t.numpy() for t in tens])
        out[p + "K_out"] = K2
        out[p + "plain"] = np.stack([t.numpy() for t in plain([im.copy() for im in imgs], np.copy(K))[0]])
        print(seed, H, W, n, "flip", flip, "scaled", sw, sh, "offset", ox, oy)
    np.savez_compressed(os.path.join(HERE, "augment.npz"), **out)
    print("wrote augment.npz", os.path.getsize(os.path.join(HERE, "augment.npz")), "bytes")


if __name__ == "__main__":
    main()
