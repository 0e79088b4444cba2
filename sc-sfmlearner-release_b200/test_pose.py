"""Absolute trajectory and rotation errors of PoseResNet on KITTI odometry snippets (the reference's test_pose.py: same flags,
defaults, printed results and <output-dir>/predictions.npy).

As in the reference: the network is PoseResNet(18, False) loaded with strict=False; snippets are 5 frames long whatever
--sequence-length says; the pair matrices come from euler pose_vec2mat whatever --rotation-mode says; only *.png frames of
<dataset-dir>/sequences/<seq>/image_2 are read, whatever --img-exts says; and the error table and predictions.npy have one row
per IMAGE, not per snippet, so they end in 4 zero rows per sequence, which the printed mean and std include.

Differences: sequences (fnmatch patterns under <dataset-dir>/sequences) are visited in sorted order, not in the order of a
Python set.  Each frame is decoded once (PIL; resized with Pillow BILINEAR when needed, as test_vo.py) and each consecutive
pair runs through the network once, in batches of --batch-size through the CUDA-graph Predictor, with pose_vec2mat on the
device; snippet j takes the matrices of pairs j..j+3 and composes them in float64 on the host as the reference does.
Added flags: --conv-mode (as train.py) and --batch-size."""
import argparse
import os

import numpy as np
import torch

parser = argparse.ArgumentParser(description='Script for PoseNet testing with corresponding groundTruth from KITTI Odometry',
                                 formatter_class=argparse.ArgumentDefaultsHelpFormatter)
parser.add_argument("pretrained_posenet", type=str, help="pretrained PoseNet path")
parser.add_argument("--img-height", default=256, type=int, help="Image height")
parser.add_argument("--img-width", default=832, type=int, help="Image width")
parser.add_argument("--no-resize", action='store_true', help="no resizing is done")
parser.add_argument("--min-depth", default=1e-3)
parser.add_argument("--max-depth", default=80)
parser.add_argument("--dataset-dir", type=str, help="Dataset directory")
parser.add_argument('--sequence-length', type=int, metavar='N', help='sequence length for testing', default=5)
parser.add_argument("--sequences", default=['09'], type=str, nargs='*', help="sequences to test")
parser.add_argument("--output-dir", default=None, type=str, help="Output directory for saving predictions in a big 3D numpy file")
parser.add_argument("--img-exts", default=['png', 'jpg', 'bmp'], nargs='*', type=str, help="images extensions to glob")
parser.add_argument("--rotation-mode", default='euler', choices=['euler', 'quat'], type=str)
parser.add_argument("--conv-mode", default="tf32x3", choices=["fp32", "tf32", "tf32x3"], help="convolution arithmetic")
parser.add_argument("--batch-size", default=1, type=int, help="image pairs per network call")

SEQ_LENGTH = 5


def evaluate(dataset_dir, sequences, pair_mats, load_frame):
    """Snippet trajectories [n_images, 5, 3, 4] and (ATE, RE) float32 [n_images, 2] over the sorted matching sequences; rows past
    the last snippet stay zero.  pair_mats(frames) -> float32 [len(frames) - 1, 3, 4], the matrix of every consecutive pair;
    load_frame(path) -> decoded frame."""
    from scsfm import inference_io as io
    names = io.kitti_sequences(dataset_dir, sequences)
    print('getting test metadata for theses sequences : {}'.format(names))
    files = [io.list_images(os.path.join(dataset_dir, "sequences", s, "image_2"), ["png"]) for s in names]
    total = sum(len(f) for f in files)
    print('{} snippets to test'.format(total))
    errors = np.zeros((total, 2), np.float32)
    predictions = np.zeros((total, SEQ_LENGTH, 3, 4))
    j = 0
    for name, imgs in zip(names, files):
        snippets = io.snippet_indices(len(imgs), SEQ_LENGTH)
        if len(snippets) == 0:
            continue
        gt = io.read_poses(os.path.join(dataset_dir, "poses", "{}.txt".format(name)))
        mats = pair_mats([load_frame(f) for f in imgs])
        for idx in snippets:
            final_poses = io.integrate(mats[idx[0]:idx[-1]]).reshape(SEQ_LENGTH, 3, 4)
            predictions[j] = final_poses
            errors[j] = io.pose_error(io.compensated_poses(gt, idx), final_poses)
            j += 1
    return predictions, errors


@torch.no_grad()
def main(argv=None):
    args = parser.parse_args(argv)
    import models
    from inverse_warp import pose_vec2mat
    from scsfm import inference_io as io
    from scsfm.infer import Predictor

    weights = torch.load(args.pretrained_posenet, map_location="cpu")
    pose_net = models.PoseResNet(18, False).to("cuda")
    pose_net.load_state_dict(weights['state_dict'], strict=False)
    pose_net.set_conv_mode(args.conv_mode).eval()
    pred = Predictor(pose_net)

    def pair_mats(frames):
        mats = []
        for i0, i1 in io.batches(len(frames) - 1, args.batch_size):
            img1 = io.network_input(np.stack(frames[i0:i1]))
            img2 = io.network_input(np.stack(frames[i0 + 1:i1 + 1]))
            mats.append(pose_vec2mat(pred(img1, img2)).cpu().numpy())
        return np.concatenate(mats)

    predictions, errors = evaluate(args.dataset_dir, args.sequences, pair_mats,
                                   lambda f: io.load_frame(f, args.img_height, args.img_width, not args.no_resize))
    mean_errors = errors.mean(0)
    std_errors = errors.std(0)
    error_names = ['ATE', 'RE']
    print('')
    print("Results")
    print("\t {:>10}, {:>10}".format(*error_names))
    print("mean \t {:10.4f}, {:10.4f}".format(*mean_errors))
    print("std \t {:10.4f}, {:10.4f}".format(*std_errors))

    if args.output_dir is not None:
        os.makedirs(args.output_dir, exist_ok=True)
        np.save(os.path.join(args.output_dir, 'predictions.npy'), predictions)
    return predictions, errors


if __name__ == '__main__':
    main()
