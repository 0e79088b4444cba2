"""KITTI trajectory of a sequence from PoseResNet (the reference's test_vo.py: same flags, defaults and output file
<output-dir><sequence>.txt, 12 columns in %1.8e).  All consecutive pairs run in batches through the fused eval forward
replayed from a CUDA graph (scsfm.infer.Predictor), pose_vec2mat runs on the device, and the integration is the reference's
float64 host loop global_pose @ inv(pose_mat), in the same order.

The network is built with pretrained=False (no ImageNet download: the checkpoint supplies the weights) and loaded with
strict=False as the reference does.  Added flags: --conv-mode (as train.py) and --batch-size (pairs per network call; 1 =
the reference's behaviour).  Images are decoded with PIL and resized with Pillow BILINEAR when needed."""
import argparse

import numpy as np
import torch

parser = argparse.ArgumentParser(description='Script for visualizing depth map and masks',
                                 formatter_class=argparse.ArgumentDefaultsHelpFormatter)
parser.add_argument("--pretrained-posenet", required=True, type=str, help="pretrained PoseNet path")
parser.add_argument("--img-height", default=256, type=int, help="Image height")
parser.add_argument("--img-width", default=832, type=int, help="Image width")
parser.add_argument("--no-resize", action='store_true', help="no resizing is done")
parser.add_argument("--dataset-dir", type=str, help="Dataset directory")
parser.add_argument("--output-dir", type=str, help="Output directory for saving predictions in a big 3D numpy file")
parser.add_argument("--img-exts", default=['png', 'jpg', 'bmp'], nargs='*', type=str, help="images extensions to glob")
parser.add_argument("--rotation-mode", default='euler', choices=['euler', 'quat'], type=str)
parser.add_argument("--sequence", default='09', type=str, help="sequence to test")
parser.add_argument("--conv-mode", default="tf32x3", choices=["fp32", "tf32", "tf32x3"], help="convolution arithmetic")
parser.add_argument("--batch-size", default=1, type=int, help="image pairs per network call")


@torch.no_grad()
def main(argv=None):
    args = parser.parse_args(argv)
    import os
    import models
    from inverse_warp import pose_vec2mat
    from scsfm import inference_io as io
    from scsfm.infer import Predictor

    weights_pose = torch.load(args.pretrained_posenet, map_location="cpu")
    pose_net = models.PoseResNet(18, False).to("cuda")
    pose_net.load_state_dict(weights_pose['state_dict'], strict=False)
    pose_net.set_conv_mode(args.conv_mode).eval()
    pred = Predictor(pose_net)

    image_dir = args.dataset_dir + args.sequence + "/image_2/"
    os.makedirs(args.output_dir, exist_ok=True)
    test_files = sorted(io.list_images(image_dir, args.img_exts))
    print('{} files to test'.format(len(test_files)))

    frames = [io.load_frame(f, args.img_height, args.img_width, not args.no_resize) for f in test_files]
    mats = []
    for i0, i1 in io.batches(len(frames) - 1, args.batch_size):
        img1 = io.network_input(np.stack(frames[i0:i1]))
        img2 = io.network_input(np.stack(frames[i0 + 1:i1 + 1]))
        mats.append(pose_vec2mat(pred(img1, img2), args.rotation_mode).cpu().numpy())
    poses = io.integrate(np.concatenate(mats) if mats else np.zeros((0, 3, 4), np.float32))
    np.savetxt(args.output_dir + args.sequence + ".txt", poses, delimiter=' ', fmt='%1.8e')


if __name__ == '__main__':
    main()
