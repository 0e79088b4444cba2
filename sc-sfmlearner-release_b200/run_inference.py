"""Depth / disparity images of a folder of pictures (the reference's run_inference.py: same flags, defaults and output
names), on the fused eval forward of DispResNet replayed from a CUDA graph (scsfm.infer.Predictor).

Added flags: --conv-mode (as train.py) and --batch-size (1 = the reference's behaviour; batching is exact in eval mode).
Images are decoded with PIL and resized with Pillow BILINEAR when needed (scsfm/inference_io.py)."""
import argparse
import os

import numpy as np
import torch

parser = argparse.ArgumentParser(description='Inference script for DispNet learned with \
                                 Structure from Motion Learner inference on KITTI Dataset',
                                 formatter_class=argparse.ArgumentDefaultsHelpFormatter)
parser.add_argument("--output-disp", action='store_true', help="save disparity img")
parser.add_argument("--output-depth", action='store_true', help="save depth img")
parser.add_argument("--pretrained", required=True, type=str, help="pretrained DispResNet path")
parser.add_argument("--img-height", default=256, type=int, help="Image height")
parser.add_argument("--img-width", default=832, type=int, help="Image width")
parser.add_argument("--no-resize", action='store_true', help="no resizing is done")
parser.add_argument("--dataset-list", default=None, type=str, help="Dataset list file")
parser.add_argument("--dataset-dir", default='.', type=str, help="Dataset directory")
parser.add_argument("--output-dir", default='output', type=str, help="Output directory")
parser.add_argument("--img-exts", default=['png', 'jpg', 'bmp'], nargs='*', type=str, help="images extensions to glob")
parser.add_argument('--resnet-layers', required=True, type=int, default=18, choices=[18, 50],
                    help='depth network architecture.')
parser.add_argument("--conv-mode", default="tf32x3", choices=["fp32", "tf32", "tf32x3"], help="convolution arithmetic")
parser.add_argument("--batch-size", default=1, type=int, help="images per network call")


@torch.no_grad()
def main(argv=None):
    args = parser.parse_args(argv)
    if not (args.output_disp or args.output_depth):
        print('You must at least output one value !')
        return
    import models
    from scsfm import inference_io as io
    from scsfm.infer import Predictor

    disp_net = models.DispResNet(args.resnet_layers, False).to("cuda")
    disp_net.load_state_dict(torch.load(args.pretrained, map_location="cpu")['state_dict'])
    disp_net.set_conv_mode(args.conv_mode).eval()
    pred = Predictor(disp_net)

    os.makedirs(args.output_dir, exist_ok=True)
    if args.dataset_list is not None:
        with open(args.dataset_list, 'r') as f:
            test_files = [os.path.join(args.dataset_dir, file) for file in f.read().splitlines()]
    else:
        test_files = io.list_images(args.dataset_dir, args.img_exts)
    print('{} files to test'.format(len(test_files)))

    for i0, i1 in io.batches(len(test_files), args.batch_size):
        frames = [io.load_frame(f, args.img_height, args.img_width, not args.no_resize) for f in test_files[i0:i1]]
        if len({fr.shape for fr in frames}) > 1:                 # --no-resize with mixed sizes: one image per call
            outs = [pred(io.network_input(fr[None]))[0] for fr in frames]
        else:
            outs = list(pred(io.network_input(np.stack(frames))))
        for file, output in zip(test_files[i0:i1], outs):
            output = output.cpu().numpy()[0]
            if args.output_disp:
                disp = io.colorize(output, output.max(), 'bone')
                io.save_png_like(os.path.join(args.output_dir, io.output_name(file, args.dataset_dir, "_disp")), disp)
            if args.output_depth:
                depth = io.colorize(1 / output, 10, 'rainbow')
                io.save_png_like(os.path.join(args.output_dir, io.output_name(file, args.dataset_dir, "_depth")), depth)


if __name__ == '__main__':
    main()
