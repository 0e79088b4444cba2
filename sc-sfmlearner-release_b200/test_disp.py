"""predictions.npy (float64 [N,H,W] of 1/disp) for the Eigen evaluation, and the inference latency (the reference's
test_disp.py: same flags, defaults, output and "Avg Time / Avg Speed" lines), on the fused eval forward of DispResNet
replayed from a CUDA graph (scsfm.infer.Predictor).

Added flags: --conv-mode (as train.py) and --batch-size (1 = the reference's behaviour; the time per image is then the time
of a batch over its size).  Images are decoded with PIL and resized with Pillow BILINEAR when needed."""
import argparse
import os
import time

import numpy as np
import torch

parser = argparse.ArgumentParser(description='Script for DispNet testing with corresponding groundTruth',
                                 formatter_class=argparse.ArgumentDefaultsHelpFormatter)
parser.add_argument("--pretrained-dispnet", required=True, type=str, help="pretrained DispNet path")
parser.add_argument("--img-height", default=256, type=int, help="Image height")
parser.add_argument("--img-width", default=832, type=int, help="Image width")
parser.add_argument("--min-depth", default=1e-3)
parser.add_argument("--max-depth", default=80)
parser.add_argument("--dataset-dir", default='.', type=str, help="Dataset directory")
parser.add_argument("--dataset-list", default=None, type=str, help="Dataset list file")
parser.add_argument("--output-dir", default=None, required=True, type=str, help="Output directory for saving predictions in a big 3D numpy file")
parser.add_argument('--resnet-layers', required=True, type=int, default=18, choices=[18, 50], help='depth network architecture.')
parser.add_argument("--conv-mode", default="tf32x3", choices=["fp32", "tf32", "tf32x3"], help="convolution arithmetic")
parser.add_argument("--batch-size", default=1, type=int, help="images per network call")


@torch.no_grad()
def main(argv=None):
    args = parser.parse_args(argv)
    import models
    from scsfm import inference_io as io
    from scsfm.infer import Predictor

    disp_net = models.DispResNet(args.resnet_layers, False).to("cuda")
    disp_net.load_state_dict(torch.load(args.pretrained_dispnet, map_location="cpu")['state_dict'])
    disp_net.set_conv_mode(args.conv_mode).eval()
    pred = Predictor(disp_net)

    if args.dataset_list is not None:
        with open(args.dataset_list, 'r') as f:
            test_files = list(f.read().splitlines())
    else:
        test_files = io.list_images(args.dataset_dir, ['png'])
    print('{} files to test'.format(len(test_files)))
    os.makedirs(args.output_dir, exist_ok=True)

    avg_time = 0
    predictions = None
    for i0, i1 in io.batches(len(test_files), args.batch_size):
        tgt_img = io.network_input(np.stack([io.load_frame(f, args.img_height, args.img_width) for f in test_files[i0:i1]]))
        torch.cuda.synchronize()
        t_start = time.time()
        output = pred(tgt_img)
        torch.cuda.synchronize()
        avg_time += time.time() - t_start
        pred_disp = output.cpu().numpy()[:, 0]
        if predictions is None:
            predictions = np.zeros((len(test_files), *pred_disp.shape[1:]))
        predictions[i0:i1] = 1 / pred_disp
    np.save(os.path.join(args.output_dir, 'predictions.npy'), predictions)

    avg_time /= len(test_files)
    print('Avg Time: ', avg_time, ' seconds.')
    print('Avg Speed: ', 1.0 / avg_time, ' fps')


if __name__ == '__main__':
    main()
