"""Dense reconstruction of a KITTI odometry sequence: DispResNet's depth for every frame, fused with the sequence's poses into a
truncated signed distance field on the device (scsfm.fusion.TSDFVolume) and meshed into a coloured PLY.

    python test_vo.py --pretrained-posenet P --dataset-dir SEQS/ --sequence 09 --output-dir OUT/
    python run_fusion.py --pretrained-dispnet D --resnet-layers 18 --dataset-dir SEQS/ --sequence 09 --poses OUT/09.txt \\
        --voxel-size 0.2 --output OUT/09.ply

Frames are <dataset-dir><sequence>/image_2/*, read and resized as test_vo.py reads them.  Depth is 1 / disp in the network's
units and the poses (test_vo.py's output, or KITTI ground truth) must be in the same scale, so --voxel-size, --sdf-trunc and
--max-depth are in that unit too: there is no default voxel size.  The intrinsics are calib.txt's P2 scaled to the frames fed
to the network, or --intrinsics FX FY CX CY given at that size.  The volume's box is the camera centres' bounding box grown by
--max-depth on every side."""
import argparse
import os
import time

import numpy as np
import torch

parser = argparse.ArgumentParser(description='Fuse a sequence\'s depth and poses into a TSDF and mesh it',
                                 formatter_class=argparse.ArgumentDefaultsHelpFormatter)
parser.add_argument("--pretrained-dispnet", required=True, type=str, help="pretrained DispResNet path")
parser.add_argument('--resnet-layers', default=18, type=int, choices=[18, 50], help='depth network architecture')
parser.add_argument("--img-height", default=256, type=int, help="Image height")
parser.add_argument("--img-width", default=832, type=int, help="Image width")
parser.add_argument("--no-resize", action='store_true', help="no resizing is done")
parser.add_argument("--dataset-dir", type=str, required=True, help="Dataset directory (the sequences' parent, ending in /)")
parser.add_argument("--sequence", default='09', type=str, help="sequence to fuse")
parser.add_argument("--img-exts", default=['png', 'jpg', 'bmp'], nargs='*', type=str, help="images extensions to glob")
parser.add_argument("--conv-mode", default="tf32x3", choices=["fp32", "tf32", "tf32x3"], help="convolution arithmetic")
parser.add_argument("--batch-size", default=16, type=int, help="frames per network call")
parser.add_argument("--poses", required=True, type=str, help="camera-to-world poses, one KITTI-format row per frame")
parser.add_argument("--voxel-size", required=True, type=float, help="voxel size, in the poses' unit")
parser.add_argument("--sdf-trunc", default=None, type=float, help="truncation distance (default: 4 voxels)")
parser.add_argument("--max-depth", default=80.0, type=float, help="depths above this are ignored")
parser.add_argument("--intrinsics", default=None, type=float, nargs=4, metavar=("FX", "FY", "CX", "CY"),
                    help="intrinsics at the network's input size (instead of the sequence's calib.txt)")
parser.add_argument("--output", required=True, type=str, help="output mesh (binary PLY)")


def intrinsics(args, seq_dir, first_frame):
    """K [3,3] at the size the frames are fed to the network."""
    from PIL import Image
    from scsfm import inference_io as io
    with Image.open(first_frame) as im:
        src = (im.height, im.width)
    dst = src if args.no_resize else (args.img_height, args.img_width)
    if args.intrinsics is not None:
        fx, fy, cx, cy = args.intrinsics
        return np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float64)
    calib = os.path.join(seq_dir, "calib.txt")
    if not os.path.isfile(calib):
        raise SystemExit("no %s: give the camera with --intrinsics FX FY CX CY" % calib)
    return io.odom_intrinsics(calib, 2, src, dst).astype(np.float64)


@torch.no_grad()
def main(argv=None):
    args = parser.parse_args(argv)
    from scsfm import inference_io as io
    if not args.voxel_size > 0:
        raise SystemExit("--voxel-size must be positive, got %g" % args.voxel_size)
    seq_dir = os.path.join(args.dataset_dir + args.sequence)
    files = sorted(io.list_images(os.path.join(seq_dir, "image_2"), args.img_exts))
    if not files:
        raise SystemExit("no images in %s" % os.path.join(seq_dir, "image_2"))
    rows = io.read_poses(args.poses)
    if len(rows) != len(files):
        raise SystemExit("%s has %d poses for %d frames in %s" % (args.poses, len(rows), len(files), os.path.join(seq_dir, "image_2")))
    K = intrinsics(args, seq_dir, files[0])
    poses = np.tile(np.eye(4), (len(rows), 1, 1))
    poses[:, :3] = rows
    centres = poses[:, :3, 3]
    lo, hi = centres.min(0) - args.max_depth, centres.max(0) + args.max_depth

    import models
    from scsfm.fusion import TSDFVolume
    from scsfm.infer import Predictor
    vol = TSDFVolume(lo, hi, args.voxel_size, trunc=args.sdf_trunc, max_depth=args.max_depth)
    disp_net = models.DispResNet(args.resnet_layers, False).to("cuda")
    disp_net.load_state_dict(torch.load(args.pretrained_dispnet, map_location="cpu")['state_dict'])
    disp_net.set_conv_mode(args.conv_mode).eval()
    pred = Predictor(disp_net)
    print('{} frames to fuse, volume {} x {} x {} voxels of {}'.format(len(files), *vol.dims, args.voxel_size))

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i0, i1 in io.batches(len(files), args.batch_size):
        frames = np.stack([io.load_frame(f, args.img_height, args.img_width, not args.no_resize) for f in files[i0:i1]])
        depth = 1 / pred(io.network_input(frames))
        vol.integrate(depth, K, poses[i0:i1], torch.from_numpy(frames).cuda())
    verts, faces, colors = vol.mesh()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    io.write_ply(args.output, verts.cpu().numpy(), faces.cpu().numpy(), colors.cpu().numpy())
    print('{} bricks, {:.1f} MB on the device; mesh {} vertices, {} faces -> {}'.format(
        vol.num_bricks, vol.memory_bytes() / 2 ** 20, len(verts), len(faces), args.output))
    print('{:.1f} frames/s (decode, depth, fusion and mesh)'.format(len(files) / dt))
    return {"frames": len(files), "seconds": dt, "bricks": vol.num_bricks, "verts": len(verts), "faces": len(faces)}


if __name__ == '__main__':
    main()
