"""Prepare the training sets (the reference's data/prepare_train_data.py: same flags and defaults, same files written).

    python data/prepare_train_data.py /path/to/raw --dataset-format kitti_raw --test-scenes test_scenes.txt \
        --static-frames static_frames.txt --with-depth --width 832 --height 256 --dump-root kitti_256

Frames are decoded and encoded on the host; the resize (Pillow BILINEAR, as scipy.misc.imresize) and the Velodyne depth maps
run on the device (scsfm.prepare).  Two deviations from the reference: --test-scenes is required for kitti_raw (the
reference reads a test_scenes.txt next to its loader; point at the original project's data/test_scenes.txt), and the 10 %
validation split is drawn over the sorted scene prefixes, so train.txt / val.txt do not depend on PYTHONHASHSEED.
--depth-size-ratio must divide --height and --width (the reference indexes out of bounds otherwise).
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

parser = argparse.ArgumentParser()
parser.add_argument("dataset_dir", metavar='DIR', help='path to original dataset')
parser.add_argument("--dataset-format", type=str, default='kitti_raw', choices=["kitti_raw", "cityscapes", "kitti_odom"])
parser.add_argument("--static-frames", default=None,
                    help="list of imgs to discard for being static, if not set will discard them based on speed "
                         "(careful, on KITTI some frames have incorrect speed)")
parser.add_argument("--test-scenes", default=None,
                    help="kitti_raw only, required: the list of drives to leave out (the original project's data/test_scenes.txt)")
parser.add_argument("--with-depth", action='store_true',
                    help="If available (e.g. with KITTI), will store depth ground truth along with images, for validation")
parser.add_argument("--with-pose", action='store_true',
                    help="If available (e.g. with KITTI), will store pose ground truth along with images, for validation")
parser.add_argument("--no-train-gt", action='store_true', help="If selected, will delete ground truth depth to save space")
parser.add_argument("--dump-root", type=str, default='dump', help="Where to dump the data")
parser.add_argument("--height", type=int, default=128, help="image height")
parser.add_argument("--width", type=int, default=416, help="image width")
parser.add_argument("--depth-size-ratio", type=int, default=1, help="will divide depth size by that ratio")
parser.add_argument("--num-threads", type=int, default=4, help="number of threads to use (decoding and encoding)")
parser.add_argument("--batch-size", type=int, default=64, help="frames per device batch")


def parse(argv=None):
    args = parser.parse_args(argv)
    if args.dataset_format == "kitti_raw" and args.test_scenes is None:
        parser.error("--test-scenes is required for kitti_raw: the list of test drives to leave out "
                     "(the original project's data/test_scenes.txt)")
    r = args.depth_size_ratio
    if r < 1 or args.height % r or args.width % r or args.width // r < 2:
        parser.error("--depth-size-ratio %d must divide --height %d and --width %d (and leave a depth map at least 2 wide)"
                     % (r, args.height, args.width))
    if args.height < 1 or args.width < 1 or args.batch_size < 1:
        parser.error("--height, --width and --batch-size must be positive")
    return args


def make_loader(args):
    from scsfm import prepare as P
    if args.dataset_format == "kitti_raw":
        return P.KittiRaw(args.dataset_dir, args.test_scenes, static_frames_file=args.static_frames, img_height=args.height,
                          img_width=args.width, get_depth=args.with_depth, get_pose=args.with_pose,
                          depth_size_ratio=args.depth_size_ratio)
    if args.dataset_format == "kitti_odom":
        return P.KittiOdom(args.dataset_dir, img_height=args.height, img_width=args.width)
    return P.Cityscapes(args.dataset_dir, img_height=args.height, img_width=args.width)


def main(argv=None, ops=None, stats=None):
    args = parse(argv)
    from scsfm import prepare as P
    loader = make_loader(args)
    if ops is None:
        ops = P.DeviceOps()
    os.makedirs(args.dump_root, exist_ok=True)
    print('Found {} potential scenes'.format(len(loader.scenes)))
    print('Retrieving frames')
    scenes = [s for drive in loader.scenes for s in loader.collect(drive)]
    P.dump(scenes, args.dump_root, args.height, args.width, args.depth_size_ratio, ops, num_threads=args.num_threads,
           batch_size=args.batch_size, stats=stats)
    print('Generating train val lists')
    P.write_split(args.dump_root, remove_train_gt=args.with_depth and args.no_train_gt)
    return args


if __name__ == '__main__':
    main()
