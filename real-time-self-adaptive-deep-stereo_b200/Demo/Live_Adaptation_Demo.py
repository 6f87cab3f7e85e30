"""Live inference and adaptation demo -- the reference's Demo/Live_Adaptation_Demo.py on the H100 engine.

The reference's flags are kept flag for flag; `-1` disables --imageShape or --cropShape as their help says (with both
disabled the network runs at the camera size).  Additions for headless machines: --output DIR writes the displayed
disparity image of every frame and a log.csv (step, loss, module, reset, step ms) instead of opening windows, and
--maxFrames N stops after N frames.  The `ImageList` grabber replays a list file; --cameraConfig then names a JSON file
{"list": "<left;right list>", "fps": <frames per second, 0 = no pacing>}.  Any camera's configuration may also name
"calibration": "<stereo calibration file>" (madstereo.rectify) when its frames are raw: they are then rectified on the
device before the rescale.

    python Demo/Live_Adaptation_Demo.py --cameraName ImageList --cameraConfig cfg.json --weights ckpt/MADNet/kitti \\
        --mode MAD --blockConfig block_config/MadNet_full.json --output out --maxFrames 300
"""
import argparse
import json
import os
import queue
import sys
import threading

HERE = os.path.dirname(os.path.abspath(__file__))
PARENT = os.path.dirname(HERE)
for p in (PARENT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import grabber  # noqa: E402
import demo_model  # noqa: E402
import Nets  # noqa: E402


def build_parser():
    """The reference's argparse definition, flag for flag, then the headless additions."""
    parser = argparse.ArgumentParser(description='Real-time stereo live demo')
    parser.add_argument("--modelName", help="name of the stereo model to be used", default="MADNet", choices=Nets.STEREO_FACTORY.keys())
    parser.add_argument("--weights", help="path to the initial weights for the disparity estimation network", default=None)
    parser.add_argument("--mode", help="online adaptation mode: NONE - perform only inference, FULL - full online backprop, MAD - backprop only on portions of the network", choices=['NONE', 'FULL', 'MAD'], default='NONE')
    parser.add_argument("--lr", help="value for learning rate", default=0.0001, type=float)
    parser.add_argument("--blockConfig", help="path to the block_config json file", default='../block_config/MadNet_full.json')
    parser.add_argument("--imageShape", help='two int, reshape input images to this shape [height,width], -1 to disable', nargs='+', type=int, default=[480, 640])
    parser.add_argument("--cropShape", help='two int, crop input images to this shape [height,width], -1 to disable', nargs='+', type=int, default=[320, 512])
    parser.add_argument("--SSIMTh", help="reset network to initial configuration if loss is above this value", type=float, default=0.5)
    parser.add_argument("--cameraConfig", help="path to a configuration file for the camera", default='/home/alessio/code/Real-time-self-adaptive-deep-stereo/Demo/configuration.json')
    parser.add_argument("--cameraName", help="name of the camera grabber to build", default="ZED_Mini", choices=grabber.get_available_camera())
    parser.add_argument("--output", help="directory for the displayed disparity of every frame and log.csv; no windows are opened", default=None)
    parser.add_argument("--maxFrames", help="stop after this many frames", type=int, default=None)
    return parser


def shape_arg(v, flag):
    """[h, w] -> [h, w]; [-1] or [-1, -1] -> [None, None] (disabled)."""
    if len(v) >= 1 and v[0] == -1:
        return [None, None]
    if len(v) != 2:
        raise SystemExit('{} takes two integers (height width) or -1'.format(flag))
    return list(v)


def resolve(path):
    """The reference's relative defaults assume the working directory is Demo/."""
    if os.path.exists(path) or os.path.isabs(path):
        return path
    alt = os.path.join(HERE, path)
    return alt if os.path.exists(alt) else path


def main(args):
    image_shape = shape_arg(args.imageShape, '--imageShape')
    crop_shape = shape_arg(args.cropShape, '--cropShape')
    if args.weights is None:
        raise SystemExit('--weights is required: the TF random initialisers of the reference are not reproduced')
    if args.cameraName not in grabber.get_available_camera():
        raise SystemExit('camera grabber {} is not available here (available: {})'.format(
            args.cameraName, ', '.join(grabber.get_available_camera())))
    camera_cls = grabber._GRABBER_FACTORY[args.cameraName]
    calibration = None
    if getattr(camera_cls, 'needs_config', True):
        assert os.path.exists(args.cameraConfig), 'camera configuration {} not found'.format(args.cameraConfig)
        with open(args.cameraConfig) as f_in:
            calibration = json.load(f_in).get('calibration')

    # setup shared queue for the grabbed frames
    camera_frames = queue.Queue(1)

    # create camera grabber and disparity network
    dd = demo_model.RealTimeStereo(
        camera_frames,
        model_name=args.modelName,
        weight_path=args.weights,
        learning_rate=args.lr,
        block_config_path=resolve(args.blockConfig),
        image_shape=image_shape,
        crop_shape=crop_shape,
        SSIMTh=args.SSIMTh,
        mode=args.mode,
        output=args.output,
        max_frames=args.maxFrames,
        calibration=calibration)
    gg = grabber.get_camera(args.cameraName, camera_frames, config=args.cameraConfig, framerate=30)

    print('Threads ready to start')
    gg.start()
    dd.start()
    if args.output is None and sys.stdin is not None and sys.stdin.isatty():
        def wait_for_key():
            input('Press something to stop')
            dd.stop()
        threading.Thread(target=wait_for_key, daemon=True).start()
    dd.join()       # ends on a key press, at the end of the stream or after --maxFrames
    print('Requesting Stops')
    gg.stop()
    gg.join()
    print('Camera grabber stopped')
    print('detector stopped')
    if dd.error is not None:
        raise dd.error
    print('Goodbye')
    return dd


if __name__ == '__main__':
    main(build_parser().parse_args())
