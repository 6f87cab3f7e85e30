"""Online adaptation of a deep stereo network -- the reference driver's command line on the H100 engine.

Mirrors Stereo_Online_Adaptation.py of the reference: the same flags (:290-307), the same output folder layout
(`config.json`, `params.sh`, `stats.csv`, `series.csv`, `disparities/disparity_<step>.png`, :262-288, :309-319) and the
same loop (:176-253).  What changed underneath: the graph construction and `sess.run` are `Nets.get_stereo_net` +
`madstereo.adaptation.OnlineAdaptation.step` (sampling, reward recurrence, reset and the CUDA step live there), the
`tf.data` reader is Data_utils/data_reader.py (host thread + pinned buffers; the next frame's copy overlaps the current
frame), `--weights` accepts a TensorFlow V2 checkpoint prefix or directory (read without TensorFlow) or an `.npz`, and
TensorBoard summaries (`--summary`) are accepted but not written.

    python Stereo_Online_Adaptation.py -l list.csv -o out --weights ckpt/MADNet/kitti/weights.ckpt \\
        --modelName MADNet --blockConfig block_config/MadNet_full.json --mode MAD --sampleMode PROBABILITY
"""
import argparse
import datetime
import json
import os
import shutil
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)

import Nets  # noqa: E402
from Data_utils import data_reader, weights_utils  # noqa: E402
from Sampler import sampler_factory  # noqa: E402

# static params
MAX_DISP = 256
PIXEL_TH = 3


def build_parser():
    """The reference's argparse definition (:290-307), flag for flag."""
    parser = argparse.ArgumentParser(description='Script for online Adaptation of a Deep Stereo Network')
    parser.add_argument("-l", "--list", help='path to the list file with frames to be processed', required=True)
    parser.add_argument("-o", "--output", help="path to the output folder where the results will be saved", required=True)
    parser.add_argument("--weights", help="path to the initial weights for the disparity estimation network", required=True)
    parser.add_argument("--modelName", help="name of the stereo model to be used", default="Dispnet", choices=Nets.STEREO_FACTORY.keys())
    parser.add_argument("--numBlocks", help="number of CNN portions to train at each iteration", type=int, default=1)
    parser.add_argument("--lr", help="value for learning rate", default=0.0001, type=float)
    parser.add_argument("--blockConfig", help="path to the block_config json file", required=True)
    parser.add_argument("--sampleMode", help="choose the sampling heuristic to use", choices=sampler_factory.AVAILABLE_SAMPLER, default='SAMPLE')
    parser.add_argument("--fixedID", help="index of the portions of network to train, used only if sampleMode=FIXED", type=int, nargs='+', default=[0])
    parser.add_argument("--reprojectionScale", help="compute all loss function at 1/reprojectionScale", default=1, type=int)
    parser.add_argument("--summary", help='flag to enable tensorboard summaries', action='store_true')
    parser.add_argument("--imageShape", help='two int for the size of the crop extracted from each image [height,width]', nargs='+', type=int, default=[320, 1216])
    parser.add_argument("--SSIMTh", help="reset network to initial configuration if loss is above this value", type=float, default=0.5)
    parser.add_argument("--sampleFrequency", help="sample new network portions to train every K frame", type=int, default=1)
    parser.add_argument("--mode", help="online adaptation mode: NONE - perform only inference, FULL - full online backprop, MAD - backprop only on portions of the network", choices=['NONE', 'FULL', 'MAD'], default='MAD')
    parser.add_argument("--logDispStep", help="save disparity every K step, -1 to disable", default=-1, type=int)
    return parser


def write_stats(path, epe_array, bad3_array, exec_time, step, reset_counter, num_predictions, fetch_counter, sample_distribution):
    """stats.csv exactly as :262-281 writes it."""
    epe_acc, bad3_acc = np.sum(epe_array), np.sum(bad3_array)
    with open(path, 'w+') as f_out:
        f_out.write('Metrics,cumulative,average\n')
        f_out.write('EPE,{},{}\n'.format(epe_acc, epe_acc / step))
        f_out.write('bad3,{},{}\n'.format(bad3_acc, bad3_acc / step))
        f_out.write('time,{},{}\n'.format(exec_time, exec_time / step))
        f_out.write('FPS,{}\n'.format(1 / (exec_time / step)))
        f_out.write('#resets,{}\n'.format(reset_counter))
        f_out.write('Blocks')
        for n in range(num_predictions):
            f_out.write(',{}'.format(n))
        f_out.write(',final\n')
        f_out.write('fetch_counter')
        for c in fetch_counter:
            f_out.write(',{}'.format(c))
        f_out.write('\n')
        for c in sample_distribution:
            f_out.write(',{}'.format(c))
        f_out.write('\n')


def write_series(path, epe_array, bad3_array, exec_time, step):
    """series.csv exactly as :283-288 writes it."""
    step_time = exec_time / step
    time_array = [str(x * step_time) for x in range(len(epe_array))]
    with open(path, 'w+') as f_out:
        f_out.write('Iteration,Time,EPE,bad3\n')
        for i, (t, e, b) in enumerate(zip(time_array, epe_array, bad3_array)):
            f_out.write('{},{},{},{}\n'.format(i, t, e, b))


def save_disparity(path, dispy):
    """uint16 PNG, disparity x 256, clipped to [0, MAX_DISP] (:247-251)."""
    import cv2
    dispy_to_save = np.clip(dispy, 0, MAX_DISP)
    dispy_to_save = (dispy_to_save * 256.0).astype(np.uint16)
    cv2.imwrite(path, dispy_to_save)


def run_loop(adapt, frames, args, max_steps, get_disparity=None, log=print):
    """The reference's while-loop (:176-253) around `adapt.step` (== one sess.run).  `frames` yields (left, right, gt)
    batches; returns the accumulators the writers need."""
    epe_accumulator, bad3_accumulator = [], []
    exec_time = 0
    step = 0
    start_time = time.time()
    it = iter(frames)
    cur = next(it, None)
    while cur is not None:
        nxt = next(it, None)
        left, right, gt = cur
        out = adapt.step(left, right, gt, want_disp_mask=0b100000 if (args.logDispStep != -1 and step % args.logDispStep == 0) else 0,
                         prefetch=None if nxt is None else (nxt[0], nxt[1]))
        epe_accumulator.append(out['epe'])
        bad3_accumulator.append(out['bad3'])
        if step % 100 == 0:
            fbTime = (time.time() - start_time)
            exec_time += fbTime
            fbTime = fbTime / 100
            missing_time = (max_steps - step) * fbTime
            log('Step:{:4d}\tbad3:{:.2f}\tEPE:{:.2f}\tSSIM:{:.2f}\tf/b time:{:3f}\tMissing time:{}'.format(
                step, out['bad3'], out['epe'], out['loss'], fbTime, datetime.timedelta(seconds=missing_time)))
            start_time = time.time()
        if args.logDispStep != -1 and step % args.logDispStep == 0 and get_disparity is not None:
            save_disparity(os.path.join(args.output, 'disparities/disparity_{}.png'.format(step)), get_disparity()[0])
        step += 1
        cur = nxt
    return epe_accumulator, bad3_accumulator, exec_time, step


def build_model(args, train_config):
    """Network + adaptation object on the current CUDA device (graph construction of the reference, :54-128)."""
    import torch
    from madstereo.adaptation import OnlineAdaptation
    if not torch.cuda.is_available():
        raise SystemExit('Stereo_Online_Adaptation.py needs a CUDA device (there is no CPU fallback)')
    h, w = args.imageShape
    dev = torch.device('cuda', torch.cuda.current_device())
    left_buf = torch.zeros(1, h, w, 3, device=dev); right_buf = torch.zeros(1, h, w, 3, device=dev)
    net_args = {'left_img': left_buf, 'right_img': right_buf, 'split_layers': [None], 'sequence': True,
                'train_portion': 'BEGIN', 'bulkhead': True if args.mode == 'MAD' else False}
    stereo_net = Nets.get_stereo_net(args.modelName, net_args)
    print('Stereo Prediction Model:\n', stereo_net)
    if args.mode == 'MAD':
        assert (len(stereo_net.get_disparities()[:-1]) == len(train_config))
    adapt = OnlineAdaptation(stereo_net, mode=args.mode, train_config=train_config, lr=args.lr, sample_mode=args.sampleMode,
                             num_blocks=args.numBlocks, fixed_id=args.fixedID, sample_frequency=args.sampleFrequency,
                             ssim_th=args.SSIMTh)
    return stereo_net, adapt


def main(args, build=build_model):
    with open(args.blockConfig) as json_data:
        train_config = json.load(json_data)
    if args.reprojectionScale != 1:
        raise SystemExit('--reprojectionScale != 1 is not supported: the engine computes every loss at full resolution')
    if len(args.imageShape) != 2:
        raise SystemExit('--imageShape takes two integers: height width')

    data_set = data_reader.dataset(args.list, batch_size=1, crop_shape=args.imageShape, num_epochs=1, augment=False,
                                   is_training=False, shuffle=False, pin_memory=(build is build_model))
    stereo_net, adapt = build(args, train_config)
    predictions = stereo_net.get_disparities()

    # restore disparity inference weights (:150-154)
    weights = args.weights
    if os.path.isdir(weights):
        weights = weights_utils.latest_checkpoint(weights)
    w_dict = weights_utils.load_weights(weights, adapt.get_variable_names())
    assert (len(w_dict) > 0)
    adapt.load_weights(w_dict, strict=False)
    print('Disparity Net Restored?: {}, number of restored variables: {}'.format(True, len(w_dict)))

    max_steps = data_set.get_max_steps()
    epe_array, bad3_array, exec_time, step = run_loop(adapt, data_set, args, max_steps,
                                                      get_disparity=lambda: predictions[-1].numpy())
    write_stats(os.path.join(args.output, 'stats.csv'), epe_array, bad3_array, exec_time, step, adapt.reset_counter,
                len(predictions[:-1]) if args.mode == 'MAD' else len(predictions), adapt.fetch_counter, adapt.sample_distribution)
    write_series(os.path.join(args.output, 'series.csv'), epe_array, bad3_array, exec_time, step)
    print('Result saved in {}'.format(args.output))
    print('All Done, Bye Bye!')


if __name__ == '__main__':
    parser = build_parser()
    args = parser.parse_args()
    if args.summary:
        print('WARNING: --summary is accepted for command-line compatibility, but no TensorBoard summaries are written')
    if not os.path.exists(args.output):
        os.makedirs(args.output)
    if args.logDispStep != -1 and not os.path.exists(os.path.join(args.output, 'disparities')):
        os.makedirs(os.path.join(args.output, 'disparities'))
    shutil.copy(args.blockConfig, os.path.join(args.output, 'config.json'))
    with open(os.path.join(args.output, 'params.sh'), 'w+') as out:
        sys.argv[0] = os.path.join(os.getcwd(), sys.argv[0])
        out.write('#!/bin/bash\n')
        out.write('python3 ')
        out.write(' '.join(sys.argv))
        out.write('\n')
    main(args)
