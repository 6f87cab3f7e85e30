"""Continual online adaptation with proxy supervision -- the reference's TPAMI driver on the H100 engine.

Mirrors Stereo_Continual_Adaptation.py of the reference: the same flags (:309-330, incl. --dilation / --decay / --uf /
--saveWeights / --eval), list files `left;right;gt;proxy`, the loss `get_proxy_loss('mean_l1')` (masked L1 to proxy
disparities, weight 0.01 on the full-resolution loss / FULL train op :75,133 and 0.1 on the MAD module losses :112), a train
op only every `--dilation` frames (:212), the reward recurrence with --decay / --uf (:232-234), the reset on --SSIMTh
(:269-271) and the output files (`overall.csv`, `series.csv`, `histogram.csv`, `disparities/disparity_<step>.png`,
`weights/`).  Underneath: Nets.get_stereo_net + madstereo.adaptation.OnlineAdaptation(loss='proxy', ...).step, the masked-L1
loss is csrc/loss.cu:proxy_loss.  --reprojectionScale s compares the MAD module disparities with the proxy resized to 1/s
and divided by s (:95-112).  --summary writes the reference's TensorBoard summaries every 100 frames (:135-145, :207-209,
:259-260): scalars `EPE` and `bad3` (the engine's masked mean |d - gt| and fraction > 3 px, computed on those frames only),
images `full_res_disp/image`, `proxy_disp/image` and `gt_disp/image`, as the online driver writes them.

    python Stereo_Continual_Adaptation.py -l list.csv -o out --weights ckpt --modelName MADNet \
        --blockConfig block_config/MadNet_full.json --mode MAD --sampleMode PROBABILITY --dilation 1
"""
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
import Stereo_Online_Adaptation as online  # noqa: E402
from madstereo.summary import AdaptationSummary  # noqa: E402

MAX_DISP = 256
PIXEL_TH = 3


def build_parser():
    """The reference's argparse definition (:309-330): the online driver's flags plus the continual ones."""
    parser = online.build_parser()
    parser.description = 'Script for online Adaptation of a Deep Stereo Network'
    parser.add_argument("--eval", help="eval mode: DISP or DEPTH", choices=['DISP', 'DEPTH', 'SSIM'], default='DISP')
    parser.add_argument("--saveWeights", help="save the adapted model", action='store_true')
    parser.add_argument("--dilation", help="save the adapted model", type=int, default=1)
    parser.add_argument("--decay", help="save the adapted model", type=float, default=0.99)
    parser.add_argument("--uf", help="save the adapted model", type=float, default=0.01)
    return parser


def frame_errors(disp, gt):
    """EPE and D1 of one frame exactly as :243-249 (valid = gt > 0; outlier = error > 3 px and >= 5 %)."""
    val = gt > 0
    if not np.any(val):
        return float('nan'), float('nan')
    disp_diff = np.abs(gt[val] - disp[val])
    outliers = np.logical_and(disp_diff > 3, (disp_diff / gt[val]) >= 0.05)
    return float(np.mean(disp_diff)), float(np.mean(outliers) * 100.)


def build_model(args, train_config):
    import torch
    from madstereo.adaptation import OnlineAdaptation
    if not torch.cuda.is_available():
        raise SystemExit('Stereo_Continual_Adaptation.py needs a CUDA device (there is no CPU fallback)')
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
                             ssim_th=args.SSIMTh, loss='proxy', decay=args.decay, uf=args.uf, dilation=args.dilation,
                             reprojection_scale=args.reprojectionScale)
    return stereo_net, adapt


def run_loop(adapt, frames, args, get_disparity, log=print, summary=None, disparity_map=None):
    """The reference's while-loop (:183-282) around `adapt.step`; `frames` yields (left, right, gt, proxy, real_width).
    `summary` (an AdaptationSummary, or None): at every 100th step the engine also computes EPE / bad3 against gt, and
    they go to the summary with `disparity_map()`, the proxy and the ground truth."""
    avg_accumulator, d1_accumulator = [], []
    step = 0
    start_time = time.time()
    for left, right, gt, proxy, _real_width in frames:
        summary_now = summary is not None and summary.due(step)
        out = adapt.step(left, right, gt if summary_now else None, want_disp_mask=0b100000, proxy=proxy)
        if summary_now:
            summary.add(step, out['epe'], out['bad3'], [('full_res_disp', disparity_map()), ('proxy_disp', proxy),
                                                        ('gt_disp', gt)])
        disp = get_disparity()[-1]
        epe, d1 = frame_errors(disp, np.asarray(gt)[-1])
        d1_accumulator.append(d1)
        avg_accumulator.append(epe)
        if step % 100 == 0:
            with open(os.path.join(args.output, 'histogram.csv'), 'a') as f_out:
                f_out.write('%s\n' % adapt.fetch_counter)
            log('Step: %04d \tEPE:%.3f\tD1:%.3f\t' % (step, epe, d1))
            start_time = time.time()
        if args.logDispStep != -1 and step % args.logDispStep == 0:
            import cv2
            dispy_to_save = np.clip(disp.astype(np.uint16), 0, MAX_DISP)                  # (:279-280: cast first, then x 256)
            cv2.imwrite(os.path.join(args.output, 'disparities/disparity_{}.png'.format(step)), dispy_to_save * 256)
        step += 1
    return avg_accumulator, d1_accumulator, step, time.time() - start_time


def write_outputs(args, avg_accumulator, d1_accumulator):
    with open(os.path.join(args.output, 'overall.csv'), 'w+') as f_out:
        f_out.write('EPE\tD1\n')
        f_out.write('%.3f\t%.3f\n' % (np.asarray(avg_accumulator).mean(), np.asarray(d1_accumulator).mean()))
    with open(os.path.join(args.output, 'series.csv'), 'w+') as f_out:
        f_out.write('step\tEPE\tD1\n')
        for i, (a, b) in enumerate(zip(avg_accumulator, d1_accumulator)):
            f_out.write('%d & %.3f & %.3f\n' % (i, a, b))


def main(args, build=build_model, colorize=None):
    """`build` and `colorize` (the summary images' colour map, default the GPU kernel) can be replaced by tests."""
    with open(args.blockConfig) as json_data:
        train_config = json.load(json_data)
    online.check_reprojection_scale(args)
    data_set = data_reader.dataset(args.list, batch_size=1, crop_shape=args.imageShape, num_epochs=1, augment=False,
                                   is_training=False, shuffle=False, proxies=True)
    stereo_net, adapt = build(args, train_config)
    predictions = stereo_net.get_disparities()
    weights = args.weights
    if os.path.isdir(weights):
        weights = weights_utils.latest_checkpoint(weights)
        if weights is None:
            raise Exception('no usable checkpoint in directory {}'.format(args.weights))
    w_dict = weights_utils.load_weights(weights, adapt.get_variable_names())
    assert (len(w_dict) > 0)
    adapt.load_weights(w_dict, strict=False)
    print('Disparity Net Restored?: {}, number of restored variables: {}'.format(True, len(w_dict)))
    summary = AdaptationSummary(args.output, colorize) if args.summary else None
    try:
        avg, d1, step, _ = run_loop(adapt, data_set, args, get_disparity=lambda: predictions[-1].numpy(), summary=summary,
                                    disparity_map=lambda: predictions[-1].tensor())
    finally:
        if summary is not None:
            summary.close()
    print(adapt.fetch_counter)
    write_outputs(args, avg, d1)
    if args.saveWeights:
        os.makedirs(os.path.join(args.output, 'weights'), exist_ok=True)
        adapt.save_weights(os.path.join(args.output, 'weights', 'model-%d' % step))
        print('Checkpoint saved in {}/weights'.format(args.output))
    print('Result saved in {}'.format(args.output))
    print('All Done, Bye Bye!')


if __name__ == '__main__':
    parser = build_parser()
    args = parser.parse_args()
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
