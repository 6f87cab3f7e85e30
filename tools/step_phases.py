"""Time graph-replayed MADNet steps per train op at the headline shape (1280x384, one frame); prints one JSON line.

Modes: NONE (forward + full-resolution loss), MAD module 0..4 (+ that module's loss, backward and momentum update) and
FULL.  Each mode's step graph is captured once and then replayed back to back; `--replays` replays per mode and round,
timed with CUDA events, the modes interleaved over `--rounds` rounds.  A step's input and scalars stay on the device.

For MAD module g the most that running its train op beside the rest of the forward can save is
min(t(MAD g) - t(NONE), the forward after module g's disparity exists).  The second term is estimated from an
instrumented NONE replay (event nodes inside the step graph): the forward convolutions after the head conv of the
module's level (module 4: none), the correlations of the later levels and the full-resolution loss.

--reprojection-scale 1 2 4 also times every MAD module with its loss at 1/2 and 1/4 resolution (`MAD<g>_s<s>`), each
scale on an engine of its own, interleaved with the rest.

    python tools/step_phases.py [--replays 300] [--rounds 3] [--height 384] [--width 1280] [--reprojection-scale 1 ...]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'real-time-self-adaptive-deep-stereo_b200')
for p in (ROOT, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, sm, sm_max = [s.strip() for s in out.split(',')]
        return {'gpu': name, 'power_limit': power, 'sm_clock': sm, 'sm_clock_max': sm_max}
    except Exception as ex:
        return {'gpu': torch.cuda.get_device_name(0), 'power_limit': 'unknown (%s)' % type(ex).__name__}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--replays', type=int, default=300)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--height', type=int, default=384)
    ap.add_argument('--width', type=int, default=1280)
    ap.add_argument('--reprojection-scale', type=int, nargs='+', default=[1],
                    help='MAD module losses at 1/s resolution; 1 (the NONE / FULL / MAD<g> modes) must be among them')
    a = ap.parse_args()
    if 1 not in a.reprojection_scale:
        ap.error('--reprojection-scale: include 1')
    import Nets
    from madstereo.adaptation import OnlineAdaptation
    from madstereo.engine import MODE_FULL, MODE_MAD, MODE_NONE
    from madstereo.synthetic import init_params, make_pair
    torch.cuda.set_device(0)
    left, right, _ = make_pair(a.height, a.width, seed=100)
    lt = torch.from_numpy(np.rint(left).clip(0, 255).astype(np.float32)).cuda()
    rt = torch.from_numpy(np.rint(right).clip(0, 255).astype(np.float32)).cuda()
    sys.stdout, real_stdout = sys.stderr, sys.stdout           # the reference-style banner stays off stdout
    net = Nets.get_stereo_net('MADNet', dict(left_img=lt, right_img=rt, split_layers=[None], sequence=True,
                                             train_portion='BEGIN', bulkhead=True, warping=True, context_net=True,
                                             radius_d=2, stride=1, is_training=False))
    cfg = json.load(open(os.path.join(PKG, 'block_config', 'MadNet_full.json')))
    ad = OnlineAdaptation(net, mode='MAD', train_config=cfg, lr=1e-4, sample_mode='SEQUENTIAL')
    eng = net.engine
    ad.load_weights(init_params(eng.layers, seed=42))
    eng.set_input(lt, rt)
    scaled = {}                                    # scale -> an engine whose MAD module losses run at 1/scale
    for sc in sorted(set(a.reprojection_scale) - {1}):
        n2 = Nets.get_stereo_net('MADNet', dict(left_img=lt, right_img=rt, split_layers=[None], sequence=True,
                                                train_portion='BEGIN', bulkhead=True, warping=True, context_net=True,
                                                radius_d=2, stride=1, is_training=False))
        ad2 = OnlineAdaptation(n2, mode='MAD', train_config=cfg, lr=1e-4, sample_mode='SEQUENTIAL', reprojection_scale=sc)
        ad2.load_weights(init_params(n2.engine.layers, seed=42))
        n2.engine.set_input(lt, rt)
        scaled[sc] = n2.engine
    sys.stdout = real_stdout

    modes = [('NONE', MODE_NONE, 0, eng)] + [('MAD%d' % g, MODE_MAD, g, eng) for g in range(eng.n_groups)] + \
        [('FULL', MODE_FULL, 0, eng)] + [('MAD%d_s%d' % (g, sc), MODE_MAD, g, e) for sc, e in scaled.items()
                                         for g in range(e.n_groups)]
    run = lambda m, g, e=eng: e.run(m, g, 0, m != MODE_NONE, 1e-4, 0.9, 1.0)
    for _, m, g, e in modes:                       # capture + warm-up
        for _ in range(5):
            run(m, g, e)
    torch.cuda.synchronize()
    times = {name: [] for name, _, _, _ in modes}
    for _ in range(a.rounds):
        for name, m, g, e in modes:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.replays):
                run(m, g, e)
            e1.record()
            e1.synchronize()
            times[name].append(1e3 * e0.elapsed_time(e1) / a.replays)

    # the forward after each module's disparity, from one instrumented NONE replay (profiling 2)
    eng.profile(2)
    for _ in range(2):
        run(MODE_NONE, 0)
    torch.cuda.synchronize()
    eng.profile(2)
    n_prof = 20
    for _ in range(n_prof):
        run(MODE_NONE, 0)
    torch.cuda.synchronize()
    cats, per_layer = eng.profile_read(), eng.profile_layers()
    eng.profile(0)
    fwd_us = {i: 1e3 * per_layer[l.name]['fwd']['ms'] / n_prof for i, l in enumerate(eng.layers)
              if 'fwd' in per_layer.get(l.name, {})}
    corr_us = 1e3 * cats['corr_fwd']['ms'] / n_prof / 5           # one correlation per level 6..2
    loss_us = 1e3 * cats['loss']['ms'] / n_prof
    head = {g: 12 + 6 * g + 5 for g in range(4)}                   # estimator disp6 of level 6 - g
    t_none = float(np.median(times['NONE']))
    ceiling = {}
    for g in range(eng.n_groups):
        after = head.get(g, len(eng.layers) - 1)
        tail = sum(v for i, v in fwd_us.items() if i > after) + corr_us * (4 - g if g < 4 else 0) + loss_us
        t_mad = float(np.median(times['MAD%d' % g]))
        ceiling['MAD%d' % g] = {'us': round(min(t_mad - t_none, tail), 1), 'train_op_us': round(t_mad - t_none, 1),
                                'forward_after_fork_us': round(tail, 1)}
    mad = [float(np.median(times['MAD%d' % g])) for g in range(eng.n_groups)]
    res = gpu_info()
    res.update({'shape': '%dx%d, batch 1' % (a.width, a.height), 'replays_per_round': a.replays, 'rounds': a.rounds,
                'step_us': {k: [round(v, 1) for v in vs] for k, vs in times.items()},
                'step_us_median': {k: round(float(np.median(vs)), 1) for k, vs in times.items()},
                'mad_mean_us': round(float(np.mean(mad)), 1),
                'ceiling': ceiling,
                'ceiling_mean_frac_of_mad_step': round(float(np.mean([c['us'] for c in ceiling.values()])) / float(np.mean(mad)), 4)})
    print(json.dumps(res))


if __name__ == '__main__':
    main()
