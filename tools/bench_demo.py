"""Throughput of the live-demo features on one GPU; prints one JSON line.

  * steady-state adaptation steps per second at 320x512 (the demo's crop) for MADNet MAD and FULL, with Adam and with
    momentum, the four configurations alternated within one call;
  * the uint8 rescale + crop kernel for a 720p frame pair -> 480x640 -> 320x512, device-resident frames;
  * the demo itself (Demo/Live_Adaptation_Demo.py, MAD, Adam) on an ImageList of synthetic 480x640 pairs at fps 0, with
    --output: frames per second including decode, host display copies, colormap and PNG writes.

Everything it writes goes to a temporary directory.

    python tools/bench_demo.py [--steps 200] [--rounds 3] [--demo-frames 200]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'real-time-self-adaptive-deep-stereo_b200')
for p in (ROOT, PKG, os.path.join(PKG, 'Demo')):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(',')]
        return {'gpu': name, 'power_limit': power}
    except Exception as ex:                         # the card name from torch is still the card name
        return {'gpu': torch.cuda.get_device_name(0), 'power_limit': 'unknown (%s)' % type(ex).__name__}


def build(mode, optimizer, h=320, w=512):
    import Nets
    from madstereo.adaptation import OnlineAdaptation
    from madstereo.synthetic import make_pair
    from oracle.madnet import init_params
    left, right, _ = make_pair(h, w, seed=3)
    lt, rt = torch.tensor(left).cuda(), torch.tensor(right).cuda()
    net = Nets.get_stereo_net('MADNet', dict(left_img=lt, right_img=rt, split_layers=[None], sequence=True,
                                             train_portion='BEGIN', bulkhead=(mode == 'MAD')))
    cfg = json.load(open(os.path.join(PKG, 'block_config', 'MadNet_full.json')))
    ad = OnlineAdaptation(net, mode=mode, train_config=cfg, lr=1e-4, sample_mode='SEQUENTIAL', optimizer=optimizer)
    ad.load_weights(init_params(seed=42))
    # a threshold no loss reaches: the timing must not include weight restores
    ad.ssim_th = float('inf')
    return ad, lt, rt


def time_steps(ad, lt, rt, steps):
    for _ in range(10):
        ad.step(lt, rt)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        ad.step(lt, rt)
    torch.cuda.synchronize()
    return steps / (time.perf_counter() - t0)


def time_resize(iters=500):
    from madstereo.engine import StereoEngine
    eng = StereoEngine('MADNet', 1, 320, 512)
    eng.set_groups([]); eng.bind(); eng.set_resize((480, 640))
    g = torch.Generator().manual_seed(0)
    l = torch.randint(0, 256, (1, 720, 1280, 3), dtype=torch.uint8, generator=g).cuda()
    r = torch.randint(0, 256, (1, 720, 1280, 3), dtype=torch.uint8, generator=g).cuda()
    for _ in range(20):
        eng.set_input(l, r)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        eng.set_input(l, r)
    b.record()
    b.synchronize()
    return 1e3 * a.elapsed_time(b) / iters


def time_demo(frames):
    import cv2
    import Live_Adaptation_Demo as demo
    from madstereo.synthetic import make_pair
    from madstereo.tf_checkpoint import write_checkpoint
    from oracle.madnet import init_params
    tmp = tempfile.mkdtemp(prefix='bench_demo_')
    try:
        lines = []
        for k in range(8):                          # 8 distinct pairs, cycled
            l, r, _ = make_pair(480, 640, seed=100 + k)
            for side, x in (('l', l), ('r', r)):
                cv2.imwrite(os.path.join(tmp, '%s%d.png' % (side, k)), np.clip(np.rint(x[0]), 0, 255).astype(np.uint8)[:, :, ::-1])
        for k in range(frames):
            lines.append('%s;%s' % (os.path.join(tmp, 'l%d.png' % (k % 8)), os.path.join(tmp, 'r%d.png' % (k % 8))))
        open(os.path.join(tmp, 'list.txt'), 'w').write('\n'.join(lines) + '\n')
        json.dump({'list': os.path.join(tmp, 'list.txt'), 'fps': 0}, open(os.path.join(tmp, 'camera.json'), 'w'))
        write_checkpoint(os.path.join(tmp, 'w.ckpt'), init_params(seed=42))
        args = demo.build_parser().parse_args([
            '--cameraName', 'ImageList', '--cameraConfig', os.path.join(tmp, 'camera.json'), '--weights',
            os.path.join(tmp, 'w.ckpt'), '--mode', 'MAD', '--blockConfig', os.path.join(PKG, 'block_config', 'MadNet_full.json'),
            '--SSIMTh', '1e9', '--output', os.path.join(tmp, 'out')])
        t0 = time.perf_counter()
        dd = demo.main(args)
        wall = time.perf_counter() - t0
        rec = dd.records
        ms = np.array([r['step_ms'] for r in rec[10:]])
        return {'demo_frames': len(rec), 'demo_fps_incl_setup': round(len(rec) / wall, 1),
                'demo_fps_steady': round((len(rec) - 11) / (rec[-1]['t'] - rec[10]['t']), 1),
                'demo_step_ms_median': round(float(np.median(ms)), 3)}
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=200)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--demo-frames', type=int, default=200)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    res = gpu_info()
    configs = [('MAD', 'adam'), ('MAD', 'momentum'), ('FULL', 'adam'), ('FULL', 'momentum')]
    built = {c: build(*c) for c in configs}
    rates = {c: [] for c in configs}
    for _ in range(a.rounds):
        for c in configs:
            rates[c].append(time_steps(*built[c], a.steps))
    res['steps_per_s_320x512'] = {'%s_%s' % c: [round(v, 1) for v in rates[c]] for c in configs}
    del built
    torch.cuda.empty_cache()
    res['resize_720p_to_320x512_us'] = round(time_resize(), 2)
    res.update(time_demo(a.demo_frames))
    print(json.dumps(res))


if __name__ == '__main__':
    main()
