"""Throughput of the live-demo features on one GPU; prints one JSON line.

  * steady-state adaptation steps per second at 320x512 (the demo's crop) for MADNet MAD and FULL, with Adam and with
    momentum, the four configurations alternated within one call;
  * the uint8 rescale + crop kernel for a 720p and a 1080p frame pair -> 480x640 -> 320x512, device-resident frames,
    alone and after on-device rectification, next to host cv2.remap of the same pair (what a grabber would otherwise do);
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


def camera_pair(h, w, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 256, (1, h, w, 3), dtype=torch.uint8, generator=g) for _ in range(2)]


def rectification_tables(h, w):
    """Tables of a plausible raw stereo rig (barrel distortion, a 2-degree rotation between the cameras)."""
    import cv2
    K = np.array([[0.7 * w, 0, w / 2], [0, 0.7 * w, h / 2], [0, 0, 1]])
    D = np.array([-0.3, 0.1, 1e-3, -5e-4, -0.02])
    R, _ = cv2.Rodrigues(np.radians([1.0, -2.0, 0.5]))
    r1, r2, p1, p2 = cv2.stereoRectify(K, D, K, D, (w, h), R, np.array([-0.12, 0.002, 0.001]),
                                       flags=cv2.CALIB_ZERO_DISPARITY, alpha=0)[:4]
    return [np.stack(cv2.initUndistortRectifyMap(K, D, r, p, (w, h), cv2.CV_32FC1), -1) for r, p in ((r1, p1), (r2, p2))]


def time_input(h, w, tables=None, iters=500):
    """Time of the camera-frame input path (optional rectify, rescale to 480x640, crop to 320x512) for one pair, in us:
    (back to back: events around `iters` calls, whatever bounds them, host or device, with frames and tables left in
    L2 from the previous call; cold: device time between events around each call, after a write of 128 MB that evicts
    L2 and keeps the device busy while the host enqueues the call, as a camera frame arriving after an adaptation
    step finds it)."""
    from madstereo.engine import StereoEngine
    eng = StereoEngine('MADNet', 1, 320, 512)
    eng.set_groups([]); eng.bind(); eng.set_resize((480, 640))
    if tables is not None:
        eng.set_rectification(*tables)
    l, r = (x.cuda() for x in camera_pair(h, w))
    for _ in range(20):
        eng.set_input(l, r)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        eng.set_input(l, r)
    b.record()
    b.synchronize()
    warm = 1e3 * a.elapsed_time(b) / iters
    flush = torch.empty(32 << 20, dtype=torch.float32, device='cuda')
    cold = []
    for _ in range(iters // 5):
        flush.fill_(1.0)
        a.record()
        eng.set_input(l, r)
        b.record()
        b.synchronize()
        cold.append(1e3 * a.elapsed_time(b))
    return warm, float(np.median(cold))


def time_host_remap(h, w, tables, iters=20):
    """What a grabber that rectifies on the host spends per pair: two cv2.remap calls (OpenCV's own threads)."""
    import cv2
    l, r = (x[0].numpy() for x in camera_pair(h, w))
    maps = [(t[..., 0].copy(), t[..., 1].copy()) for t in tables]
    def pair():
        return [cv2.remap(img, mx, my, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT) for img, (mx, my) in zip((l, r), maps)]
    pair()
    t0 = time.perf_counter()
    for _ in range(iters):
        pair()
    return 1e6 * (time.perf_counter() - t0) / iters


def input_paths():
    """Rescale + crop alone and with rectification for a 720p and a 1080p pair, plus host cv2.remap of the same pair.
    Traffic of the rectify pass: raw frames read, tables read, rectified frames written (then re-read by the rescale,
    counted once more), in MB."""
    import cv2
    out = {'host_cv2_threads': cv2.getNumThreads()}
    for name, (h, w) in (('720p', (720, 1280)), ('1080p', (1080, 1920))):
        tables = rectification_tables(h, w)
        warm, cold = time_input(h, w)
        out['resize_%s_to_320x512_us' % name] = round(warm, 2)
        out['resize_%s_to_320x512_cold_l2_us' % name] = round(cold, 2)
        warm, cold = time_input(h, w, tables)
        out['rectify_resize_%s_to_320x512_us' % name] = round(warm, 2)
        out['rectify_resize_%s_to_320x512_cold_l2_us' % name] = round(cold, 2)
        out['rectify_traffic_%s_mb' % name] = round(2 * h * w * (3 + 8 + 3 + 3) / 1e6, 1)
        out['host_cv2_remap_%s_pair_us' % name] = round(time_host_remap(h, w, tables), 1)
    return out


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
    res.update(input_paths())
    res.update(time_demo(a.demo_frames))
    print(json.dumps(res))


if __name__ == '__main__':
    main()
