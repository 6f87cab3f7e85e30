"""Cost of the adaptation drivers' --summary at 1280x384 (MADNet, MAD, one module per frame).

Times, on the current CUDA device:
  * a plain step (OnlineAdaptation.step with ground truth, as the online driver runs every frame) and a summary step (the
    same plus AdaptationSummary.add: the colorize kernels of the disparity and the ground truth, the device-to-host copies,
    PNG encoding and the event write), host clock around work that ends in a device synchronise;
  * the device time of the colorize kernels (ms_colorize_summary_u8 and ms_colorize) with CUDA events over many launches;
  * the host time of PNG encoding and of writing one event to the file.

    python tools/bench_summary.py [--iters 50] [--out /tmp/bench_summary.json]

Prints one JSON line; the GPU name and power limit are part of it.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'real-time-self-adaptive-deep-stereo_b200')
for p in (ROOT, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def gpu_info():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        q = torch.cuda.get_device_name()
    return q


def median_ms(fn, iters):
    times = []
    for _ in range(iters):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(times))


def event_ms(fn, iters):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    start.record()
    for _ in range(iters):
        fn()
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_summary.py needs a CUDA device')
    import Nets
    from madstereo import ops
    from madstereo.adaptation import OnlineAdaptation
    from madstereo.summary import AdaptationSummary, _image_value
    from madstereo.synthetic import make_pair
    from oracle.madnet import init_params

    h, w = 384, 1280
    torch.cuda.set_device(0)
    left, right, gt = make_pair(h, w, seed=3)
    lt, rt, gtt = torch.from_numpy(left).cuda(), torch.from_numpy(right).cuda(), torch.from_numpy(gt).cuda()
    net = Nets.get_stereo_net('MADNet', dict(left_img=lt, right_img=rt, split_layers=[None], sequence=True,
                                             train_portion='BEGIN', bulkhead=True))
    cfg = json.load(open(os.path.join(PKG, 'block_config', 'MadNet_full.json')))
    ad = OnlineAdaptation(net, mode='MAD', train_config=cfg, lr=1e-4, sample_mode='FIXED', fixed_id=2)
    ad.load_weights(init_params(seed=42))
    disp = net.get_disparities()[-1]

    with tempfile.TemporaryDirectory() as logdir:
        summ = AdaptationSummary(logdir)

        def plain():
            ad.step(lt, rt, gtt)

        def with_summary():
            out = ad.step(lt, rt, gtt)
            summ.add(0, out['epe'], out['bad3'], [('full_res_disp', disp.tensor()), ('gt_disp', gtt)])

        for _ in range(10):
            plain(); with_summary()
        t_plain, t_summary = [], []
        for _ in range(3):                        # alternate, so drifts of a shared host hit both alike
            t_plain.append(median_ms(plain, a.iters))
            t_summary.append(median_ms(with_summary, a.iters))

        d = disp.tensor()
        k_u8 = event_ms(lambda: ops.colorize_summary_image(d, cmap='jet'), 200)
        k_f32 = event_ms(lambda: ops.colorize_img(d, cmap='jet'), 200)
        img = ops.colorize_summary_image(d, cmap='jet').cpu().numpy()
        png_ms = median_ms(lambda: _image_value('full_res_disp/image', img), a.iters)
        writer = summ.writer

        def write_event():
            writer.add_scalar('EPE', 1.0, 0); writer.add_image('full_res_disp/image', img, 0); writer.flush()
        write_ms = median_ms(write_event, a.iters) - png_ms
        summ.close()

    res = {'gpu': gpu_info(), 'shape': [h, w], 'plain_step_ms': min(t_plain), 'summary_step_ms': min(t_summary),
           'summary_extra_ms': min(t_summary) - min(t_plain),
           'colorize_summary_u8_device_ms': k_u8, 'colorize_f32_device_ms': k_f32,
           'png_encode_host_ms': png_ms, 'event_write_host_ms': write_ms,
           'note': 'step times: median over --iters, best of 3 alternated rounds; kernel times: CUDA events over 200 calls '
                   '(including the Python wrapper\'s LUT upload and workspace allocation)'}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, 'w').write(line + '\n')


if __name__ == '__main__':
    main()
