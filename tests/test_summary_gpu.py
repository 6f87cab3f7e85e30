"""TensorBoard summaries on the H100: the colorize kernels (csrc/summary.cu) against the host restatement
(tests/colorize_oracle.py, pinned to the reference's colorize_img by tests/golden/reference_colorize.npz), and both
adaptation drivers end to end with --summary."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import PKG, ROOT

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import colorize_oracle as CO  # noqa: E402

pytestmark = pytest.mark.gpu


def _golden(key):
    return np.load(os.path.join(ROOT, 'tests', 'golden', 'reference_colorize.npz'))[key]


def _maps(batch):
    """(name, value [batch,H,W,1], vmin, vmax) cases: smooth maps with the batch max in the last image, exact .5 ties,
    a given range narrower than the data (out-of-range pixels), a constant map, and a full-resolution map."""
    rng = np.random.default_rng(batch)
    smooth = (rng.standard_normal((batch, 48, 80, 1)) * 20 + 40).astype(np.float32)
    smooth[-1, 5, 7, 0] = 500.0
    ties = np.repeat(_golden('ties_auto__jet__value'), batch, axis=0)
    big = (rng.uniform(0, 200, (batch, 384, 1280, 1))).astype(np.float32)
    return [('smooth', smooth, None, None), ('ties_auto', ties, None, None), ('ties_given', ties, 0.0, 1.0),
            ('narrow_range', smooth, 20.0, 60.0), ('vmin_only', smooth, 30.0, None), ('vmax_only', smooth, None, 45.0),
            ('constant', np.full((batch, 16, 24, 1), 3.25, np.float32), None, None), ('full_res', big, None, None)]


@pytest.mark.parametrize('batch', [1, 2])
@pytest.mark.parametrize('cmap', ['jet', None])
def test_colorize_kernels_equal_the_restatement(batch, cmap):
    from madstereo import ops
    lut = ops.colormap_lut(cmap)
    for name, value, vmin, vmax in _maps(batch):
        t = torch.from_numpy(value).cuda()
        got = ops.colorize_img(t, vmin=vmin, vmax=vmax, cmap=cmap).cpu().numpy()
        want = CO.colorize(value, lut, vmin, vmax)
        assert got.shape == (batch,) + value.shape[1:3] + (3,)
        assert np.array_equal(got, want), (name, int((got != want).any(-1).sum()))
        img = ops.colorize_summary_image(t, vmin=vmin, vmax=vmax, cmap=cmap).cpu().numpy()
        assert img.dtype == np.uint8 and img.shape == value.shape[1:3] + (3,)
        assert np.array_equal(img, CO.summary_image(value, lut, vmin, vmax)), name
        if name == 'constant':
            assert not got.any() and not img.any()
    # the batch-wide range: image 0 alone would be scaled differently
    if batch == 2:
        _, smooth, _, _ = _maps(2)[0]
        alone = ops.colorize_summary_image(torch.from_numpy(smooth[:1]).cuda(), cmap=cmap).cpu().numpy()
        both = ops.colorize_summary_image(torch.from_numpy(smooth).cuda(), cmap=cmap).cpu().numpy()
        assert not np.array_equal(alone, both)


def test_colorize_refuses_bad_arguments():
    from madstereo import ops
    from madstereo._lib import MadStereoError
    with pytest.raises(MadStereoError):
        ops.colorize_img(torch.zeros(1, 4, 4, 3, device='cuda'))
    with pytest.raises(MadStereoError):
        ops.colorize_img(torch.zeros(1, 4, 4, 1, device='cuda'), cmap='viridis')


# ---- drivers end to end -----------------------------------------------------------------------------------------------
def _dataset(tmp_path, continual):
    import cv2
    from madstereo.synthetic import make_pair
    from oracle.madnet import init_params
    lines = []
    for i in range(3):
        left, right, gt = make_pair(64, 128, seed=20 + i)
        names = []
        for tag, img in (('l', left[0]), ('r', right[0])):
            p = str(tmp_path / ('%s%d.png' % (tag, i)))
            cv2.imwrite(p, np.clip(img, 0, 255).astype(np.uint8)[..., ::-1]); names.append(p)
        for tag, scale in (('gt', 1.0), ('px', 1.1)):
            p = str(tmp_path / ('%s%d.png' % (tag, i)))
            cv2.imwrite(p, (np.clip(gt[0, ..., 0] * scale, 0, 255) * 256).astype(np.uint16)); names.append(p)
        lines.append(';'.join(names if continual else names[:3]))
    lst = tmp_path / 'list.csv'
    lst.write_text(''.join(lines[i % 3] + '\n' for i in range(201)))
    np.savez(str(tmp_path / 'w.npz'), **init_params(seed=42))
    return str(lst)


def _run(d, tmp_path, lst, out, summary):
    argv = ['-l', lst, '-o', str(out), '--weights', str(tmp_path / 'w.npz'), '--modelName', 'MADNet', '--blockConfig',
            os.path.join(PKG, 'block_config', 'MadNet_full.json'), '--mode', 'MAD', '--sampleMode', 'SEQUENTIAL',
            '--imageShape', '64', '128', '--logDispStep', '100'] + (['--summary'] if summary else [])
    os.makedirs(os.path.join(str(out), 'disparities'))
    rec = {'out': [], 'disp': {}, 'gt': {}, 'proxy': {}}

    def build(a, cfg):
        net, adapt = d.build_model(a, cfg)
        step = adapt.step

        def recording_step(left, right, gt=None, *args, **kw):
            r = step(left, right, gt, *args, **kw)
            k = len(rec['out'])
            rec['out'].append(r)
            if k % 100 == 0:
                rec['disp'][k] = net.get_disparities()[-1].numpy()
                rec['proxy'][k] = None if kw.get('proxy') is None else np.asarray(kw['proxy']).copy()
            return r
        adapt.step = recording_step
        return net, adapt
    d.main(d.build_parser().parse_args(argv), build=build)
    torch.cuda.synchronize()
    return rec


def _gt_frames(lst, continual):
    """The ground truth of steps 0, 100, 200 as the data reader yields it."""
    from Data_utils import data_reader
    frames = list(data_reader.dataset(lst, batch_size=1, crop_shape=[64, 128], num_epochs=1, augment=False, is_training=False,
                                      shuffle=False, proxies=continual))
    return {s: np.asarray(frames[s][2]) for s in (0, 100, 200)}


@pytest.mark.parametrize('driver', ['Stereo_Online_Adaptation', 'Stereo_Continual_Adaptation'])
def test_driver_summary_end_to_end(driver, tmp_path):
    import importlib
    import cv2
    from madstereo import ops
    from tensorboard.backend.event_processing import event_accumulator as ea
    d = importlib.import_module(driver)
    continual = 'Continual' in driver
    lst = _dataset(tmp_path, continual)
    plain, with_summary = tmp_path / 'plain', tmp_path / 'summary'
    _run(d, tmp_path, lst, plain, False)
    rec = _run(d, tmp_path, lst, with_summary, True)

    assert not [f for f in os.listdir(str(plain)) if f.startswith('events.out')]
    acc = ea.EventAccumulator(str(with_summary), size_guidance={ea.SCALARS: 0, ea.IMAGES: 0})
    acc.Reload()
    images = ['full_res_disp/image', 'proxy_disp/image', 'gt_disp/image'] if continual else ['full_res_disp/image', 'gt_disp/image']
    assert sorted(acc.Tags()['scalars']) == ['EPE', 'bad3'] and sorted(acc.Tags()['images']) == sorted(images)
    assert [e.step for e in acc.Scalars('EPE')] == [0, 100, 200]
    series = open(str(with_summary / 'series.csv')).read().splitlines()[1:]
    for e, b in zip(acc.Scalars('EPE'), acc.Scalars('bad3')):
        out = rec['out'][e.step]
        assert e.value == np.float32(out['epe']) and b.value == np.float32(out['bad3'])
        if continual:          # series.csv: the host EPE of the same frame, to 3 decimals
            assert abs(float(series[e.step].split(' & ')[1]) - e.value) <= 5e-4 + 1e-4 * e.value
        else:
            row = series[e.step].split(',')
            assert float(row[2]) == float(np.float32(out['epe'])) and float(row[3]) == float(np.float32(out['bad3']))
    jet = ops.colormap_lut('jet')
    gts = _gt_frames(lst, continual)

    def decoded(tag):
        return {e.step: cv2.imdecode(np.frombuffer(e.encoded_image_string, np.uint8), cv2.IMREAD_UNCHANGED)[..., ::-1]
                for e in acc.Images(tag)}
    for step, img in decoded('full_res_disp/image').items():
        assert np.array_equal(img, CO.summary_image(rec['disp'][step], jet)), step
    for step, img in decoded('gt_disp/image').items():
        assert np.array_equal(img, CO.summary_image(gts[step], jet)), step
    if continual:
        for step, img in decoded('proxy_disp/image').items():
            assert np.array_equal(img, CO.summary_image(rec['proxy'][step], jet)), step

    # everything the run wrote without --summary is unchanged (timings aside)
    files = ['overall.csv', 'series.csv', 'histogram.csv'] if continual else []
    for f in files + ['disparities/disparity_%d.png' % s for s in (0, 100, 200)]:
        assert open(str(plain / f), 'rb').read() == open(str(with_summary / f), 'rb').read(), f
    if not continual:
        a = open(str(plain / 'stats.csv')).read().splitlines()
        b = open(str(with_summary / 'stats.csv')).read().splitlines()
        assert [l for l in a if not l.startswith(('time', 'FPS'))] == [l for l in b if not l.startswith(('time', 'FPS'))]
        sa = [l.split(',') for l in open(str(plain / 'series.csv')).read().splitlines()]
        sb = [l.split(',') for l in open(str(with_summary / 'series.csv')).read().splitlines()]
        assert [r[:1] + r[2:] for r in sa] == [r[:1] + r[2:] for r in sb]
