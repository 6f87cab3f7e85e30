"""GPU tests of stereo rectification: the ms_rectify_u8 kernel against the float64 rule of test_rectify_cpu, its border,
NaN and identity cases, the engine's rectify + rescale + crop input path, prefetch, and the demo end to end with a
calibration."""
import json
import os

import numpy as np
import pytest
import torch

from conftest import PKG
from test_demo_gpu import GEOMS, LR, _demo_modules, _madnet, _note, _release, _resize_ref, _Seq, _write_image_list, \
    _write_weights
from test_rectify_cpu import remap_rule, synthetic_calibration, write_calibration

pytestmark = pytest.mark.gpu

# Bound on |fp32 blend - float64 blend|: the kernel's blend is at most eight fp32 roundings (three lerps of a difference,
# a product and a sum) of values below 256, each off by at most 2^-24 * 256 = 1.5e-5, and the fractions fx, fy are exact
# (m - floor(m) of an fp32 m >= 0 is exact; the tests' tables stay inside the frame).  So the rounded results can differ
# only where the float64 blend lies within 1.25e-4 of k + 1/2, and then by 1.
TIE = 1.25e-4


def _rectify(src, table):
    """ms_rectify_u8 of uint8 CUDA frames [B,h,w,3] through one float32 CUDA table [h,w,2]."""
    from madstereo._lib import check, lib
    b, h, w, _ = src.shape
    dst = torch.full_like(src, 77)
    check(lib().ms_rectify_u8(src.data_ptr(), table.data_ptr(), b, h, w, dst.data_ptr(),
                              torch.cuda.current_stream().cuda_stream), 'ms_rectify_u8')
    torch.cuda.synchronize()
    return dst


def _tables(h, w, seed=0, alpha=0.0):
    from madstereo.rectify import rectification_maps
    calib = synthetic_calibration(h, w, seed=seed)
    calib['alpha'] = alpha
    return rectification_maps(calib, (h, w))


def _frames(batch, h, w, seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (batch, h, w, 3), dtype=np.uint8) for _ in range(2)]


@pytest.mark.parametrize('size', [(720, 1280), (375, 1242), (1080, 1920)], ids=['720p', 'kitti', '1080p'])
@pytest.mark.parametrize('batch', [1, 2])
def test_rectify_matches_the_rule(size, batch):
    h, w = size
    tables = _tables(h, w, seed=h + batch)
    for cam, (img, table) in enumerate(zip(_frames(batch, h, w, seed=w + batch), tables)):
        got = _rectify(torch.from_numpy(img).cuda(), torch.from_numpy(table).cuda()).cpu().numpy()
        ref, blend = remap_rule(img, table)
        d = np.abs(got.astype(np.int64) - ref.astype(np.int64))
        near_tie = np.abs(blend - np.floor(blend) - 0.5) <= TIE
        assert d.max() <= 1 and near_tie[d > 0].all(), (cam, int(d.max()))
        _note(test='rectify_vs_rule', size=size, batch=batch, camera=cam, values_differing=int((d > 0).sum()),
              values_near_tie=int(near_tie.sum()), values=int(d.size))


def test_rectify_zero_outside_the_frame_and_for_bad_entries():
    h, w = 375, 1242
    # alpha 1 keeps every source pixel: the corners of the rectified frame come from outside the raw frame
    table = _tables(h, w, seed=7, alpha=1.0)[0].copy()
    img = _frames(2, h, w, seed=8)[0] | 1                  # no source value is 0
    bad = [(np.nan, 10.0), (10.0, np.nan), (np.nan, np.nan), (np.inf, 5.0), (5.0, -np.inf), (1e30, 1e30), (-1e30, 3.0),
           (-1.0001, 3.0), (w + 0.001, 3.0), (3.0, h + 0.5), (3.0, -2.0), (w + 1e9, -1e9), (float(w), float(h)), (-1.0, -1.0)]
    for k, v in enumerate(bad):
        table[h // 2, 100 + k] = v
    got = _rectify(torch.from_numpy(img).cuda(), torch.from_numpy(table).cuda()).cpu().numpy()
    mx, my = table[..., 0].astype(np.float64), table[..., 1].astype(np.float64)
    with np.errstate(invalid='ignore'):
        ok = (mx >= -1) & (mx <= w) & (my >= -1) & (my <= h)
    mx, my = np.where(ok, mx, 0.0), np.where(ok, my, 0.0)
    x0, y0 = np.floor(mx), np.floor(my)
    fx, fy = mx - x0, my - y0
    reach = np.zeros(mx.shape, bool)              # some tap with a non-zero weight lies inside the frame
    for dx, wx in ((0, 1 - fx), (1, fx)):
        for dy, wy in ((0, 1 - fy), (1, fy)):
            reach |= (x0 + dx >= 0) & (x0 + dx < w) & (y0 + dy >= 0) & (y0 + dy < h) & (wx * wy > 0)
    outside = ~ok | ~reach
    assert outside[h // 2, 100:100 + len(bad)].all()
    n_out = int(outside.sum())
    assert n_out > 1000, 'the alpha=1 tables should reach outside the frame'
    assert (got[:, outside] == 0).all()
    ref = remap_rule(img, table)[0]
    assert (np.abs(got.astype(np.int64) - ref.astype(np.int64)) <= 1).all()
    _note(test='rectify_outside', pixels_all_taps_outside=n_out, pixels=h * w)


def test_rectify_identity_is_exact():
    for (b, h, w) in ((1, 720, 1280), (2, 375, 1242), (1, 7, 9)):
        ys, xs = np.mgrid[0:h, 0:w].astype(np.float32)
        ident = torch.from_numpy(np.stack([xs, ys], -1)).cuda()
        img = torch.from_numpy(_frames(b, h, w, seed=h)[0]).cuda()
        assert torch.equal(_rectify(img, ident), img)


def _identity(h, w):
    ys, xs = np.mgrid[0:h, 0:w].astype(np.float32)
    return np.stack([xs, ys], -1)


@pytest.mark.parametrize('geom', GEOMS, ids=['720p-480x640-320x512', '375x1242-pad', '375x1242-odd-pad-crop', 'upscale', 'identity'])
def test_engine_identity_rectification_equals_the_plain_resize(geom):
    from madstereo.engine import StereoEngine
    (h, w), rs, (H, W) = geom
    eng = StereoEngine('MADNet', 2, H, W)
    eng.set_groups([]); eng.bind()
    eng.set_resize(rs if rs is not None else (-1, -1))
    left, right = (torch.from_numpy(x).cuda() for x in _frames(2, h, w, seed=h + w))
    eng.set_input(left, right)
    plain = [eng.tensor(n).cpu().numpy().view(np.uint32) for n in ('raw_left', 'raw_right')]
    eng.set_rectification(_identity(h, w), torch.from_numpy(_identity(h, w)))      # numpy and torch tables
    eng.tensor('raw_left').fill_(-1); eng.tensor('raw_right').fill_(-1)
    eng.set_input(left, right)
    torch.cuda.synchronize()
    for n, p in zip(('raw_left', 'raw_right'), plain):
        assert np.array_equal(eng.tensor(n).cpu().numpy().view(np.uint32), p), n
    del eng
    _release()


def test_engine_rectify_rescale_crop_equals_the_oracle_on_the_rectified_frames():
    from madstereo.engine import StereoEngine
    (h, w), rs, (H, W) = (720, 1280), (480, 640), (320, 512)
    tables = _tables(h, w, seed=11)
    eng = StereoEngine('MADNet', 2, H, W)
    eng.set_groups([]); eng.bind(); eng.set_resize(rs)
    eng.set_rectification(*tables)
    left, right = _frames(2, h, w, seed=12)
    for kind, (l, r) in (('pageable', (torch.from_numpy(left), torch.from_numpy(right))),
                         ('device', (torch.from_numpy(left).cuda(), torch.from_numpy(right).cuda()))):
        eng.set_input(l, r)
        torch.cuda.synchronize()
        scratch = eng._rect[2].cpu().numpy().reshape(2, 2, h, w, 3)      # the device's own rectified frames
        for cam, (src, table) in enumerate(((left, tables[0]), (right, tables[1]))):
            one = _rectify(torch.from_numpy(src).cuda(), torch.from_numpy(table).cuda()).cpu().numpy()
            assert np.array_equal(scratch[cam], one), (kind, cam)             # both cameras in one launch == one by one
        for cam, name in enumerate(('raw_left', 'raw_right')):
            ref = _resize_ref(scratch[cam], rs, (H, W))
            got = eng.tensor(name).cpu().numpy().astype(np.float64)
            assert np.abs(got - ref).max() <= 1e-4, (kind, name)
        assert not np.array_equal(scratch[0], left), 'the tables should move pixels'
    del eng
    _release()


def test_engine_rectification_refusals_and_switching_off():
    from madstereo import MadStereoError
    from madstereo.engine import StereoEngine
    h, w = 240, 320
    tables = _tables(h, w, seed=13)
    eng = StereoEngine('MADNet', 1, 320, 512)
    eng.set_groups([]); eng.bind()
    with pytest.raises(MadStereoError, match='set_resize'):
        eng.set_rectification(*tables)
    eng.set_resize((480, 640))
    with pytest.raises(MadStereoError, match='float32'):
        eng.set_rectification(tables[0].astype(np.float64), tables[1])
    with pytest.raises(MadStereoError, match='differ in size'):
        eng.set_rectification(tables[0], tables[1][:-1])
    eng.set_rectification(*tables)
    with pytest.raises(MadStereoError, match='rectification off first'):
        eng.set_resize(None)
    left, right = _frames(1, h + 10, w, seed=14)
    with pytest.raises(MadStereoError, match='frames are 250x320, the rectification tables 240x320'):
        eng.set_input(left, right)
    left, right = (torch.from_numpy(x).cuda() for x in _frames(1, h, w, seed=15))
    eng.set_input(left, right)
    rectified = eng.tensor('raw_left').cpu().numpy()
    eng.set_rectification(None)
    eng.set_input(left, right)
    plain = eng.tensor('raw_left').cpu().numpy()
    assert np.abs(plain.astype(np.float64) - _resize_ref(left.cpu().numpy(), (480, 640), (320, 512))).max() <= 1e-4
    assert not np.array_equal(plain, rectified)
    eng.set_resize(None)
    del eng
    _release()


def test_rectified_prefetch_matches_serial_path():
    """prefetch() stages camera-size uint8 frames; the step then rectifies and rescales from the staging buffers."""
    from madstereo.synthetic import make_pair
    frames = []
    for k in range(4):
        l, r, _ = make_pair(240, 320, seed=40 + k)
        frames.append((np.clip(np.rint(l), 0, 255).astype(np.uint8), np.clip(np.rint(r), 0, 255).astype(np.uint8)))
    tables = _tables(240, 320, seed=16)
    losses = {}
    for pipelined in (False, True):
        net, ad, _ = _madnet(320, 512, 'MAD', seq=[0, 3, 1, 4])
        ad.engine.set_resize((480, 640))
        ad.engine.set_rectification(*tables)
        res = []
        for k, (l, r) in enumerate(frames):
            nxt = frames[k + 1] if pipelined and k + 1 < len(frames) else None
            res.append(ad.step(l, r, prefetch=nxt)['loss'])
        losses[pipelined] = res
        del net, ad
        _release()
    assert losses[False] == losses[True]
    _note(test='rectified_prefetch', losses=losses[False])


def test_demo_end_to_end_with_a_calibration(tmp_path):
    demo, demo_model = _demo_modules()
    frames = _write_image_list(tmp_path, 4, h=480, w=640)
    calib = synthetic_calibration(480, 640, seed=17)
    cal_path = write_calibration(tmp_path / 'stereo.yml', calib, ('K1', 'D1', 'K2', 'D2', 'R', 'T'))
    cfg = json.loads((tmp_path / 'camera.json').read_text())
    cfg['calibration'] = cal_path
    (tmp_path / 'camera.json').write_text(json.dumps(cfg))
    weights, _ = _write_weights(tmp_path, with_adam=False)
    args = demo.build_parser().parse_args([
        '--cameraName', 'ImageList', '--cameraConfig', str(tmp_path / 'camera.json'), '--weights', weights, '--mode', 'MAD',
        '--blockConfig', os.path.join(PKG, 'block_config', 'MadNet_full.json'),
        '--SSIMTh', '10', '--output', str(tmp_path / 'out')])
    dd = demo.main(args)
    rows = [l.split(',') for l in open(str(tmp_path / 'out' / 'log.csv')).read().splitlines()[1:]]
    assert len(rows) == len(frames) and all(os.path.exists(str(tmp_path / 'out' / ('disparity_%06d.png' % k))) for k in range(4))
    assert dd._adapt.engine._rect is not None
    losses, modules = [float(r[1]) for r in rows], [int(r[2]) for r in rows]
    del dd
    _release()
    # the same frames through OnlineAdaptation.step, rectified with the loader's tables, then without rectification
    from madstereo.rectify import load_calibration, rectification_maps
    train_config = json.load(open(args.blockConfig))
    direct = {}
    for rectify in (True, False):
        ad, _ = demo_model.build_engine('MADNet', 320, 512, 'MAD', train_config, LR, 10.0, [480, 640])
        demo_model.restore_weights(ad, weights)
        if rectify:
            ad.engine.set_rectification(*rectification_maps(load_calibration(cal_path), (480, 640)))
        ad.sampler = _Seq(modules)
        direct[rectify] = [ad.step(l, r)['loss'] for l, r in frames]
        del ad
        _release()
    assert direct[True] == losses
    assert direct[False] != losses
    _note(test='demo_with_calibration', losses=losses, unrectified=direct[False])
