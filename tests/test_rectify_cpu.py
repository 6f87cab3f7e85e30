"""CPU tests of stereo rectification: the calibration loader against OpenCV called directly, its refusals, the float64
statement of the device kernel's rule against cv2.remap, and the demo's calibration plumbing with a stub adapter.

The rule (`remap_rule`) is what csrc/elementwise.cu rectify_u8_kernel computes, in float64; the GPU tests compare the kernel
with it."""
import json
import os
import queue
import sys

import numpy as np
import pytest

from conftest import PKG

DEMO = os.path.join(PKG, 'Demo')
if DEMO not in sys.path:
    sys.path.insert(0, DEMO)


def remap_rule(src, m):
    """src uint8 [..., h, w, 3], m float32 [h, w, 2] = (src_x, src_y) -> (uint8 result, float64 blend before rounding).
    Taps at floor(m) and +1, 0 outside the frame, blended x then y; rounded to nearest, ties to even, clamped to
    [0, 255].  An entry that is NaN or outside [-1, w] x [-1, h] gives 0."""
    src = np.asarray(src)
    h, w = src.shape[-3], src.shape[-2]
    mx, my = m[..., 0].astype(np.float64), m[..., 1].astype(np.float64)
    ok = (mx >= -1) & (mx <= w) & (my >= -1) & (my <= h)            # False for NaN
    mx, my = np.where(ok, mx, 0.0), np.where(ok, my, 0.0)
    x0, y0 = np.floor(mx), np.floor(my)
    fx, fy = (mx - x0)[..., None], (my - y0)[..., None]
    x0, y0 = x0.astype(np.int64) + 1, y0.astype(np.int64) + 1       # indices into the zero-padded frame
    pad = np.zeros(src.shape[:-3] + (h + 3, w + 3, 3))
    pad[..., 1:h + 1, 1:w + 1, :] = src
    tl, tr = pad[..., y0, x0, :], pad[..., y0, x0 + 1, :]
    bl, br = pad[..., y0 + 1, x0, :], pad[..., y0 + 1, x0 + 1, :]
    top, bot = tl + (tr - tl) * fx, bl + (br - bl) * fx
    v = np.where(ok[..., None], top + (bot - top) * fy, 0.0)
    return np.clip(np.rint(v), 0, 255).astype(np.uint8), v


def synthetic_calibration(h, w, seed=0):
    """A plausible stereo rig for (h, w) frames: two slightly different pinhole cameras with barrel distortion (5
    coefficients), the right one rotated by a few degrees and 12 cm to the right."""
    import cv2
    rng = np.random.default_rng(seed)
    f = 0.7 * w
    cams = []
    for _ in range(2):
        K = np.array([[f * rng.uniform(0.98, 1.02), 0, w / 2 + rng.uniform(-8, 8)],
                      [0, f * rng.uniform(0.98, 1.02), h / 2 + rng.uniform(-8, 8)], [0, 0, 1]])
        D = np.array([[-0.3 + rng.uniform(-0.02, 0.02), 0.1, rng.uniform(-1e-3, 1e-3), rng.uniform(-1e-3, 1e-3), -0.02]])
        cams.append((K, D))
    R, _ = cv2.Rodrigues(np.radians(rng.uniform(-3, 3, 3)).reshape(3, 1))
    T = np.array([[-0.12], [rng.uniform(-0.005, 0.005)], [rng.uniform(-0.005, 0.005)]])
    return {'K1': cams[0][0], 'D1': cams[0][1], 'K2': cams[1][0], 'D2': cams[1][1], 'R': R, 'T': T, 'size': (h, w)}


def write_calibration(path, calib, keys, alpha=None):
    import cv2
    fs = cv2.FileStorage(str(path), cv2.FILE_STORAGE_WRITE)
    fs.write('image_width', int(calib['size'][1]))
    fs.write('image_height', int(calib['size'][0]))
    for k in keys:
        fs.write(k, np.asarray(calib[k], np.float64))
    if alpha is not None:
        fs.write('alpha', float(alpha))
    fs.release()
    return str(path)


def direct_maps(calib, R1, R2, P1, P2):
    import cv2
    h, w = calib['size']
    out = []
    for K, D, R, P in ((calib['K1'], calib['D1'], R1, P1), (calib['K2'], calib['D2'], R2, P2)):
        mx, my = cv2.initUndistortRectifyMap(K, D, R, P, (w, h), cv2.CV_32FC1)
        out.append(np.stack([mx, my], axis=-1))
    return out


@pytest.mark.parametrize('ext', ['yml', 'xml', 'json'])
@pytest.mark.parametrize('alpha', [None, 0.5])
def test_loader_computes_the_rectification_from_R_T(tmp_path, ext, alpha):
    import cv2
    from madstereo.rectify import load_calibration, rectification_maps
    calib = synthetic_calibration(120, 160, seed=1)
    path = write_calibration(tmp_path / ('stereo.' + ext), calib, ('K1', 'D1', 'K2', 'D2', 'R', 'T'), alpha)
    got = rectification_maps(load_calibration(path), (120, 160))
    R1, R2, P1, P2 = cv2.stereoRectify(calib['K1'], calib['D1'], calib['K2'], calib['D2'], (160, 120), calib['R'],
                                       calib['T'], flags=cv2.CALIB_ZERO_DISPARITY, alpha=alpha or 0)[:4]
    for g, ref in zip(got, direct_maps(calib, R1, R2, P1, P2)):
        assert g.dtype == np.float32 and g.shape == (120, 160, 2) and g.flags['C_CONTIGUOUS']
        assert np.array_equal(g, ref)
    if alpha is not None:        # alpha reaches stereoRectify: the default (0) gives other tables
        R1, R2, P1, P2 = cv2.stereoRectify(calib['K1'], calib['D1'], calib['K2'], calib['D2'], (160, 120), calib['R'],
                                           calib['T'], flags=cv2.CALIB_ZERO_DISPARITY, alpha=0)[:4]
        assert not np.array_equal(got[0], direct_maps(calib, R1, R2, P1, P2)[0])


def test_loader_uses_a_given_rectification_as_it_is(tmp_path):
    import cv2
    from madstereo.rectify import load_calibration, rectification_maps
    calib = synthetic_calibration(90, 130, seed=2)
    # a rectification that stereoRectify would not produce (alpha 1, no zero-disparity flag), with R T present too:
    # R1 R2 P1 P2 win
    R1, R2, P1, P2 = cv2.stereoRectify(calib['K1'], calib['D1'], calib['K2'], calib['D2'], (130, 90), calib['R'],
                                       calib['T'], flags=0, alpha=1)[:4]
    calib.update(R1=R1, R2=R2, P1=P1, P2=P2)
    for keys in (('K1', 'D1', 'K2', 'D2', 'R1', 'R2', 'P1', 'P2'), ('K1', 'D1', 'K2', 'D2', 'R', 'T', 'R1', 'R2', 'P1', 'P2')):
        path = write_calibration(tmp_path / 'given.yml', calib, keys)
        got = rectification_maps(load_calibration(path), (90, 130))
        for g, ref in zip(got, direct_maps(calib, R1, R2, P1, P2)):
            assert np.array_equal(g, ref)


def test_loader_refuses_missing_keys_and_other_frame_sizes(tmp_path):
    from madstereo import MadStereoError
    from madstereo.rectify import load_calibration, rectification_maps
    calib = synthetic_calibration(60, 80)
    calib.update(R1=np.eye(3), R2=np.eye(3), P1=np.eye(3, 4))
    for keys, missing in ((('K1', 'D1', 'K2', 'R', 'T'), 'D2'), (('K1', 'D1', 'K2', 'D2', 'R'), 'T'),
                          (('K1', 'D1', 'K2', 'D2', 'R1', 'R2', 'P1'), 'T')):
        path = write_calibration(tmp_path / 'c.yml', calib, keys)
        with pytest.raises(MadStereoError, match='missing .*%s' % missing):
            load_calibration(path)
    import cv2
    fs = cv2.FileStorage(str(tmp_path / 'nosize.yml'), cv2.FILE_STORAGE_WRITE)
    for k in ('K1', 'D1', 'K2', 'D2', 'R', 'T'):
        fs.write(k, calib[k])
    fs.release()
    with pytest.raises(MadStereoError, match='missing image_width image_height'):
        load_calibration(str(tmp_path / 'nosize.yml'))
    with pytest.raises(MadStereoError, match='cannot be opened'):
        load_calibration(str(tmp_path / 'absent.yml'))
    good = load_calibration(write_calibration(tmp_path / 'ok.yml', calib, ('K1', 'D1', 'K2', 'D2', 'R', 'T')))
    for size in ((80, 60), (120, 160), (60, 81)):
        with pytest.raises(MadStereoError, match='calibration is for 60x80'):
            rectification_maps(good, size)


def _neighbourhood_slope(img, m):
    """Per output pixel: the largest |difference| of horizontally (Lx) and vertically (Ly) adjacent taps of the zero-padded
    frame in rows floor(my)-1 .. +2 and columns floor(mx)-1 .. +2, which bounds the slope of the bilinear interpolant on
    every cell a step of at most 1/64 pixel from m can reach."""
    h, w = img.shape[:2]
    pad = np.zeros((h + 6, w + 6, 3))
    pad[3:h + 3, 3:w + 3] = img
    x0 = np.floor(m[..., 0]).astype(np.int64) + 3
    y0 = np.floor(m[..., 1]).astype(np.int64) + 3
    lx = np.zeros(m.shape[:2] + (3,)); ly = np.zeros(m.shape[:2] + (3,))
    for dy in range(-1, 3):
        for dx in range(-1, 3):
            if dx < 2:
                lx = np.maximum(lx, np.abs(pad[y0 + dy, x0 + dx + 1] - pad[y0 + dy, x0 + dx]))
            if dy < 2:
                ly = np.maximum(ly, np.abs(pad[y0 + dy + 1, x0 + dx] - pad[y0 + dy, x0 + dx]))
    return lx, ly


@pytest.mark.parametrize('size', [(240, 320), (375, 1242)])
def test_rule_agrees_with_cv2_remap(size):
    """OpenCV's remap (INTER_LINEAR, 8-bit) rounds each coordinate to the nearest 1/32 pixel (cvRound(m * 32)) and blends
    with integer weights in units of 2^-15.  On that grid the bilinear weights are products of multiples of 1/32, i.e.
    multiples of 2^-10, so they are exact in 2^-15 units and sum to 1 with no correction.  Hence:
      * maps on the 1/32 grid: OpenCV's blend equals the rule's blend exactly; the results differ only where the blend is
        exactly k + 1/2 (OpenCV's (s + 2^14) >> 15 rounds half up, the rule half to even), and then by 1;
      * any maps: the coordinates move by at most 1/64 pixel per axis, so the blends differ by at most
        (Lx + Ly) / 64 (Lipschitz bound of the interpolant, _neighbourhood_slope); the two roundings add at most 1, and
        |rule - cv2| <= floor((Lx + Ly) / 64 + 1) per pixel and channel."""
    import cv2
    h, w = size
    calib = synthetic_calibration(h, w, seed=h)
    from madstereo.rectify import rectification_maps
    calib['alpha'] = 0.0
    rng = np.random.default_rng(w)
    img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    for m in rectification_maps(calib, size):
        for snapped in (True, False):
            mm = (np.rint(m * 32) / 32).astype(np.float32) if snapped else m
            ref = cv2.remap(img, mm[..., 0], mm[..., 1], cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
            got, blend = remap_rule(img, mm)
            d = np.abs(got.astype(np.int64) - ref.astype(np.int64))
            if snapped:
                assert d.max() <= 1 and (blend[d > 0] - np.floor(blend[d > 0]) == 0.5).all()
                assert (got[d > 0] % 2 == 0).all() and (got[d > 0] + 1 == ref[d > 0]).all()
            else:
                lx, ly = _neighbourhood_slope(img, mm)
                assert (d <= np.floor((lx + ly) / 64 + 1)).all()
            print('MEASURED', json.dumps({'size': size, 'snapped': snapped, 'max_diff': int(d.max()),
                                          'pixels_differing': int((d > 0).any(-1).sum()), 'pixels': h * w}))


def test_rule_border_nan_and_identity():
    rng = np.random.default_rng(5)
    img = rng.integers(0, 256, (2, 7, 9, 3), dtype=np.uint8)
    ys, xs = np.mgrid[0:7, 0:9].astype(np.float32)
    ident = np.stack([xs, ys], -1)
    assert np.array_equal(remap_rule(img, ident)[0], img)
    m = ident.copy()
    m[0, 0] = (np.nan, 3); m[0, 1] = (2, np.nan); m[0, 2] = (-1.5, 2); m[0, 3] = (4, 7.25); m[0, 4] = (1e30, -1e30)
    m[1, 0] = (-1, 3)              # on the edge of the range: the only tap inside has weight 0
    m[1, 1] = (-0.5, 3)            # half of column 0
    got = remap_rule(img, m)[0]
    assert (got[:, 0, :5] == 0).all() and (got[:, 1, 0] == 0).all()
    assert np.array_equal(got[:, 1, 1], np.rint(img[:, 3, 0] * 0.5).astype(np.uint8))


def _stub_demo(tmp_path, monkeypatch, calib_size, frame_size=(24, 32)):
    """The demo's main() with the engine replaced by a stub that records set_rectification."""
    import cv2
    import demo_model
    import Live_Adaptation_Demo as demo
    h, w = frame_size
    rng = np.random.default_rng(0)
    lines = []
    for k in range(2):
        for side in 'lr':
            cv2.imwrite(str(tmp_path / ('%s%d.png' % (side, k))), rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
        lines.append('%s;%s' % (tmp_path / ('l%d.png' % k), tmp_path / ('r%d.png' % k)))
    (tmp_path / 'list.txt').write_text('\n'.join(lines) + '\n')
    calib = synthetic_calibration(*calib_size, seed=3)
    cal_path = write_calibration(tmp_path / 'stereo.yml', calib, ('K1', 'D1', 'K2', 'D2', 'R', 'T'))
    (tmp_path / 'camera.json').write_text(json.dumps({'list': str(tmp_path / 'list.txt'), 'fps': 0,
                                                      'calibration': cal_path}))

    class Engine(object):
        def __init__(self):
            self.tables = []

        def set_rectification(self, map_left, map_right):
            self.tables.append((map_left, map_right))

    class Adapt(object):
        def __init__(self):
            self.engine, self.sample_distribution, self.frames = Engine(), None, 0

        def step(self, left, right):
            assert self.engine.tables, 'a frame reached the engine before its rectification was set'
            self.frames += 1
            return {'loss': 0.1, 'blocks': [0], 'reset': False}

    stub = Adapt()
    disp = np.zeros((1, 16, 24, 1), np.float32)
    monkeypatch.setattr(demo_model, 'build_engine', lambda *a: (stub, lambda: (disp, disp, disp)))
    monkeypatch.setattr(demo_model, 'restore_weights', lambda adapt, path: None)
    args = demo.build_parser().parse_args(['--cameraName', 'ImageList', '--cameraConfig', str(tmp_path / 'camera.json'),
                                           '--weights', 'unused', '--mode', 'NONE', '--imageShape', '-1',
                                           '--cropShape', '16', '24', '--output', str(tmp_path / 'out')])
    return demo, args, stub, calib, cal_path


def test_demo_sets_the_calibration_tables_on_the_engine(tmp_path, monkeypatch):
    from madstereo.rectify import load_calibration, rectification_maps
    demo, args, stub, calib, cal_path = _stub_demo(tmp_path, monkeypatch, (24, 32))
    dd = demo.main(args)
    assert dd.error is None and stub.frames == 2 and len(stub.engine.tables) == 1
    ref = rectification_maps(load_calibration(cal_path), (24, 32))
    for got, r in zip(stub.engine.tables[0], ref):
        assert np.array_equal(got, r)


def test_demo_refuses_frames_of_another_size_than_the_calibration(tmp_path, monkeypatch):
    from madstereo import MadStereoError
    demo, args, stub, _, _ = _stub_demo(tmp_path, monkeypatch, (30, 40))
    with pytest.raises(MadStereoError, match='frames are 24x32 but the calibration is for 30x40'):
        demo.main(args)
    assert stub.frames == 0


def test_demo_without_calibration_sets_no_tables(tmp_path):
    import demo_model
    q = queue.Queue()
    q.put(np.zeros((2, 8, 12, 3), np.uint8))
    q.put(None)

    class Adapt(object):
        engine, sample_distribution = None, None        # any engine call would fail

        def step(self, left, right):
            return {'loss': 0.1, 'blocks': [0], 'reset': False}
    disp = np.zeros((1, 8, 12, 1), np.float32)
    dd = demo_model.RealTimeStereo(q, weight_path='unused', mode='NONE', image_shape=[None, None], crop_shape=[8, 12],
                                   output=str(tmp_path / 'o'), build=lambda h, w: (Adapt(), lambda: (disp, disp, disp)),
                                   log=lambda s: None)
    dd.run()
    assert dd.error is None and len(dd.records) == 1
