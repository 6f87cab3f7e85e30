"""CPU tests of the live demo: command line vs the reference, grabbers, the demo loop with a stub adapter, Adam-state
loading from a checkpoint, and the Adam known answers of the float64 restatement."""
import argparse
import ctypes
import json
import os
import queue
import sys

import numpy as np
import pytest

from conftest import PKG, ROOT

DEMO = os.path.join(PKG, 'Demo')
for _p in (DEMO,):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import grabber  # noqa: E402


def _actions(parser):
    out = []
    for a in parser._actions:
        if a.dest == 'help':
            continue
        out.append({'flags': list(a.option_strings), 'dest': a.dest, 'required': bool(a.required), 'default': a.default,
                    'type': getattr(a.type, '__name__', None), 'nargs': a.nargs, 'choices': sorted(a.choices) if a.choices else None,
                    'store_true': isinstance(a, argparse._StoreTrueAction)})
    return out


def test_demo_flags_equal_the_reference():
    """tests/golden/reference_demo_cli.json: the reference's argparse actions (tests/golden/make_demo_golden.py)."""
    import Live_Adaptation_Demo as demo
    golden = json.load(open(os.path.join(ROOT, 'tests', 'golden', 'reference_demo_cli.json')))['actions']
    mine = _actions(demo.build_parser())
    ref_dests = [a['dest'] for a in golden]
    assert [a['dest'] for a in mine[:len(golden)]] == ref_dests
    for a, g in zip(mine, golden):
        if a['dest'] == 'cameraName':
            # the grabbers available here differ: ZED_Mini needs the ZED SDK, ImageList is new
            assert g['choices'] == ['ZED_Mini'] and 'ImageList' in a['choices']
            a, g = dict(a, choices=None), dict(g, choices=None)
        assert a == g, a['dest']
    # the headless additions
    extra = {a['dest']: a for a in mine[len(golden):]}
    assert sorted(extra) == ['maxFrames', 'output']
    assert extra['output']['flags'] == ['--output'] and extra['output']['default'] is None
    assert extra['maxFrames']['flags'] == ['--maxFrames'] and extra['maxFrames']['type'] == 'int'
    assert demo.shape_arg([-1], '--x') == [None, None] and demo.shape_arg([-1, -1], '--x') == [None, None]
    assert demo.shape_arg([480, 640], '--x') == [480, 640]
    with pytest.raises(SystemExit):
        demo.shape_arg([480], '--x')


def test_demo_refuses_missing_weights_and_checks_camera_config(tmp_path):
    import Live_Adaptation_Demo as demo
    args = demo.build_parser().parse_args(['--cameraName', 'ImageList'])
    with pytest.raises(SystemExit, match='--weights'):
        demo.main(args)
    args = demo.build_parser().parse_args(['--cameraName', 'ImageList', '--weights', 'w', '--cameraConfig',
                                           str(tmp_path / 'missing.json')])
    with pytest.raises(AssertionError, match='camera configuration'):
        demo.main(args)


def test_grabber_factory():
    with pytest.raises(Exception, match='Unrecognized camera type'):
        grabber.get_camera('nope', queue.Queue(1))
    assert 'ImageList' in grabber.get_available_camera()
    try:
        import pyzed.sl  # noqa: F401
        has_zed = True
    except ImportError:
        has_zed = False
    assert ('ZED_Mini' in grabber.get_available_camera()) == has_zed

    @grabber.register_camera_to_factory()
    class Constant(grabber.ImageGrabber):
        _name = 'TestConstant'

        def _connect_to_camera(self):
            self.n = 0

        def _read_frame(self):
            self.n += 1
            return (np.full((2, 3, 3), self.n, np.uint8), np.zeros((2, 3, 3), np.uint8)) if self.n <= 2 else None

        def _disconnect_from_camera(self):
            self.closed = True

    try:
        q = queue.Queue(1)
        g = grabber.get_camera('TestConstant', q, config=None, framerate=0)
        assert isinstance(g, Constant)
        g.start()
        got = [q.get(timeout=10) for _ in range(3)]
        g.join(10)
        assert got[0].shape == (2, 2, 3, 3) and got[0][0, 0, 0, 0] == 1 and got[1][0, 0, 0, 0] == 2
        assert got[2] is grabber.END_OF_STREAM and g.closed
    finally:
        del grabber._GRABBER_FACTORY['TestConstant']


def _image_list(tmp_path, n, h=6, w=10):
    import cv2
    rng = np.random.default_rng(0)
    lines, frames = [], []
    for k in range(n):
        l = rng.integers(0, 256, (h, w, 3), dtype=np.uint8); r = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        pl, pr = str(tmp_path / ('l%d.png' % k)), str(tmp_path / ('r%d.png' % k))
        cv2.imwrite(pl, l[:, :, ::-1]); cv2.imwrite(pr, r[:, :, ::-1])
        lines.append('%s;%s' % (pl, pr))
        frames.append((l, r))
    (tmp_path / 'list.txt').write_text('# comment\n' + '\n'.join(lines) + '\n')
    cfg = tmp_path / 'camera.json'
    cfg.write_text(json.dumps({'list': str(tmp_path / 'list.txt'), 'fps': 0}))
    return str(cfg), frames


def test_image_list_grabber_yields_frames_in_order_then_ends(tmp_path):
    cfg, frames = _image_list(tmp_path, 3)
    q = queue.Queue(1)
    g = grabber.get_camera('ImageList', q, config=cfg, framerate=30)
    assert g._sleeptime == 0.0                 # fps 0: no pacing
    g.start()
    for l, r in frames:
        f = q.get(timeout=10)
        assert f.dtype == np.uint8 and f.shape == (2,) + l.shape
        assert np.array_equal(f[0], l) and np.array_equal(f[1], r)
    assert q.get(timeout=10) is grabber.END_OF_STREAM
    g.join(10)
    assert not g.is_alive()


class _StubAdapt(object):
    """Stands in for OnlineAdaptation: records the sample distribution each step saw and returns scripted losses."""

    def __init__(self, losses, th):
        self.losses, self.th, self.k = losses, th, 0
        self.sample_distribution = None
        self.seen = []
        self.reset_counter = 0

    def step(self, left, right):
        assert left.shape[0] == 1 and right.shape[0] == 1 and left.dtype == np.uint8
        self.seen.append(np.array(self.sample_distribution, copy=True))
        loss = self.losses[self.k]
        self.k += 1
        reset = loss > self.th
        self.reset_counter += int(reset)
        # uniform draw from softmax(zeros): any module; the stub picks k % 5
        return {'loss': loss, 'blocks': [self.k % 5], 'reset': reset}


def test_demo_loop_with_stub_adapter(tmp_path):
    import cv2
    import demo_model
    losses = [0.3, 0.7, 0.2, 0.9, 0.1]
    stub = _StubAdapt(losses, 0.5)
    disp = np.linspace(0, 300, 8 * 12, dtype=np.float32).reshape(1, 8, 12, 1)
    lefty = np.full((1, 8, 12, 3), 7.6, np.float32)

    def build(h, w):
        assert (h, w) == (8, 12)
        return stub, lambda: (lefty, lefty, disp)

    q = queue.Queue()
    for _ in losses:
        q.put(np.zeros((2, 16, 20, 3), np.uint8))
    q.put(grabber.END_OF_STREAM)
    out = tmp_path / 'out'
    dd = demo_model.RealTimeStereo(q, weight_path='unused', mode='MAD', image_shape=[None, None], crop_shape=[8, 12],
                                   SSIMTh=0.5, output=str(out), build=build, log=lambda s: None,
                                   block_config_path=os.path.join(PKG, 'block_config', 'MadNet_full.json'))
    dd.run()
    assert dd.error is None
    # the reference never sets `first` to False: the gain is always 0 and the distribution stays at zero
    assert all(s.shape == (5,) and not s.any() for s in stub.seen) and not dd.sample_distribution.any()
    rows = [l.split(',') for l in open(str(out / 'log.csv')).read().splitlines()]
    assert rows[0] == ['step', 'loss', 'module', 'reset', 'step_ms']
    assert [float(r[1]) for r in rows[1:]] == losses
    assert [int(r[2]) for r in rows[1:]] == [1, 2, 3, 4, 0]
    assert [r[3] for r in rows[1:]] == ['0', '1', '0', '1', '0'] and stub.reset_counter == 2
    img = cv2.imread(str(out / 'disparity_000003.png'))
    assert np.array_equal(img, cv2.applyColorMap(disp[0].astype(np.uint8), cv2.COLORMAP_JET))
    assert len([f for f in os.listdir(str(out)) if f.endswith('.png')]) == len(losses)
    # --maxFrames stops early
    q2 = queue.Queue()
    for _ in range(3):
        q2.put(np.zeros((2, 8, 12, 3), np.uint8))
    stub2 = _StubAdapt([0.1] * 3, 0.5)
    dd2 = demo_model.RealTimeStereo(q2, weight_path='unused', mode='NONE', image_shape=[None, None], crop_shape=[None, None],
                                    output=str(tmp_path / 'o2'), max_frames=2, build=lambda h, w: (stub2, lambda: (lefty, lefty, disp)),
                                    log=lambda s: None)
    dd2.run()
    assert len(dd2.records) == 2 and stub2.k == 2 and q2.qsize() == 1


def test_network_shape():
    import demo_model
    assert demo_model.network_shape([480, 640], [320, 512], (720, 1280)) == (320, 512)
    assert demo_model.network_shape([480, 640], [None, None], (720, 1280)) == (480, 640)
    assert demo_model.network_shape([None, None], [None, None], (720, 1280)) == (720, 1280)


def _layers():
    """MADNet layer table from the library (no device needed)."""
    from madstereo import _lib
    from madstereo.engine import LayerInfo
    L = _lib.lib()
    e = L.ms_engine_create(b'MADNet', 1, 64, 128, 2, 1, 1)
    out = []
    for i in range(L.ms_engine_num_layers(e)):
        nm, sc, bn = (ctypes.create_string_buffer(128) for _ in range(3))
        dims = (ctypes.c_int * 7)(); alpha = ctypes.c_float()
        assert L.ms_engine_layer_info(e, i, nm, 128, sc, 128, bn, 128, dims, ctypes.byref(alpha)) == 0
        out.append(LayerInfo(i, nm.value.decode(), sc.value.decode(), bn.value.decode(), *list(dims), alpha.value))
    L.ms_engine_destroy(e)
    return out


def test_adam_slots_load_only_for_trained_variables(tmp_path):
    from Data_utils import weights_utils
    from madstereo.adaptation import trained_variable_names
    from madstereo.tf_checkpoint import write_checkpoint
    from oracle.madnet import param_shapes
    shapes = param_shapes()
    layers = _layers()
    cfg = json.load(open(os.path.join(PKG, 'block_config', 'MadNet_piramid_only.json')))
    by_name = {l.name: l.index for l in layers}
    groups = [sorted({by_name[n] for n in g if n in by_name}) for g in cfg]
    rng = np.random.default_rng(3)
    tensors = {}
    for n, s in shapes.items():
        tensors[n] = rng.normal(0, 0.1, s).astype(np.float32)
        tensors[n + '/Adam'] = rng.normal(0, 1e-3, s).astype(np.float32)
        tensors[n + '/Adam_1'] = rng.uniform(0, 1e-6, s).astype(np.float32)
    tensors['beta1_power'] = np.float32(0.5)
    tensors['beta2_power'] = np.float32(0.25)
    prefix = str(tmp_path / 'model.ckpt')
    write_checkpoint(prefix, tensors)

    mad = trained_variable_names('MAD', groups, layers)
    assert mad and all('fgc-volume-filtering' in n or 'context' in n for n in mad)        # estimators + refinement only
    assert not any('gc-read-pyramid' in n for n in mad)
    st = weights_utils.load_adam_state(prefix, {n: shapes[n] for n in mad})
    assert sorted(st['m']) == sorted(mad) and sorted(st['v']) == sorted(mad)
    for n in mad:
        assert np.array_equal(st['m'][n], tensors[n + '/Adam']) and np.array_equal(st['v'][n], tensors[n + '/Adam_1'])
    assert st['powers'] == (0.5, 0.25) and st['found'] == 2 * len(mad) + 2

    full = trained_variable_names('FULL', groups, layers)
    assert sorted(full) == sorted(shapes)
    assert weights_utils.load_adam_state(prefix, {n: shapes[n] for n in full})['found'] == 2 * len(shapes) + 2

    assert trained_variable_names('NONE', groups, layers) == []
    none = weights_utils.load_adam_state(prefix, {})
    assert none == {'m': {}, 'v': {}, 'powers': None, 'found': 0}

    # a checkpoint without optimizer state (weights only): zeros and powers (beta1, beta2)
    plain = str(tmp_path / 'plain.ckpt')
    write_checkpoint(plain, {n: tensors[n] for n in shapes})
    st = weights_utils.load_adam_state(plain, {n: shapes[n] for n in mad}, 0.9, 0.999)
    assert st['found'] == 0 and st['powers'] == (float(np.float32(0.9)), float(np.float32(0.999)))
    assert all(not st['m'][n].any() and not st['v'][n].any() and st['m'][n].shape == tuple(shapes[n]) for n in mad)


def test_adam_requires_a_single_gpu(monkeypatch):
    """OnlineAdaptation(optimizer='adam') refuses a data-parallel run before it touches the device."""
    import torch
    from madstereo._lib import MadStereoError
    from madstereo.adaptation import OnlineAdaptation
    monkeypatch.setattr(torch.distributed, 'is_available', lambda: True)
    monkeypatch.setattr(torch.distributed, 'is_initialized', lambda: True)
    monkeypatch.setattr(torch.distributed, 'get_world_size', lambda g=None: 2)
    monkeypatch.setattr(torch.distributed, 'get_rank', lambda g=None: 0)

    class _Net(object):
        engine = None
    with pytest.raises(MadStereoError, match='single GPU'):
        OnlineAdaptation(_Net(), mode='FULL', optimizer='adam')


def test_adam_oracle_known_answer():
    """At t = 1 (powers beta1, beta2, zero slots) ApplyAdam moves w by lr * g / (|g| + eps): lr_t = lr sqrt(1-b2)/(1-b1),
    m = (1-b1) g, sqrt(v) = sqrt(1-b2) |g|."""
    from adam_oracle import BETA1, BETA2, EPS, adam_reference, advance_powers
    g = np.array([1e-3, -2.5, 3e-9, 0.0, 7.0])
    w0 = np.zeros(5)
    w, m, v = adam_reference(w0, g, np.zeros(5), np.zeros(5), (np.float32(BETA1), np.float32(BETA2)), 1e-4)
    one_m_b1 = float(np.float32(1) - np.float32(BETA1)); one_m_b2 = float(np.float32(1) - np.float32(BETA2))
    sc = np.sqrt(1 - float(np.float32(BETA2))) / (1 - float(np.float32(BETA1))) * one_m_b1 / np.sqrt(one_m_b2)
    expect = -float(np.float32(1e-4)) * sc * g / (np.abs(g) + float(np.float32(EPS)) / np.sqrt(one_m_b2))
    assert np.allclose(w, expect, rtol=1e-12, atol=0)
    # with fp32's (1 - beta) the factor sc is 1 to within 1e-6: the step is lr * g / (|g| + eps') for every gradient size
    assert abs(sc - 1) < 1e-6
    assert np.allclose(-w[[1, 4]], 1e-4 * np.sign(g[[1, 4]]), rtol=1e-5)      # |g| >> eps': a step of lr exactly
    assert w[3] == 0 and abs(w[2]) < 1e-4 * 0.01                              # |g| << eps': hardly any step
    assert advance_powers((np.float32(BETA1), np.float32(BETA2))) == (np.float32(np.float32(0.9) * np.float32(0.9)),
                                                                      np.float32(np.float32(0.999) * np.float32(0.999)))
