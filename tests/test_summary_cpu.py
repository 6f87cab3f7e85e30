"""TensorBoard summaries of the adaptation drivers without a GPU: the event-file writer read back by TensorBoard's own
reader, TFRecord framing, the jet / gray colour maps, the colorize restatement against the reference's colorize_img, and
both drivers' --summary around a stub engine."""
import os
import struct
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'real-time-self-adaptive-deep-stereo_b200')
sys.path.insert(0, ROOT)
sys.path.insert(0, PKG)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import colorize_oracle as CO  # noqa: E402
from madstereo import ops, summary as S  # noqa: E402
from madstereo import tf_checkpoint as tfc  # noqa: E402


def _events(logdir):
    from tensorboard.backend.event_processing import event_accumulator as ea
    acc = ea.EventAccumulator(str(logdir), size_guidance={ea.SCALARS: 0, ea.IMAGES: 0})
    acc.Reload()
    return acc


def _decode_png(encoded):
    import cv2
    return cv2.imdecode(np.frombuffer(encoded, np.uint8), cv2.IMREAD_UNCHANGED)[..., ::-1]


def test_event_file_reads_back_in_tensorboard(tmp_path):
    rng = np.random.default_rng(0)
    imgs = {s: rng.integers(0, 256, (5, 7, 3), dtype=np.uint8) for s in (0, 100)}
    w = S.SummaryWriter(str(tmp_path))
    for s in (0, 100):
        w.add_scalar('EPE', 1.5 + s, s)
        w.add_scalar('bad3', 0.25, s)
        w.add_image('full_res_disp/image', imgs[s], s)
    w.close()
    assert os.path.basename(w.path).startswith('events.out.tfevents.')
    acc = _events(tmp_path)
    tags = acc.Tags()
    assert sorted(tags['scalars']) == ['EPE', 'bad3'] and tags['images'] == ['full_res_disp/image']
    assert [(e.step, e.value) for e in acc.Scalars('EPE')] == [(0, 1.5), (100, 101.5)]
    assert [e.value for e in acc.Scalars('bad3')] == [0.25, 0.25]
    for e in acc.Images('full_res_disp/image'):
        assert (e.width, e.height) == (7, 5)
        assert np.array_equal(_decode_png(e.encoded_image_string), imgs[e.step])      # RGB order survives
    assert acc.file_version == 2.0                                        # parsed from 'brain.Event:2'


def test_values_of_one_step_share_one_event(tmp_path):
    from tensorboard.backend.event_processing import event_file_loader
    w = S.SummaryWriter(str(tmp_path))
    w.add_scalar('EPE', 1.0, 0); w.add_scalar('bad3', 0.5, 0)
    w.add_scalar('EPE', 2.0, 100)
    w.close()
    evs = list(event_file_loader.EventFileLoader(w.path).Load())
    assert evs[0].file_version == 'brain.Event:2' and not evs[0].HasField('summary')
    assert [(e.step, [v.tag for v in e.summary.value]) for e in evs[1:]] == [(0, ['EPE', 'bad3']), (100, ['EPE'])]


def test_tfrecord_length_and_crc_fields():
    data = b'\x09' + bytes(8) + b'\x1a\x0dbrain.Event:2'
    rec = S.tfrecord(data)
    assert len(rec) == 8 + 4 + len(data) + 4
    assert struct.unpack('<Q', rec[:8])[0] == len(data)
    assert tfc.unmask_crc(struct.unpack('<I', rec[8:12])[0]) == tfc.crc32c(rec[:8])
    assert rec[12:12 + len(data)] == data
    assert tfc.unmask_crc(struct.unpack('<I', rec[-4:])[0]) == tfc.crc32c(data)
    # masked CRC32C of the 8 length bytes, computed from the definitions: CRC-32C (reflected 0x82F63B78) then LevelDB's mask
    crc = 0xFFFFFFFF
    for b in rec[:8]:
        crc ^= b
        for _ in range(8):
            crc = (crc >> 1) ^ (0x82F63B78 if crc & 1 else 0)
    crc ^= 0xFFFFFFFF
    assert struct.unpack('<I', rec[8:12])[0] == ((((crc >> 15) | (crc << 17)) + 0xa282ead8) & 0xFFFFFFFF)


def test_jet_and_gray_luts_on_matplotlib_breakpoints():
    """Entries computed by hand from matplotlib's segment data, entry i at x = i / 255, linear between breakpoints."""
    jet, gray = ops.colormap_lut('jet'), ops.colormap_lut()
    assert jet.shape == (256, 3) and jet.dtype == np.float32
    assert np.array_equal(jet[0], np.float32([0, 0, 0.5])) and np.array_equal(jet[255], np.float32([0.5, 0, 0]))
    # red: 0 up to x = 0.35, 1 from 0.66 to 0.89, then down to 0.5 at x = 1
    assert jet[89, 0] == 0 and jet[170, 0] == 1 and jet[226, 0] == 1
    assert jet[200, 0] == np.float32(1.0) and abs(jet[240, 0] - (1 - 0.5 * (240 / 255 - 0.89) / 0.11)) < 1e-7
    # green: 0 below 0.125, 1 on [0.375, 0.64]; blue rises 0.5 -> 1 on [0, 0.11]
    assert jet[31, 1] == 0 and jet[96, 1] == 1 and jet[163, 1] == 1 and jet[233, 1] == 0
    assert abs(jet[16, 2] - (0.5 + 0.5 * (16 / 255) / 0.11)) < 1e-7
    assert abs(jet[64, 1] - (64 / 255 - 0.125) / 0.25) < 1e-7
    assert abs(jet[128, 0] - (128 / 255 - 0.35) / 0.31) < 1e-7
    assert np.array_equal(gray[:, 0], gray[:, 2]) and np.array_equal(gray[:, 1], gray[:, 2])
    assert gray[0, 0] == 0 and gray[255, 0] == 1 and abs(gray[51, 0] - 0.2) < 1e-7
    with pytest.raises(Exception, match='viridis'):
        ops.colormap_lut('viridis')


def test_colorize_restatement_equals_the_reference_colorize_img():
    """tests/golden/reference_colorize.npz: the reference's colorize_img through the TF shim (make_colorize_golden.py)."""
    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'reference_colorize.npz'))
    assert np.array_equal(g['lut_jet'], ops.colormap_lut('jet'))
    keys = sorted(k[:-len('__out')] for k in g.files if k.endswith('__out'))
    assert len(keys) == 10
    for key in keys:
        lut = g['lut_' + key.split('__')[1]]
        vmin, vmax = [None if np.isnan(x) else float(x) for x in g[key + '__range']]
        got = CO.colorize(g[key + '__value'], lut, vmin, vmax)
        assert np.array_equal(got, g[key + '__out']), key
    # the tie cases hold exact .5 products that rint sends to the even neighbour
    v = g['ties_auto__jet__value'][..., 0].ravel()
    x = v * np.float32(255)
    assert np.sum(x - np.floor(x) == 0.5) >= 100


def test_restatement_out_of_range_constant_and_normalization():
    lut = ops.colormap_lut('jet')
    v = np.array([-1, 0, 5, 10, 11], np.float32).reshape(1, 1, 5, 1)
    idx = CO.colorize_index(v, 0.0, 10.0)
    assert idx.ravel().tolist() == [256, 0, 128, 255, 256]               # 127.5 -> 128; outside the range: zeros
    c = CO.colorize(v, lut, 0.0, 10.0)
    assert np.array_equal(c[0, 0, 0], [0, 0, 0]) and np.array_equal(c[0, 0, 4], [0, 0, 0])
    assert not CO.colorize(np.full((2, 3, 3, 1), 4.0, np.float32), lut).any()       # constant map: black
    assert not CO.summary_image(np.full((1, 3, 3, 1), 4.0, np.float32), lut).any()
    u8 = CO.summary_u8(np.array([[[0.0, 0.25, 0.5]]], np.float32))
    assert u8.tolist() == [[[0, 127, 255]]]                              # 255 / 0.5 = 510: 0.25 * 510 = 127.5 truncated
    u8 = CO.summary_u8(np.array([[[-1.0, 0.0, 0.5]], [[np.nan, 0, 0]]], np.float32))
    assert u8.tolist() == [[[1, 128, 191]], [[255, 0, 0]]]               # centred on 128, non-finite pixel red


# ---- drivers with a stub engine ---------------------------------------------------------------------------------------
class _Map:
    def __init__(self, h, w):
        self.h, self.w, self.value = h, w, None

    def numpy(self):
        return self.value.copy()

    def tensor(self):
        return self.value


class _Net:
    def __init__(self, h, w):
        self.d = [_Map(h, w) for _ in range(6)]

    def get_disparities(self):
        return self.d


class _Adapt:
    def __init__(self, net):
        self.net, self.calls = net, []
        self.reset_counter, self.fetch_counter, self.sample_distribution = 0, [0] * 5, np.zeros(5)

    def get_variable_names(self):
        return ['model/context-1/weights']

    def load_weights(self, w, strict=True):
        pass

    def step(self, left, right, gt=None, want_disp_mask=0, prefetch=None, proxy=None):
        k = len(self.calls)
        h, w = left.shape[1:3]
        self.net.d[-1].value = (np.arange(h * w, dtype=np.float32).reshape(1, h, w, 1) + k)
        self.calls.append(gt is not None)
        return {'loss': 0.1, 'train_loss': 0.0, 'epe': 1.0 + k, 'bad3': 0.001 * k, 'blocks': [0], 'reset': False}


def _dataset(tmp_path, n, continual):
    import cv2
    rng = np.random.default_rng(5)
    l = rng.integers(0, 256, (12, 20, 3), dtype=np.uint8)
    names = [str(tmp_path / n_) for n_ in ('l.png', 'r.png', 'g.png', 'p.png')]
    cv2.imwrite(names[0], l); cv2.imwrite(names[1], l)
    cv2.imwrite(names[2], (rng.uniform(1, 30, (12, 20)) * 256).astype(np.uint16))
    cv2.imwrite(names[3], (rng.uniform(1, 30, (12, 20)) * 256).astype(np.uint16))
    lst = tmp_path / 'list.csv'
    lst.write_text(''.join(';'.join(names if continual else names[:3]) + '\n' for _ in range(n)))
    tfc.write_checkpoint(str(tmp_path / 'w.ckpt'), {'model/context-1/weights': np.zeros((3, 3, 2, 2), np.float32)})
    return str(lst)


@pytest.mark.parametrize('driver', ['Stereo_Online_Adaptation', 'Stereo_Continual_Adaptation'])
@pytest.mark.parametrize('with_summary', [True, False])
def test_driver_summary_with_a_stub_engine(driver, with_summary, tmp_path):
    import importlib
    d = importlib.import_module(driver)
    continual = 'Continual' in driver
    lst = _dataset(tmp_path, 201, continual)
    out = tmp_path / 'out'
    out.mkdir()
    argv = ['-l', lst, '-o', str(out), '--weights', str(tmp_path / 'w.ckpt'), '--modelName', 'MADNet', '--blockConfig',
            os.path.join(PKG, 'block_config', 'MadNet_full.json'), '--imageShape', '8', '16'] + (['--summary'] if with_summary else [])
    made = {}
    lut = ops.colormap_lut('jet')

    def build(a, cfg):
        made['net'] = _Net(8, 16)
        made['adapt'] = _Adapt(made['net'])
        return made['net'], made['adapt']

    seen = []

    def colorize(value):
        seen.append(np.asarray(value).copy())
        return CO.summary_image(np.asarray(value, np.float32), lut)

    d.main(d.build_parser().parse_args(argv), build=build, colorize=colorize)
    events = [f for f in os.listdir(str(out)) if f.startswith('events.out.tfevents.')]
    calls = made['adapt'].calls
    assert len(calls) == 201
    if not with_summary:
        assert events == [] and not seen
        assert not any(calls) if continual else all(calls)
        return
    assert len(events) == 1
    acc = _events(out)
    images = ['full_res_disp/image', 'proxy_disp/image', 'gt_disp/image'] if continual else ['full_res_disp/image', 'gt_disp/image']
    assert sorted(acc.Tags()['scalars']) == ['EPE', 'bad3'] and sorted(acc.Tags()['images']) == sorted(images)
    assert [e.step for e in acc.Scalars('EPE')] == [0, 100, 200]
    assert [e.value for e in acc.Scalars('EPE')] == [1.0, 101.0, 201.0]
    assert [e.value for e in acc.Scalars('bad3')] == [np.float32(0.0), np.float32(0.1), np.float32(0.2)]
    if continual:                                    # gt goes to the engine on summary frames only
        assert [i for i, c in enumerate(calls) if c] == [0, 100, 200]
    assert len(seen) == 3 * len(images)
    for k, step in enumerate((0, 100, 200)):
        disp = seen[k * len(images)]
        assert np.array_equal(disp[0, ..., 0], np.arange(128, dtype=np.float32).reshape(8, 16) + step)
    for e in acc.Images('full_res_disp/image'):
        disp = np.arange(128, dtype=np.float32).reshape(1, 8, 16, 1) + e.step
        assert (e.width, e.height) == (16, 8)
        assert np.array_equal(_decode_png(e.encoded_image_string), CO.summary_image(disp, lut))
