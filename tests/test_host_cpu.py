"""CPU tests of the host side: C-ABI exports, layer/group tables through the engine (no kernels run),
samplers and the reward recurrence against the oracle transcription."""
import ctypes
import importlib.util
import json
import os
import re

import numpy as np
import pytest

from conftest import PKG, ROOT
from madstereo import _lib
from oracle import adaptation as OA
from oracle.madnet import param_shapes, mad_groups_full
from Sampler import sampler_factory

_spec = importlib.util.spec_from_file_location('make_engine_kernels', os.path.join(ROOT, 'tests', 'golden', 'make_engine_kernels.py'))
_mk = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(_mk)


def test_library_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, 'include', 'madstereo.h')).read()
    declared = set(re.findall(r'\b(ms_\w+)\s*\(', hdr))
    assert len(declared) >= 30
    h = ctypes.CDLL(_lib.LIB_PATH)
    for name in declared:
        assert hasattr(h, name), 'missing export %s' % name
    assert declared == set(_lib.EXPORTS)
    assert _lib.lib().ms_version() >= 100


def test_ctypes_table_matches_the_header_prototypes():
    """Every prototype of include/madstereo.h against madstereo/_lib.py:_SIGS -- argument count and the C type class of each
    argument and of the return value (a mismatch here is a silent stack / register mix-up at call time)."""
    hdr = open(os.path.join(ROOT, 'include', 'madstereo.h')).read()
    hdr = re.sub(r'/\*.*?\*/', ' ', hdr, flags=re.S)
    hdr = re.sub(r'//[^\n]*', ' ', hdr)
    hdr = re.sub(r'^\s*#[^\n]*', ' ', hdr, flags=re.M)           # preprocessor lines
    hdr = re.sub(r'extern\s+"C"\s*\{', ' ', hdr)
    protos = re.findall(r'([A-Za-z_][\w\s\*]*?)\b(ms_\w+)\s*\(([^;{]*?)\)\s*;', hdr)
    assert len(protos) >= 30

    def cls(t):
        t = t.strip()
        if '*' in t:
            return 'char*' if re.match(r'(const\s+)?char\s*\*$', t) else 'ptr'
        base = re.sub(r'\bconst\b', '', t).strip()
        return {'int': 'int', 'float': 'float', 'size_t': 'size_t', 'long long': 'll', 'double': 'double', 'void': 'void',
                'unsigned int': 'uint'}.get(base, base)

    want_cls = {ctypes.c_int: 'int', ctypes.c_float: 'float', ctypes.c_size_t: 'size_t', ctypes.c_void_p: 'ptr',
                ctypes.c_char_p: 'char*', ctypes.c_longlong: 'll', ctypes.c_double: 'double', ctypes.c_uint: 'uint', None: 'void'}
    seen = set()
    for ret, name, args in protos:
        assert name in _lib._SIGS, 'header declares %s, the ctypes table does not know it' % name
        seen.add(name)
        restype, argtypes = _lib._SIGS[name]
        params = [a.strip() for a in args.split(',')] if args.strip() not in ('', 'void') else []
        ptypes = []
        for a in params:
            a = re.sub(r'\[[^\]]*\]', '*', a)                       # array parameter = pointer
            m = re.match(r'(.*?)(\b\w+)?\s*$', a)                   # strip the parameter name
            t = a if a.rstrip().endswith('*') else m.group(1)
            ptypes.append(cls(t))
        got = [want_cls.get(t, 'ptr' if hasattr(t, 'contents') or getattr(t, '__name__', '').startswith('LP_') else str(t)) for t in argtypes]
        got = ['ptr' if g == 'char*' else g for g in got]
        exp = ['ptr' if g == 'char*' else g for g in ptypes]
        assert len(got) == len(exp), '%s: header has %d parameters, ctypes table %d' % (name, len(exp), len(got))
        assert got == exp, '%s: header %s vs ctypes %s' % (name, exp, got)
        r = cls(ret.split(';')[-1].split('}')[-1])
        assert ('ptr' if r in ('char*', 'ptr') else r) == ('ptr' if want_cls.get(restype, str(restype)) in ('char*', 'ptr') else want_cls.get(restype, str(restype))), name
    assert seen == set(_lib._SIGS), sorted(set(_lib._SIGS) - seen)


def _engine_tables(groups_cfg, net='MADNet', batch=1, h=384, w=1280, variant=(2, 1, True)):
    L = _lib.lib()
    radius_d, stride, warping = variant
    e = L.ms_engine_create(net.encode(), batch, h, w, radius_d, stride, int(warping))
    assert e, L.ms_last_error()
    n = L.ms_engine_num_layers(e)
    layers = []
    for i in range(n):
        nm, sc, bn = (ctypes.create_string_buffer(128) for _ in range(3))
        dims = (ctypes.c_int * 7)(); alpha = ctypes.c_float()
        assert L.ms_engine_layer_info(e, i, nm, 128, sc, 128, bn, 128, dims, ctypes.byref(alpha)) == 0
        layers.append((nm.value.decode(), sc.value.decode(), bn.value.decode(), list(dims), alpha.value))
    name_to_idx = {l[0]: i for i, l in enumerate(layers)}
    arr = (ctypes.c_int * n)(*([-1] * n))
    for g, names in enumerate(groups_cfg):
        for nm in names:
            if nm in name_to_idx:
                arr[name_to_idx[nm]] = g
    assert L.ms_engine_set_groups(e, arr, n, len(groups_cfg)) == 0
    npar, nws = ctypes.c_size_t(), ctypes.c_size_t()
    assert L.ms_engine_sizes(e, ctypes.byref(npar), ctypes.byref(nws)) == 0, L.ms_last_error()
    ranges = []
    for g in range(len(groups_cfg)):
        b, en = ctypes.c_size_t(), ctypes.c_size_t()
        assert L.ms_engine_group_range(e, g, ctypes.byref(b), ctypes.byref(en)) == 0
        ranges.append((b.value, en.value))
    offs = []
    for i in range(n):
        wo, bo = ctypes.c_size_t(), ctypes.c_size_t()
        L.ms_engine_param_offsets(e, i, ctypes.byref(wo), ctypes.byref(bo))
        offs.append((wo.value, bo.value))
    L.ms_engine_destroy(e)
    return layers, npar.value, nws.value, ranges, offs


def test_engine_layer_table_matches_reference_variable_names():
    cfg = json.load(open(os.path.join(PKG, 'block_config', 'MadNet_full.json')))
    layers, npar, nws, ranges, offs = _engine_tables(cfg)
    shapes = param_shapes()
    names = []
    for nm, sc, bn, d, alpha in layers:
        assert shapes[sc + '/weights'] == (d[0], d[1], d[2], d[3])
        assert shapes[sc + '/' + bn] == (d[3],)
        names += [sc + '/weights', sc + '/' + bn]
    assert set(names) == set(shapes)
    # module sizes of SURVEY §8(a) a15 (arena ranges include <=3 floats of alignment padding per tensor)
    expect = [1112801, 745185, 588449, 468577, 911058]
    for (b, e), ex, grp in zip(ranges, expect, mad_groups_full()):
        assert ex <= e - b <= ex + 4 * len(grp)
    assert 3826070 <= npar <= 3826070 + 4 * 98
    assert nws > 0
    # groups are contiguous, ordered and disjoint
    for (b0, e0), (b1, e1) in zip(ranges, ranges[1:]):
        assert e0 == b1
    # 16-byte alignment of every tensor (float4 loads)
    assert all(w % 4 == 0 and b % 4 == 0 for w, b in offs)


@pytest.mark.parametrize('cfg', _mk.CONFIGS, ids=[c[0] for c in _mk.CONFIGS])
def test_engine_sizes_every_kernel_sequence_config(cfg):
    """ms_engine_sizes lays the engine out without a device, and the layout checks every layer's planned views against
    the layer: MADNet with its MAD modules at the radius / stride / warping variants, and DispNet."""
    _name, net, batch, h, w, variant, _steps = cfg
    groups = json.load(open(os.path.join(PKG, 'block_config', 'MadNet_full.json'))) if net == 'MADNet' else []
    layers, npar, nws, _ranges, _offs = _engine_tables(groups, net, batch, h, w, variant or (2, 1, True))
    assert len(layers) == (49 if net == 'MADNet' else 32)
    assert npar > 0 and nws > 0


def test_unknown_network_name():
    L = _lib.lib()
    assert not L.ms_engine_create(b'NoSuchNet', 1, 64, 64, 2, 1, 1)
    assert b'Unrecognized network name' in L.ms_last_error()


def test_samplers_match_reference_semantics():
    d = np.ones(5) / 5
    s = sampler_factory.get_sampler('SEQUENTIAL', 2)
    assert [s.sample(d) for _ in range(3)] == [[0, 1], [1, 2], [2, 3]]
    o = OA.SequentialSampler(2)
    assert [o.sample(d) for _ in range(3)] == [[0, 1], [1, 2], [2, 3]]
    assert sampler_factory.get_sampler('FIXED', 1, [3]).sample(d) == [3]
    assert sampler_factory.get_sampler('FIXED', 1, 2).sample(d) == [2]
    a = sampler_factory.get_sampler('ARGMAX', 2).sample(np.array([0.1, 0.5, 0.05, 0.3, 0.05]))
    assert set(int(x) for x in a) == {1, 3}
    for name in ('RANDOM', 'PROBABILITY'):
        np.random.seed(7)
        mine = sampler_factory.get_sampler(name, 2).sample(d)
        np.random.seed(7)
        ref = OA.sample(name, 2, d)
        assert list(mine) == list(ref)
    with pytest.raises(AssertionError):
        sampler_factory.get_sampler('SAMPLE', 1)          # the reference's invalid default (:303)
    assert set(sampler_factory.AVAILABLE_SAMPLER) == {'FIXED', 'RANDOM', 'ARGMAX', 'SEQUENTIAL', 'PROBABILITY'}


def test_reward_recurrence_matches_transcription():
    from madstereo.adaptation import softmax
    tr = OA.RewardTracker(5)
    losses = [0.3, 0.28, 0.31, 0.25, 0.2]
    blocks = [[0], [1], [2], [3], [4]]
    h = np.zeros(5); l1 = l2 = 0.0; last = []
    for t, (L, b) in enumerate(zip(losses, blocks)):
        tr.update(L, b)
        if t == 0:
            l2 = l1 = L
        gain = (2 * l1 - l2) - L
        h = 0.99 * h
        for i in last:
            h[i] += 0.01 * gain
        last = b; l2, l1 = l1, L
        assert np.allclose(tr.h, h)
    assert np.allclose(softmax(h).sum(), 1.0)


def test_sampler_and_block_configs_match_reference_golden_vectors():
    """Vectors produced by the reference's OWN Sampler/sampler_factory.py and block_config/*.json (imported in the build
    container by tests/golden/make_reference_golden.py): the mirror must reproduce every draw with the same numpy seed."""
    import json
    g = json.load(open(os.path.join(ROOT, 'tests', 'golden', 'reference_sampler.json')))
    assert sorted(sampler_factory.AVAILABLE_SAMPLER) == g['available_sampler']
    for c in g['cases']:
        d = np.array(c['distribution'])
        np.random.seed(c['seed'])
        s = sampler_factory.get_sampler(c['name'], c['blocks'], fixed_id=2)
        draws = [[int(v) for v in s.sample(d)] for _ in range(len(c['draws']))]
        if c['name'] == 'ARGMAX':
            draws = [sorted(v) for v in draws]
        assert draws == c['draws'], (c['name'], c['blocks'], c['seed'])
    pkg = os.path.join(ROOT, 'real-time-self-adaptive-deep-stereo_b200', 'block_config')
    for fn, ref_cfg in g['block_config'].items():
        assert json.load(open(os.path.join(pkg, fn))) == ref_cfg, fn


def test_loss_factory_entry_point_errors_like_the_reference():
    from Losses import loss_factory
    with pytest.raises(Exception, match='Unknown loss function selected'):
        loss_factory.get_reprojection_loss('no_such_loss')
    with pytest.raises(NotImplementedError):
        loss_factory.get_reprojection_loss('mean_l1')
    assert callable(loss_factory.get_reprojection_loss('mean_SSIM_l1', reduced=True))
    assert set(loss_factory.ALL_LOSSES) >= {'mean_SSIM_l1', 'ssim_l1', 'ZNCC'}


def test_stereonet_base_class_protocol(capsys):
    """The construction protocol, printed lines, defaults and getters of Nets.Stereo_net.StereoNet (reference
    Nets/Stereo_net.py:26-46, 99-107, 131-222) on a network without an engine."""
    from Nets import Stereo_net

    class Shape(object):
        def __init__(self, shape): self.shape = shape

    class Toy(Stereo_net.StereoNet):
        _netName = 'Toy'

        def _validate_args(self, args):
            super(Toy, self)._validate_args(args)
            return args

        def _preprocess_inputs(self, args):
            self.seen = dict(args)

        def _build_network(self, args):
            a, b, d = Shape((1, 4, 8, 16)), Shape((1, 2, 4, 32)), Shape((1, 4, 8, 1))
            self._add_to_layers('left/conv1', a, ['w1:0', 'b1:0'])
            self._add_to_layers('right/conv1', b)
            self._add_to_layers('final_disp', d, ['w1:0', 'b1:0', 'w2:0'])
            self._layers['rescaled_prediction'] = d
            self._disparities.append(d)

    net = Toy(left_img=0, right_img=0)
    out = capsys.readouterr().out.splitlines()
    assert out[0] == '=' * 50 and out[1] == 'Starting Creation of Toy' and out[2] == '=' * 50
    assert [l for l in out if l.startswith('WARNING')] == [
        'WARNING: no split points selected, the network will flow without interruption',
        'WARNING: train_portion not specified, using default END',
        'WARNING: sequence flag not setted, configuring the network for single image adaptation',
        'WARNING: flag for trainign not setted, using default False']
    assert out[-4:] == ['Args Validated, setting up graph', 'Meta op to preprocess data created', 'Network ready', '=' * 50]
    assert net.seen['split_layers'] == [None] and net.seen['train_portion'] == 'BEGIN' and net.seen['sequence'] is False
    assert str(net) == ('Layer left/conv1: (1, 4, 8, 16)\nLayer right/conv1: (1, 2, 4, 32)\n'
                        'Prediction Layer final_disp: (1, 4, 8, 1)\nPrediction Layer rescaled_prediction: (1, 4, 8, 1)\n')
    assert repr(net) == str(net)
    assert list(net.get_layers_names()) == ['left/conv1', 'right/conv1', 'final_disp', 'rescaled_prediction']
    assert net.get_variables('left/conv1') == ['w1:0', 'b1:0'] and net.get_variables('right/conv1') == []
    assert net.get_variables('rescaled_prediction') == [] and len(net.get_variables('final_disp')) == 3
    assert net.get_trainable_variables() == ['w1:0', 'b1:0', 'w2:0']
    assert net.get_disparities() == [net['final_disp']] and net.get_all_layers() is net._layers and net.get_placeholders() == []
    with pytest.raises(KeyError):
        net.get_variables('nope')
    with pytest.raises(Exception, match='Unable to find placeholder'):
        net.get_placeholder('x')
    with pytest.raises(Exception, match='Invalid portion'):
        Toy(left_img=0, right_img=0, train_portion='MIDDLE')
    with pytest.raises(Exception, match='split_layers'):
        Toy(left_img=0, right_img=0, split_layers=['left/conv1'])
    quiet = Toy(left_img=0, right_img=0, split_layers=[None], sequence=True, train_portion='BEGIN', is_training=False)
    assert quiet.seen['sequence'] is True
    assert dict(Toy.getPossibleArsg())['sequence'].startswith('flag to use network')


class _NoCudaCtx(object):
    def __init__(self, *_a, **_k): pass
    def __enter__(self): return self
    def __exit__(self, *_a): return False


class _Buf(object):
    """What the drivers pass as left_img / right_img: only .shape (and optionally .device) is consulted at build time."""
    def __init__(self, shape): self.shape = shape


def _build_mirror_on_cpu(monkeypatch, name, h, w):
    import torch
    import Nets
    monkeypatch.setattr(torch.cuda, 'is_available', lambda: True)
    monkeypatch.setattr(torch.cuda, 'current_device', lambda: 0)
    monkeypatch.setattr(torch.cuda, 'device', _NoCudaCtx)
    return Nets.get_stereo_net(name, dict(left_img=_Buf((1, h, w, 3)), right_img=_Buf((1, h, w, 3)), split_layers=[None],
                                          sequence=True, train_portion='BEGIN', bulkhead=True))


def test_madnet_mirror_matches_reference_graph_layers_and_variable_lists(monkeypatch, capsys):
    """The host mirror built without a device (engine handle only, nothing bound) against what the reference's own
    Nets/MadNet.py produced over the TF shim: layer names in order, `str(net)`, the variable list of every layer a
    block_config names, trainable-variable order."""
    import json
    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'reference_graph_madnet_64x128.npz'))
    net = _build_mirror_on_cpu(monkeypatch, 'MADNet', 64, 128)
    assert list(net.get_layers_names()) == [str(s) for s in g['layer_names']]
    assert str(net) == str(g['str_net'])
    ref_vars = json.loads(str(g['get_variables']))
    for layer, names in ref_vars.items():
        assert [v.name for v in net.get_variables(layer)] == names, layer
    assert [v.name[:-2] for v in net.get_trainable_variables()] == [str(s) for s in g['variable_names']]
    assert len(net.get_disparities()) == 6 and net.get_disparities()[-1] is net['rescaled_prediction']


def test_dispnet_mirror_matches_reference_graph_layers(monkeypatch, capsys):
    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'reference_graph_dispnet_64x128.npz'))
    net = _build_mirror_on_cpu(monkeypatch, 'Dispnet', 64, 128)
    assert list(net.get_layers_names()) == [str(s) for s in g['layer_names']]
    assert [v.name[:-2] for v in net.get_trainable_variables()] == [str(s) for s in g['variable_names']]
    assert len(net.get_disparities()) == 7


def test_mad_groups_of_the_product_equal_the_reference_var_lists(monkeypatch, capsys):
    """OnlineAdaptation resolves block_config/MadNet_full.json through net.get_variables() exactly like
    Stereo_Online_Adaptation.py:109-118; the layer sets it hands to the engine must own the variables the reference's own
    train ops got (tests/golden/reference_graph_madnet_64x128.npz: mad<k>_vars)."""
    import json
    from madstereo import engine as eng_mod
    from madstereo.adaptation import OnlineAdaptation
    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'reference_graph_madnet_64x128.npz'))
    net = _build_mirror_on_cpu(monkeypatch, 'MADNet', 64, 128)
    monkeypatch.setattr(eng_mod.StereoEngine, 'bind', lambda self: None)
    cfg = json.load(open(os.path.join(ROOT, 'real-time-self-adaptive-deep-stereo_b200', 'block_config', 'MadNet_full.json')))
    ad = OnlineAdaptation(net, mode='MAD', train_config=cfg, sample_mode='SEQUENTIAL')
    assert len(ad.groups) == 5 and ad.num_actions == 5
    layers = net.engine.layers
    for k, idxs in enumerate(ad.groups):
        mine = set()
        for i in idxs:
            mine |= {layers[i].scope + '/weights', layers[i].scope + '/' + layers[i].bias_name}
        assert mine == set(str(s) for s in g['mad%d_vars' % k]), k
    flat = [i for idxs in ad.groups for i in idxs]
    assert len(flat) == len(set(flat)) == len(layers)            # a partition of the 49 conv layers
