"""MAD module losses at 1/s resolution (--reprojectionScale), without a GPU: the oracle against the reference's own graph code
(tests/golden/reference_graph_madnet_rs_64x128.npz, written by tests/golden/make_reference_rs_golden.py), and the drivers'
handling of the flag."""
import json
import os

import numpy as np
import pytest
import torch

from conftest import PKG, ROOT
from reprojection_scale_oracle import RsOracleAdapter, module_loss

GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'reference_graph_madnet_rs_64x128.npz')


def _rel(a, b):
    a = np.asarray(a, dtype=np.float64); b = np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def _sub(a, n=4096):
    a = np.asarray(a).ravel()
    return a[::max(1, a.size // n)]


def _inputs(g, tag=''):
    return tuple(g[k + tag].astype(np.float32) for k in ('left', 'right', 'proxy'))


@pytest.mark.parametrize('loss', ['reprojection', 'proxy'])
def test_oracle_module_losses_and_gradients_match_reference_graph(loss):
    """Every module loss at s = 2, 3, 4 and module 0 / 2 / 4 gradients at s = 2, 3, at the bars test_oracle_cpu applies
    at s = 1 (losses 2e-6 absolute, subsampled gradients 2e-4 relative)."""
    from oracle.madnet import init_params
    g = np.load(GOLDEN)
    left, right, proxy = _inputs(g)
    params = init_params(seed=42)
    for s in (2, 3, 4):
        for k in range(5):
            orc = RsOracleAdapter(params, reprojection_scale=s, loss=loss, lr=0.0)
            out = orc.step(left, right, k, proxy=proxy)
            assert abs(out['train_loss'] - float(g['rs%d_%s_mad%d_loss' % (s, loss, k)])) < 2e-6, (s, k)
            keys = [x for x in g.files if x.startswith('rs%d_%s_mad%d_grad:' % (s, loss, k))]
            assert bool(keys) == (s in (2, 3) and k in (0, 2, 4))
            for key in keys:
                assert _rel(_sub(out['grads'][key.split(':', 1)[1]]), g[key]) < 2e-4, key


def test_oracle_module_losses_match_reference_graph_with_crop():
    """100x200 pads to 128x256: the first resize's centre crop is active before the second resize."""
    from oracle.madnet import MadNetOracle, init_params
    g = np.load(GOLDEN)
    left, right, proxy = (torch.as_tensor(x) for x in _inputs(g, '100'))
    disps, _ = MadNetOracle(init_params(seed=42)).forward(left, right)
    for k in range(5):
        for loss in ('reprojection', 'proxy'):
            got = float(module_loss(disps[k], left, right, 3, loss, proxy))
            assert abs(got - float(g['p100_rs3_%s_mad%d_loss' % (loss, k)])) < 2e-6, (loss, k)


def test_scale_one_is_the_full_resolution_module_loss():
    from oracle.adaptation import OracleAdapter
    from oracle.madnet import init_params
    g = np.load(GOLDEN)
    left, right, proxy = _inputs(g)
    params = init_params(seed=42)
    a = RsOracleAdapter(params, reprojection_scale=1).step(left, right, 2)
    b = OracleAdapter(params, mode='MAD').step(left, right, 2)
    assert a['train_loss'] == b['train_loss'] and a['full_loss'] == b['full_loss']
    for n in b['grads']:
        assert np.array_equal(a['grads'][n], b['grads'][n]), n


# ---------------------------------------------------------------------------------------------------- drivers
def _driver(name):
    import importlib
    return importlib.import_module(name)


def _args(d, lst, out, *extra):
    cfg = os.path.join(PKG, 'block_config', 'MadNet_full.json')
    return d.build_parser().parse_args(['-l', lst, '-o', str(out), '--weights', 'x', '--blockConfig', cfg] + list(extra))


class _Built(Exception):
    pass


@pytest.mark.parametrize('driver', ['Stereo_Online_Adaptation', 'Stereo_Continual_Adaptation'])
def test_drivers_pass_the_scale_through_and_refuse_bad_ones(driver, tmp_path, monkeypatch):
    d = _driver(driver)
    monkeypatch.setattr(d.data_reader, 'dataset', lambda *a, **k: None)
    lst = str(tmp_path / 'list.csv')
    seen = {}

    def build(a, train_config):           # stops main() right after the network would have been built
        seen['scale'] = a.reprojectionScale
        raise _Built()

    with pytest.raises(_Built):
        d.main(_args(d, lst, tmp_path, '--modelName', 'MADNet', '--mode', 'MAD', '--reprojectionScale', '2'), build=build)
    assert seen['scale'] == 2
    for bad in ('0', '-1'):
        with pytest.raises(SystemExit):
            d.main(_args(d, lst, tmp_path, '--modelName', 'MADNet', '--reprojectionScale', bad), build=build)
    with pytest.raises(SystemExit):
        d.main(_args(d, lst, tmp_path, '--modelName', 'Dispnet', '--mode', 'MAD', '--reprojectionScale', '2'), build=build)
    seen.clear()
    with pytest.raises(_Built):
        d.main(_args(d, lst, tmp_path, '--modelName', 'Dispnet', '--mode', 'FULL', '--reprojectionScale', '2'), build=build)
    assert seen['scale'] == 2


@pytest.mark.parametrize('driver', ['Stereo_Online_Adaptation', 'Stereo_Continual_Adaptation'])
def test_build_model_hands_the_scale_to_online_adaptation(driver, monkeypatch):
    """MADNet + MAD + --reprojectionScale 2 reaches OnlineAdaptation(reprojection_scale=2)."""
    import madstereo.adaptation
    d = _driver(driver)
    got = {}

    class FakeAdaptation(object):
        def __init__(self, net, **kw):
            got.update(kw)

    monkeypatch.setattr(madstereo.adaptation, 'OnlineAdaptation', FakeAdaptation)
    monkeypatch.setattr(torch.cuda, 'is_available', lambda: True)
    monkeypatch.setattr(torch.cuda, 'current_device', lambda: 0)
    monkeypatch.setattr(torch, 'zeros', lambda *a, **k: None)
    monkeypatch.setattr(d.Nets, 'get_stereo_net', lambda name, args: _FakeStereo())
    cfg = json.load(open(os.path.join(PKG, 'block_config', 'MadNet_full.json')))
    args = _args(d, 'l', 'o', '--modelName', 'MADNet', '--mode', 'MAD', '--reprojectionScale', '2', '--imageShape', '16', '32')
    d.build_model(args, cfg)
    assert got['reprojection_scale'] == 2


class _FakeStereo(object):
    def get_disparities(self):
        return [None] * 6

    def __str__(self):
        return 'fake'
