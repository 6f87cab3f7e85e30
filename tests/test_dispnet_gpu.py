"""GPU parity of DispNet-C (BASELINE config 4): forward and one/two FULL adaptation steps vs the CPU oracle."""
import json
import os

import numpy as np
import pytest
import torch

from conftest import PKG

pytestmark = pytest.mark.gpu


def rel_linf(a, b):
    a = np.asarray(a, dtype=np.float64); b = np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def build(left, right, mode):
    import Nets
    from madstereo.adaptation import OnlineAdaptation
    from oracle.dispnet import init_params
    lt = torch.as_tensor(left).cuda(); rt = torch.as_tensor(right).cuda()
    net = Nets.get_stereo_net('Dispnet', dict(left_img=lt, right_img=rt, split_layers=[None], sequence=True,
                                              train_portion='BEGIN', bulkhead=False, correlation=True))
    ad = OnlineAdaptation(net, mode=mode, lr=1e-4)
    params = init_params(seed=7)
    ad.load_weights(params)
    return net, ad, params, lt, rt


# (h, w) or (h, w, batch): batch 3 (odd, every frame seeded separately) compares every frame of the batched step
@pytest.mark.parametrize('hw', [(64, 128), (100, 200), pytest.param((64, 128, 3), id='64x128-b3')])
def test_dispnet_forward_parity(hw):
    from madstereo.synthetic import make_pair
    from oracle.dispnet import DispNetOracle
    h, w, batch = (tuple(hw) + (1,))[:3]
    left, right, _ = make_pair(h, w, seed=5, batch=batch)
    net, ad, params, lt, rt = build(left, right, 'NONE')
    assert len(net.get_disparities()) == 7
    names = list(net.get_layers_names())
    assert names[:6] == ['conv1a', 'conv1b', 'conv2a', 'conv2b', 'conv_redir', 'corr'] and names[-1] == 'rescaled_prediction'
    assert [v.name for v in net.get_variables('conv3/1')] == ['model/conv3/1/weights:0', 'model/conv3/1/bias:0']
    assert net.get_variables('conv1b') == [] and net.get_variables('up5/deconv')[0].shape == (4, 4, 512, 1024)
    out = ad.step(lt, rt, want_disp_mask=0b1111111)
    disps, layers = DispNetOracle(params).forward(left, right)
    for name in ('conv1a', 'conv1b', 'conv2a', 'conv_redir', 'corr', 'conv3', 'conv4/1', 'conv6/1', 'up5/deconv', 'up5/predict',
                 'up5/up_predict', 'up5/concat', 'up3/concat', 'up1/concat', 'prediction'):
        assert rel_linf(net[name].numpy(), layers[name].numpy()) < 2e-4, name
    for i, (d, ref) in enumerate(zip(net.get_disparities(), disps)):
        assert rel_linf(d.numpy(), ref.numpy()) < 1e-3, 'disparity %d' % i
    from oracle import tf1_ops as T
    ref_loss = float(T.reprojection_loss(disps[-1], torch.tensor(left), torch.tensor(right)))
    assert abs(out['loss'] - ref_loss) < 2e-5


def test_dispnet_full_step_parity():
    _check_full_step(batch=1)


def test_dispnet_full_step_parity_batch3():
    _check_full_step(batch=3)


def _check_full_step(batch):
    from madstereo.synthetic import make_pair
    from oracle.dispnet import DispNetAdapter
    left, right, _ = make_pair(64, 128, seed=5, batch=batch)
    net, ad, params, lt, rt = build(left, right, 'FULL')
    orc = DispNetAdapter(params, mode='FULL', lr=1e-4)
    out = ad.step(lt, rt)
    ref = orc.step(left, right)
    assert abs(out['loss'] - ref['full_loss']) < 2e-5
    g = net.engine.param_views(net.engine.grads)
    for n, gr in ref['grads'].items():
        assert rel_linf(g[n].cpu().numpy(), gr) < 1e-2, n
    wv = net.engine.export_params()
    for n in ref['grads']:
        dref = orc.net.p[n].detach().numpy() - params[n]
        assert np.abs((wv[n] - params[n]) - dref).max() <= 0.15 * np.abs(dref).max() + 1e-7, n


def test_dispnet_mad_asserts_like_the_reference():
    from madstereo.synthetic import make_pair
    import Nets
    from madstereo.adaptation import OnlineAdaptation
    left, right, _ = make_pair(64, 128, seed=5)
    lt = torch.as_tensor(left).cuda(); rt = torch.as_tensor(right).cuda()
    net = Nets.get_stereo_net('Dispnet', dict(left_img=lt, right_img=rt, split_layers=[None], sequence=True,
                                              train_portion='BEGIN'))
    cfg = json.load(open(os.path.join(PKG, 'block_config', 'dispnet_full.json')))
    with pytest.raises(AssertionError):       # 6 side predictions vs 5 groups (Stereo_Online_Adaptation.py:97)
        OnlineAdaptation(net, mode='MAD', train_config=cfg)
