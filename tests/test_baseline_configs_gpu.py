"""Parity at the BASELINE.json configurations (what one sess.run returns, Stereo_Online_Adaptation.py:194-208).

  config 1  MADNet forward, 640x384                      -> test_madnet_forward_baseline[384x640]
  config 2  MADNet FULL adaptation step, 1280x384        -> test_madnet_full_step_1280x384
  config 3  MADNet MAD step per module, 1280x384         -> test_madnet_mad_step_1280x384[0..4]
  config 4  DispNet forward + FULL step, 1280x384        -> test_dispnet_forward_1280x384 / test_dispnet_full_step_1280x384
  config 5  MADNet 1920x1056 (padded 1920x1088)          -> test_madnet_forward_1920x1056 (oracle forward takes seconds)

At these sizes every level-2/3 map has more than 74 output tiles, i.e. the convolutions run the non-split-K kernels
with the engine's fused epilogue options (channel-stride views, residual, dgrad mask, accumulate) that the small
(<=128x256) engine tests never reach.  Gradients are judged by tests/parity_metrics.py (relative L2 against the fp64
oracle, bounded by twice the fp32 oracle's own distance to fp64 or the stated floor).
"""
import json
import os

import numpy as np
import pytest
import torch

from conftest import PKG
from parity_metrics import assert_grads, grad_report, rel_l2, rel_linf, summarize

pytestmark = pytest.mark.gpu

TOL_DISP = 1e-3          # north star: relative L-inf of every disparity output
TOL_LAYER = 2e-4
TOL_LOSS = 2e-5
TOL_GRAD_L2 = 1e-4       # floor of the per-tensor relative L2 bound (see parity_metrics.assert_grads)
TOL_GRAD_LINF = 1e-2     # secondary bound, not looser than round 1's
TOL_DW_L2 = 1e-3         # adapted weights: |dw_gpu - dw_64|_2 <= max(TOL_DW_L2, 2 x fp32-oracle noise) * |dw_64|_2

# MS_TEST_REPORT_DIR=<dir>: the measured distances are appended to <dir>/baseline_parity.jsonl (nothing is written otherwise)
REPORT = os.path.join(os.environ['MS_TEST_REPORT_DIR'], 'baseline_parity.jsonl') if os.environ.get('MS_TEST_REPORT_DIR') else None


def _log(rec):
    if REPORT is None:
        return
    try:
        os.makedirs(os.path.dirname(REPORT), exist_ok=True)
        with open(REPORT, 'a') as f:
            f.write(json.dumps(rec) + '\n')
    except OSError:
        pass


def build_madnet(left, right, mode):
    import Nets
    from madstereo.adaptation import OnlineAdaptation
    from oracle.madnet import init_params
    lt = torch.as_tensor(left).cuda(); rt = torch.as_tensor(right).cuda()
    args = dict(left_img=lt, right_img=rt, split_layers=[None], sequence=True, train_portion='BEGIN',
                bulkhead=(mode == 'MAD'), warping=True, context_net=True, radius_d=2, stride=1, is_training=False)
    net = Nets.get_stereo_net('MADNet', args)
    cfg = json.load(open(os.path.join(PKG, 'block_config', 'MadNet_full.json')))
    ad = OnlineAdaptation(net, mode=mode, train_config=cfg, lr=1e-4, sample_mode='FIXED', fixed_id=0)
    params = init_params(seed=42)
    ad.load_weights(params)
    return net, ad, params, lt, rt


MADNET_PROBES = ('left/conv2', 'left/conv4', 'right/conv4', 'left/conv6', 'left/conv12', 'right/conv12',
                 'fgc-volume-filtering-6/disp6', 'fgc-volume-filtering-4/disp3', 'fgc-volume-filtering-3/disp1',
                 'fgc-volume-filtering-3/disp6', 'fgc-volume-filtering-2/disp1', 'fgc-volume-filtering-2/disp2',
                 'fgc-volume-filtering-2/disp5', 'fgc-volume-filtering-2/disp6', 'context1', 'context2', 'context3',
                 'context4', 'context5', 'context6', 'final_disp')


def _check_madnet_forward(h, w, seed):
    from madstereo.synthetic import make_pair
    from oracle.madnet import MadNetOracle
    from oracle import tf1_ops as T
    left, right, _ = make_pair(h, w, seed=seed)
    net, ad, params, lt, rt = build_madnet(left, right, 'NONE')
    out = ad.step(lt, rt, want_disp_mask=0b111111)
    disps, layers = MadNetOracle(params).forward(left, right)
    worst_layer = 0.0
    for name in MADNET_PROBES:
        r = rel_linf(net[name].numpy(), layers[name].numpy())
        worst_layer = max(worst_layer, r)
        assert r < TOL_LAYER, (name, r)
    for k in (6, 5, 4, 3, 2):
        c = net.engine.tensor('cost%d' % k).cpu().numpy()
        C = layers['left/conv%d' % (2 * k)].shape[-1]
        assert rel_linf(c[..., C:C + 5], layers['corr%d' % k].numpy()) < TOL_LAYER, 'corr%d' % k
    worst = 0.0
    for i, (d, ref) in enumerate(zip(net.get_disparities(), disps)):
        assert d.shape == tuple(ref.shape)
        r = rel_linf(d.numpy(), ref.numpy())
        worst = max(worst, r)
        assert r < TOL_DISP, ('disparity %d' % i, r)
    ref_loss = float(T.reprojection_loss(disps[-1], torch.tensor(left), torch.tensor(right)))
    assert abs(out['loss'] - ref_loss) < TOL_LOSS
    _log({'test': 'madnet_forward', 'hw': [h, w], 'worst_disp_rel_linf': worst, 'worst_layer_rel_linf': worst_layer,
          'loss': out['loss'], 'ref_loss': ref_loss})


@pytest.mark.parametrize('hw', [(384, 640), (384, 1280)])
def test_madnet_forward_baseline(hw):
    _check_madnet_forward(hw[0], hw[1], seed=3)


def test_madnet_forward_1920x1056():
    """config 5 resolution: the oracle forward at 1920x1088 takes a few seconds on the host cores."""
    _check_madnet_forward(1056, 1920, seed=5)


def _oracle_steps(params, mode, left, right, module):
    from oracle.adaptation import OracleAdapter
    o32 = OracleAdapter(params, mode=mode, lr=1e-4)
    o64 = OracleAdapter(params, mode=mode, lr=1e-4, dtype=torch.float64)
    r32 = o32.step(left, right, module)
    r64 = o64.step(left, right, module)
    return o32, r32, o64, r64


def _check_step(net, ad, params, out, o32, r32, o64, r64, tag):
    assert abs(out['loss'] - r64['full_loss']) < TOL_LOSS
    if tag.startswith('mad'):                       # FULL trains on the full-resolution loss itself (slot 1 unused)
        assert abs(out['train_loss'] - r64['train_loss']) < TOL_LOSS
    gv = net.engine.param_views(net.engine.grads)
    got = {n: gv[n].cpu().numpy() for n in r64['grads']}
    rep = grad_report(got, r32['grads'], r64['grads'])
    _log(dict(test=tag, **summarize(rep)))
    assert_grads(rep, TOL_GRAD_L2, TOL_GRAD_LINF, tag)
    wv = net.engine.export_params()
    worst = 0.0
    for n in r64['grads']:
        d64 = o64.net.p[n].detach().numpy() - params[n].astype(np.float64)
        d32 = o32.net.p[n].detach().numpy().astype(np.float64) - params[n]
        dg = wv[n].astype(np.float64) - params[n]
        e, noise = rel_l2(dg, d64), rel_l2(d32, d64)
        worst = max(worst, e)
        assert e <= max(TOL_DW_L2, 2.0 * noise), (tag, n, e, noise)
    _log({'test': tag + ':dw', 'max_rel_l2': worst})
    trained = set(r64['grads'])
    for n, v in wv.items():
        if n not in trained:
            assert np.array_equal(v, params[n]), n


@pytest.mark.parametrize('module', [0, 1, 2, 3, 4])
def test_madnet_mad_step_1280x384(module):
    from madstereo.synthetic import make_pair
    left, right, _ = make_pair(384, 1280, seed=3)
    net, ad, params, lt, rt = build_madnet(left, right, 'MAD')
    ad.sampler._fixed_id = module
    out = ad.step(lt, rt)
    assert out['blocks'] == [module]
    o32, r32, o64, r64 = _oracle_steps(params, 'MAD', left, right, module)
    _check_step(net, ad, params, out, o32, r32, o64, r64, 'mad%d_1280x384' % module)


def test_madnet_full_step_1280x384():
    from madstereo.synthetic import make_pair
    left, right, _ = make_pair(384, 1280, seed=3)
    net, ad, params, lt, rt = build_madnet(left, right, 'FULL')
    out = ad.step(lt, rt)
    o32, r32, o64, r64 = _oracle_steps(params, 'FULL', left, right, None)
    _check_step(net, ad, params, out, o32, r32, o64, r64, 'full_1280x384')


@pytest.mark.parametrize('mode,module', [('MAD', 0), ('MAD', 4), ('FULL', None)])
def test_madnet_step_640x384_batch2(mode, module):
    """Two distinct frames at 640x384: the non-split-K convolutions and their fused epilogues with two images per
    launch (the image count enters the tile and split choice), every frame against the fp64 oracle at batch 2."""
    from madstereo.synthetic import make_pair
    # (seed 5: with seed 3, frame 1003 alone, at batch 1, already sits on the edge of the fp64-anchored bound for module 4)
    left, right, _ = make_pair(384, 640, seed=5, batch=2)
    net, ad, params, lt, rt = build_madnet(left, right, mode)
    if mode == 'MAD':
        ad.sampler._fixed_id = module
    out = ad.step(lt, rt, want_disp_mask=0b111111)
    o32, r32, o64, r64 = _oracle_steps(params, mode, left, right, module)
    for i, (d, ref) in enumerate(zip(net.get_disparities(), r64['disparities'])):
        assert d.shape == ref.shape
        assert rel_linf(d.numpy(), ref) < TOL_DISP, ('disparity %d' % i)
    tag = ('mad%d' % module if mode == 'MAD' else 'full') + '_640x384_b2'
    _check_step(net, ad, params, out, o32, r32, o64, r64, tag)


# ---------------------------------------------------------------------------------------------------- DispNet
def build_dispnet(left, right, mode):
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


def test_dispnet_forward_1280x384():
    from madstereo.synthetic import make_pair
    from oracle.dispnet import DispNetOracle
    from oracle import tf1_ops as T
    left, right, _ = make_pair(384, 1280, seed=5)
    net, ad, params, lt, rt = build_dispnet(left, right, 'NONE')
    out = ad.step(lt, rt, want_disp_mask=0b1111111)
    disps, layers = DispNetOracle(params).forward(left, right)
    for name in ('conv1a', 'conv1b', 'conv2a', 'conv_redir', 'corr', 'conv3', 'conv3/1', 'conv4/1', 'conv5/1', 'conv6/1',
                 'up5/deconv', 'up5/predict', 'up5/up_predict', 'up5/concat', 'up3/concat', 'up1/concat', 'prediction'):
        assert rel_linf(net[name].numpy(), layers[name].numpy()) < TOL_LAYER, name
    worst = 0.0
    for i, (d, ref) in enumerate(zip(net.get_disparities(), disps)):
        r = rel_linf(d.numpy(), ref.numpy())
        worst = max(worst, r)
        assert r < TOL_DISP, ('disparity %d' % i, r)
    ref_loss = float(T.reprojection_loss(disps[-1], torch.tensor(left), torch.tensor(right)))
    assert abs(out['loss'] - ref_loss) < TOL_LOSS
    _log({'test': 'dispnet_forward_1280x384', 'worst_disp_rel_linf': worst})


def test_dispnet_full_step_1280x384():
    from madstereo.synthetic import make_pair
    from oracle.dispnet import DispNetAdapter
    left, right, _ = make_pair(384, 1280, seed=5)
    net, ad, params, lt, rt = build_dispnet(left, right, 'FULL')
    out = ad.step(lt, rt)
    o32 = DispNetAdapter(params, mode='FULL', lr=1e-4)
    o64 = DispNetAdapter(params, mode='FULL', lr=1e-4, dtype=torch.float64)
    r32 = o32.step(left, right); r64 = o64.step(left, right)
    _check_step(net, ad, params, out, o32, r32, o64, r64, 'dispnet_full_1280x384')
