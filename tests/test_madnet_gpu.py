"""GPU parity of the whole path: MADNet forward, every MAD module step and the FULL step vs the CPU oracle,
through the reference-shaped Python API (Nets.get_stereo_net / OnlineAdaptation) and the C-ABI engine."""
import json
import os

import numpy as np
import pytest
import torch

from conftest import PKG

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), 'golden', 'madnet_64x128.npz')

# tolerances (north_star: disparities within 1e-3 relative L-inf of the fp32 reference forward)
TOL_DISP = 1e-3
TOL_LAYER = 2e-4
# Gradients pass through non-smooth ops (leaky/relu masks, floor() in both warps, the SSIM clip).  A pre-activation
# within ~1e-7 of a kink can land on either side under a different fp32 summation order, which perturbs a whole
# weight-gradient tensor by ~1/#pixels.  The fp32 oracle vs the fp64 oracle shows exactly this: <=1e-5 when no
# mask flips, up to 1.7e-3 (MAD) / 1.8e-2 (FULL) relative L-inf when one does (measured at 100x200, step 2).
# Op-level tests (test_ops_gpu.py) pin every kernel at 2e-5..5e-5; the bounds here are the kink-noise envelope.
TOL_GRAD = 1e-2          # relative L-inf per tensor, first step
TOL_GRAD_2 = 1.5e-1      # second step (weights already differ by the first step's noise; flips compound)
TOL_DW = 1.5e-1            # adapted weights: |dw_gpu - dw_ref|_inf <= TOL_DW * |dw_ref|_inf + 1e-7 per tensor


def rel_linf(a, b):
    a = np.asarray(a, dtype=np.float64); b = np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def hwb(shape):
    """(h, w) or (h, w, batch) test parameter -> h, w, batch; make_pair(batch=B) seeds every frame separately."""
    h, w, batch = (tuple(shape) + (1,))[:3]
    return h, w, batch


# batch 3 (odd, distinct frames): every frame of the batched engine step is compared with the oracle at batch 3
B3 = pytest.param((64, 128, 3), id='64x128-b3')


def build(left, right, mode, cfg='MadNet_full.json', **kw):
    import Nets
    from madstereo.adaptation import OnlineAdaptation
    from oracle.madnet import init_params
    lt = torch.as_tensor(left).cuda(); rt = torch.as_tensor(right).cuda()
    args = dict(left_img=lt, right_img=rt, split_layers=[None], sequence=True, train_portion='BEGIN',
                bulkhead=(mode == 'MAD'), warping=True, context_net=True, radius_d=2, stride=1, is_training=False)
    net = Nets.get_stereo_net('MADNet', args)
    train_config = json.load(open(os.path.join(PKG, 'block_config', cfg)))
    ad = OnlineAdaptation(net, mode=mode, train_config=train_config, lr=1e-4, sample_mode='FIXED', fixed_id=0, **kw)
    params = init_params(seed=42)
    ad.load_weights(params)
    return net, ad, params, lt, rt


def test_api_surface():
    from madstereo.synthetic import make_pair
    left, right, _ = make_pair(64, 128, seed=3)
    net, ad, params, lt, rt = build(left, right, 'MAD')
    assert len(net.get_disparities()) == 6
    names = list(net.get_layers_names())
    assert names[0] == 'left/conv1' and 'right/conv12' in names and names[-1] == 'rescaled_prediction'
    vs = net.get_variables('left/conv1')
    assert [v.name for v in vs] == ['model/gc-read-pyramid/conv1/weights:0', 'model/gc-read-pyramid/conv1/biases:0']
    assert vs[0].shape == (3, 3, 3, 16)
    assert net.get_variables('right/conv1') == [] and net.get_variables('rescaled_prediction') == []
    assert len(net.get_variables('final_disp')) == 98
    assert len(net.get_trainable_variables()) == 98
    assert 'Prediction Layer rescaled_prediction: (1, 64, 128, 1)' in str(net)
    with pytest.raises(Exception):
        import Nets
        Nets.get_stereo_net('nope', {})


@pytest.mark.parametrize('hw', [(64, 128), (128, 256), (100, 200), B3, pytest.param((100, 200, 3), id='100x200-b3')])
def test_forward_parity(hw):
    from madstereo.synthetic import make_pair
    from oracle.madnet import MadNetOracle
    h, w, batch = hwb(hw)
    left, right, _ = make_pair(h, w, seed=3, batch=batch)
    net, ad, params, lt, rt = build(left, right, 'NONE')
    eng = net.engine
    eng.set_input(lt, rt)
    eng.forward(0b111111)
    torch.cuda.synchronize()
    disps, layers = MadNetOracle(params).forward(left, right)
    for name in ('left/conv1', 'left/conv4', 'right/conv4', 'left/conv12', 'right/conv12',
                 'fgc-volume-filtering-6/disp1', 'fgc-volume-filtering-6/disp6', 'fgc-volume-filtering-4/disp3',
                 'fgc-volume-filtering-2/disp6', 'context1', 'context5', 'final_disp'):
        got = net[name].numpy()
        assert rel_linf(got, layers[name].numpy()) < TOL_LAYER, name
    for k in (6, 5, 4, 3, 2):
        c = eng.tensor('cost%d' % k).cpu().numpy()
        C = layers['left/conv%d' % (2 * k)].shape[-1]
        assert rel_linf(c[..., C:C + 5], layers['corr%d' % k].numpy()) < TOL_LAYER, 'corr%d' % k
    for i, (d, ref) in enumerate(zip(net.get_disparities(), disps)):
        assert d.shape == tuple(ref.shape)
        assert rel_linf(d.numpy(), ref.numpy()) < TOL_DISP, 'disparity %d' % i


REF_GRAPH_GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference_graph_madnet_64x128.npz')
SAFE_LAYER_KEYS = ('layer:left/conv4', 'layer:right/conv12', 'layer:fgc-volume-filtering-4/disp3', 'layer:context5', 'layer:final_disp')


@pytest.mark.parametrize('which', ['oracle', 'reference_graph'])
def test_forward_matches_golden_fixture(which):
    """'oracle': vectors written by the CPU oracle; 'reference_graph': vectors written by the reference's own graph code
    executed over oracle/tf1_shim.py (oracle/run_reference_graph.py) -- same inputs, same seeded weights."""
    g = np.load(GOLDEN if which == 'oracle' else REF_GRAPH_GOLDEN)
    left = g['left'].astype(np.float32); right = g['right'].astype(np.float32)
    net, ad, params, lt, rt = build(left, right, 'NONE')
    out = ad.step(lt, rt, want_disp_mask=0b111111)
    for i, d in enumerate(net.get_disparities()):
        assert rel_linf(d.numpy(), g['disp%d' % i]) < TOL_DISP
    for key in g.files:
        if key.startswith('layer:') and not key.startswith('layer:corr') and (which == 'oracle' or key in SAFE_LAYER_KEYS):
            assert rel_linf(net[key[6:]].numpy(), g[key]) < TOL_LAYER, key
    assert abs(out['loss'] - float(g['full_loss'])) < 2e-5


@pytest.mark.parametrize('module', [0, 1, 2, 3, 4])
@pytest.mark.parametrize('hw', [(64, 128), (100, 200), B3])
def test_mad_step_parity(module, hw):
    from madstereo.synthetic import make_pair
    from oracle.adaptation import OracleAdapter
    h, w, batch = hwb(hw)
    left, right, _ = make_pair(h, w, seed=3, batch=batch)
    net, ad, params, lt, rt = build(left, right, 'MAD')
    ad.sampler._fixed_id = module
    orc = OracleAdapter(params, mode='MAD', lr=1e-4)
    prev = params
    for it in range(2):                                   # second step exercises the momentum slots
        out = ad.step(lt, rt)
        ref = orc.step(left, right, module)
        assert out['blocks'] == [module]
        assert abs(out['loss'] - ref['full_loss']) < 2e-5
        assert abs(out['train_loss'] - ref['train_loss']) < 2e-5
        gviews = net.engine.param_views(net.engine.grads)
        for n, gr in ref['grads'].items():
            assert rel_linf(gviews[n].cpu().numpy(), gr) < (TOL_GRAD if it == 0 else TOL_GRAD_2), (it, n)
        wviews = net.engine.export_params()
        for n in ref['grads']:
            dw_ref = orc.net.p[n].detach().numpy() - prev[n]
            dw = wviews[n] - prev[n]
            assert np.abs(dw - dw_ref).max() <= TOL_DW * np.abs(dw_ref).max() + 1e-7, (it, n)
        prev = {n: orc.net.p[n].detach().numpy().copy() for n in ref['grads']}
    # parameters outside the module are untouched
    trained = set(ref['grads'])
    for n, v in net.engine.export_params().items():
        if n not in trained:
            assert np.array_equal(v, params[n]), n


def test_mad_two_blocks_per_frame():
    """--numBlocks 2 (Stereo_Online_Adaptation.py:181-189,199: several train ops in ONE sess.run): the first block runs
    inside the captured step (fused update), the second one eagerly on the same forward.  Both gradients must be those of
    the PRE-update weights: the groups are disjoint and every u_k is stop-gradiented (bulkhead), which only holds if the
    first block's backward / update leaves the forward activations and the disparity buffers alone."""
    from madstereo.adaptation import OnlineAdaptation
    from madstereo.synthetic import make_pair
    from oracle.adaptation import OracleAdapter
    from Sampler import sampler_factory
    left, right, _ = make_pair(64, 128, seed=3)
    net, ad, params, lt, rt = build(left, right, 'MAD')
    ad.sampler = sampler_factory.get_sampler('SEQUENTIAL', 2, 0)      # first draw: blocks [0, 1]
    out = ad.step(lt, rt)
    assert sorted(out['blocks']) == [0, 1]
    gviews = net.engine.param_views(net.engine.grads)
    wviews = net.engine.export_params()
    trained = set()
    for module in out['blocks']:
        orc = OracleAdapter(params, mode='MAD', lr=1e-4)             # fresh: gradients of the pre-update weights
        ref = orc.step(left, right, module)
        if module == out['blocks'][0]:
            assert abs(out['loss'] - ref['full_loss']) < 2e-5
        for n, gr in ref['grads'].items():
            assert rel_linf(gviews[n].cpu().numpy(), gr) < TOL_GRAD, (module, n)
            dw_ref = orc.net.p[n].detach().numpy() - params[n]
            assert np.abs((wviews[n] - params[n]) - dw_ref).max() <= TOL_DW * np.abs(dw_ref).max() + 1e-7, (module, n)
            trained.add(n)
    for n, v in wviews.items():
        if n not in trained:
            assert np.array_equal(v, params[n]), n


@pytest.mark.parametrize('mode,module,batch', [pytest.param('MAD', 1, 1, id='MAD-1'), pytest.param('MAD', 4, 1, id='MAD-4'),
                                               pytest.param('FULL', None, 1, id='FULL-None'),
                                               pytest.param('MAD', 4, 3, id='MAD-4-b3'),
                                               pytest.param('FULL', None, 3, id='FULL-None-b3')])
def test_continual_proxy_loss_step(mode, module, batch):
    """SURVEY 8f-3: one adaptation step supervised by proxy disparities (Stereo_Continual_Adaptation.py:75,112,133;
    get_proxy_loss('mean_l1'), weights 0.01 / 0.1) against the oracle: losses, gradients, adapted weights; plus --dilation."""
    from madstereo.adaptation import OnlineAdaptation
    from madstereo.synthetic import make_pair
    from oracle.adaptation import OracleAdapter
    from oracle.madnet import init_params
    import Nets
    left, right, gt = make_pair(64, 128, seed=3, batch=batch)
    proxy = gt.copy()
    proxy[:, ::7, ::5] = 0.0                           # holes, as in SGM proxies
    proxy[:, 3, 4] = 200.0                             # >= 192: invalid
    proxy[1:, :, :24] = 0.0                            # batch: frames with different numbers of holes
    lt = torch.as_tensor(left).cuda(); rt = torch.as_tensor(right).cuda()
    net = Nets.get_stereo_net('MADNet', dict(left_img=lt, right_img=rt, split_layers=[None], sequence=True, train_portion='BEGIN',
                                             bulkhead=(mode == 'MAD'), warping=True, context_net=True, radius_d=2, stride=1))
    cfg = json.load(open(os.path.join(PKG, 'block_config', 'MadNet_full.json')))
    ad = OnlineAdaptation(net, mode=mode, train_config=cfg, lr=1e-4, sample_mode='FIXED', fixed_id=module or 0, loss='proxy',
                          ssim_th=1e9, dilation=2)
    params = init_params(seed=42)
    ad.load_weights(params)
    out = ad.step(lt, rt, proxy=proxy)
    orc = OracleAdapter(params, mode=mode, lr=1e-4, loss='proxy')
    ref = orc.step(left, right, module, proxy=proxy)
    assert abs(out['loss'] - ref['full_loss']) < 2e-5 * max(1.0, abs(ref['full_loss']))
    if mode == 'MAD':
        assert abs(out['train_loss'] - ref['train_loss']) < 2e-5 * max(1.0, abs(ref['train_loss']))
    gviews = net.engine.param_views(net.engine.grads)
    for n, gr in ref['grads'].items():
        assert rel_linf(gviews[n].cpu().numpy(), gr) < TOL_GRAD, n
    w1 = net.engine.export_params()
    for n in ref['grads']:
        dw_ref = orc.net.p[n].detach().numpy() - params[n]
        assert np.abs((w1[n] - params[n]) - dw_ref).max() <= TOL_DW * np.abs(dw_ref).max() + 1e-7, n
    ad.step(lt, rt, proxy=proxy)                       # step 1 with --dilation 2: inference only, no train op
    w2 = net.engine.export_params()
    assert all(np.array_equal(w1[n], w2[n]) for n in w1)


def test_mad_golden_gradients():
    g = np.load(GOLDEN)
    left = g['left'].astype(np.float32); right = g['right'].astype(np.float32)
    for module in range(5):
        net, ad, params, lt, rt = build(left, right, 'MAD')
        ad.sampler._fixed_id = module
        out = ad.step(lt, rt)
        assert abs(out['train_loss'] - float(g['MAD%d:train_loss' % module])) < 2e-5
        gviews = net.engine.param_views(net.engine.grads)
        for key in g.files:
            if key.startswith('MAD%d:grad:' % module):
                assert rel_linf(gviews[key.split(':', 2)[2]].cpu().numpy(), g[key]) < TOL_GRAD, key
            if key.startswith('MAD%d:gslice:' % module):
                got = gviews[key.split(':', 2)[2]].reshape(-1)[:64].cpu().numpy()
                ref_norm = float(g[key.replace('gslice', 'gnorm')])
                assert np.abs(got - g[key]).max() < TOL_GRAD * max(np.abs(g[key]).max(), 1e-3 * ref_norm), key


@pytest.mark.parametrize('hw', [(64, 128), (100, 200), B3])
def test_full_step_parity(hw):
    from madstereo.synthetic import make_pair
    from oracle.adaptation import OracleAdapter
    h, w, batch = hwb(hw)
    left, right, _ = make_pair(h, w, seed=3, batch=batch)
    net, ad, params, lt, rt = build(left, right, 'FULL')
    orc = OracleAdapter(params, mode='FULL', lr=1e-4)
    prev = params
    for it in range(2):
        out = ad.step(lt, rt)
        ref = orc.step(left, right)
        assert abs(out['loss'] - ref['full_loss']) < 2e-5
        gviews = net.engine.param_views(net.engine.grads)
        worst = 0.0
        for n, gr in ref['grads'].items():
            r = rel_linf(gviews[n].cpu().numpy(), gr)
            worst = max(worst, r)
            assert r < (TOL_GRAD if it == 0 else TOL_GRAD_2), (it, n, r)
        wviews = net.engine.export_params()
        for n in ref['grads']:
            dw_ref = orc.net.p[n].detach().numpy() - prev[n]
            dw = wviews[n] - prev[n]
            assert np.abs(dw - dw_ref).max() <= TOL_DW * np.abs(dw_ref).max() + 1e-7, (it, n)
        prev = {n: orc.net.p[n].detach().numpy().copy() for n in ref['grads']}


def test_piramid_only_config_trains_estimators_only():
    from madstereo.synthetic import make_pair
    from oracle.adaptation import OracleAdapter
    left, right, _ = make_pair(64, 128, seed=3)
    net, ad, params, lt, rt = build(left, right, 'MAD', cfg='MadNet_piramid_only.json')
    ad.sampler._fixed_id = 4
    cfg = json.load(open(os.path.join(PKG, 'block_config', 'MadNet_piramid_only.json')))
    groups = []
    for names in cfg:
        g = []
        for nm in names:
            for v in net.get_variables(nm):
                g.append(v.op_name)
        groups.append(g)
    orc = OracleAdapter(params, mode='MAD', lr=1e-4, groups=groups)
    out = ad.step(lt, rt)
    ref = orc.step(left, right, 4)
    gviews = net.engine.param_views(net.engine.grads)
    for n, gr in ref['grads'].items():
        assert rel_linf(gviews[n].cpu().numpy(), gr) < TOL_GRAD, n
    exported = net.engine.export_params()
    for n in params:
        if n not in ref['grads']:
            assert np.array_equal(exported[n], params[n]), n


def test_divergence_reset_restores_weights_not_momentum():
    from madstereo.synthetic import make_pair
    left, right, _ = make_pair(64, 128, seed=3)
    net, ad, params, lt, rt = build(left, right, 'MAD', ssim_th=0.0)      # every frame "diverges"
    out = ad.step(lt, rt)
    assert out['reset'] and ad.reset_counter == 1
    for n, v in net.engine.export_params().items():
        assert np.array_equal(v, params[n]), n
    assert float(net.engine.momentum.abs().max()) > 0.0                    # slots survive (weights_utils.py:4-38)


def test_sequential_sampler_and_reward_bookkeeping():
    from madstereo.synthetic import make_pair
    left, right, _ = make_pair(64, 128, seed=3)
    import Nets
    from madstereo.adaptation import OnlineAdaptation
    from oracle.madnet import init_params
    lt = torch.as_tensor(left).cuda(); rt = torch.as_tensor(right).cuda()
    net = Nets.get_stereo_net('MADNet', dict(left_img=lt, right_img=rt, split_layers=[None], sequence=True,
                                             train_portion='BEGIN', bulkhead=True))
    cfg = json.load(open(os.path.join(PKG, 'block_config', 'MadNet_full.json')))
    ad = OnlineAdaptation(net, mode='MAD', train_config=cfg, sample_mode='SEQUENTIAL')
    ad.load_weights(init_params(seed=42))
    seen = [ad.step(lt, rt)['blocks'][0] for _ in range(7)]
    assert seen == [0, 1, 2, 3, 4, 0, 1]
    assert ad.fetch_counter == [2, 2, 1, 1, 1]
    assert ad.sample_distribution.shape == (5,) and np.isfinite(ad.sample_distribution).all()


def test_prefetch_pipeline_matches_serial_input_path():
    """step(prefetch=next) stages the next frame's host buffers on a side stream while the current frame computes;
    the sequence of losses and the adapted weights must be identical to the serial path (same kernels, same order)."""
    _check_prefetch_pipeline(np.float32)


def test_prefetch_pipeline_matches_serial_input_path_uint8():
    """The same with uint8 frames: the staging buffers are uint8 and the conversion runs after the device copy."""
    _check_prefetch_pipeline(np.uint8)


def _check_prefetch_pipeline(dtype):
    from madstereo.synthetic import make_pair
    import Nets
    from madstereo.adaptation import OnlineAdaptation
    from oracle.madnet import init_params
    frames = [make_pair(64, 128, seed=10 + i)[:2] for i in range(3)]
    if dtype == np.uint8:
        frames = [(np.round(l).astype(np.uint8), np.round(r).astype(np.uint8)) for l, r in frames]
    host = [(torch.from_numpy(l).pin_memory(), torch.from_numpy(r).pin_memory()) for l, r in frames]
    cfg = json.load(open(os.path.join(PKG, 'block_config', 'MadNet_full.json')))

    def run(pipelined):
        net = Nets.get_stereo_net('MADNet', dict(left_img=host[0][0].float().cuda(), right_img=host[0][1].float().cuda(), split_layers=[None],
                                                 sequence=True, train_portion='BEGIN', bulkhead=True))
        ad = OnlineAdaptation(net, mode='MAD', train_config=cfg, sample_mode='SEQUENTIAL')
        ad.load_weights(init_params(seed=42))
        losses = []
        for i in range(6):
            cur, nxt = host[i % 3], host[(i + 1) % 3]
            out = ad.step(*cur, prefetch=nxt) if pipelined else ad.step(*cur)
            losses.append((out['loss'], out['train_loss']))
        return losses, net.engine.weights.clone().cpu().numpy()

    l0, w0 = run(False)
    l1, w1 = run(True)
    assert l0 == l1
    assert np.array_equal(w0, w1)


def test_config5_1920x1056_size_independent_properties():
    """BASELINE config 5 resolution (1920x1056 -> REFLECT-padded to 1920x1088, preprocessing.py:7-29), where the CPU oracle
    is too slow to be a checker: properties that do not depend on size.
      * forward is deterministic (bit-identical disparities on a second run) and the output has the un-padded shape;
      * the final disparity is relu'd (>= 0) and finite;
      * one MAD step per module (SEQUENTIAL sampler): finite losses, exactly the sampled module's variables change
        (bulkhead + var_list, Stereo_Online_Adaptation.py:112-118), every other parameter is bit-identical."""
    from madstereo.synthetic import make_pair
    H, W = 1056, 1920
    left, right, _ = make_pair(H, W, seed=5)
    net, ad, params, lt, rt = build(left, right, 'MAD')
    ad.sampler = __import__('Sampler.sampler_factory', fromlist=['x']).get_sampler('SEQUENTIAL', 1)
    eng = net.engine
    eng.set_input(lt, rt)
    eng.forward()
    d0 = net.get_disparities()[-1].numpy().copy()
    eng.forward()
    d1 = net.get_disparities()[-1].numpy()
    assert d0.shape == (1, H, W, 1)
    assert np.array_equal(d0, d1)
    assert np.isfinite(d0).all() and d0.min() >= 0.0 and d0.max() > 0.0
    ranges = eng.group_ranges
    for k in range(5):
        before = eng.weights.clone()
        out = ad.step(lt, rt)
        assert out['blocks'] == [k] and np.isfinite(out['loss']) and np.isfinite(out['train_loss'])
        changed = (eng.weights != before)
        lo, hi = ranges[k]
        assert bool(changed[lo:hi].any()), 'module %d did not move' % k
        changed[lo:hi] = False
        assert not bool(changed.any()), 'parameters outside module %d moved' % k
