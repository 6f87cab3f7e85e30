"""MAD module losses at 1/s resolution (--reprojectionScale) on the engine: the step against the CPU oracle
(tests/reprojection_scale_oracle.py), what must not change (slot 0, the full-resolution disparity, other modules' weights,
scale 1), the fused disparity kernel against the two existing resizes, graph replay, determinism, batching, Adam, the
refusals and both drivers end to end."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import PKG, ROOT
from reprojection_scale_oracle import RsOracleAdapter

pytestmark = pytest.mark.gpu

# the bars test_madnet_gpu applies at s = 1
TOL_GRAD = 1e-2
TOL_DW = 1.5e-1
# ... and its kink bar (TOL_GRAD_2) where the loss-resolution map is small enough for one kink to show: at 100x200, s = 3
# (66x66 loss pixels, 8x16 level-4 pixels) a 1e-6 relative perturbation of the weights moves the CPU oracle's own
# module-2 gradients by up to 16 % (disp-6 biases), against 1e-4 at s = 1 -- one pre-activation or warp tap crossing its
# kink.  The engine's forward differs from the oracle's by about that much (fp32 summation order).
TOL_GRAD_KINK = 1.5e-1


def rel_linf(a, b):
    a = np.asarray(a, dtype=np.float64); b = np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def synthetic(h, w, batch=1, seed=3):
    from madstereo.synthetic import make_pair
    left, right, gt = make_pair(h, w, seed=seed, batch=batch)
    proxy = gt.copy()
    proxy[:, ::7, ::5] = 0.0
    proxy[:, 3::11, 4::13] = 200.0
    return left, right, proxy


def build(left, right, scale=1, loss='reprojection', module=0, **kw):
    import Nets
    from madstereo.adaptation import OnlineAdaptation
    from oracle.madnet import init_params
    lt = torch.as_tensor(left).cuda(); rt = torch.as_tensor(right).cuda()
    net = Nets.get_stereo_net('MADNet', dict(left_img=lt, right_img=rt, split_layers=[None], sequence=True,
                                             train_portion='BEGIN', bulkhead=True, warping=True, context_net=True,
                                             radius_d=2, stride=1, is_training=False))
    cfg = json.load(open(os.path.join(PKG, 'block_config', 'MadNet_full.json')))
    ad = OnlineAdaptation(net, mode='MAD', train_config=cfg, lr=1e-4, sample_mode='FIXED', fixed_id=module, loss=loss,
                          ssim_th=1e9, reprojection_scale=scale, **kw)
    params = init_params(seed=42)
    ad.load_weights(params)
    return net, ad, params, lt, rt


CASES = [(64, 128, s, m, l) for s in (2, 3, 4) for m in range(5) for l in ('reprojection', 'proxy')] + \
        [(100, 200, 3, m, l) for m in range(5) for l in ('reprojection', 'proxy')]


@pytest.mark.parametrize('h,w,scale,module,loss', CASES)
def test_mad_step_matches_oracle(h, w, scale, module, loss):
    left, right, proxy = synthetic(h, w)
    net, ad, params, lt, rt = build(left, right, scale, loss, module)
    out = ad.step(lt, rt, proxy=proxy if loss == 'proxy' else None)
    orc = RsOracleAdapter(params, reprojection_scale=scale, loss=loss)
    ref = orc.step(left, right, module, proxy=proxy)
    assert out['blocks'] == [module]
    assert abs(out['loss'] - ref['full_loss']) < 2e-5 * max(1.0, abs(ref['full_loss']))
    assert abs(out['train_loss'] - ref['train_loss']) < 2e-5 * max(1.0, abs(ref['train_loss']))
    gviews = net.engine.param_views(net.engine.grads)
    tol = TOL_GRAD_KINK if (h, w) == (100, 200) else TOL_GRAD
    for n, gr in ref['grads'].items():
        assert rel_linf(gviews[n].cpu().numpy(), gr) < tol, n
    wv = net.engine.export_params()
    for n in ref['grads']:
        dw_ref = orc.net.p[n].detach().numpy() - params[n]
        assert np.abs((wv[n] - params[n]) - dw_ref).max() <= max(TOL_DW, tol) * np.abs(dw_ref).max() + 1e-7, n
    for n, v in wv.items():
        if n not in ref['grads']:
            assert np.array_equal(v, params[n]), n


def _state(net):
    e = net.engine
    return {'w': e.weights.clone(), 'g': e.grads.clone(), 'm': e.momentum.clone(),
            'disp': net.get_disparities()[-1].numpy().copy()}


@pytest.mark.parametrize('module', [0, 2, 4])
def test_scale_leaves_slot0_full_disparity_and_other_modules_alone(module):
    left, right, _ = synthetic(64, 128)
    outs, states, nets = [], [], []
    for scale in (1, 2):
        net, ad, params, lt, rt = build(left, right, scale, module=module)
        outs.append(ad.step(lt, rt, want_disp_mask=0b100000)); states.append(_state(net)); nets.append(net)
    assert outs[0]['loss'] == outs[1]['loss']                         # slot 0, bit for bit
    assert np.array_equal(states[0]['disp'], states[1]['disp'])
    lo, hi = nets[0].engine.group_ranges[module]
    for k in ('w', 'm'):
        a, b = states[0][k].clone(), states[1][k].clone()
        a[lo:hi] = 0; b[lo:hi] = 0
        assert torch.equal(a, b), k
    assert not torch.equal(states[0]['g'][lo:hi], states[1]['g'][lo:hi])


def test_scale_one_is_bitwise_the_default_path():
    left, right, _ = synthetic(64, 128)
    res = []
    for call in (False, True):
        net, ad, params, lt, rt = build(left, right, 1, module=3)
        if call:
            net.engine.set_reprojection_scale(2)
            net.engine.set_reprojection_scale(1)
        for _ in range(2):
            out = ad.step(lt, rt, want_disp_mask=0b111111)
        res.append((out, _state(net), [d.numpy().copy() for d in net.get_disparities()]))
    (o0, s0, d0), (o1, s1, d1) = res
    assert o0['loss'] == o1['loss'] and o0['train_loss'] == o1['train_loss']
    for k in ('w', 'g', 'm'):
        assert torch.equal(s0[k], s1[k]), k
    assert all(np.array_equal(a, b) for a, b in zip(d0, d1))


@pytest.mark.parametrize('h,w,scale', [(384, 1280, 2), (384, 1280, 3), (100, 200, 3)])
def test_fused_disparity_and_inputs_equal_the_existing_resizes(h, w, scale):
    """rs_disp (one pass from the coarse head) against ms_resize_bilinear to H x W (the engine's disparity) and then to
    h x w; rs_left / rs_right against ms_resize_bilinear per channel (the same arithmetic: bit for bit)."""
    from madstereo import ops
    from madstereo.engine import MODE_MAD
    left, right, _ = synthetic(h, w)
    net, ad, params, lt, rt = build(left, right, scale)
    eng = net.engine
    eng.set_input(lt, rt)
    hs, ws = h // scale, w // scale
    for module in range(5):
        eng.run(MODE_MAD, module, 1 << module, 0)
        torch.cuda.synchronize()
        full = eng.tensor('disp%d' % module).contiguous()
        want = ops.resize_bilinear(full, hs, ws)
        got = eng.tensor('rs_disp')
        assert got.shape == (1, hs, ws, 1)
        err = (got - want).abs().max().item()
        assert err <= 4e-6 * max(want.abs().max().item(), 1.0), (module, err)
    for name, src in (('rs_left', lt), ('rs_right', rt)):
        got = eng.tensor(name)
        for c in range(3):
            want = ops.resize_bilinear(src[..., c:c + 1].contiguous(), hs, ws)
            assert torch.equal(got[..., c:c + 1], want), (name, c)


def test_graph_replay_equals_eager_first_step_and_follows_scale_changes():
    from madstereo.engine import MODE_MAD
    left, right, proxy = synthetic(64, 128)
    runs = {}
    for kind in ('eager', 'graph'):
        net, ad, params, lt, rt = build(left, right, 2, module=1)
        eng = net.engine
        eng.set_input(lt, rt)
        if kind == 'graph':
            eng.run(MODE_MAD, 1, 0, 0)                               # capture (+ first replay)
            eng.set_input(lt, rt)
            eng.grads.zero_()
        if kind == 'eager':
            eng.profile(1)                                           # run() steps eagerly while profiling 1
        eng.run(MODE_MAD, 1, 0, 0)
        eng.profile(0)
        torch.cuda.synchronize()
        runs[kind] = (eng.read_scalars()[:2], eng.grads.clone())
    assert runs['eager'][0] == runs['graph'][0]
    assert torch.equal(runs['eager'][1], runs['graph'][1])
    # a new scale reaches the next (re-captured) step
    orc3 = RsOracleAdapter(params, reprojection_scale=3, lr=0.0)
    eng.set_reprojection_scale(3)
    eng.set_input(lt, rt)
    eng.run(MODE_MAD, 1, 0, 0)
    ref = orc3.step(left, right, 1)
    assert abs(eng.read_scalars()[1] - ref['train_loss']) < 2e-5
    assert eng.tensor('rs_disp').shape == (1, 64 // 3, 128 // 3, 1)


def test_two_replays_give_bitwise_identical_gradients():
    from madstereo.engine import MODE_MAD
    left, right, _ = synthetic(384, 1280)
    net, ad, params, lt, rt = build(left, right, 2)
    eng = net.engine
    eng.set_input(lt, rt)
    grads = []
    for module in (0, 4):
        for _ in range(3):
            eng.run(MODE_MAD, module, 0, 0)
            torch.cuda.synchronize()
            grads.append(eng.grads.clone())
        assert torch.equal(grads[-1], grads[-2]) and torch.equal(grads[-2], grads[-3]), module


def test_batch_of_two_is_the_mean_of_its_frames():
    """Each frame's loss-resolution images are its own: batch 2 = the mean of two batch-1 steps, at the bars of
    test_batch_gpu (loss 1e-6 relative; per tensor |g_batch - mean g_b|_2 <= 1e-2 * mean |g_b|_2)."""
    left, right, _ = synthetic(64, 128, batch=2)
    net, ad, params, lt, rt = build(left, right, 2, module=2)
    out = ad.step(lt, rt)
    gb = {n: v.cpu().numpy().astype(np.float64) for n, v in net.engine.param_views(net.engine.grads).items()}
    losses, frames = [], []
    for b in range(2):
        n1, ad1, _, l1, r1 = build(left[b:b + 1], right[b:b + 1], 2, module=2)
        losses.append(ad1.step(l1, r1)['train_loss'])
        frames.append({n: v.cpu().numpy().astype(np.float64) for n, v in n1.engine.param_views(n1.engine.grads).items()})
    assert abs(out['train_loss'] - np.mean(losses)) <= 1e-6 * abs(np.mean(losses))
    for n in gb:
        scale = 0.5 * (np.linalg.norm(frames[0][n]) + np.linalg.norm(frames[1][n]))
        if scale > 0:
            assert np.linalg.norm(gb[n] - 0.5 * (frames[0][n] + frames[1][n])) <= 1e-2 * scale, n


def test_adam_update_matches_oracle():
    """Adam at s = 2 against adam_oracle's ApplyAdam, at the bounds of test_demo_gpu's Adam parity: Adam's first step moves
    every trained weight by about +-lr whatever the gradient's size, so a gradient within kink noise of zero may flip;
    every weight within 1 lr per step, 95 % within 0.05 lr per step."""
    lr = 1e-4
    left, right, _ = synthetic(64, 128)
    net, ad, params, lt, rt = build(left, right, 2, module=2, optimizer='adam')
    orc = RsOracleAdapter(params, reprojection_scale=2, optimizer='adam', lr=lr)
    steps = 3
    for it in range(steps):
        out = ad.step(lt, rt)
        ref = orc.step(left, right, 2)
        assert abs(out['train_loss'] - ref['train_loss']) < 2e-5, it
    wv = net.engine.export_params()
    diffs = np.concatenate([np.abs(wv[n].astype(np.float64) - orc.net.p[n].detach().numpy().astype(np.float64)).ravel()
                            for n in wv]) / lr
    assert diffs.max() <= 1.0 * steps
    assert float(np.mean(diffs <= 0.05 * steps)) >= 0.95


def test_refusals_return_an_error_and_launch_nothing():
    from ctypes import c_void_p
    import Nets
    from madstereo._lib import MadStereoError
    from madstereo.adaptation import OnlineAdaptation
    left, right, _ = synthetic(64, 128)
    net, ad, params, lt, rt = build(left, right, 1)
    eng = net.engine
    L = eng._lib
    scratch = torch.empty(L.ms_engine_reprojection_scratch_floats(eng._h, 2), device='cuda')
    n0 = eng.launch_count()
    for scale, buf, n in ((0, scratch, scratch.numel()), (-1, scratch, scratch.numel()), (22, scratch, scratch.numel()),
                          (2, scratch, scratch.numel() - 1)):
        rc = L.ms_engine_set_reprojection_scale(eng._h, scale, c_void_p(buf.data_ptr()), n)
        assert rc < 0 and L.ms_last_error().decode(), scale
    assert L.ms_engine_reprojection_scratch_floats(eng._h, 22) == 0          # 64 // 22 = 2 < 3
    assert eng.launch_count() == n0 and eng.reprojection_scale == 1
    with pytest.raises(MadStereoError):
        eng.set_reprojection_scale(0)
    # DispNet has no MAD train ops
    dn = Nets.get_stereo_net('Dispnet', dict(left_img=lt, right_img=rt, split_layers=[None], sequence=True,
                                             train_portion='BEGIN', bulkhead=False))
    OnlineAdaptation(dn, mode='FULL', train_config=None, lr=1e-4)
    d = dn.engine
    n0 = d.launch_count()
    assert d._lib.ms_engine_set_reprojection_scale(d._h, 2, c_void_p(scratch.data_ptr()), scratch.numel()) < 0
    assert 'MADNet' in d._lib.ms_last_error().decode()
    assert d.launch_count() == n0


@pytest.mark.parametrize('driver', ['Stereo_Online_Adaptation.py', 'Stereo_Continual_Adaptation.py'])
def test_drivers_end_to_end(driver, tmp_path):
    import cv2
    from oracle.madnet import init_params
    frames = []
    for i in range(3):
        left, right, gt = synthetic(64, 128, seed=10 + i)
        names = []
        for tag, img in (('l', left[0]), ('r', right[0])):
            p = str(tmp_path / ('%s%d.png' % (tag, i)))
            cv2.imwrite(p, np.clip(img, 0, 255).astype(np.uint8)[..., ::-1]); names.append(p)
        for tag in ('gt', 'px'):
            p = str(tmp_path / ('%s%d.png' % (tag, i)))
            cv2.imwrite(p, (np.clip(gt[0, ..., 0], 0, 255) * 256).astype(np.uint16)); names.append(p)
        frames.append(names)
    lst = str(tmp_path / 'list.csv')
    with open(lst, 'w') as f:
        for n in frames:
            f.write(';'.join(n if 'Continual' in driver else n[:3]) + '\n')
    np.savez(str(tmp_path / 'w.npz'), **init_params(seed=42))
    out = tmp_path / 'out'
    cmd = [sys.executable, os.path.join(PKG, driver), '-l', lst, '-o', str(out), '--weights', str(tmp_path / 'w.npz'),
           '--modelName', 'MADNet', '--blockConfig', os.path.join(PKG, 'block_config', 'MadNet_full.json'), '--mode', 'MAD',
           '--sampleMode', 'SEQUENTIAL', '--imageShape', '64', '128', '--reprojectionScale', '2']
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    want = ('overall.csv', 'series.csv') if 'Continual' in driver else ('stats.csv', 'series.csv')
    for f in want:
        assert (out / f).exists(), f
