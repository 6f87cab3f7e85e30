"""GPU tests of the live demo's engine features: the Adam update (operator, engine step, graph replays, oracle parity,
DispNet), optimizer switching, the on-device rescale + crop of uint8 camera frames, and the demo end to end."""
import gc
import json
import os
import sys

import numpy as np
import pytest
import torch

from conftest import PKG
from adam_oracle import BETA1, BETA2, EPS, AdamOracleAdapter, adam_reference, advance_powers

pytestmark = pytest.mark.gpu
LR = 1e-4
DEMO = os.path.join(PKG, 'Demo')


def _note(**kw):
    """Measured deviations, printed for the record (pytest -s)."""
    print('MEASURED', json.dumps(kw))


def _release():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


class _Seq(object):
    """Module sampler that replays a fixed sequence."""

    def __init__(self, seq):
        self.seq, self.i = list(seq), 0

    def sample(self, dist):
        b = self.seq[self.i % len(self.seq)]
        self.i += 1
        return [b]


def _madnet(h, w, mode, optimizer='adam', cfg='MadNet_full.json', batch=1, seq=None, **kw):
    import Nets
    from madstereo.adaptation import OnlineAdaptation
    from oracle.madnet import init_params
    lt = torch.zeros(batch, h, w, 3, device='cuda'); rt = torch.zeros(batch, h, w, 3, device='cuda')
    net = Nets.get_stereo_net('MADNet', dict(left_img=lt, right_img=rt, split_layers=[None], sequence=True,
                                             train_portion='BEGIN', bulkhead=(mode == 'MAD')))
    train_config = json.load(open(os.path.join(PKG, 'block_config', cfg)))
    ad = OnlineAdaptation(net, mode=mode, train_config=train_config, lr=LR, sample_mode='FIXED', fixed_id=0,
                          optimizer=optimizer, **kw)
    params = init_params(seed=42)
    ad.load_weights(params)
    if seq is not None:
        ad.sampler = _Seq(seq)
    return net, ad, params


def _f32(x):
    return x.detach().cpu().numpy().astype(np.float32)


def _check_adam_range(w0, m0, v0, p0, g, w1, m1, v1, what):
    """Engine result (w1, m1, v1) vs float64 ApplyAdam from the engine's own pre-step state and gradient arena.
    Bound: the engine rounds every intermediate to fp32 (about 6e-8 relative each), so w may differ by one fp32 spacing of
    w plus 1e-5 lr (the update term itself is at most a few lr); m by 3e-7 of |m| + |g| and v by 3e-7 of v + g^2 (the
    fp32 roundings of the difference, the product and the sum, each relative to the larger of the operands)."""
    wr, mr, vr = adam_reference(w0, g, m0, v0, p0, LR)
    dw = np.abs(w1.astype(np.float64) - wr)
    bw = np.spacing(np.abs(w1)).astype(np.float64) + 1e-5 * LR
    assert (dw <= bw).all(), '%s: w off by %g (bound %g)' % (what, (dw - bw).max(), bw[np.argmax(dw - bw)])
    g64 = np.asarray(g, np.float64)
    for a, r, scale, nm in ((m1, mr, np.abs(m0) + np.abs(g64), 'm'), (v1, vr, np.asarray(v0, np.float64) + g64 * g64, 'v')):
        d = np.abs(a.astype(np.float64) - r)
        assert (d <= 3e-7 * scale + 1e-37).all(), '%s: %s off by %g' % (what, nm, (d - 3e-7 * scale).max())
    return float((dw / LR).max())


# ---- 1. operator ---------------------------------------------------------------------------------------------
def test_adam_operator_matches_float64_formula():
    from madstereo._lib import check, lib
    n = 4099                                       # n % 4 != 0: the scalar tail of the vectorised kernel runs
    rng = np.random.default_rng(1)
    w = torch.tensor(rng.normal(0, 0.1, n), dtype=torch.float32, device='cuda')
    m = torch.zeros(n, device='cuda'); v = torch.zeros(n, device='cuda')
    powers = torch.tensor([BETA1, BETA2], dtype=torch.float32, device='cuda')
    gs = 0.5
    wh, mh, vh = _f32(w).astype(np.float64), np.zeros(n), np.zeros(n)
    p = (np.float32(BETA1), np.float32(BETA2))
    worst = 0.0
    for step in range(5):
        g = torch.tensor(rng.normal(0, 1e-3, n) * (10.0 ** rng.integers(-4, 2, n)), dtype=torch.float32, device='cuda')
        check(lib().ms_adam_update(w.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), powers.data_ptr(), n, LR, BETA1,
                                   BETA2, EPS, gs, torch.cuda.current_stream().cuda_stream), 'adam')
        torch.cuda.synchronize()
        # float64 restatement carried in float64 across the 5 steps (not re-seeded from the kernel's state)
        wh, mh, vh = adam_reference(wh, _f32(g), mh, vh, p, LR, grad_scale=gs)
        p = advance_powers(p)
        # bound in units of lr: each step moves w by at most ~lr (|m| / sqrt(v) <= (1 - b1) / sqrt(1 - b2) times the
        # bias correction); fp32 rounding of m, v and the quotient is ~1e-7 relative of that, plus the fp32 spacing of w
        # itself (|w| < 0.5: 3e-8 = 3e-4 lr), accumulated over 5 steps -> 2e-3 lr
        err = np.abs(_f32(w).astype(np.float64) - wh).max() / LR
        worst = max(worst, err)
        assert err < 2e-3, (step, err)
        assert _f32(powers)[0] == p[0] and _f32(powers)[1] == p[1]
    _note(test='adam_operator', worst_w_err_in_lr=worst)


# ---- 2. engine step ------------------------------------------------------------------------------------------
def test_engine_adam_step_shared_powers_and_graph_replays():
    from madstereo.synthetic import make_pair
    seq = [2, 0, 2, 4]
    net, ad, _ = _madnet(64, 128, 'MAD', seq=seq * 3)
    eng = ad.engine
    p_chain = (np.float32(BETA1), np.float32(BETA2))
    worst = 0.0
    for k in range(len(seq) * 3):                  # rounds 2 and 3 replay the captured graphs
        left, right, _ = make_pair(64, 128, seed=10 + k)
        w0, m0, v0, p0 = _f32(eng.weights), _f32(eng.momentum), _f32(eng.adam_v), _f32(eng.adam_powers)
        assert p0[0] == p_chain[0] and p0[1] == p_chain[1], 'step %d: powers are not beta^(t+1) (t = %d train ops)' % (k, k)
        out = ad.step(torch.tensor(left).cuda(), torch.tensor(right).cuda())
        g = seq[k % len(seq)]
        assert out['blocks'] == [g]
        torch.cuda.synchronize()
        w1, m1, v1, p1 = _f32(eng.weights), _f32(eng.momentum), _f32(eng.adam_v), _f32(eng.adam_powers)
        gr = _f32(eng.grads)
        lo, hi = eng.group_ranges[g]
        worst = max(worst, _check_adam_range(w0[lo:hi], m0[lo:hi], v0[lo:hi], p0, gr[lo:hi], w1[lo:hi], m1[lo:hi],
                                             v1[lo:hi], 'step %d module %d' % (k, g)))
        assert np.any(w1[lo:hi] != w0[lo:hi])
        mask = np.ones(eng.n_params, bool); mask[lo:hi] = False
        for a, b, nm in ((w0, w1, 'w'), (m0, m1, 'm'), (v0, v1, 'v')):
            assert np.array_equal(a[mask].view(np.uint32), b[mask].view(np.uint32)), 'step %d: %s of other modules moved' % (k, nm)
        p_chain = advance_powers(p_chain)
        assert p1[0] == p_chain[0] and p1[1] == p_chain[1], 'powers advanced more or less than once'
    _note(test='engine_adam', worst_w_err_in_lr=worst)
    del net, ad, eng
    _release()


def test_dispnet_full_step_with_adam():
    import Nets
    from madstereo.adaptation import OnlineAdaptation
    from madstereo.synthetic import make_pair
    from oracle.dispnet import init_params
    left, right, _ = make_pair(64, 128, seed=5)
    lt = torch.tensor(left).cuda(); rt = torch.tensor(right).cuda()
    net = Nets.get_stereo_net('Dispnet', dict(left_img=lt, right_img=rt, split_layers=[None], sequence=True,
                                              train_portion='BEGIN', bulkhead=False, correlation=True))
    ad = OnlineAdaptation(net, mode='FULL', lr=LR, optimizer='adam')
    ad.load_weights(init_params(seed=7))
    eng = ad.engine
    for k in range(2):
        w0, m0, v0, p0 = _f32(eng.weights), _f32(eng.momentum), _f32(eng.adam_v), _f32(eng.adam_powers)
        ad.step(lt, rt)
        torch.cuda.synchronize()
        _check_adam_range(w0, m0, v0, p0, _f32(eng.grads), _f32(eng.weights), _f32(eng.momentum), _f32(eng.adam_v),
                          'DispNet FULL step %d' % k)
        assert tuple(_f32(eng.adam_powers)) == advance_powers(p0)
    del net, ad, eng
    _release()


# ---- 3. parity against the oracle ----------------------------------------------------------------------------
@pytest.mark.parametrize('hw', [(64, 128), (320, 512)])
@pytest.mark.parametrize('mode', ['MAD', 'FULL'])
def test_adam_parity_against_oracle(hw, mode):
    from madstereo.synthetic import make_pair
    from oracle.madnet import mad_groups_full
    h, w = hw
    seq = [1, 3, 0, 4, 2]
    steps = 5 if mode == 'MAD' else 3
    net, ad, params = _madnet(h, w, mode, seq=seq)
    orc = AdamOracleAdapter(params, mode=mode, lr=LR, groups=mad_groups_full())
    loss_err = disp_err = 0.0
    for k in range(steps):
        left, right, _ = make_pair(h, w, seed=20 + k)
        out = ad.step(torch.tensor(left).cuda(), torch.tensor(right).cuda())
        ref = orc.step(left, right, seq[k] if mode == 'MAD' else None)
        loss_err = max(loss_err, abs(out['loss'] - ref['full_loss']))
        if mode == 'MAD':                          # (FULL trains on the full-resolution loss: the engine fills slot 0 only)
            loss_err = max(loss_err, abs(out['train_loss'] - ref['train_loss']))
        d = net.get_disparities()[-1].numpy()
        disp_err = max(disp_err, float(np.abs(d - ref['disparities'][-1]).max() / np.abs(ref['disparities'][-1]).max()))
    eng_w = ad.engine.export_params()
    diffs = np.concatenate([np.abs(eng_w[n].astype(np.float64) - orc.net.p[n].detach().numpy().astype(np.float64)).ravel()
                            for n in eng_w]) / LR
    frac_small = float(np.mean(diffs <= 0.05 * steps))
    _note(test='adam_parity', hw=list(hw), mode=mode, loss_err=loss_err, disp_rel_err=disp_err, w_max_in_lr=float(diffs.max()),
          w_p999_in_lr=float(np.quantile(diffs, 0.999)), frac_within_0p05lr_per_step=frac_small)
    # Bounds.  Weights: Adam's first step moves every trained weight by about +-lr whatever the gradient's size, so a
    # gradient within kink noise of zero (see test_madnet_gpu.py) can flip sign and put the weight up to 2 lr away; later
    # steps move a weight by at most a few lr.  Every weight is held to 1 lr per step, and 95 % of them to 0.05 lr per
    # step.  Measured on an H100 SXM (400 W): worst weight 1.13 lr (MAD 64x128, 5 steps), 1.27 lr (MAD 320x512), 0.36 lr
    # (FULL 64x128, 3 steps), 2.28 lr (FULL 320x512); fraction within 0.05 lr per step >= 0.9999 at 64x128, 0.995 (MAD)
    # and 0.965 (FULL) at 320x512.  Loss / disparity: measured worst cases 4.5e-6 / 1.9e-3 relative L-inf (320x512 FULL),
    # bounds with ~3x margin.
    assert diffs.max() <= 1.0 * steps
    assert frac_small >= 0.95
    assert loss_err < 2e-5
    assert disp_err < 6e-3
    del net, ad
    _release()


# ---- 5. optimizer switches -----------------------------------------------------------------------------------
def test_optimizer_switch_drops_graphs():
    from madstereo.engine import MODE_MAD
    from madstereo._lib import MadStereoError
    from madstereo.synthetic import make_pair
    left, right, _ = make_pair(64, 128, seed=3)
    lt, rt = torch.tensor(left).cuda(), torch.tensor(right).cuda()
    net_a, ad_a, _ = _madnet(64, 128, 'MAD', optimizer='momentum', seq=[1])
    ea = ad_a.engine
    w_init = ea.weights.clone()
    ad_a.step(lt, rt)                              # momentum graph captured
    ea.set_optimizer('adam')
    w_before = ea.weights.clone()
    ad_a.step(lt, rt)                              # must not replay the momentum graph
    lo, hi = ea.group_ranges[1]
    assert torch.count_nonzero(ea.adam_v[lo:hi]) > 0, 'the Adam step did not run Adam'
    with pytest.raises(MadStereoError, match='momentum only'):
        ea.run(MODE_MAD, 1, 0, 2, LR, 0.9, 1.0)    # the fused data-parallel update is momentum-only
    assert not torch.equal(ea.weights, w_before)
    ea.set_optimizer('momentum')
    ea.weights.copy_(w_init); ea.momentum.zero_(); ea.weights_changed()
    ad_a.step(lt, rt)                              # must not replay the Adam graph
    net_b, ad_b, _ = _madnet(64, 128, 'MAD', optimizer='momentum', seq=[1])
    ad_b.step(lt, rt)
    torch.cuda.synchronize()
    assert torch.equal(ea.weights, ad_b.engine.weights)
    assert torch.equal(ea.momentum, ad_b.engine.momentum)
    del net_a, ad_a, net_b, ad_b, ea
    _release()


# ---- 6. rescale + crop ---------------------------------------------------------------------------------------
GEOMS = [((720, 1280), (480, 640), (320, 512)),     # the demo's defaults on 720p frames
         ((375, 1242), None, (384, 1280)),          # no rescale: KITTI frame padded on both axes
         ((375, 1242), None, (384, 1241)),          # no rescale: odd row padding (9), odd column crop (1)
         ((240, 320), (480, 640), (320, 512)),      # upscale
         ((320, 512), None, (320, 512))]            # identity


def _resize_ref(x, rs, out):
    from oracle import tf1_ops as T
    t = torch.tensor(x, dtype=torch.float64)
    if rs is not None:
        t = T.resize_bilinear(t, rs[0], rs[1])
    return T.crop_or_pad(t, out[0], out[1]).numpy()


@pytest.mark.parametrize('geom', GEOMS, ids=['720p-480x640-320x512', '375x1242-pad', '375x1242-odd-pad-crop', 'upscale', 'identity'])
@pytest.mark.parametrize('batch', [1, 2])
def test_resize_and_crop(geom, batch):
    from madstereo.engine import StereoEngine
    (h, w), rs, (H, W) = geom
    eng = StereoEngine('MADNet', batch, H, W)
    eng.set_groups([]); eng.bind()
    eng.set_resize(rs if rs is not None else (-1, -1))
    rng = np.random.default_rng(h + batch)
    left = rng.integers(0, 256, (batch, h, w, 3), dtype=np.uint8)
    right = rng.integers(0, 256, (batch, h, w, 3), dtype=np.uint8)
    ref_l, ref_r = _resize_ref(left, rs, (H, W)), _resize_ref(right, rs, (H, W))
    sources = {'pageable': (torch.from_numpy(left), torch.from_numpy(right)),
               'pinned': (torch.from_numpy(left).pin_memory(), torch.from_numpy(right).pin_memory()),
               'device': (torch.from_numpy(left).cuda(), torch.from_numpy(right).cuda())}
    outs = {}
    for kind, (l, r) in sources.items():
        eng.tensor('raw_left').fill_(-1); eng.tensor('raw_right').fill_(-1)
        eng.set_input(l, r)
        torch.cuda.synchronize()
        gl, gr = eng.tensor('raw_left').cpu().numpy(), eng.tensor('raw_right').cpu().numpy()
        for g, ref, side in ((gl, ref_l, 'left'), (gr, ref_r, 'right')):
            assert np.abs(g.astype(np.float64) - ref).max() <= 1e-4, (kind, side)
        outs[kind] = (gl, gr)
    for kind in ('pinned', 'device'):
        assert np.array_equal(outs[kind][0], outs['pageable'][0]) and np.array_equal(outs[kind][1], outs['pageable'][1])
    rh, rw = rs if rs is not None else (h, w)
    if rh < H:                                     # zero padding, exactly
        pt = (H - rh) // 2
        assert (outs['device'][0][:, :pt] == 0).all() and (outs['device'][0][:, pt + rh:] == 0).all()
    if rw < W:
        pl = (W - rw) // 2
        assert (outs['device'][0][:, :, :pl] == 0).all() and (outs['device'][0][:, :, pl + rw:] == 0).all()
    if (h, w) == (H, W) and rs is None:            # identity == the plain uint8 path, bit for bit
        eng.set_resize(None)
        eng.set_input(torch.from_numpy(left), torch.from_numpy(right))
        torch.cuda.synchronize()
        assert np.array_equal(eng.tensor('raw_left').cpu().numpy().view(np.uint32), outs['device'][0].view(np.uint32))
        assert np.array_equal(eng.tensor('raw_right').cpu().numpy().view(np.uint32), outs['device'][1].view(np.uint32))
    del eng
    _release()


def test_resized_prefetch_matches_serial_path():
    """prefetch() stages camera-size uint8 frames; the step then rescales from the staging buffers."""
    from madstereo.synthetic import make_pair
    frames = []
    for k in range(4):
        l, r, _ = make_pair(240, 320, seed=40 + k)
        frames.append((np.clip(np.rint(l), 0, 255).astype(np.uint8), np.clip(np.rint(r), 0, 255).astype(np.uint8)))
    losses = {}
    for pipelined in (False, True):
        net, ad, _ = _madnet(320, 512, 'MAD', seq=[0, 3, 1, 4])
        ad.engine.set_resize((480, 640))
        res = []
        for k, (l, r) in enumerate(frames):
            nxt = frames[k + 1] if pipelined and k + 1 < len(frames) else None
            res.append(ad.step(l, r, prefetch=nxt)['loss'])
        losses[pipelined] = res
        del net, ad
        _release()
    assert losses[False] == losses[True]


# ---- 7. the demo end to end ----------------------------------------------------------------------------------
def _demo_modules():
    for p in (PKG, DEMO):
        if p not in sys.path:
            sys.path.insert(0, p)
    import Live_Adaptation_Demo
    import demo_model
    return Live_Adaptation_Demo, demo_model


def _write_image_list(tmp, n, h=480, w=640):
    import cv2
    from madstereo.synthetic import make_pair
    lines, frames = [], []
    for k in range(n):
        l, r, _ = make_pair(h, w, seed=60 + k)
        l8, r8 = (np.clip(np.rint(x[0]), 0, 255).astype(np.uint8) for x in (l, r))
        pl, pr = str(tmp / ('l%d.png' % k)), str(tmp / ('r%d.png' % k))
        cv2.imwrite(pl, l8[:, :, ::-1]); cv2.imwrite(pr, r8[:, :, ::-1])      # stored BGR, read back as RGB
        lines.append('%s;%s' % (pl, pr))
        frames.append((l8[None], r8[None]))
    (tmp / 'list.txt').write_text('\n'.join(lines) + '\n')
    (tmp / 'camera.json').write_text(json.dumps({'list': str(tmp / 'list.txt'), 'fps': 0}))
    return frames


def _write_weights(tmp, with_adam):
    from madstereo.tf_checkpoint import write_checkpoint
    from oracle.madnet import init_params
    params = init_params(seed=42)
    tensors = dict(params)
    if with_adam:
        rng = np.random.default_rng(9)
        for n, a in params.items():
            tensors[n + '/Adam'] = rng.normal(0, 1e-3, a.shape).astype(np.float32)
            tensors[n + '/Adam_1'] = rng.uniform(0, 1e-5, a.shape).astype(np.float32)
        tensors['beta1_power'] = np.float32(0.9 ** 11)
        tensors['beta2_power'] = np.float32(0.999 ** 11)
    prefix = str(tmp / 'weights.ckpt')
    write_checkpoint(prefix, tensors)
    return prefix, tensors


def _run_demo(tmp, mode, weights, ssim_th, out_name):
    demo, _ = _demo_modules()
    args = demo.build_parser().parse_args([
        '--cameraName', 'ImageList', '--cameraConfig', str(tmp / 'camera.json'), '--weights', weights, '--mode', mode,
        '--blockConfig', os.path.join(PKG, 'block_config', 'MadNet_full.json'), '--SSIMTh', str(ssim_th),
        '--output', str(tmp / out_name)])
    dd = demo.main(args)
    rows = [l.split(',') for l in open(str(tmp / out_name / 'log.csv')).read().splitlines()[1:]]
    return dd, rows


@pytest.mark.parametrize('mode', ['MAD', 'FULL', 'NONE'])
def test_demo_end_to_end(tmp_path, mode):
    _, demo_model = _demo_modules()
    frames = _write_image_list(tmp_path, 5)
    weights, tensors = _write_weights(tmp_path, with_adam=False)
    dd, rows = _run_demo(tmp_path, mode, weights, 10.0, 'out')
    assert len(rows) == len(frames) and all(os.path.exists(str(tmp_path / 'out' / ('disparity_%06d.png' % k))) for k in range(5))
    losses = [float(r[1]) for r in rows]
    modules = [int(r[2]) for r in rows]
    assert not np.any(dd.sample_distribution), 'the demo quirk keeps the sample distribution at zero'
    if mode == 'NONE':
        w = dd._adapt.engine.export_params()
        for n, a in w.items():
            assert np.array_equal(a, tensors[n].reshape(a.shape)), n
    del dd
    _release()
    # the same frames and module sequence through OnlineAdaptation.step directly
    train_config = json.load(open(os.path.join(PKG, 'block_config', 'MadNet_full.json')))
    ad, _fetch = demo_model.build_engine('MADNet', 320, 512, mode, train_config, LR, 10.0, [480, 640])
    demo_model.restore_weights(ad, weights)
    if mode == 'MAD':
        ad.sampler = _Seq(modules)
    direct = [ad.step(l, r)['loss'] for l, r in frames]
    assert direct == losses
    del ad
    _release()


def test_demo_reset_restores_weights_and_adam_state(tmp_path):
    _write_image_list(tmp_path, 3)
    weights, tensors = _write_weights(tmp_path, with_adam=True)
    dd, rows = _run_demo(tmp_path, 'MAD', weights, 0.0, 'out')
    assert [r[3] for r in rows] == ['1', '1', '1'] and dd._adapt.reset_counter == 3
    eng = dd._adapt.engine
    w, m, v = eng.export_params(), eng.export_params(eng.momentum), eng.export_params(eng.adam_v)
    trained = set(dd._adapt.trained_variable_names())
    for n in w:
        assert np.array_equal(w[n], tensors[n].reshape(w[n].shape)), n
        if n in trained:
            assert np.array_equal(m[n], tensors[n + '/Adam'].reshape(m[n].shape)), n
            assert np.array_equal(v[n], tensors[n + '/Adam_1'].reshape(v[n].shape)), n
    p = _f32(eng.adam_powers)
    assert p[0] == tensors['beta1_power'] and p[1] == tensors['beta2_power']
    del dd, eng
    _release()
