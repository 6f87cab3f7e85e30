"""The engine at batch B > 1, the uint8 input path and the EPE / bad3 metrics.

Batch properties need no oracle, so they also run where the CPU oracle is too slow (BASELINE config 5: MADNet at
1920x1056 -> padded 1920x1088, 8 frames).  Forward kernels use no float atomics and split-K reduces in a fixed order, so a
frame's forward values and activation gradients depend on that frame's data only:
  * frame independence: changing frame k of a batch leaves every per-frame tensor of every other frame bit-identical;
  * identical frames: a batch of B copies of one frame gives B bit-identical slots;
  * batch = mean of frames: batch B against B batch-1 runs.  The image count changes the convolution tiling (split-K,
    tile shape), hence the fp32 summation order, so these are bounded, not exact.
Every step is a FULL step without update: the whole backward chain writes its gradient tensors, the weights stay fixed.
"""
import functools
import gc
import json
import math
import os

import numpy as np
import pytest
import torch

from conftest import PKG

pytestmark = pytest.mark.gpu

TOL_BATCH_DISP = 2e-5       # relative L-inf, per frame and per disparity output, batch B vs batch 1
TOL_BATCH_LOSS = 1e-6       # relative, batch loss vs the mean of the per-frame losses
TOL_BATCH_GRAD = 1e-2       # per weight-gradient tensor: |g_batch - mean_b g_b|_2 <= TOL * mean_b |g_b|_2
# The image count changes the convolution tiling and hence the fp32 summation order of the forward; a pre-activation within
# ~1e-7 of a relu/leaky kink or of a floor() in the warps then lands on the other side and moves a whole gradient chain
# (the known noise source, see tests/dp_check.py).  The weight-gradient reduction itself is not the cause: reversing the
# frame order of the batch moves the gradients by < 6e-6 relative, and the bias gradient of a 1-channel head equals the
# fp64 sum of the engine's own activation gradient.  Measured on an H100 SXM (400 W power limit): up to 4.2e-3 (MADNet
# 1920x1088 b8, level-6 head bias), 3.1e-3 (DispNet 384x1280 b2) and 2.3e-5 (MADNet 64x128 b4) of the per-frame scale; the
# fp32 CPU oracle's own distance to the fp64 oracle on a FULL step at 640x384 b2 is up to 1.2e-2 relative L2.  The scale is
# the mean per-frame norm, not the norm of the mean: the coarse heads' gradients cancel across frames (config 5, level-5
# disp-6 bias: per-frame values of +-2e-6 average to 9e-9), and relative to such a mean any per-frame rounding looks large.

# MS_TEST_REPORT_DIR=<dir>: measured distances are appended to <dir>/batch.jsonl (nothing is written otherwise)
_LOG = os.path.join(os.environ['MS_TEST_REPORT_DIR'], 'batch.jsonl') if os.environ.get('MS_TEST_REPORT_DIR') else None


def _log(rec):
    if _LOG is None:
        return
    try:
        os.makedirs(os.path.dirname(_LOG), exist_ok=True)
        with open(_LOG, 'a') as f:
            f.write(json.dumps(rec) + '\n')
    except OSError:
        pass


# (net, H, W, B): config 5; a small size where the level-4..6 convolutions run split-K; DispNet at config 4's size
BATCH_CASES = [
    pytest.param('MADNet', 1056, 1920, 8, id='madnet-1056x1920-b8'),
    pytest.param('MADNet', 64, 128, 4, id='madnet-64x128-b4'),
    pytest.param('Dispnet', 384, 1280, 2, id='dispnet-384x1280-b2'),
]


@functools.lru_cache(maxsize=16)
def _frame(h, w, seed):
    """One synthetic frame (left, right, gt), each [1,h,w,c]; make_pair(batch=B, seed=s) frame b == _frame(h, w, s + 1000 b)."""
    from madstereo.synthetic import make_pair
    return make_pair(h, w, seed=seed)


def _frames(h, w, seeds):
    fs = [_frame(h, w, s) for s in seeds]
    return tuple(np.ascontiguousarray(np.concatenate([f[i] for f in fs])) for i in range(3))


def _build(net_name, left, right, mode='FULL', **kw):
    import Nets
    from madstereo.adaptation import OnlineAdaptation
    lt = torch.as_tensor(left).cuda(); rt = torch.as_tensor(right).cuda()
    if net_name == 'MADNet':
        from oracle.madnet import init_params
        net = Nets.get_stereo_net('MADNet', dict(left_img=lt, right_img=rt, split_layers=[None], sequence=True,
                                                 train_portion='BEGIN', bulkhead=(mode == 'MAD'), warping=True,
                                                 context_net=True, radius_d=2, stride=1, is_training=False))
        cfg = json.load(open(os.path.join(PKG, 'block_config', 'MadNet_full.json')))
        ad = OnlineAdaptation(net, mode=mode, train_config=cfg, lr=1e-4, **kw)
        params = init_params(seed=42)
    else:
        from oracle.dispnet import init_params
        net = Nets.get_stereo_net('Dispnet', dict(left_img=lt, right_img=rt, split_layers=[None], sequence=True,
                                                  train_portion='BEGIN', bulkhead=False, correlation=True))
        ad = OnlineAdaptation(net, mode=mode, lr=1e-4, **kw)
        params = init_params(seed=7)
    ad.load_weights(params)
    return net, ad


def _release():
    """Free the engines the caller has dropped (nets hold reference cycles through their layer handles) before the next
    one is built: at 1920x1088 x 8 frames one engine's workspace is several GB."""
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _full_step_no_update(net, left, right):
    from madstereo.engine import MODE_FULL
    eng = net.engine
    eng.set_input(left, right)
    eng.run(MODE_FULL, 0, (1 << len(net.get_disparities())) - 1, with_update=0)


def _per_frame(eng):
    """name -> device copy [B,...] of every named engine view with one slot per frame; a view over 2B images (left frames
    first, then right frames: the MADNet input image, the DispNet conv1/conv2 gradients) is split into its two halves."""
    out = {}
    for name in eng.tensor_names():
        t = eng.tensor(name)
        if t.shape[0] == eng.B:
            out[name] = t.clone()
        elif t.shape[0] == 2 * eng.B:
            out[name + '[left]'] = t[:eng.B].clone()
            out[name + '[right]'] = t[eng.B:].clone()
    return out


def _bits(t):
    return t.contiguous().view(torch.int32)


def _zero_per_frame(eng):
    for name in eng.tensor_names():
        t = eng.tensor(name)
        if t.shape[0] in (eng.B, 2 * eng.B):
            t.zero_()


# ---------------------------------------------------------------------------------------------------- batch properties
@pytest.mark.parametrize('net_name,h,w,B', BATCH_CASES)
def test_frame_independence(net_name, h, w, B):
    """Changing one frame of the batch (the last one, then the first one) leaves every forward and gradient view of every
    other frame bit-identical, and does change that frame's full-resolution disparity."""
    seeds = [3 + 1000 * b for b in range(B)]
    left, right, _ = _frames(h, w, seeds)
    net, ad = _build(net_name, left, right)
    eng = net.engine
    _full_step_no_update(net, left, right)
    base = _per_frame(eng)
    assert 'rescaled_prediction' in base and any(n.startswith('grad/') for n in base)
    for k in (B - 1, 0):
        l2, r2, _ = _frames(h, w, [777 if b == k else s for b, s in enumerate(seeds)])
        _full_step_no_update(net, l2, r2)
        cur = _per_frame(eng)
        for name, t in base.items():
            for b in range(B):
                if b != k:
                    assert torch.equal(_bits(t[b]), _bits(cur[name][b])), (k, name, b)
        assert not torch.equal(base['rescaled_prediction'][k], cur['rescaled_prediction'][k]), k
        del cur
    del net, ad, eng, base
    _release()


@pytest.mark.parametrize('net_name,h,w,B', BATCH_CASES)
def test_identical_frames_give_identical_slots(net_name, h, w, B):
    l1, r1, _ = _frame(h, w, 11)
    left, right = np.repeat(l1, B, axis=0), np.repeat(r1, B, axis=0)
    net, ad = _build(net_name, left, right)
    eng = net.engine
    _zero_per_frame(eng)           # views a step does not write hold the same value in every slot
    _full_step_no_update(net, left, right)
    snap = _per_frame(eng)
    for name, t in snap.items():
        for b in range(1, B):
            assert torch.equal(_bits(t[0]), _bits(t[b])), (name, b)
    del net, ad, eng, snap
    _release()


def _step_results(net, left, right):
    _full_step_no_update(net, left, right)
    eng = net.engine
    loss = eng.read_scalars()[0]
    disps = [d.numpy() for d in net.get_disparities()]
    grads = {n: g.detach().cpu().numpy().astype(np.float64) for n, g in eng.param_views(eng.grads).items()}
    return loss, disps, grads


@pytest.mark.parametrize('net_name,h,w,B', BATCH_CASES)
def test_batch_equals_mean_of_frames(net_name, h, w, B):
    """Every loss is a mean over the batch, so batch B = the mean of B batch-1 steps: per-frame disparities, the loss and
    every weight gradient (relative to the per-frame gradient scale, see TOL_BATCH_GRAD).  This is the equivalence
    data-parallel training rests on (N ranks x 1 frame == batch N)."""
    left, right, _ = _frames(h, w, [5 + 1000 * b for b in range(B)])
    net, ad = _build(net_name, left, right)
    loss_b, disps_b, grads_b = _step_results(net, left, right)
    del net, ad
    _release()
    net, ad = _build(net_name, left[:1], right[:1])
    losses, disps_1, grads_sum, grads_scale = [], [], {}, {}
    for b in range(B):
        loss, disps, grads = _step_results(net, left[b:b + 1], right[b:b + 1])
        losses.append(loss); disps_1.append(disps)
        for n, g in grads.items():
            grads_sum[n] = grads_sum.get(n, 0.0) + g
            grads_scale[n] = grads_scale.get(n, 0.0) + float(np.linalg.norm(g))
    del net, ad
    _release()
    worst_disp = 0.0
    for b in range(B):
        for i, (db, d1) in enumerate(zip(disps_b, disps_1[b])):
            r = float(np.abs(db[b].astype(np.float64) - d1[0]).max() / max(np.abs(d1[0]).max(), 1e-30))
            worst_disp = max(worst_disp, r)
            assert r < TOL_BATCH_DISP, ('frame', b, 'disparity', i, r)
    mean_loss = float(np.mean(np.asarray(losses, np.float64)))
    loss_err = abs(loss_b - mean_loss) / abs(mean_loss)
    worst_grad, worst_name = 0.0, None
    for n, gs in grads_sum.items():
        gm = gs / B
        r = float(np.linalg.norm(grads_b[n] - gm) / max(grads_scale[n] / B, 1e-30))
        if r > worst_grad:
            worst_grad, worst_name = r, n
    _log({'test': 'batch_equals_mean_of_frames', 'net': net_name, 'hw': [h, w], 'B': B, 'worst_disp_rel_linf': worst_disp,
          'loss_rel': loss_err, 'worst_grad_rel_l2': worst_grad, 'worst_grad_tensor': worst_name})
    assert loss_err < TOL_BATCH_LOSS, (loss_b, losses)
    assert worst_grad < TOL_BATCH_GRAD, (worst_name, worst_grad)


# ---------------------------------------------------------------------------------------------------- uint8 input
def _u8_frames(h, w, B, seed):
    left, right, _ = _frames(h, w, [seed + 1000 * b for b in range(B)])
    return np.round(left).astype(np.uint8), np.round(right).astype(np.uint8)


def _two_mad_steps(left, right):
    """Two MAD steps (modules 0, 1) from the same weights: raw inputs, losses, all disparities, adapted weights."""
    shape_only = np.zeros(tuple(left.shape), np.float32)
    net, ad = _build('MADNet', shape_only, shape_only, mode='MAD', sample_mode='SEQUENTIAL')
    eng = net.engine
    out = {'loss': [], 'disp': []}
    for it in range(2):
        r = ad.step(left, right, want_disp_mask=0b111111)
        assert r['blocks'] == [it]
        if it == 0:
            out['raw_left'] = eng.tensor('raw_left').cpu().numpy()
            out['raw_right'] = eng.tensor('raw_right').cpu().numpy()
        out['loss'].append((r['loss'], r['train_loss']))
        out['disp'].append([d.numpy() for d in net.get_disparities()])
    out['weights'] = eng.weights.cpu().numpy()
    del net, ad, eng
    _release()
    return out


@pytest.mark.parametrize('hwb', [(64, 128, 3), (375, 1242, 1), (1056, 1920, 2)], ids=['64x128-b3', 'kitti-375x1242-b1', '1056x1920-b2'])
def test_uint8_input_matches_float_input(hwb):
    """uint8 frames from pageable host, pinned host and device memory give bit-identically the step of the same pixels
    given as float32.  375x1242 (KITTI) has B*H*W*3 = 1397250, not a multiple of 4."""
    h, w, B = hwb
    lu, ru = _u8_frames(h, w, B, seed=21)
    ref = _two_mad_steps(lu.astype(np.float32), ru.astype(np.float32))
    sources = {'pageable': lambda x: torch.from_numpy(x),
               'pinned': lambda x: torch.from_numpy(x).pin_memory(),
               'device': lambda x: torch.from_numpy(x).cuda()}
    for src, conv in sources.items():
        got = _two_mad_steps(conv(lu), conv(ru))
        assert np.array_equal(got['raw_left'].view(np.int32), ref['raw_left'].view(np.int32)), src
        assert np.array_equal(got['raw_right'].view(np.int32), ref['raw_right'].view(np.int32)), src
        assert got['loss'] == ref['loss'], src
        for it in range(2):
            for i, (a, b) in enumerate(zip(got['disp'][it], ref['disp'][it])):
                assert np.array_equal(a, b), (src, it, i)
        assert np.array_equal(got['weights'], ref['weights']), src


# ---------------------------------------------------------------------------------------------------- EPE / bad3
def _epe_bad3_reference(disp, gt):
    """Stereo_Online_Adaptation.py:76-82 in float64, with |d - gt| taken in float32 as the kernel does."""
    abs_err = np.abs(disp.astype(np.float32) - gt.astype(np.float32)).astype(np.float64)
    valid = (gt != 0).astype(np.float64)
    filtered = abs_err * valid
    with np.errstate(invalid='ignore', divide='ignore'):
        epe = filtered.sum() / valid.sum()
        bad3 = (filtered > 3.0).astype(np.float64).sum() / valid.sum()
    return epe, bad3


def test_epe_bad3_match_reference_metric():
    h, w, B = 64, 128, 3
    left, right, _ = _frames(h, w, [31 + 1000 * b for b in range(B)])
    net, ad = _build('MADNet', left, right, mode='NONE')
    lt, rt = torch.as_tensor(left).cuda(), torch.as_tensor(right).cuda()
    ad.step(lt, rt)
    d = net.get_disparities()[-1].numpy()
    rng = np.random.default_rng(0)
    # |d - gt| spread over [0, 8] px: about half the valid pixels above the 3 px threshold, some exactly at it
    gt = (d + rng.uniform(-8.0, 8.0, d.shape)).astype(np.float32)
    gt[:, ::9, ::4] = d[:, ::9, ::4] + np.float32(3.0)
    gt[:, 5:9] = d[:, 5:9] + np.float32(40.0)              # far off: well above 3 px
    gt[0, ::7, ::5] = 0.0                                   # holes, a different pattern and count in every frame
    gt[1, :, :50] = 0.0
    gt[2][rng.random((h, w, 1)) < 0.1] = 0.0
    gt_before = gt.copy()
    out = ad.step(lt, rt, gt=gt)
    d2 = net.get_disparities()[-1].numpy()
    assert np.array_equal(gt, gt_before)
    epe, bad3 = _epe_bad3_reference(d2, gt)
    assert 0.2 < bad3 < 0.9 and epe > 3.0
    assert abs(out['epe'] - epe) <= 1e-6 * epe, (out['epe'], epe)
    assert out['bad3'] == np.float32(bad3), (out['bad3'], bad3)
    # one frame without ground truth: the batch metric counts only the valid pixels of the others
    gt[1] = 0.0
    out = ad.step(lt, rt, gt=gt)
    epe, bad3 = _epe_bad3_reference(net.get_disparities()[-1].numpy(), gt)
    assert abs(out['epe'] - epe) <= 1e-6 * epe and out['bad3'] == np.float32(bad3)
    # no valid pixel at all: 0 / 0 = NaN for both, as in the reference
    out = ad.step(lt, rt, gt=np.zeros_like(gt))
    assert math.isnan(out['epe']) and math.isnan(out['bad3'])
