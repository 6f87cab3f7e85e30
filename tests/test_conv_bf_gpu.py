"""GPU parity of the split-16-bit wgmma convolution kernels (csrc/conv_bf.cu, csrc/wgrad_bf.cu) vs the CPU oracle.

Three 16-bit MMAs per K step on hi/lo planes, accumulated in fp32:
  forward  : fp16 planes (22 mantissa bits)  -> per-product relative error <= ~3 * 2^-22; tolerance 2e-5 relative L-inf
  gradients: bf16 planes (16 mantissa bits)  -> per-product relative error <= ~3 * 2^-16; tolerance 1e-4 relative L-inf
Measured errors can be logged (MS_TEST_REPORT_DIR, below).
"""
import json
import os
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
TOL = 1e-4          # bf16-plane kernels (dgrad, wgrad)
TOL_FWD = 2e-5      # fp16-plane forward
# MS_TEST_REPORT_DIR=<dir>: measured errors are appended to <dir>/conv_bf_errors.jsonl (nothing is written otherwise)
_LOG = os.path.join(os.environ['MS_TEST_REPORT_DIR'], 'conv_bf_errors.jsonl') if os.environ.get('MS_TEST_REPORT_DIR') else None


def _log(rec):
    if _LOG is None:
        return
    try:
        os.makedirs(os.path.dirname(_LOG), exist_ok=True)
        with open(_LOG, 'a') as f:
            f.write(json.dumps(rec) + '\n')
    except OSError:
        pass


def rel_linf(a, b):
    a = np.asarray(a, dtype=np.float64); b = np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def cu(x):
    return torch.as_tensor(np.ascontiguousarray(x, dtype=np.float32)).cuda()


CASES = [
    # n, h, w, cin, cout, k, stride, dil, alpha
    (1, 32, 8, 32, 32, 3, 1, 1, 0.2),           # exactly one 8x32 tile
    (1, 16, 32, 64, 64, 3, 1, 1, 0.2),
    (2, 24, 40, 128, 128, 3, 1, 1, 0.2),        # partial tiles, batch 2
    (1, 24, 48, 128, 96, 3, 1, 4, 0.2),         # dilated (context net)
    (1, 24, 48, 96, 64, 3, 1, 16, 0.2),         # dilation > tile height: one patch per tap
    (1, 96, 320, 96, 64, 3, 1, 16, 0.2),        # dilation 16 on a full level-2 map (N = 256, halo patch)
    (1, 12, 40, 136, 128, 3, 1, 1, 0.2),        # K not a multiple of 32 (TMA zero-fills the channels)
    (1, 6, 20, 192, 192, 3, 1, 1, 0.2),         # level 6: two M blocks, split-K
    (1, 12, 40, 133, 128, 3, 1, 1, 0.2),        # level 5 estimator input (odd channel count), split-K
    (2, 20, 36, 16, 16, 3, 1, 1, 0.2),
    (1, 16, 16, 128, 64, 1, 1, 1, 0.1),         # 1x1 (DispNet conv_redir)
    (1, 96, 320, 128, 128, 3, 1, 1, 0.2),       # the dominant MADNet layer shape (N = 256 tiles, 120 CTAs)
    (1, 96, 320, 38, 128, 3, 1, 1, 0.2),        # estimator-2 disp-1
    (1, 48, 160, 70, 128, 3, 1, 1, 0.2),        # estimator-3 disp-1
    (2, 192, 640, 16, 32, 3, 2, 1, 0.2),        # pyramid conv3: stride 2 through TMA element strides
    (2, 48, 160, 64, 96, 3, 2, 1, 0.2),         # pyramid conv7
    (1, 24, 80, 96, 128, 3, 2, 1, 0.2),         # pyramid conv9
    (1, 96, 320, 64, 128, 5, 2, 1, 0.1),        # DispNet conv2 (5x5 stride 2)
    (1, 24, 80, 256, 512, 3, 2, 1, 0.1),        # DispNet conv4: 4 M blocks
]


@pytest.mark.parametrize('case', CASES)
def test_conv_bf_forward(case):
    from madstereo import ops
    from oracle import tf1_ops as T
    n, h, w, cin, cout, k, stride, dil, alpha = case
    rng = np.random.default_rng(sum(case[:8]))
    x = rng.standard_normal((n, h, w, cin)).astype(np.float32)
    wt = (rng.standard_normal((k, k, cin, cout)) / np.sqrt(k * k * cin)).astype(np.float32)
    b = rng.uniform(-0.1, 0.1, cout).astype(np.float32)
    ref = T.conv2d(torch.tensor(x), torch.tensor(wt), torch.tensor(b), stride=stride, dilation=dil, alpha=alpha)
    out = ops.conv2d_bf(cu(x), cu(wt), cu(b), stride, dil, alpha)           # fp16 planes of x / 16 (the MADNet setting)
    torch.cuda.synchronize()
    assert out.shape == tuple(ref.shape)
    err = rel_linf(out.cpu().numpy(), ref.numpy())
    _log({'op': 'fwd', 'case': list(case), 'rel_linf': err})
    assert err < TOL_FWD


@pytest.mark.parametrize('case', CASES)
def test_conv_bf_dgrad(case):
    """stride 1: one launch; stride 2: the four output-parity classes as dense launches (conv_bf.cu)."""
    from madstereo import ops
    from oracle import tf1_ops as T
    n, h, w, cin, cout, k, stride, dil, alpha = case
    rng = np.random.default_rng(sum(case[:8]) + 1)
    x = rng.standard_normal((n, h, w, cin)).astype(np.float32)
    wt = (rng.standard_normal((k, k, cin, cout)) / np.sqrt(k * k * cin)).astype(np.float32)
    xt = torch.tensor(x, requires_grad=True)
    pre = T.conv2d(xt, torch.tensor(wt), torch.zeros(cout), stride=stride, dilation=dil, alpha=None)
    g = rng.standard_normal(pre.shape).astype(np.float32)
    (gx,) = torch.autograd.grad(pre, xt, grad_outputs=torch.tensor(g))
    dx = ops.conv2d_dgrad_bf(cu(g), cu(wt), (h, w), stride, dil)
    torch.cuda.synchronize()
    err = rel_linf(dx.cpu().numpy(), gx.numpy())
    _log({'op': 'dgrad', 'case': list(case), 'rel_linf': err})
    assert err < TOL


WGRAD_CASES = [c for c in CASES if c[3] >= 16 and c[4] >= 16 and c[4] % 4 == 0] + [
    (1, 6, 20, 197, 128, 3, 1, 1, 0.2),         # estimator-6 disp-1: two ci blocks, odd channel count
    (2, 6, 20, 192, 192, 3, 1, 1, 0.2),         # pyramid conv12 (both towers): two co blocks
    (1, 96, 320, 33, 128, 3, 1, 1, 0.2),        # context-1
    (1, 96, 320, 128, 128, 3, 1, 2, 0.2),       # context-2 (dilation 2: shared halo patch)
    (1, 96, 320, 128, 96, 3, 1, 8, 0.2),        # context-4 (dilation 8: one box per tap)
]


@pytest.mark.parametrize('case', WGRAD_CASES)
def test_wgrad_bf(case):
    """dW, db of csrc/wgrad_bf.cu (MN-major UMMA operands straight from the NHWC planes) vs autograd over the oracle conv."""
    from madstereo import ops
    from oracle import tf1_ops as T
    n, h, w, cin, cout, k, stride, dil, alpha = case
    rng = np.random.default_rng(sum(case[:8]) + 2)
    x = rng.standard_normal((n, h, w, cin)).astype(np.float32)
    wt = torch.tensor((rng.standard_normal((k, k, cin, cout)) / np.sqrt(k * k * cin)).astype(np.float32), requires_grad=True)
    b = torch.zeros(cout, requires_grad=True)
    pre = T.conv2d(torch.tensor(x), wt, b, stride=stride, dilation=dil, alpha=None)
    g = rng.standard_normal(pre.shape).astype(np.float32)
    gw, gb = torch.autograd.grad(pre, (wt, b), grad_outputs=torch.tensor(g))
    dw, db = ops.conv2d_wgrad_bf(cu(x), cu(g), k, k, stride, dil)
    torch.cuda.synchronize()
    e1, e2 = rel_linf(dw.cpu().numpy(), gw.numpy()), rel_linf(db.cpu().numpy(), gb.numpy())
    _log({'op': 'wgrad', 'case': list(case), 'rel_linf_dw': e1, 'rel_linf_db': e2})
    assert e1 < TOL and e2 < TOL


@pytest.mark.parametrize('mag,scale', [(1e-3, 64.0), (1e-3, 0.0625), (300.0, 0.0625), (2.0e5, 0.0625)])
def test_conv_bf_forward_activation_range(mag, scale):
    """fp16 forward planes hold x * act_scale: small activations need a large scale (DispNet: 64), large ones a small one
    (MADNet: 1/16); out-of-range values saturate (graceful degradation), they never become inf / nan."""
    from madstereo import ops
    from oracle import tf1_ops as T
    n, h, w, cin, cout, k = 1, 24, 40, 64, 64, 3
    rng = np.random.default_rng(11)
    x = (rng.standard_normal((n, h, w, cin)) * mag).astype(np.float32)
    wt = (rng.standard_normal((k, k, cin, cout)) / np.sqrt(k * k * cin)).astype(np.float32)
    b = np.zeros(cout, np.float32)
    ref = T.conv2d(torch.tensor(x), torch.tensor(wt), torch.tensor(b), stride=1, dilation=1, alpha=0.2)
    out = ops.conv2d_bf(cu(x), cu(wt), cu(b), 1, 1, 0.2, act_scale=scale)
    torch.cuda.synchronize()
    err = rel_linf(out.cpu().numpy(), ref.numpy())
    _log({'op': 'fwd_range', 'mag': mag, 'scale': scale, 'rel_linf': err})
    assert np.isfinite(out.cpu().numpy()).all()
    good_range = 6e-5 * 64 < mag * scale < 6e4 / 8
    assert err < (TOL_FWD if good_range else 5e-3), (mag, scale, err)


# conv2d_transpose (DispNet's 4x4 stride-2 up-convolutions, Nets/DispNet.py:45-57) and its two gradients on the wgmma path.
# The gradients are checked against autograd THROUGH the oracle's conv2d_transpose (tf.gradients of the same op).
TCASES = [
    # n, h, w, cin, cout
    (1, 6, 20, 1024, 512),        # up5/deconv at 1280x384 (8 output-channel blocks in the input gradient)
    (1, 12, 40, 512, 256),        # up4/deconv
    (1, 48, 160, 128, 64),        # up2/deconv
    (1, 96, 320, 64, 32),         # up1/deconv
    (2, 10, 12, 64, 32),          # ragged tiles, batch 2
    (1, 7, 9, 96, 48),            # odd sizes
]


def _transpose_case(case):
    from oracle import tf1_ops as T
    n, h, w, cin, cout = case
    rng = np.random.default_rng(sum(case))
    x = rng.standard_normal((n, h, w, cin)).astype(np.float32)
    wt = (rng.standard_normal((4, 4, cout, cin)) / np.sqrt(4.0 * cin)).astype(np.float32)
    b = rng.uniform(-0.1, 0.1, cout).astype(np.float32)
    g = rng.standard_normal((n, 2 * h, 2 * w, cout)).astype(np.float32)
    xt, wtt, bt = (torch.tensor(v, requires_grad=True) for v in (x, wt, b))
    pre = T.conv2d_transpose(xt, wtt, bt, 2, None)
    gx, gw, gb = torch.autograd.grad(pre, [xt, wtt, bt], grad_outputs=torch.tensor(g))
    return x, wt, b, g, pre.detach().numpy(), gx.numpy(), gw.numpy(), gb.numpy()


@pytest.mark.parametrize('case', TCASES)
def test_conv_transpose_bf_forward(case):
    from madstereo import ops
    x, wt, b, g, ref, _, _, _ = _transpose_case(case)
    out = ops.conv2d_transpose_bf(cu(x), cu(wt), cu(b), 2, 1.0)
    torch.cuda.synchronize()
    err = rel_linf(out.cpu().numpy(), ref)
    _log({'op': 'transpose_fwd', 'case': list(case), 'rel_linf': err})
    assert err < TOL_FWD


@pytest.mark.parametrize('case', TCASES)
def test_conv_transpose_bf_dgrad(case):
    from madstereo import ops
    x, wt, b, g, _, gx, _, _ = _transpose_case(case)
    dx = ops.conv2d_transpose_dgrad_bf(cu(g), cu(wt), 2)
    torch.cuda.synchronize()
    err = rel_linf(dx.cpu().numpy(), gx)
    _log({'op': 'transpose_dgrad', 'case': list(case), 'rel_linf': err})
    assert err < TOL


@pytest.mark.parametrize('case', TCASES)
def test_conv_transpose_bf_wgrad(case):
    from madstereo import ops
    x, wt, b, g, _, _, gw, gb = _transpose_case(case)
    dw, db = ops.conv2d_transpose_wgrad_bf(cu(x), cu(g), 4, 4, 2)
    torch.cuda.synchronize()
    e_w = rel_linf(dw.cpu().numpy(), gw); e_b = rel_linf(db.cpu().numpy(), gb)
    _log({'op': 'transpose_wgrad', 'case': list(case), 'rel_linf': e_w, 'rel_linf_bias': e_b})
    assert e_w < TOL and e_b < 5e-5
