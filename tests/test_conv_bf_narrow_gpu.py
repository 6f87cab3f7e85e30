"""Pixel-major conv_bf tiles (csrc/conv_bf.cu): layers whose output channels round up to 16, 32, 64 or 96 issue their MMAs
with M = pixels and N = that channel count instead of padding M to 128 output channels.  Same split-16-bit arithmetic
and tolerances as tests/test_conv_bf_gpu.py (2e-5 forward, 1e-4 gradients), against the CPU oracle."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
TOL = 1e-4
TOL_FWD = 2e-5


def rel_linf(a, b):
    a = np.asarray(a, dtype=np.float64); b = np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def cu(x):
    return torch.as_tensor(np.ascontiguousarray(x, dtype=np.float32)).cuda()


CASES = [
    # n, h, w, cin, cout, k, stride, dil, alpha
    (2, 192, 640, 16, 16, 3, 1, 1, 0.2),        # MADNet conv2 shape, both towers (its dgrad: M = 16)
    (2, 192, 640, 16, 32, 3, 2, 1, 0.2),        # conv3: dgrad is M = 16 at 192x640 (four parity launches)
    (2, 96, 320, 32, 32, 3, 1, 1, 0.2),         # conv4
    (1, 96, 320, 128, 96, 3, 1, 1, 0.2),        # estimator-2 disp3
    (1, 96, 320, 96, 64, 3, 1, 1, 0.2),         # estimator-2 disp4 / context5 (dgrad M = 96)
    (1, 96, 320, 64, 32, 3, 1, 1, 0.2),         # estimator-2 disp5 / context6
    (1, 96, 320, 128, 96, 3, 1, 8, 0.2),        # context4 (dilation 8)
    (1, 96, 320, 96, 64, 3, 1, 16, 0.2),        # context5 (dilation 16: one patch per tap)
    (1, 96, 320, 33, 128, 3, 1, 1, 0.2),        # context1: dgrad M = 33 -> 64
    (1, 96, 320, 38, 128, 3, 1, 1, 0.2),        # estimator-2 disp1: dgrad M = 38 -> 64
    (1, 6, 20, 64, 32, 3, 1, 1, 0.2),           # level 6 disp5: split-K
    (1, 12, 40, 96, 64, 3, 1, 2, 0.2),          # split-K, dilation 2
    (2, 23, 37, 32, 16, 3, 1, 1, 0.2),          # partial tiles, odd width, batch 2
    (2, 25, 41, 16, 33, 3, 2, 1, 0.2),          # stride 2 with odd sizes, cout 33 -> 64
    (1, 30, 50, 38, 38, 3, 1, 2, 0.2),          # odd channel counts both ways
    (1, 40, 72, 64, 96, 3, 2, 1, 0.2),          # pyramid conv7 shape, stride 2
    (1, 16, 16, 128, 8, 1, 1, 1, 0.1),          # 1x1, cout 8 -> 16
]


@pytest.mark.parametrize('case', CASES)
def test_conv_bf_narrow_forward(case):
    from madstereo import ops
    from oracle import tf1_ops as T
    n, h, w, cin, cout, k, stride, dil, alpha = case
    rng = np.random.default_rng(sum(case[:8]) + 7)
    x = rng.standard_normal((n, h, w, cin)).astype(np.float32)
    wt = (rng.standard_normal((k, k, cin, cout)) / np.sqrt(k * k * cin)).astype(np.float32)
    b = rng.uniform(-0.1, 0.1, cout).astype(np.float32)
    ref = T.conv2d(torch.tensor(x), torch.tensor(wt), torch.tensor(b), stride=stride, dilation=dil, alpha=alpha)
    out = ops.conv2d_bf(cu(x), cu(wt), cu(b), stride, dil, alpha)
    torch.cuda.synchronize()
    assert out.shape == tuple(ref.shape)
    assert rel_linf(out.cpu().numpy(), ref.numpy()) < TOL_FWD


@pytest.mark.parametrize('case', CASES)
def test_conv_bf_narrow_dgrad(case):
    from madstereo import ops
    from oracle import tf1_ops as T
    n, h, w, cin, cout, k, stride, dil, alpha = case
    rng = np.random.default_rng(sum(case[:8]) + 8)
    x = rng.standard_normal((n, h, w, cin)).astype(np.float32)
    wt = (rng.standard_normal((k, k, cin, cout)) / np.sqrt(k * k * cin)).astype(np.float32)
    xt = torch.tensor(x, requires_grad=True)
    pre = T.conv2d(xt, torch.tensor(wt), torch.zeros(cout), stride=stride, dilation=dil, alpha=None)
    g = rng.standard_normal(pre.shape).astype(np.float32)
    (gx,) = torch.autograd.grad(pre, xt, grad_outputs=torch.tensor(g))
    dx = ops.conv2d_dgrad_bf(cu(g), cu(wt), (h, w), stride, dil)
    torch.cuda.synchronize()
    assert rel_linf(dx.cpu().numpy(), gx.numpy()) < TOL


TCASES = [
    # n, h, w, cin, cout: forward M = cout, dgrad M = cin
    (1, 96, 320, 64, 32),         # DispNet up1/deconv
    (2, 11, 13, 96, 16),          # ragged tiles, batch 2
    (1, 24, 40, 32, 96),
]


@pytest.mark.parametrize('case', TCASES)
def test_conv_transpose_bf_narrow(case):
    from madstereo import ops
    from oracle import tf1_ops as T
    n, h, w, cin, cout = case
    rng = np.random.default_rng(sum(case))
    x = rng.standard_normal((n, h, w, cin)).astype(np.float32)
    wt = (rng.standard_normal((4, 4, cout, cin)) / np.sqrt(4.0 * cin)).astype(np.float32)
    b = rng.uniform(-0.1, 0.1, cout).astype(np.float32)
    g = rng.standard_normal((n, 2 * h, 2 * w, cout)).astype(np.float32)
    xt = torch.tensor(x, requires_grad=True)
    pre = T.conv2d_transpose(xt, torch.tensor(wt), torch.tensor(b), 2, None)
    (gx,) = torch.autograd.grad(pre, xt, grad_outputs=torch.tensor(g))
    out = ops.conv2d_transpose_bf(cu(x), cu(wt), cu(b), 2, 1.0)
    dx = ops.conv2d_transpose_dgrad_bf(cu(g), cu(wt), 2)
    torch.cuda.synchronize()
    assert rel_linf(out.cpu().numpy(), pre.detach().numpy()) < TOL_FWD
    assert rel_linf(dx.cpu().numpy(), gx.numpy()) < TOL


def test_madnet_narrow_weight_tiles():
    """The weight tiles the engine prepares (sized by ms_bf_weight_halfs) are CN rows for the narrow MADNet layers at
    1280x384: forward of estimator disp3-disp5, context4-context6 and pyramid conv3-conv4; dgrad of pyramid conv2-conv3
    (M = cin = 16) and of estimator-2 disp1 / context1 (cin 38 / 33 -> 64)."""
    from madstereo import _lib
    lib = _lib.lib()

    def rows(m, k):
        kpad = 32 if k <= 32 else -(-k // 64) * 64
        halfs = lib.ms_bf_weight_halfs(9, m, k)
        assert halfs % (2 * 9 * kpad) == 0
        return halfs // (2 * 9 * kpad)

    fwd = {'disp3': (128, 96), 'disp4': (96, 64), 'disp5': (64, 32), 'context4': (128, 96), 'context5': (96, 64),
           'context6': (64, 32), 'conv3': (16, 32), 'conv4': (32, 32)}
    for name, (cin, cout) in fwd.items():
        assert rows(cout, cin) == {16: 16, 32: 32, 64: 64, 96: 96}[cout], name
    for name, (cin, cout) in {'conv2': (16, 16), 'conv3': (16, 32), 'disp1': (38, 128), 'context1': (33, 128)}.items():
        assert rows(cin, cout) == (16 if cin <= 16 else 64), name
    assert rows(128, 128) == 128 and rows(192, 128) == 256 and rows(97, 64) == 128
