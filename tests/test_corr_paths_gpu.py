"""Every correlation kernel the dispatch in csrc/corr.cu (corr_fwd / corr_bwd) can pick, against the float64 oracle.

The engine's default setting (radius 2, stride 1, warped) sends every MADNet cost volume to one kernel, corr_fwd4_kernel.
The other kernels serve other radius_d / stride values, narrow or odd channel counts and wide windows; each case below
names the kernel its shape must reach, and test_dispatch_reaches_named_kernel checks that with torch.profiler so the
table cannot silently stop covering a kernel when the dispatch heuristics change.

Forward: out = concat(left, corr(left, warp(right, u)), u, 0...) written through ms_corr_fwd into a buffer wider than
the concat, pre-filled with a sentinel, with left / right as channel-strided views into wider tensors where the case
says so.  The channel contract checked is the one stated next to ms_corr_fwd in include/madstereo.h.
Backward: ms_corr_bwd against autograd over the oracle, with dcost laid out as the engine's [left | corr | u | pad].
"""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

SENTINEL = 1234.5


def rel_linf(a, b):
    a = np.asarray(a, dtype=np.float64); b = np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def ndisp(d, s):
    return len(range(-d, d + 1, s))


def pad4(c):
    return (c + 3) // 4 * 4


@pytest.fixture(scope='module')
def lib():
    from madstereo._lib import lib as _l
    return _l()


def _check(rc, what):
    from madstereo._lib import check
    check(rc, what)


def _p(t):
    return ctypes.c_void_p(t.data_ptr() if t is not None else 0)


def _s():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _view(x, cs, fill):
    """x [b,h,w,c] float32 numpy -> CUDA view [..., :c] of a [b,h,w,cs] tensor whose other channels hold `fill`."""
    b, h, w, c = x.shape
    wide = torch.full((b, h, w, cs), fill, dtype=torch.float32, device='cuda')
    wide[..., :c] = torch.from_numpy(x).cuda()
    return wide, wide[..., :c]


def _warp_offsets(rng, b, h, w, umax):
    u = rng.uniform(-umax, umax, (b, h, w, 1)).astype(np.float32)
    for i in range(b):                                   # taps outside both borders, in every image
        u[i, 0, 0, 0] = -7.25
        u[i, -1, -1, 0] = 9.5
        if w > 8:
            u[i, h // 2, w // 2, 0] = -(w // 2) - 3.5      # lands left of column 0
            u[i, h // 2, w // 2 - 1, 0] = w / 2 + 2.25     # lands right of column w-1
    return u


def _oracle_corr(x, y, u, d, s):
    from oracle import tf1_ops as T
    xt = torch.tensor(x, dtype=torch.float64); yt = torch.tensor(y, dtype=torch.float64)
    if u is not None:
        yt = T.linear_warp(yt, torch.tensor(u, dtype=torch.float64))
    return T.correlation(xt, yt, d, s).numpy()


# ---------------------------------------------------------------------------------------------------------- forward
# name: (B, h, w, C, max_disp, stride, warp, copy_left, u_chan, extra left/right channels, kernel it must reach)
FWD_CASES = {
    'v4_c32_cat_u': (2, 3, 100, 32, 2, 1, True, True, True, 0, 'corr_fwd4_kernel<1>'),
    'v4_c64_cat_views': (1, 4, 72, 64, 2, 1, False, True, False, 8, 'corr_fwd4_kernel<2>'),
    'v4_c96_plain': (2, 3, 100, 96, 2, 1, True, False, False, 4, 'corr_fwd4_kernel<0>'),
    'v3_nd3_s2_cat_u': (2, 3, 150, 32, 2, 2, True, True, True, 0, 'corr_fwd3_kernel<0>'),
    'v3_nd2_s3_views': (2, 4, 37, 16, 2, 3, True, False, False, 4, 'corr_fwd3_kernel<0>'),
    'v3_c8_d1_cat': (1, 5, 300, 8, 1, 1, False, True, False, 0, 'corr_fwd3_kernel<0>'),
    'v3_nd5_pack8_cat_u': (2, 3, 140, 32, 4, 2, True, True, True, 0, 'corr_fwd3_kernel<5>'),
    'v3_nd5_pack8_unwarped': (1, 4, 20, 32, 4, 2, False, True, False, 4, 'corr_fwd3_kernel<5>'),
    'v3_nd5_c20_plain': (2, 3, 45, 20, 2, 1, False, False, False, 0, 'corr_fwd3_kernel<5>'),
    'v2_nd5_pack8_cat_u': (2, 3, 100, 64, 4, 2, True, True, True, 4, 'corr_fwd2_kernel<5>'),
    'v2_nd5_c48_plain': (1, 3, 24, 48, 2, 1, True, False, False, 0, 'corr_fwd2_kernel<5>'),
    'v2_nd3_s2_cat_u': (2, 3, 90, 64, 2, 2, True, True, True, 0, 'corr_fwd2_kernel<0>'),
    'v2_nd9_cat_u_views': (2, 3, 150, 32, 4, 1, True, True, True, 8, 'corr_fwd2_kernel<0>'),
    'v2_nd3_s3_c128_cat': (1, 3, 70, 128, 4, 3, True, True, False, 0, 'corr_fwd2_kernel<0>'),
    'v2_nd3_s3_unwarped': (2, 2, 33, 128, 4, 3, False, False, False, 0, 'corr_fwd2_kernel<0>'),
    'v1_c400_d40': (1, 2, 64, 400, 40, 1, False, False, False, 0, 'corr_fwd_kernel('),
    'v1_c192_d40_warp_cat_u': (1, 2, 64, 192, 40, 1, True, True, True, 0, 'corr_fwd_kernel('),
}


def _fwd_setup(case, seed):
    b, h, w, c, d, s, warp, cat, uch, extra, _ = case
    nd = ndisp(d, s)
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((b, h, w, c)).astype(np.float32)
    y = rng.standard_normal((b, h, w, c)).astype(np.float32)
    u = _warp_offsets(rng, b, h, w, 3.0) if warp else None
    lw, lv = _view(x, c + extra, -3.0)
    rw, rv = _view(y, c + extra, 5.0)
    used = (c if cat else 0) + nd + (1 if uch else 0)
    ocs = pad4(used) + 8                                 # wider than the concat: the pad channels are visible
    out = torch.full((b, h, w, ocs), SENTINEL, dtype=torch.float32, device='cuda')
    if warp and uch:                                     # the engine's layout: u lives in the concat buffer
        out[..., c + nd] = torch.from_numpy(u[..., 0]).cuda()
        up, ucs = out[..., c + nd:], ocs
    elif warp:
        uw, up = _view(u, 3, 0.0)
        ucs = 3
    else:
        up, ucs = None, 1
    return dict(x=x, y=y, u=u, nd=nd, ocs=ocs, lw=lw, rw=rw, lv=lv, rv=rv, out=out, up=up, ucs=ucs,
                keep=[lw, rw] + ([uw] if warp and not uch else []))


def _fwd_call(lib, case, t):
    b, h, w, c, d, s, warp, cat, uch, extra, _ = case
    _check(lib.ms_corr_fwd(_p(t['lv']), c + extra, _p(t['rv']), c + extra, _p(t['up']), t['ucs'], _p(t['out']), t['ocs'],
                           b, h, w, c, d, s, int(cat), int(uch), _s()), 'ms_corr_fwd')


@pytest.mark.parametrize('name', list(FWD_CASES))
def test_corr_fwd_concat_contract(lib, name):
    case = FWD_CASES[name]
    b, h, w, c, d, s, warp, cat, uch, extra, _ = case
    t = _fwd_setup(case, seed=sum(case[:6]))
    _fwd_call(lib, case, t)
    torch.cuda.synchronize()
    out = t['out'].cpu().numpy()
    nd = t['nd']
    ref = _oracle_corr(t['x'], t['y'], t['u'], d, s)
    coff = c if cat else 0
    assert rel_linf(out[..., coff:coff + nd], ref) < 2e-5
    if cat:
        assert np.array_equal(out[..., :c], t['x']), 'left copy is not bit-identical'
        tail = c + nd
        if uch:
            assert np.array_equal(out[..., tail], t['u'][..., 0]), 'u channel changed'
            tail += 1
        assert (out[..., tail:] == 0.0).all(), 'pad channels after the concat must be zero'
    else:
        assert (out[..., nd:] == SENTINEL).all(), 'channels after the correlation must be left as they were'
    # the views' neighbouring channels are inputs only
    if extra:
        assert bool((t['lw'][..., c:] == -3.0).all()) and bool((t['rw'][..., c:] == 5.0).all())


def test_corr_wide_window_entry():
    """ms_corr_fwd_wide (DispNet's banded tensor-core kernel) at a ragged width, batch 2."""
    from madstereo import ops
    rng = np.random.default_rng(40)
    x = rng.standard_normal((2, 3, 100, 64)).astype(np.float32)
    y = rng.standard_normal((2, 3, 100, 64)).astype(np.float32)
    out = ops.correlation_wide(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), 40, act_scale=64.0)
    torch.cuda.synchronize()
    assert rel_linf(out.cpu().numpy(), _oracle_corr(x, y, None, 40, 1)) < 2e-5


# --------------------------------------------------------------------------------------------------------- backward
# name: (B, h, w, C, max_disp, stride, warp, add_left_slice, extra channels of every strided view, kernel, tolerance)
BWD_CASES = {
    'tma_s1_warp_du': (2, 3, 64, 32, 2, 1, True, True, 0, 'corr_bwd_kernel(', 2e-5),
    'views_s1_warp_du_slice': (2, 3, 64, 32, 2, 1, True, True, 4, 'corr_bwd_kernel(', 2e-5),
    'views_s2_unwarped_slice': (2, 3, 50, 32, 2, 2, False, True, 8, 'corr_bwd_kernel(', 2e-5),
    'views_s3_warp_du_slice': (2, 3, 40, 64, 4, 3, True, True, 4, 'corr_bwd_kernel(', 2e-5),
    'tma_s3_warp_du': (1, 4, 37, 16, 2, 3, True, False, 0, 'corr_bwd_kernel(', 2e-5),
    'tma_s2_nd5_unwarped': (1, 3, 60, 48, 4, 2, False, False, 0, 'corr_bwd_kernel(', 2e-5),
    'views_s2_nd5_warp_du_slice': (2, 3, 45, 32, 4, 2, True, True, 4, 'corr_bwd_kernel(', 2e-5),
    # C = 192, radius 4: the row no longer fits one tile (TW = 64 for w = 150: two full tiles, a ragged third, halos)
    'tiled_tma_unwarped': (2, 2, 150, 192, 4, 1, False, True, 0, 'corr_bwd_kernel(', 2e-5),
    'tiled_views_s2_unwarped_slice': (1, 3, 150, 192, 4, 2, False, True, 4, 'corr_bwd_kernel(', 2e-5),
    'mma_d40_slice': (1, 4, 100, 64, 40, 1, False, True, 0, 'corr_mma_bwd_kernel', 1e-4),
}


def _bwd_setup(case, seed):
    b, h, w, c, d, s, warp, slc, extra, _, _ = case
    nd = ndisp(d, s)
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((b, h, w, c)).astype(np.float32)
    y = rng.standard_normal((b, h, w, c)).astype(np.float32)
    u = _warp_offsets(rng, b, h, w, 3.0) if warp else None
    dcs = pad4(c + nd + (1 if warp else 0))
    # [left | corr | u | pad]: every channel holds data, so reading the wrong one shows
    gscale = 1e-3 if d >= 8 else 1.0
    dcost = (rng.standard_normal((b, h, w, dcs)) * gscale).astype(np.float32)
    lw, lv = _view(x, c + extra, -3.0)
    rw, rv = _view(y, c + extra, 5.0)
    dlw, dlv = _view(np.zeros_like(x), c + extra, SENTINEL)
    drw, drv = _view(np.zeros_like(y), c + extra, SENTINEL)
    t = dict(x=x, y=y, u=u, nd=nd, dcs=dcs, dcost_np=dcost, dcost=torch.from_numpy(dcost).cuda(), lw=lw, lv=lv, rw=rw, rv=rv,
             dlw=dlw, dlv=dlv, drw=drw, drv=drv, cs=c + extra)
    if warp:
        t['uw'], t['uv'] = _view(u, 2, 0.0)
        t['duw'], t['duv'] = _view(np.zeros_like(u), 3, SENTINEL)
    else:
        t['uv'] = t['duv'] = None
    return t


def _bwd_call(lib, case, t):
    b, h, w, c, d, s, warp, slc, extra, _, _ = case
    cs = t['cs']
    _check(lib.ms_corr_bwd(_p(t['lv']), cs, _p(t['rv']), cs, _p(t['uv']), 2, _p(t['dcost']), t['dcs'], _p(t['dlv']), cs,
                           _p(t['drv']), cs, _p(t['duv']), 3, b, h, w, c, d, s, int(slc), _s()), 'ms_corr_bwd')


@pytest.mark.parametrize('name', list(BWD_CASES))
def test_corr_bwd(lib, name):
    from oracle import tf1_ops as T
    case = BWD_CASES[name]
    b, h, w, c, d, s, warp, slc, extra, _, tol = case
    t = _bwd_setup(case, seed=sum(case[:6]) + 7)
    _bwd_call(lib, case, t)
    torch.cuda.synchronize()
    nd = t['nd']
    xt = torch.tensor(t['x'], dtype=torch.float64, requires_grad=True)
    yt = torch.tensor(t['y'], dtype=torch.float64, requires_grad=True)
    ut = torch.tensor(t['u'], dtype=torch.float64, requires_grad=True) if warp else None
    ref = T.correlation(xt, T.linear_warp(yt, ut) if warp else yt, d, s)
    g = torch.tensor(t['dcost_np'][..., c:c + nd], dtype=torch.float64)
    grads = torch.autograd.grad(ref, [xt, yt] + ([ut] if warp else []), grad_outputs=g)
    gx = grads[0].numpy() + (t['dcost_np'][..., :c] if slc else 0.0)
    dlw, drw = t['dlw'].cpu().numpy(), t['drw'].cpu().numpy()
    assert rel_linf(dlw[..., :c], gx) < tol
    assert rel_linf(drw[..., :c], grads[1].numpy()) < tol
    assert (dlw[..., c:] == SENTINEL).all() and (drw[..., c:] == SENTINEL).all(), 'wrote outside the gradient views'
    if warp:
        duw = t['duw'].cpu().numpy()
        assert rel_linf(duw[..., 0], grads[2].numpy()[..., 0]) < 1e-4
        assert (duw[..., 1:] == SENTINEL).all()


# --------------------------------------------------------------------------------------------------------- dispatch
def _cuda_kernels(fn, sessions=4):
    """Names of the CUDA kernels one call of fn launches (torch.profiler, CUDA activity); None if the profiler records none.

    A session can miss its first activities when the profiler has run before in the same process -- for a call that
    launches one kernel, all of it -- so fn runs twice with a torch kernel in between as a marker, and only what follows
    the marker counts (as in cuda_activities of tests/golden/make_engine_kernels.py; fn only rewrites its outputs).  Now
    and then a session records no CUDA activity at all; it is repeated before concluding that the profiler sees none."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(sessions):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
            torch.ones(1, device='cuda').add_(1)
            torch.cuda.synchronize()
            fn()
            torch.cuda.synchronize()
        ev = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA),
                    key=lambda e: e.time_range.start)
        names = [e.name for e in ev]
        marks = [i for i, n in enumerate(names) if 'ms::' not in n]
        if marks:
            return names[marks[-1] + 1:]
    return None


CORR_KERNELS = ('corr_fwd_kernel(', 'corr_fwd2_kernel<', 'corr_fwd3_kernel<', 'corr_fwd4_kernel<', 'corr_mma_kernel',
                'corr_bwd_kernel(', 'corr_mma_bwd_kernel')


@pytest.mark.parametrize('name', ['fwd:' + k for k in FWD_CASES] + ['bwd:' + k for k in BWD_CASES] + ['wide'])
def test_dispatch_reaches_named_kernel(lib, name):
    if name == 'wide':
        from madstereo import ops
        x = torch.randn(1, 2, 64, 64, device='cuda'); y = torch.randn(1, 2, 64, 64, device='cuda')
        want, fn = 'corr_mma_kernel', lambda: ops.correlation_wide(x, y, 40, act_scale=64.0)
    elif name.startswith('fwd:'):
        case = FWD_CASES[name[4:]]
        t = _fwd_setup(case, seed=1)
        want, fn = case[-1], lambda: _fwd_call(lib, case, t)
    else:
        case = BWD_CASES[name[4:]]
        t = _bwd_setup(case, seed=1)
        want, fn = case[-2], lambda: _bwd_call(lib, case, t)
    names = _cuda_kernels(fn)
    if names is None:
        pytest.skip('torch.profiler recorded no CUDA kernel events on this machine: the kernel choice cannot be observed')
    corr = [n for n in names if any(k in n for k in CORR_KERNELS)]
    assert len(corr) == 1 and want in corr[0], (want, corr)
