"""Every node of a real engine step against float64 of the inputs the engine gave it.

One step is run as production runs it (a replayed CUDA graph with its momentum or Adam update), then the engine's own
buffers are read back.  For every layer, Engine.layer_plan() names the views it read and wrote and the kernels planned
for it; each output is recomputed in float64 on the device from the engine's fp32 inputs with the oracle's ops
(oracle/tf1_ops.py), adjoints with torch.autograd.  No leaky-ReLU kink can flip between the two, because every mask is
taken from the engine's own post-activation tensor, so each kernel is held to the bound its per-op test uses and a
failure names the layer, the direction, the planned kernel and the (n, h, w, c) of the worst element.

What a step writes is checked to be written: before it, the parameter elements of the gradient arena and the valid
channels of every grad/* view are set to NaN.  Afterwards every gradient the train op owns must be finite and match,
and the arena entries of layers it does not train must still be NaN.

The momentum arena of the trained layers is seeded before each momentum step, so that the update moves every trained
weight tensor by a known fraction of its largest weight whatever the size of its gradient: the update check then
covers the momentum term too, and a module whose 16-bit weight tiles were not refreshed after its update fails the
forward check of the next step.
"""
import json
import os

import numpy as np
import pytest
import torch

from conftest import PKG

pytestmark = pytest.mark.gpu

D = torch.float64
TOL_FWD = 2e-5          # fp32 and fp16-plane forward kernels, correlation forward (relative L-inf per tensor)
TOL_GRAD = 1e-4         # input, weight and bias gradients
TOL_RESIZE_FWD = 1e-5
TOL_RESIZE_ADJ = 2e-5
TOL_LOSS = 5e-4
# scale of the engine's fp16 forward planes (ms_engine_create) and the range of max|x| * scale in which
# test_conv_bf_forward_activation_range holds conv_bf to TOL_FWD
ACT_SCALE = {'MADNet': 1.0 / 16, 'Dispnet': 64.0}
BF_RANGE = (6e-5 * 64, 6e4 / 8)
LR, MU = 1e-4, 0.9
MOVE = 5e-3             # the seeded momentum moves each trained weight tensor by up to MOVE x its max |w|
MIN_MOVE = 1e-3         # ... and the check requires at least MIN_MOVE

MINIMUM_PAIRS = {('fwd', k) for k in ('HEAD', 'ONE_CHANNEL', 'STEM', 'SMALL', 'BF', 'GEMM')} | \
                {('dgrad', k) for k in ('HEAD', 'BF', 'GEMM')} | {('wgrad', k) for k in ('BF', 'STEM', 'HEAD', 'FP32')}
PLANNED, CHECKED, WORST = {}, {}, {}    # configuration -> planned (direction, kind) pairs / pairs that passed / worst error


def f64(t):
    return t.detach().to(D).contiguous()


def slope(x, alpha):
    """leaky-ReLU derivative taken from the post-activation tensor x"""
    return torch.where(x > 0, torch.ones_like(x), torch.full_like(x, alpha))


def adjoint(fn, x, g):
    x = f64(x).requires_grad_(True)
    return torch.autograd.grad(fn(x), x, f64(g))[0]


def reprojection_loss(disp, left, right, ambiguous=None):
    """T.reprojection_loss of a disparity at the frames' size, in float64 from the warp coordinate x - d as the loss
    kernel forms it in fp32.  In fp64 that coordinate would pick the other neighbour wherever x - d lies within an fp32
    rounding of an integer (at x ~ 1000 the rounding is 6e-5), and d(loss)/dd, the difference of the two neighbours,
    jumps there.  ambiguous: a list that receives the [B,H,W,1] mask of pixels whose |warped - left| is within a few fp32
    roundings of zero, where the sign of the L1 term's derivative is the rounding's choice."""
    from oracle import tf1_ops as T
    right, left = right / 256.0, left / 256.0
    b, h, w, c = right.shape
    xs = torch.arange(w, dtype=D, device=right.device).view(1, 1, w, 1)
    cx32 = (xs.float() - disp.detach().float()).to(D)
    cx = cx32 + (disp.detach() - disp)            # the fp32 value, d cx / dd = -1
    x0 = torch.floor(cx32)
    i0 = torch.clamp(x0, 0, w - 1).long().expand(b, h, w, c)
    i1 = torch.clamp(x0 + 1, 0, w - 1).long().expand(b, h, w, c)
    warped = (x0 + 1 - cx) * torch.gather(right, 2, i0) + (cx - x0) * torch.gather(right, 2, i1)
    if ambiguous is not None:
        with torch.no_grad():
            gap = (warped - left).abs() <= 2.0 ** -21 * torch.maximum(warped.abs(), left.abs())
            ambiguous.append(gap.any(dim=3, keepdim=True))
    return T.mean_ssim_l1(warped, left)


def check_loss_grad(c, s, which):
    """grad/disp against the fp64 adjoint of the loss on disp<which>; pixels whose L1 sign is the rounding's choice are
    left out, and must be rare"""
    eng = c.eng
    left, right = f64(eng.tensor('raw_left')), f64(eng.tensor('raw_right'))
    amb = []
    ref = adjoint(lambda d: reprojection_loss(d, left, right, amb), eng.tensor('disp%d' % which),
                  torch.ones((), dtype=D, device=eng.device))
    got = torch.where(amb[0], ref, f64(eng.tensor('grad/disp')))
    n = int(amb[0].sum())
    if n > 1e-4 * amb[0].numel():
        s.fail('grad/disp: %d pixels with |warped - left| at fp32 rounding level' % n)
    s.check('grad/disp (%d pixels at an L1 kink left out)' % n, [('loss_grad', 'reprojection')], got, ref, TOL_LOSS)


def rel_err(got, ref):
    """relative L-inf of got vs ref, and the index of the worst element (the first non-finite one if any)"""
    got = got.detach().to(D)
    bad = ~torch.isfinite(got)
    if bool(bad.any()):
        return float('inf'), tuple(int(v) for v in bad.nonzero()[0])
    d = (got - ref.detach()).abs()
    i = int(d.argmax())
    den = float(ref.abs().max())
    err = float(d.max()) / den if den > 0 else float(d.max()) * 1e30
    return err, tuple(int(v) for v in np.unravel_index(i, tuple(d.shape)))


class Checks:
    """failures and worst errors of one configuration; keys are (direction, kernel kind) pairs"""

    def __init__(self, cfg):
        self.cfg, self.step, self.fails = cfg, '', []
        PLANNED.setdefault(cfg, set()); CHECKED.setdefault(cfg, set()); WORST.setdefault(cfg, {})

    def check(self, what, keys, got, ref, tol):
        assert tuple(got.shape) == tuple(ref.shape), (self.step, what, tuple(got.shape), tuple(ref.shape))
        err, at = rel_err(got, ref)
        for k in keys:
            WORST[self.cfg][k] = max(WORST[self.cfg].get(k, 0.0), err)
        if err < tol:
            CHECKED[self.cfg].update(keys)
        else:
            self.fails.append('%s: %s %s: rel L-inf %.3g > %.0e at %s %s of %s' % (
                self.step, what, ' + '.join('%s[%s]' % k for k in keys), err, tol,
                '(n,h,w,c)' if len(at) == 4 else 'index', at, tuple(got.shape)))

    def fail(self, msg):
        self.fails.append('%s: %s' % (self.step, msg))

    def done(self):
        assert not self.fails, '%d failures:\n' % len(self.fails) + '\n'.join(self.fails[:40])


# ---------------------------------------------------------------------------------------------------------------------
# engine set-up and one step
# ---------------------------------------------------------------------------------------------------------------------
class Ctx:
    pass


def make(net_name, H, W, B, radius_d=2, stride=1, warping=True, optimizer='momentum'):
    import Nets
    from madstereo.adaptation import OnlineAdaptation
    from madstereo.synthetic import make_pair
    left, right, _ = make_pair(H, W, seed=3, batch=B)
    lt, rt = torch.as_tensor(left).cuda(), torch.as_tensor(right).cuda()
    c = Ctx()
    c.net_name, c.radius_d, c.stride, c.warping = net_name, radius_d, stride, warping
    if net_name == 'MADNet':
        from oracle.madnet import init_params
        net = Nets.get_stereo_net('MADNet', dict(left_img=lt, right_img=rt, split_layers=[None], sequence=True,
                                                 train_portion='BEGIN', bulkhead=True, warping=warping, context_net=True,
                                                 radius_d=radius_d, stride=stride, is_training=False))
        cfg = json.load(open(os.path.join(PKG, 'block_config', 'MadNet_full.json')))
        c.ad = OnlineAdaptation(net, mode='MAD', train_config=cfg, lr=LR, sample_mode='FIXED', optimizer=optimizer,
                                ssim_th=1e9)
        c.ad.load_weights(init_params(seed=42, radius_d=radius_d, stride=stride))
    else:
        from oracle.dispnet import init_params
        net = Nets.get_stereo_net('Dispnet', dict(left_img=lt, right_img=rt, split_layers=[None], sequence=True,
                                                  train_portion='BEGIN', bulkhead=False, correlation=True))
        c.ad = OnlineAdaptation(net, mode='FULL', lr=LR, optimizer=optimizer, ssim_th=1e9)
        c.ad.load_weights(init_params(seed=7))
    eng = c.eng = net.engine
    eng.set_input(lt, rt)
    c.plan = [eng.layer_plan(l.index) for l in eng.layers]
    c.L = {l.name: l for l in eng.layers}
    c.grad_names = [n for n in eng.tensor_names() if n.startswith('grad/')]
    c.n_disp = 6 if net_name == 'MADNet' else 7
    c.Hp, c.Wp = eng.tensor('img').shape[1:3]
    return c


def planned_pairs(c):
    out = set()
    for P in c.plan:
        out |= {('fwd', P['fwd']), ('wgrad', P['wgrad'])}
        if P['dx'] is not None:
            out.add(('dgrad', P['dgrad']))
    return out


def param_ranges(c, idxs):
    eng = c.eng
    out = []
    for i in idxs:
        l = eng.layers[i]
        wo, bo = eng.param_offsets[i]
        out += [(wo, wo + l.kh * l.kw * l.cin * l.cout), (bo, bo + l.cout)]
    return out


def element_mask(c, idxs):
    m = torch.zeros(c.eng.n_params, dtype=torch.bool, device=c.eng.device)
    for a, b in param_ranges(c, idxs):
        m[a:b] = True
    return m


def run_step(c, s, mode, group, trained, seed_momentum):
    """one graph-replayed step with its update; returns the arenas before it"""
    from madstereo.engine import MODE_NONE
    eng = c.eng
    s.step = {0: 'NONE', 1: 'MAD %d' % group, 2: 'FULL'}[mode]
    if mode != MODE_NONE and seed_momentum:
        gen = torch.Generator(device=eng.device).manual_seed(1000 + 10 * mode + group)
        for i in trained:
            l = eng.layers[i]
            wo = eng.param_offsets[i][0]
            n = l.kh * l.kw * l.cin * l.cout
            amp = MOVE * float(eng.weights[wo:wo + n].abs().max()) / (LR * MU)
            eng.momentum[wo:wo + n] = (torch.rand(n, generator=gen, device=eng.device) * 2 - 1) * amp
    before = {'W': eng.weights.clone(), 'M': eng.momentum.clone()}
    if eng.optimizer == 'adam':
        before['V'], before['powers'] = eng.adam_v.clone(), eng.adam_powers.clone()
    if mode != MODE_NONE:
        for a, b in param_ranges(c, range(len(eng.layers))):
            eng.grads[a:b] = float('nan')
        for n in c.grad_names:
            eng.tensor(n).fill_(float('nan'))
    eng.run(mode, group, (1 << c.n_disp) - 1, mode != MODE_NONE, LR, MU)
    torch.cuda.synchronize()
    return before


# ---------------------------------------------------------------------------------------------------------------------
# every layer: forward, and the fp64 adjoints of its (x, dpre)
# ---------------------------------------------------------------------------------------------------------------------
def pre_activation(l, x, w, b):
    from oracle import tf1_ops as T
    if l.transposed:
        return T.conv2d_transpose(x, w, b, l.stride, None)
    return T.conv2d(x, w, b, stride=l.stride, dilation=l.dilation, alpha=None)


def layer_pass(c, s, W, dx_layers=(), trained=()):
    """checks every layer's forward from the weights W it ran with; returns {layer: fp64 adjoint wrt its input x} of the
    layers in dx_layers and checks the weight and bias gradients of the layers in `trained`"""
    from oracle import tf1_ops as T
    eng = c.eng
    views, gviews = eng.param_views(W), eng.param_views(eng.grads)
    dx = {}
    for l in eng.layers:
        P = c.plan[l.index]
        want_dx, train = l.index in dx_layers, l.index in trained
        x = f64(P['x']).requires_grad_(want_dx)
        kw, kb = l.scope + '/weights', l.scope + '/' + l.bias_name
        w, b = f64(views[kw]).requires_grad_(train), f64(views[kb]).requires_grad_(train)
        pre = pre_activation(l, x, w, b)
        with torch.no_grad():
            y = T.leaky(pre, l.alpha)
            if l.name == 'context7':                 # final_disp = V[2] + context7
                y = y + f64(eng.tensor('fgc-volume-filtering-2/disp6'))
            s.check(l.name, [('fwd', P['fwd'])], P['y'], y, TOL_FWD)
            if P['fwd'] == 'BF':
                r = float(x.abs().max()) * ACT_SCALE[c.net_name]
                if not BF_RANGE[0] < r < BF_RANGE[1]:
                    s.fail('%s: max|x| * act_scale = %.3g outside the fp16 plane range %s' % (l.name, r, BF_RANGE))
        if want_dx or train:
            ins = ([x] if want_dx else []) + ([w, b] if train else [])
            g = torch.autograd.grad(pre, ins, f64(P['dpre']))
            if want_dx:
                dx[l.index] = g[0]
            if train:
                s.check(l.name + ' weights', [('wgrad', P['wgrad'])], gviews[kw], g[-2], TOL_GRAD)
                s.check(l.name + ' bias', [('wgrad', P['wgrad'])], gviews[kb], g[-1], TOL_GRAD)
        del pre
    return dx


# ---------------------------------------------------------------------------------------------------------------------
# MADNet
# ---------------------------------------------------------------------------------------------------------------------
def _mad(c):
    from oracle.madnet import PYRAMID_CH, num_displacements
    return PYRAMID_CH, num_displacements(c.radius_d, c.stride)


def madnet_disp_fns(c, i):
    from oracle import tf1_ops as T
    H, W, Hp, Wp = c.eng.H, c.eng.W, c.Hp, c.Wp
    if i < 5:
        return lambda v: T.crop_or_pad(T.resize_bilinear(torch.relu(v * -20.0), Hp, Wp), H, W)
    return lambda v: T.crop_or_pad(torch.relu(T.resize_bilinear(v, Hp, Wp) * -20.0), H, W)


def madnet_head(i):
    return 'fgc-volume-filtering-%d/disp6' % (6 - i) if i < 4 else 'final_disp'


def madnet_forward_extra(c, s):
    """correlation levels (left copy, u channel, correlation of the warped right features), ctxin's copy, the heads"""
    from oracle import tf1_ops as T
    eng = c.eng
    PYR, nd = _mad(c)
    t = lambda n: f64(eng.tensor(n))
    with torch.no_grad():
        for k in (6, 5, 4, 3, 2):
            C = PYR[2 * k]
            cost = eng.tensor('cost%d' % k)
            lf, rf = t('left/conv%d' % (2 * k)), t('right/conv%d' % (2 * k))
            s.check('cost%d left copy' % k, [('fwd', 'corr')], cost[..., :C], lf, TOL_FWD)
            u = None
            if k < 6:
                h, w = cost.shape[1:3]
                uref = T.resize_bilinear(t('fgc-volume-filtering-%d/disp6' % (k + 1)), h, w) * (20.0 / 2 ** k)
                s.check('cost%d u' % k, [('fwd', 'resize')], cost[..., C + nd:C + nd + 1], uref, TOL_RESIZE_FWD)
                u = f64(cost[..., C + nd:C + nd + 1])
            r = T.linear_warp(rf, u) if (u is not None and c.warping) else rf
            s.check('corr%d' % k, [('fwd', 'corr')], cost[..., C:C + nd], T.correlation(lf, r, c.radius_d, c.stride), TOL_FWD)
        s.check('ctxin left copy', [('fwd', 'corr')], eng.tensor('ctxin')[..., :PYR[4]], t('left/conv4'), TOL_FWD)
        for i in range(6):
            s.check('disp%d' % i, [('fwd', 'resize')], eng.tensor('disp%d' % i), madnet_disp_fns(c, i)(t(madnet_head(i))),
                    TOL_RESIZE_FWD)


def madnet_schedule(c, mode, group):
    """(layers whose input gradient the step computes, layers it trains, pyramid levels lo..top of its gradients),
    as the reference graph's train op differentiates (oracle/madnet.py, Stereo_Online_Adaptation.py:87-128)"""
    from madstereo.engine import MODE_FULL
    L = c.L
    if mode == MODE_FULL:
        return {i for i, P in enumerate(c.plan) if P['dx'] is not None}, set(range(len(c.plan))), 1, 12
    trained = set(c.ad.groups[group])
    k = 6 - group
    top = 2 * k
    lo = min([i for i in range(1, 13) if L['left/conv%d' % i].index in trained] + [13])
    assert lo <= top, 'module %d trains no pyramid level below its features: its correlation gradient is not computed' % group
    dx = {L['fgc-volume-filtering-%d/disp%d' % (k, j)].index for j in range(1, 7)}
    dx |= {L['left/conv%d' % i].index for i in range(lo + 1, top + 1)}
    if group == 4:
        dx |= {L['context%d' % j].index for j in range(1, 8)}
    return dx, trained, lo, top


def madnet_corr_adjoint(c, k, want_du):
    """fp64 adjoint of [left copy | correlation(left, warp(right, u))] of level k from the engine's grad/cost<k>"""
    from oracle import tf1_ops as T
    eng = c.eng
    PYR, nd = _mad(c)
    C = PYR[2 * k]
    g = f64(eng.tensor('grad/cost%d' % k))
    lf = f64(eng.tensor('left/conv%d' % (2 * k))).requires_grad_(True)
    rf = f64(eng.tensor('right/conv%d' % (2 * k))).requires_grad_(True)
    u = None
    ins = [lf, rf]
    if k < 6 and c.warping:
        u = f64(eng.tensor('cost%d' % k)[..., C + nd:C + nd + 1]).requires_grad_(want_du)
        if want_du:
            ins.append(u)
    corr = T.correlation(lf, T.linear_warp(rf, u) if u is not None else rf, c.radius_d, c.stride)
    gs = torch.autograd.grad(corr, ins, g[..., C:C + nd])
    return gs[0] + g[..., :C], gs[1], (gs[2] if len(gs) > 2 else None)


def madnet_backward_checks(c, s, mode, group, dx, lo, top):
    from madstereo.engine import MODE_FULL
    from oracle import tf1_ops as T
    from oracle.madnet import ALPHA
    eng = c.eng
    P, L, B = c.plan, c.L, eng.B
    PYR, nd = _mad(c)
    t = lambda n: f64(eng.tensor(n))
    full = mode == MODE_FULL
    levels = (2, 3, 4, 5, 6) if full else (6 - group,)
    ctx_ran = full or group == 4
    corr = {k: madnet_corr_adjoint(c, k, full) for k in levels}
    # loss gradient and the disparity head's resize adjoint
    which = 5 if full else group
    check_loss_grad(c, s, which)
    head = madnet_head(which)
    s.check('grad/' + head, [('resize_bwd', 'resize')], eng.tensor('grad/' + head),
            adjoint(madnet_disp_fns(c, which), eng.tensor(head), eng.tensor('grad/disp')), TOL_RESIZE_ADJ)
    with torch.no_grad():
        if ctx_ran:      # V[2] feeds both the context net's input and its residual
            s.check('grad/fgc-volume-filtering-2/disp6', [('ctx_tail', 'add')], eng.tensor('grad/fgc-volume-filtering-2/disp6'),
                    t('grad/final_disp') + t('grad/ctxin')[..., PYR[4]:PYR[4] + 1], TOL_GRAD)
            for j in range(1, 8):
                li = L['context%d' % j].index
                ref = dx[li] if j == 1 else dx[li] * slope(f64(P[li]['x']), ALPHA)
                s.check('context%d' % j, [('dgrad', P[li]['dgrad'])], P[li]['dx'], ref, TOL_GRAD)
        for k in levels:
            for j in range(1, 7):
                li = L['fgc-volume-filtering-%d/disp%d' % (k, j)].index
                ref = dx[li] if j == 1 else dx[li] * slope(f64(P[li]['x']), ALPHA)
                s.check('fgc-volume-filtering-%d/disp%d' % (k, j), [('dgrad', P[li]['dgrad'])], P[li]['dx'], ref, TOL_GRAD)
        if full:         # u_k: warp-coordinate adjoint + the estimator-input slice, then the resize adjoint into V[k+1]
            for k in (2, 3, 4, 5):
                C = PYR[2 * k]
                ref = t('grad/cost%d' % k)[..., C + nd:C + nd + 1]
                if c.warping:
                    ref = ref + corr[k][2]
                s.check('grad/u%d' % k, [('corr_bwd', 'corr')], eng.tensor('grad/u%d' % k), ref, TOL_GRAD)
        # pyramid: d(pre-activation) of conv j = slope(pyr_j) x (conv j+1's input gradient + correlation adjoint +
        # left-feature slices of the cost volume and of the context input)
        for j in range(lo, top + 1):
            pre = P[j - 1]
            acc = torch.zeros_like(f64(pre['y']))
            if j < top:
                li = L['left/conv%d' % (j + 1)].index
                acc += dx[li]
                what, keys = 'left/conv%d' % (j + 1), [('dgrad', P[li]['dgrad'])]
            else:
                what, keys = 'correlation adjoint into left/conv%d' % j, []
            if j % 2 == 0 and j // 2 in corr:
                gl, gr, _ = corr[j // 2]
                acc[:B] += gl
                acc[B:] += gr
                keys = keys + [('corr_bwd', 'corr')]
            if j == 4 and ctx_ran:
                acc[:B] += t('grad/ctxin')[..., :PYR[4]]
            s.check(what, keys, pre['dpre'], acc * slope(f64(pre['y']), ALPHA), TOL_GRAD)
    if full:
        for k in (3, 4, 5, 6):
            h, w = eng.tensor('cost%d' % (k - 1)).shape[1:3]
            ref = adjoint(lambda v: T.resize_bilinear(v, h, w) * (20.0 / 2 ** (k - 1)),
                          eng.tensor('fgc-volume-filtering-%d/disp6' % k), eng.tensor('grad/u%d' % (k - 1)))
            s.check('grad/fgc-volume-filtering-%d/disp6' % k, [('resize_bwd', 'resize')],
                    eng.tensor('grad/fgc-volume-filtering-%d/disp6' % k), ref, TOL_RESIZE_ADJ)


# ---------------------------------------------------------------------------------------------------------------------
# DispNet
# ---------------------------------------------------------------------------------------------------------------------
def dispnet_disp_fn(c, i, op_w):
    from oracle import tf1_ops as T
    H, W, Hp, Wp = c.eng.H, c.eng.W, c.Hp, c.Wp
    if i < 6:
        return lambda v: T.crop_or_pad(T.resize_bilinear(torch.relu(v * (Wp / op_w)), Hp, Wp), H, W)
    return lambda v: T.crop_or_pad(T.resize_bilinear(v, Hp, Wp) * 2, H, W)


def dispnet_heads(c):
    from oracle.dispnet import UPS
    return [u[0] + '/predict' for u in UPS] + ['prediction', 'prediction']


def dispnet_forward_extra(c, s):
    from oracle import tf1_ops as T
    from oracle.dispnet import MAX_DISP, UPS
    eng = c.eng
    P, L, B = c.plan, c.L, eng.B
    with torch.no_grad():
        c2 = f64(P[L['conv2a'].index]['y'])
        s.check('corr', [('fwd', 'corr')], eng.tensor('corr'), T.correlation(c2[:B], c2[B:], MAX_DISP), TOL_FWD)
        srcs = {'conv2a': c2[:B], 'conv1a': f64(P[L['conv1a'].index]['y'])[:B]}
        for name, _, skip, _, _, sc in UPS:
            src = srcs[skip] if skip in srcs else f64(P[L[skip].index]['y'])
            s.check(name + '/cat skip copy', [('fwd', 'copy')], eng.tensor(name + '/cat')[..., :sc], src, TOL_FWD)
        for i, h in enumerate(dispnet_heads(c)):
            v = eng.tensor(h)
            s.check('disp%d' % i, [('fwd', 'resize')], eng.tensor('disp%d' % i), dispnet_disp_fn(c, i, v.shape[2])(f64(v)),
                    TOL_RESIZE_FWD)


def dispnet_backward_checks(c, s, dx):
    from oracle import tf1_ops as T
    from oracle.dispnet import ALPHA, MAX_DISP, UPS
    eng = c.eng
    P, L, B = c.plan, c.L, eng.B
    nd = 2 * MAX_DISP + 1
    t = lambda n: f64(eng.tensor(n))
    check_loss_grad(c, s, 6)
    pred = eng.tensor('prediction')
    s.check('grad/prediction', [('resize_bwd', 'resize')], eng.tensor('grad/prediction'),
            adjoint(dispnet_disp_fn(c, 6, pred.shape[2]), pred, eng.tensor('grad/disp')), TOL_RESIZE_ADJ)
    c2 = f64(P[L['conv2a'].index]['y'])
    ca, cb = c2[:B].clone().requires_grad_(True), c2[B:].clone().requires_grad_(True)
    g_corr = torch.autograd.grad(T.correlation(ca, cb, MAX_DISP), [ca, cb], t('grad/cat3')[..., :nd])
    with torch.no_grad():
        li = L['prediction'].index
        s.check('prediction', [('dgrad', P[li]['dgrad'])], P[li]['dx'], dx[li], TOL_GRAD)
        for u, (name, _, _, _, cout, sc) in enumerate(UPS):
            cat = L[name + '/concat'].index
            xin = f64(P[cat]['x'])
            mask = torch.ones_like(xin)            # the deconv slice's leaky-ReLU is applied in place
            mask[..., sc:sc + cout] = slope(xin[..., sc:sc + cout], ALPHA)
            s.check(name + '/concat', [('dgrad', P[cat]['dgrad'])], P[cat]['dx'], dx[cat] * mask, TOL_GRAD)
            up = L[name + '/up_predict'].index
            s.check(name + '/up_predict', [('dgrad', P[up]['dgrad'])], P[up]['dx'], dx[up], TOL_GRAD)
            pr, de = L[name + '/predict'].index, L[name + '/deconv'].index
            ref = dx[pr] + dx[de]                  # both read the block's bottom
            if u == 0:
                ref = ref * slope(f64(P[pr]['x']), ALPHA)
            s.check(name + '/predict + deconv', [('dgrad', P[pr]['dgrad']), ('dgrad', P[de]['dgrad'])], P[pr]['dx'], ref,
                    TOL_GRAD)
        # encoder: skip slices of the decoder's concatenations seed conv5/1, conv4/1 and conv3/1
        skip_of = {UPS[u][2]: (UPS[u][0], UPS[u][5]) for u in range(3)}
        for name in ('conv6/1', 'conv6', 'conv5/1', 'conv5', 'conv4/1', 'conv4', 'conv3/1'):
            li = L[name].index
            below = eng.layers[li - 1].name
            ref = dx[li].clone()
            if below in skip_of:
                up, sc = skip_of[below]
                ref += t('grad/%s/cat' % up)[..., :sc]
            s.check(name, [('dgrad', P[li]['dgrad'])], P[li]['dx'], ref * slope(f64(P[li]['x']), ALPHA), TOL_GRAD)
        li = L['conv3'].index
        xin = f64(P[li]['x'])
        mask = torch.ones_like(xin)                # [corr | conv_redir]: only conv_redir is leaky
        mask[..., nd:] = slope(xin[..., nd:], ALPHA)
        s.check('conv3', [('dgrad', P[li]['dgrad'])], P[li]['dx'], dx[li] * mask, TOL_GRAD)
        # conv2's output: conv_redir's input gradient, the correlation adjoint and the up2 skip slice (left), correlation (right)
        li = L['conv_redir'].index
        ref = torch.zeros_like(c2)
        ref[:B] = dx[li] + g_corr[0] + t('grad/up2/cat')[..., :UPS[3][5]]
        ref[B:] = g_corr[1]
        s.check('conv_redir', [('dgrad', P[li]['dgrad']), ('corr_bwd', 'corr')], eng.tensor('grad/conv2'),
                ref * slope(c2, ALPHA), TOL_GRAD)
        li = L['conv2a'].index
        c1 = f64(P[li]['x'])
        ref = dx[li].clone()
        ref[:B] += t('grad/up1/cat')[..., :UPS[4][5]]
        s.check('conv2a', [('dgrad', P[li]['dgrad'])], eng.tensor('grad/conv1'), ref * slope(c1, ALPHA), TOL_GRAD)


# ---------------------------------------------------------------------------------------------------------------------
# updates
# ---------------------------------------------------------------------------------------------------------------------
def check_update(c, s, before, trained, lr=LR, mu=MU):
    eng = c.eng
    tm = element_mask(c, trained)
    rest = element_mask(c, set(range(len(eng.layers))) - set(trained))
    W0, M0, W1, M1, G = before['W'], before['M'], eng.weights, eng.momentum, eng.grads
    if not bool(torch.isfinite(G[tm]).all()):
        s.fail('non-finite gradient in the trained range')
    if bool(rest.any()) and not bool(torch.isnan(G[rest]).all()):
        s.fail('the gradient arena of untrained layers was written')
    if not (torch.equal(W1[~tm], W0[~tm]) and torch.equal(M1[~tm], M0[~tm])):
        s.fail('weights or optimizer state outside the trained range changed')
    w0, g = W0[tm].to(D), G[tm].to(D)
    if eng.optimizer == 'adam':
        from adam_oracle import adam_reference, advance_powers
        p0 = before['powers'].cpu().numpy()
        wr, mr, vr = adam_reference(w0.cpu().numpy(), g.cpu().numpy(), M0[tm].to(D).cpu().numpy(),
                                    before['V'][tm].to(D).cpu().numpy(), p0, lr)
        w1 = W1[tm].cpu().numpy().astype(np.float64)
        bw = np.spacing(np.abs(W1[tm].cpu().numpy())).astype(np.float64) + 1e-5 * lr
        if not (np.abs(w1 - wr) <= bw).all():
            s.fail('Adam update: w off by %g (bound %g)' % ((np.abs(w1 - wr) - bw).max(), bw[np.argmax(np.abs(w1 - wr) - bw)]))
        v0 = before['V'][tm].to(D).cpu().numpy()
        m0 = M0[tm].to(D).cpu().numpy()
        g64 = g.cpu().numpy()
        for got, ref, scale, nm in ((eng.momentum[tm], mr, np.abs(m0) + np.abs(g64), 'm'),
                                    (eng.adam_v[tm], vr, v0 + g64 * g64, 'v')):
            d = np.abs(got.to(D).cpu().numpy() - ref)
            if not (d <= 1e-6 * scale + 1e-30).all():
                s.fail('Adam update: %s off by %g relative' % (nm, (d / np.maximum(scale, 1e-30)).max()))
        if tuple(eng.adam_powers.cpu().numpy()) != tuple(advance_powers(p0)):
            s.fail('Adam powers not advanced once')
        return
    lr32, mu32 = float(np.float32(lr)), float(np.float32(mu))
    m0 = M0[tm].to(D)
    m_ref = mu32 * m0 + g
    w_ref = w0 - lr32 * m_ref
    tol_m = 2.0 ** -22 * (mu32 * m0.abs() + g.abs()) + 1e-40
    tol_w = 2.0 ** -22 * (w0.abs() + lr32 * m_ref.abs()) + lr32 * tol_m + 1e-40
    for nm, got, ref, tol in (('momentum', M1[tm].to(D), m_ref, tol_m), ('weights', W1[tm].to(D), w_ref, tol_w)):
        over = (got - ref).abs() - tol
        if not bool((over <= 0).all()):
            i = int(over.argmax())
            s.fail('momentum update: %s off by %g at arena element %d (bound %g)' % (nm, float((got - ref).abs()[i]), i,
                                                                                     float(tol[i])))


def check_moved(c, s, before, trained):
    eng = c.eng
    for i in trained:
        l = eng.layers[i]
        wo = eng.param_offsets[i][0]
        n = l.kh * l.kw * l.cin * l.cout
        w0 = before['W'][wo:wo + n]
        moved = float((eng.weights[wo:wo + n] - w0).abs().max()) / float(w0.abs().max())
        if not moved > MIN_MOVE:
            s.fail('%s moved by %.2g of its max |w| (the tile check needs > %g)' % (l.name, moved, MIN_MOVE))


# ---------------------------------------------------------------------------------------------------------------------
# steps
# ---------------------------------------------------------------------------------------------------------------------
def checked_step(c, s, mode, group=0, seed_momentum=True):
    from madstereo.engine import MODE_NONE
    if mode == MODE_NONE:
        run_step(c, s, mode, group, (), False)
        layer_pass(c, s, c.eng.weights)
        (madnet_forward_extra if c.net_name == 'MADNet' else dispnet_forward_extra)(c, s)
        return
    if c.net_name == 'MADNet':
        dx_layers, trained, lo, top = madnet_schedule(c, mode, group)
    else:
        dx_layers, trained = {i for i, P in enumerate(c.plan) if P['dx'] is not None}, set(range(len(c.plan)))
    trained = sorted(trained)
    before = run_step(c, s, mode, group, trained, seed_momentum and c.eng.optimizer == 'momentum')
    dx = layer_pass(c, s, before['W'], dx_layers, trained)
    if c.net_name == 'MADNet':
        madnet_forward_extra(c, s)
        madnet_backward_checks(c, s, mode, group, dx, lo, top)
    else:
        dispnet_forward_extra(c, s)
        dispnet_backward_checks(c, s, dx)
    check_update(c, s, before, trained)
    if seed_momentum and c.eng.optimizer == 'momentum':
        check_moved(c, s, before, trained)
    del dx
    torch.cuda.empty_cache()


def report(cfg):
    print('\n%s: worst relative L-inf per (direction, kernel)' % cfg)
    for k in sorted(WORST[cfg]):
        print('  %-12s %-12s %.2e' % (k[0], k[1], WORST[cfg][k]))


def test_madnet_bench_size_every_module_two_rounds():
    """384x1280, batch 1 (the benchmark's configuration): FULL, then MAD 0..4; then a second forward, whose checks fail
    for a module whose weight tiles were not refreshed after its update"""
    from madstereo.engine import MODE_FULL, MODE_MAD, MODE_NONE
    cfg = 'MADNet 384x1280 B1'
    c = make('MADNet', 384, 1280, 1)
    PLANNED[cfg] = planned_pairs(c)
    s = Checks(cfg)
    checked_step(c, s, MODE_FULL)
    for g in range(5):
        checked_step(c, s, MODE_MAD, g)
    s.step = 'round 2'
    checked_step(c, s, MODE_NONE)
    report(cfg)
    s.done()


def test_madnet_kitti_size_batch2():
    """375x1242 (the KITTI frame size, reflect-padded to 384x1280), two distinct frames: FULL and MAD 4"""
    from madstereo.engine import MODE_FULL, MODE_MAD
    cfg = 'MADNet 375x1242 B2'
    c = make('MADNet', 375, 1242, 2)
    PLANNED[cfg] = planned_pairs(c)
    s = Checks(cfg)
    checked_step(c, s, MODE_FULL)
    checked_step(c, s, MODE_MAD, 4)
    report(cfg)
    s.done()


def test_madnet_radius4_stride2_no_warping():
    from madstereo.engine import MODE_FULL
    cfg = 'MADNet 384x640 radius_d=4 stride=2 warping=False'
    c = make('MADNet', 384, 640, 1, radius_d=4, stride=2, warping=False)
    PLANNED[cfg] = planned_pairs(c)
    s = Checks(cfg)
    checked_step(c, s, MODE_FULL)
    report(cfg)
    s.done()


def test_madnet_small_frame_gemm_forward():
    """128x320: the 1/64 maps (2x5 pixels) are below conv_bf's 32-pixel minimum, so conv11, conv12 and the level-6
    estimator run their forward on the CUDA-core gather GEMM, which no frame of 384x640 or more plans"""
    from madstereo.engine import MODE_FULL
    cfg = 'MADNet 128x320 B1'
    c = make('MADNet', 128, 320, 1)
    PLANNED[cfg] = planned_pairs(c)
    assert ('fwd', 'GEMM') in PLANNED[cfg]
    s = Checks(cfg)
    checked_step(c, s, MODE_FULL)
    report(cfg)
    s.done()


def test_dispnet_bench_size():
    from madstereo.engine import MODE_FULL
    cfg = 'DispNet 384x1280 B1'
    c = make('Dispnet', 384, 1280, 1)
    PLANNED[cfg] = planned_pairs(c)
    s = Checks(cfg)
    checked_step(c, s, MODE_FULL)
    report(cfg)
    s.done()


def test_madnet_adam_updates():
    """Adam (the live demo's optimizer): one MAD module, then FULL, each checked against the float64 ApplyAdam"""
    from madstereo.engine import MODE_FULL, MODE_MAD
    c = make('MADNet', 384, 640, 1, optimizer='adam')
    s = Checks('MADNet 384x640 Adam')
    for mode, g in ((MODE_MAD, 2), (MODE_FULL, 0)):
        dx_layers, trained, _, _ = madnet_schedule(c, mode, g)
        before = run_step(c, s, mode, g, trained, False)
        check_update(c, s, before, sorted(trained))
    s.done()


def test_every_planned_kernel_was_checked():
    """The configurations above together check every (direction, kernel) pair their plans use, and these include every
    kernel kind of the engine's plan."""
    cfgs = ('MADNet 384x1280 B1', 'MADNet 375x1242 B2', 'MADNet 384x640 radius_d=4 stride=2 warping=False',
            'MADNet 128x320 B1', 'DispNet 384x1280 B1')
    if not all(k in PLANNED for k in cfgs):
        pytest.skip('needs the configuration tests of this file to have run in this session')
    planned = set().union(*(PLANNED[k] for k in cfgs))
    checked = set().union(*(CHECKED[k] for k in cfgs))
    assert MINIMUM_PAIRS <= planned, 'never planned: %s' % sorted(MINIMUM_PAIRS - planned)
    assert planned <= checked, 'planned but not checked within bounds: %s' % sorted(planned - checked)
