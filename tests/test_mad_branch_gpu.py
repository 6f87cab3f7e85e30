"""A MAD step's train op runs on a branch of the captured step graph, beside the rest of the forward (Engine::mad_branch).
The same kernels run with the same arguments, so a graph-replayed step must equal an eager step (engine.profile(1): one
stream, launch order) bit for bit: both losses, all six disparities, the weights, the optimizer state and the gradients --
for every module, over consecutive replays, with momentum and Adam, with the proxy loss, without the in-graph update, and
with two modules per frame."""
import gc
import json
import os

import numpy as np
import pytest
import torch

from conftest import PKG

pytestmark = pytest.mark.gpu
LR = 1e-4


class _Seq(object):
    """Module sampler that replays a fixed sequence of block lists."""

    def __init__(self, seq):
        self.seq, self.i = list(seq), 0

    def sample(self, dist):
        b = self.seq[self.i % len(self.seq)]
        self.i += 1
        return list(b)


def _adapter(h, w, batch, seq, eager, **kw):
    import Nets
    from madstereo.adaptation import OnlineAdaptation
    from oracle.madnet import init_params
    lt = torch.zeros(batch, h, w, 3, device='cuda'); rt = torch.zeros(batch, h, w, 3, device='cuda')
    net = Nets.get_stereo_net('MADNet', dict(left_img=lt, right_img=rt, split_layers=[None], sequence=True,
                                             train_portion='BEGIN', bulkhead=True))
    cfg = json.load(open(os.path.join(PKG, 'block_config', 'MadNet_full.json')))
    ad = OnlineAdaptation(net, mode='MAD', train_config=cfg, lr=LR, sample_mode='FIXED', fixed_id=0, **kw)
    ad.load_weights(init_params(seed=42))
    ad.sampler = _Seq(seq)
    ad.ssim_th = float('inf')         # no weight restore: both sides must adapt through every step
    if eager:
        ad.engine.profile(1)
    return net, ad


def _state(net, ad):
    eng = ad.engine
    s = {'disp%d' % i: d.numpy() for i, d in enumerate(net.get_disparities())}
    s.update(weights=eng.weights, grads=eng.grads, momentum=eng.momentum)
    if ad.optimizer == 'adam':
        s.update(adam_v=eng.adam_v, adam_powers=eng.adam_powers)
    return {k: (v.detach().cpu().numpy() if torch.is_tensor(v) else np.asarray(v)).astype(np.float32) for k, v in s.items()}


def _assert_same(a, b, what):
    assert a.keys() == b.keys()
    for k in a:
        assert a[k].shape == b[k].shape and np.array_equal(a[k].view(np.uint32), b[k].view(np.uint32)), '%s: %s differs' % (what, k)


def _release():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _run_pair(h, w, batch, seq, **kw):
    from madstereo.synthetic import make_pair
    sides = [_adapter(h, w, batch, seq, eager, **kw) for eager in (True, False)]
    for k in range(len(seq)):
        left, right, disp = make_pair(h, w, seed=20 + k, batch=batch)
        extra = {'proxy': torch.tensor(disp, dtype=torch.float32).reshape(batch, h, w, 1).cuda()} if kw.get('loss') == 'proxy' else {}
        outs, states = [], []
        for net, ad in sides:
            outs.append(ad.step(torch.tensor(left).cuda(), torch.tensor(right).cuda(), want_disp_mask=0b111111, **extra))
            torch.cuda.synchronize()
            states.append(_state(net, ad))
        what = 'step %d, modules %s' % (k, outs[0]['blocks'])
        assert outs[0]['blocks'] == outs[1]['blocks'] == list(seq[k])
        for key in ('loss', 'train_loss'):
            assert np.float32(outs[0][key]).view(np.uint32) == np.float32(outs[1][key]).view(np.uint32), '%s: %s differs' % (what, key)
        _assert_same(states[0], states[1], what)
    del sides
    _release()


# every module, three consecutive replays of its graph
SEQ = [(g,) for g in range(5) for _ in range(3)]


@pytest.mark.parametrize('h,w,batch', [(384, 1280, 1), (64, 128, 2)])
@pytest.mark.parametrize('optimizer', ['momentum', 'adam'])
def test_graph_step_equals_eager_step(h, w, batch, optimizer):
    _run_pair(h, w, batch, SEQ, optimizer=optimizer)


def test_graph_step_equals_eager_step_proxy_loss():
    _run_pair(64, 128, 2, SEQ, loss='proxy')


def test_graph_step_equals_eager_step_two_modules_per_frame():
    # the first module's train op runs in the step graph, the second eagerly after it (OnlineAdaptation.step)
    _run_pair(64, 128, 2, [(0, 3), (4, 1), (2, 4), (3, 0), (1, 2)] * 2, num_blocks=2)


@pytest.mark.parametrize('h,w,batch', [(384, 1280, 1), (64, 128, 2)])
def test_graph_step_without_update_equals_eager_step(h, w, batch):
    """with_update=0: the branch joins after the backward; gradients and losses as eager, weights untouched."""
    from madstereo.engine import MODE_MAD
    from madstereo.synthetic import make_pair
    sides = [_adapter(h, w, batch, SEQ, eager) for eager in (True, False)]
    w0 = sides[0][1].engine.weights.detach().cpu().numpy()
    for k, (g,) in enumerate(SEQ):
        left, right, _ = make_pair(h, w, seed=40 + k, batch=batch)
        states, scalars = [], []
        for net, ad in sides:
            eng = ad.engine
            eng.set_input(torch.tensor(left).cuda(), torch.tensor(right).cuda())
            eng.run(MODE_MAD, g, 0b111111, 0, LR, 0.9, 1.0)
            scalars.append(np.asarray(eng.read_scalars()[:2], np.float32))
            states.append(_state(net, ad))
        what = 'step %d, module %d' % (k, g)
        assert np.array_equal(scalars[0].view(np.uint32), scalars[1].view(np.uint32)), what
        _assert_same(states[0], states[1], what)
        assert np.array_equal(states[1]['weights'], w0), what
    del sides
    _release()
