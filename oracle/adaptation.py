"""CPU oracle — online-adaptation step restated from Stereo_Online_Adaptation.py (TEST INFRASTRUCTURE).

Follows /root/reference/Stereo_Online_Adaptation.py:25-27 (softmax), :68-70 (full-res loss),
:85-128 (Momentum optimizer, MAD per-module train ops, FULL train op), :166-224 (sampling + reward
recurrence) and /root/reference/Sampler/sampler_factory.py:23-90.  Gradients = torch autograd.
"""
import numpy as np
import torch

from . import tf1_ops as T
from .madnet import MadNetOracle, mad_groups_full


def softmax(x):
    """Stereo_Online_Adaptation.py:25-27."""
    return np.exp(x) / np.sum(np.exp(x), axis=0)


class OracleAdapter:
    """One tf.train.MomentumOptimizer(lr, 0.9) shared by all train ops (one slot per variable)."""

    def __init__(self, params, mode='MAD', lr=1e-4, mu=0.9, dtype=torch.float32, groups=None, loss='reprojection',
                 radius_d=2, stride=1, warping=True, kink_signs=None):
        self.loss_kind = loss          # 'proxy': Stereo_Continual_Adaptation.py:75,112,133 (weights 0.01 / 0.1)
        assert mode in ('NONE', 'MAD', 'FULL')
        self.mode, self.lr, self.mu = mode, lr, mu
        self.net = MadNetOracle(params, dtype=dtype, radius_d=radius_d, stride=stride, warping=warping,
                                bulkhead=(mode == 'MAD'), kink_signs=kink_signs)
        self.groups = groups if groups is not None else mad_groups_full()
        self.momentum = {k: torch.zeros_like(v) for k, v in self.net.p.items()}

    def step(self, left, right, module=None, proxy=None):
        """One sess.run: forward, full-res loss, optional train op. Returns dict of numpy results."""
        net = self.net
        if self.mode == 'NONE':
            names = []
        elif self.mode == 'FULL':
            names = list(net.p.keys())
        else:
            names = self.groups[module]
        net.requires_grad_(set(names))
        left_t = torch.as_tensor(left).to(net.dtype)
        right_t = torch.as_tensor(right).to(net.dtype)
        with torch.set_grad_enabled(bool(names)):
            disps, layers = net.forward(left_t, right_t)
            if self.loss_kind == 'proxy':
                px = torch.as_tensor(proxy).to(net.dtype)
                full_loss = T.proxy_loss(disps[-1], px, 0.01)
                loss = T.proxy_loss(disps[module], px, 0.1) if self.mode == 'MAD' else full_loss
            else:
                full_loss = T.reprojection_loss(disps[-1], left_t, right_t)
                if self.mode == 'MAD':
                    loss = T.reprojection_loss(disps[module], left_t, right_t)
                else:
                    loss = full_loss
        out = {'full_loss': float(full_loss.detach()), 'train_loss': float(loss.detach()),
               'disparities': [d.detach().numpy() for d in disps]}
        grads = {}
        if names:
            gl = torch.autograd.grad(loss, [net.p[n] for n in names], allow_unused=True)
            with torch.no_grad():
                for n, g in zip(names, gl):
                    if g is None:
                        continue
                    grads[n] = g.numpy().copy()
                    w, m = T.momentum_update(net.p[n], g, self.momentum[n], self.lr, self.mu)
                    net.p[n].copy_(w)
                    self.momentum[n] = m
        out['grads'] = grads
        net.requires_grad_(set())
        return out


# ---- samplers (Sampler/sampler_factory.py:23-90) -------------------------------------------
class SequentialSampler:
    def __init__(self, k):
        self.k, self.c = k, 0

    def sample(self, dist):
        n = dist.shape[0]
        r = [(self.c % n + i) % n for i in range(self.k)]
        self.c += 1
        return r


def sample(name, k, dist, fixed_id=0, state=None):
    if name == 'FIXED':
        return [fixed_id]
    if name == 'RANDOM':
        return np.random.choice(range(dist.shape[0]), size=k, replace=False)
    if name == 'ARGMAX':
        return np.argpartition(np.squeeze(dist), -k)[-k:]
    if name == 'PROBABILITY':
        return np.random.choice(range(dist.shape[0]), size=k, replace=False, p=np.squeeze(dist))
    raise AssertionError(name)


class RewardTracker:
    """Stereo_Online_Adaptation.py:166-173, :211-224."""

    def __init__(self, n):
        self.h = np.zeros(n)
        self.l1 = self.l2 = 0.0
        self.last = []
        self.step = 0

    def update(self, new_loss, blocks):
        if self.step == 0:
            self.l2 = self.l1 = new_loss
        expected = 2 * self.l1 - self.l2
        gain = expected - new_loss
        self.h = 0.99 * self.h
        for i in self.last:
            self.h[i] += 0.01 * gain
        self.last = blocks
        self.l2, self.l1 = self.l1, new_loss
        self.step += 1
