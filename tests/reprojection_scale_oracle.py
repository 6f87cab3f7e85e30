"""Test helpers: the MAD step with its module losses at 1/s resolution (--reprojectionScale), restated on the CPU oracle.

Stereo_Online_Adaptation.py:22-23,91-107 and Stereo_Continual_Adaptation.py:95-112 of the reference: with h = H // s and
w = W // s, the frames (and the proxy, then divided by s) are resized to h x w with preprocessing.rescale_image (legacy
bilinear), and module i's disparity -- already full resolution -- with resize_to_prediction to h x w, times
multiplier = H // H = 1.  So the disparity keeps its full-resolution units while it warps the 1/s frames or meets the
proxy / s: the reference's arithmetic, kept as it is.  The full-resolution loss and everything that reads it do not change.
Gradients are torch autograd through the two resizes.
"""
import numpy as np
import torch

from oracle import tf1_ops as T
from oracle.adaptation import OracleAdapter

from adam_oracle import BETA1, BETA2, EPS, adam_reference, advance_powers


def module_loss(disp, left, right, scale, loss='reprojection', proxy=None):
    """Module loss of one full-resolution module disparity [B,H,W,1] at 1/scale resolution."""
    h, w = left.shape[1] // scale, left.shape[2] // scale
    p = T.resize_bilinear(disp, h, w) * 1.0                       # resize_to_prediction(p, left_s) * multiplier (1)
    if loss == 'proxy':
        return T.proxy_loss(p, T.resize_bilinear(proxy, h, w) / scale, 0.1)
    return T.reprojection_loss(p, T.resize_bilinear(left, h, w), T.resize_bilinear(right, h, w))


class RsOracleAdapter(OracleAdapter):
    """OracleAdapter (momentum, or optimizer='adam' as adam_oracle.AdamOracleAdapter applies it) whose MAD module losses
    run at 1/reprojection_scale resolution."""

    def __init__(self, params, reprojection_scale=1, optimizer='momentum', lr=1e-4, **kw):
        OracleAdapter.__init__(self, params, mode='MAD', lr=lr, **kw)
        self.scale, self.optimizer = int(reprojection_scale), optimizer
        if optimizer == 'adam':
            self.m = {k: np.zeros(v.shape, np.float64) for k, v in self.net.p.items()}
            self.v = {k: np.zeros(v.shape, np.float64) for k, v in self.net.p.items()}
            self.powers = (np.float32(BETA1), np.float32(BETA2))

    def step(self, left, right, module=None, proxy=None):
        net = self.net
        names = self.groups[module]
        net.requires_grad_(set(names))
        left_t = torch.as_tensor(left).to(net.dtype)
        right_t = torch.as_tensor(right).to(net.dtype)
        px = None if proxy is None else torch.as_tensor(proxy).to(net.dtype)
        with torch.enable_grad():
            disps, _ = net.forward(left_t, right_t)
            if self.loss_kind == 'proxy':
                full_loss = T.proxy_loss(disps[-1], px, 0.01)
            else:
                full_loss = T.reprojection_loss(disps[-1], left_t, right_t)
            loss = module_loss(disps[module], left_t, right_t, self.scale, self.loss_kind, px)
        out = {'full_loss': float(full_loss.detach()), 'train_loss': float(loss.detach()),
               'disparities': [d.detach().numpy() for d in disps], 'grads': {}}
        gl = torch.autograd.grad(loss, [net.p[n] for n in names], allow_unused=True)
        with torch.no_grad():
            for n, g in zip(names, gl):
                if g is None:
                    continue
                out['grads'][n] = g.numpy().copy()
                if self.optimizer == 'adam':
                    w = net.p[n].detach().numpy()
                    w, self.m[n], self.v[n] = adam_reference(w, g.numpy(), self.m[n], self.v[n], self.powers, self.lr,
                                                             BETA1, BETA2, EPS)
                    net.p[n].copy_(torch.as_tensor(w, dtype=net.dtype))
                else:
                    w, m = T.momentum_update(net.p[n], g, self.momentum[n], self.lr, self.mu)
                    net.p[n].copy_(w)
                    self.momentum[n] = m
        if self.optimizer == 'adam':
            self.powers = advance_powers(self.powers)
        net.requires_grad_(set())
        return out
