"""Test helpers: TF1 AdamOptimizer (ApplyAdam) restated in float64, and the CPU oracle adaptation step with it.

tf.train.AdamOptimizer keeps one pair of non-slot variables beta1_power / beta2_power per graph (every train op of the
demo shares them; both start at beta1 / beta2 and every train op multiplies them by beta1 / beta2 in fp32 after its
update) and one m / v slot per variable.
"""
import numpy as np
import torch

from oracle.adaptation import OracleAdapter

BETA1, BETA2, EPS = 0.9, 0.999, 1e-8


def adam_reference(w, g, m, v, powers, lr, beta1=BETA1, beta2=BETA2, eps=EPS, grad_scale=1.0):
    """One ApplyAdam in float64 from the given (fp32) state -> (w, m, v) float64.  powers = (beta1_power, beta2_power)."""
    f = lambda x: np.asarray(x, dtype=np.float64)
    b1p, b2p = float(powers[0]), float(powers[1])
    one_m_b1 = float(np.float32(1.0) - np.float32(beta1))     # the kernel forms (1 - beta) in fp32, as TF does
    one_m_b2 = float(np.float32(1.0) - np.float32(beta2))
    g = f(g) * float(np.float32(grad_scale))
    lr_t = float(np.float32(lr)) * np.sqrt(1.0 - b2p) / (1.0 - b1p)
    m = f(m) + (g - f(m)) * one_m_b1
    v = f(v) + (g * g - f(v)) * one_m_b2
    w = f(w) - lr_t * m / (float(np.float32(eps)) + np.sqrt(v))
    return w, m, v


def advance_powers(powers, beta1=BETA1, beta2=BETA2):
    """beta1_power *= beta1, beta2_power *= beta2 in fp32."""
    return (np.float32(np.float32(powers[0]) * np.float32(beta1)), np.float32(np.float32(powers[1]) * np.float32(beta2)))


class AdamOracleAdapter(OracleAdapter):
    """OracleAdapter whose train ops apply Adam with one pair of powers shared by all of them."""

    def __init__(self, params, mode='MAD', lr=1e-4, dtype=torch.float32, groups=None, beta1=BETA1, beta2=BETA2, eps=EPS):
        OracleAdapter.__init__(self, params, mode=mode, lr=0.0, mu=0.0, dtype=dtype, groups=groups)
        self.adam_lr, self.beta1, self.beta2, self.eps = lr, beta1, beta2, eps
        self.m = {k: np.zeros(v.shape, np.float64) for k, v in self.net.p.items()}
        self.v = {k: np.zeros(v.shape, np.float64) for k, v in self.net.p.items()}
        self.powers = (np.float32(beta1), np.float32(beta2))

    def step(self, left, right, module=None, proxy=None):
        # the parent computes the gradients of the train op; with lr = mu = 0 its momentum update leaves every weight as is
        out = OracleAdapter.step(self, left, right, module=module, proxy=proxy)
        if self.mode == 'NONE':
            return out
        with torch.no_grad():
            for n, g in out['grads'].items():
                w = self.net.p[n].detach().numpy()
                w, self.m[n], self.v[n] = adam_reference(w, g, self.m[n], self.v[n], self.powers, self.adam_lr, self.beta1,
                                                         self.beta2, self.eps)
                self.net.p[n].copy_(torch.as_tensor(w, dtype=self.net.dtype))
        self.powers = advance_powers(self.powers, self.beta1, self.beta2)
        return out
