"""CPU oracle — MADNet forward restated from Nets/MadNet.py (TEST INFRASTRUCTURE).

Pinned against the reference's own Nets/MadNet.py executed over oracle/tf1_shim.py (tests/golden/reference_graph_madnet_64x128.npz,
tests/test_oracle_cpu.py); TF's conv-padding / resize kernels themselves stay unpinned (see oracle/tf1_ops.py).

Follows /root/reference/Nets/MadNet.py:56-71 (_preprocess_inputs, _make_disp), :73-120 (estimator),
:122-171 (context net), :173-249 (pyramid), :251-364 (_build_network), :370-375 (cost volume).
Backward comes from torch-CPU autograd over this forward (tf.gradients equivalent); `bulkhead`
maps tf.stop_gradient to .detach().
"""
from collections import OrderedDict

import numpy as np
import torch

from . import tf1_ops as T

PYRAMID_CH = [3, 16, 16, 32, 32, 64, 64, 96, 96, 128, 128, 192, 192]   # MadNet.py:173-249
EST_CH = [128, 128, 96, 64, 32, 1]                                      # MadNet.py:73-120
CTX_CH = [128, 128, 128, 96, 64, 32, 1]                                 # MadNet.py:122-171
CTX_RATE = [1, 2, 4, 8, 16, 1, 1]
LEVEL_FEAT = {6: 12, 5: 10, 4: 8, 3: 6, 2: 4}                            # level -> pyramid conv index
ALPHA = 0.2                                                              # MadNet.py:366-367


def num_displacements(radius_d=2, stride=1):
    """Channels of sharedLayers.correlation_tf: one per displacement in range(-d, d+1, stride) (sharedLayers.py:46)."""
    return len(range(-radius_d, radius_d + 1, stride))


def param_shapes(radius_d=2, stride=1):
    """OrderedDict TF-variable-name -> shape, in graph-construction order."""
    p = OrderedDict()
    for i in range(1, 13):
        s = 'model/gc-read-pyramid/conv%d' % i
        p[s + '/weights'] = (3, 3, PYRAMID_CH[i - 1], PYRAMID_CH[i])
        p[s + '/biases'] = (PYRAMID_CH[i],)
    nd = num_displacements(radius_d, stride)
    for k in (6, 5, 4, 3, 2):
        cin = PYRAMID_CH[LEVEL_FEAT[k]] + nd + (0 if k == 6 else 1)
        for j, co in enumerate(EST_CH):
            s = 'model/G%d/fgc-volume-filtering-%d/disp-%d' % (k, k, j + 1)
            p[s + '/weights'] = (3, 3, cin, co)
            p[s + '/biases'] = (co,)
            cin = co
    cin = PYRAMID_CH[4] + 1
    for j, co in enumerate(CTX_CH):
        s = 'model/context-%d' % (j + 1)
        p[s + '/weights'] = (3, 3, cin, co)
        p[s + '/biases'] = (co,)
        cin = co
    return p


def init_params(seed=42, bias_range=0.1, radius_d=2, conditioned=True, stride=1):
    """Seeded xavier-uniform weights + small non-zero biases (SURVEY §8d).

    conditioned=True additionally rescales the draw so that a random net behaves like a trained one
    (activations O(1) on 0..255 inputs, every disparity head alive under relu(-20*V)); otherwise a
    raw xavier net is chaotic (fp32-vs-fp64 differences get amplified ~100x) and most heads are dead,
    which makes the MAD gradients identically zero.  Pure test-vector conditioning, no reference
    counterpart (the reference always starts from a pretrained checkpoint, README.MD:47).
    """
    rng = np.random.default_rng(seed)
    out = OrderedDict()
    for name, shp in param_shapes(radius_d, stride).items():
        head = name.endswith('disp-6/weights') or name.endswith('context-7/weights')
        head_b = name.endswith('disp-6/biases') or name.endswith('context-7/biases')
        if len(shp) == 4:
            w = T.xavier_uniform(rng, shp)
            if conditioned:
                if name == 'model/gc-read-pyramid/conv1/weights':
                    w = w * np.float32(1.0 / 48.0)
                elif head:
                    w = w * np.float32(0.5)
                else:
                    w = w * np.float32(1.3)
            out[name] = w
        else:
            b = rng.uniform(-bias_range, bias_range, size=shp).astype('float32')
            if conditioned and head_b:
                b = b - np.float32(0.05 if name.endswith('context-7/biases') else 0.35)
            out[name] = b
    return out


class MadNetOracle:
    def __init__(self, params, dtype=torch.float32, radius_d=2, stride=1, warping=True,
                 context_net=True, bulkhead=False, kink_signs=None, kink_band=1e-4):
        self.p = OrderedDict((k, (v if torch.is_tensor(v) else torch.tensor(np.asarray(v))).to(dtype))
                             for k, v in params.items())
        self.dtype = dtype
        self.radius_d, self.stride = radius_d, stride
        self.warping, self.context_net, self.bulkhead = warping, context_net, bulkhead
        assert context_net, "context_net=False path is broken in the reference (MadNet.py:360)"
        # kink_signs: {layer name: bool array, True where another implementation's output of that leaky-ReLU layer is
        # > 0}.  Where this oracle's pre-activation lies within kink_band x the layer's largest |pre-activation| of zero,
        # the slope follows that sign instead of its own; everywhere else the oracle is unchanged.  Two correct fp32
        # computations can land on opposite sides of a kink for such an element, and then every gradient upstream of it
        # differs by that element's share; with the other side's choice at those elements only, the float64 oracle
        # measures the remaining arithmetic.  None (default): plain oracle.
        self.kink_signs, self.kink_band = kink_signs, kink_band
        self.kink_overrides = {}                      # layer name -> number of elements whose slope was taken over

    def requires_grad_(self, names=None):
        for k, v in self.p.items():
            v.requires_grad_(names is None or k in names)

    def _conv(self, x, scope, stride=1, rate=1, alpha=ALPHA, name=None):
        if alpha is None or self.kink_signs is None or name not in self.kink_signs:
            return T.conv2d(x, self.p[scope + '/weights'], self.p[scope + '/biases'],
                            stride=stride, dilation=rate, alpha=alpha)
        pre = T.conv2d(x, self.p[scope + '/weights'], self.p[scope + '/biases'], stride=stride, dilation=rate, alpha=None)
        with torch.no_grad():
            near = pre.abs() <= self.kink_band * pre.abs().max()
            pos = torch.where(near, torch.as_tensor(np.asarray(self.kink_signs[name]), dtype=torch.bool), pre > 0)
            self.kink_overrides[name] = int((near & (pos != (pre > 0))).sum())
        return torch.where(pos, pre, pre * alpha)

    def pyramid(self, img, prefix, layers):
        x = img
        for i in range(1, 13):
            name = '%s/conv%d' % (prefix, i)
            x = self._conv(x, 'model/gc-read-pyramid/conv%d' % i, stride=2 if i % 2 == 1 else 1, name=name)
            layers[name] = x

    def estimator(self, cost, u, k, layers):
        x = cost if u is None else torch.cat([cost, u], -1)
        for j in range(6):
            name = 'fgc-volume-filtering-%d/disp%d' % (k, j + 1)
            x = self._conv(x, 'model/G%d/fgc-volume-filtering-%d/disp-%d' % (k, k, j + 1),
                           alpha=ALPHA if j < 5 else None, name=name)
            layers[name] = x
        return x

    def context(self, feat, disp, layers):
        x = torch.cat([feat, disp], -1)
        for j in range(7):
            x = self._conv(x, 'model/context-%d' % (j + 1), rate=CTX_RATE[j],
                           alpha=ALPHA if j < 6 else None, name='context%d' % (j + 1))
            layers['context%d' % (j + 1)] = x
        final = disp + x
        layers['final_disp'] = final
        return final

    def make_disp(self, v, hp, wp, h, w):
        """MadNet._make_disp (MadNet.py:68-71)."""
        return T.crop_or_pad(T.resize_bilinear(torch.relu(v * -20.0), hp, wp), h, w)

    def forward(self, left, right):
        """left/right [B,H,W,3] (0..255). Returns (disparities list of 6, layers dict)."""
        left = torch.as_tensor(left).to(self.dtype)
        right = torch.as_tensor(right).to(self.dtype)
        h, w = left.shape[1], left.shape[2]
        lp = T.pad_reflect_to_multiple(left, 64)
        rp = T.pad_reflect_to_multiple(right, 64)
        hp, wp = lp.shape[1], lp.shape[2]
        layers = OrderedDict()
        self.pyramid(lp, 'left', layers)
        self.pyramid(rp, 'right', layers)
        disps = []
        v = None
        for k in (6, 5, 4, 3, 2):
            lf = layers['left/conv%d' % LEVEL_FEAT[k]]
            rf = layers['right/conv%d' % LEVEL_FEAT[k]]
            u = None
            if k < 6:
                u = T.resize_bilinear(v, hp // 2 ** k, wp // 2 ** k) * 20.0 / 2 ** k
                if self.bulkhead:
                    u = u.detach()
                layers['u%d' % k] = u
                if self.warping:
                    rf = T.linear_warp(rf, u)
                    layers['right_warped_%d' % k] = rf
            corr = T.correlation(lf, rf, self.radius_d, self.stride)
            layers['corr%d' % k] = corr
            cost = torch.cat([lf, corr], -1)
            v = self.estimator(cost, u, k, layers)
            if k > 2:
                disps.append(self.make_disp(v, hp, wp, h, w))
        final = self.context(layers['left/conv4'], v, layers)
        disps.append(self.make_disp(final, hp, wp, h, w))
        resc = torch.relu(T.resize_bilinear(final, hp, wp) * -20.0)
        resc = T.crop_or_pad(resc, h, w)
        layers['rescaled_prediction'] = resc
        disps.append(resc)
        return disps, layers


# MAD module -> variable scopes trained (block_config/MadNet_full.json + Stereo_net.get_variables)
def mad_groups_full():
    groups = []
    for k in (6, 5, 4, 3, 2):
        scopes = ['model/G%d/fgc-volume-filtering-%d/disp-%d' % (k, k, j) for j in range(1, 7)]
        if k > 2:
            scopes += ['model/gc-read-pyramid/conv%d' % LEVEL_FEAT[k],
                       'model/gc-read-pyramid/conv%d' % (LEVEL_FEAT[k] - 1)]
        else:
            scopes += ['model/gc-read-pyramid/conv%d' % i for i in (4, 3, 2, 1)]
            scopes += ['model/context-%d' % j for j in range(1, 8)]
        names = []
        for s in scopes:
            names += [s + '/weights', s + '/biases']
        groups.append(names)
    return groups
