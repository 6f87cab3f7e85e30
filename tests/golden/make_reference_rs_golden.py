"""MAD module losses at 1/s resolution (--reprojectionScale) computed by the REFERENCE's own graph code -- TEST INFRASTRUCTURE.

Runs in the build container only (it needs /root/reference).  Over the eager TF shim (oracle/tf1_shim.py) it builds
MADNet exactly as oracle/run_reference_graph.py does, then the MAD train ops at scale s with the reference's own
preprocessing.rescale_image, preprocessing.resize_to_prediction, loss_factory.get_reprojection_loss and
loss_factory.get_proxy_loss.  The glue of Stereo_Online_Adaptation.py:87-118 is oracle/run_reference_graph.py's
mad_train_ops; the glue of Stereo_Continual_Adaptation.py:95-112 (proxy loss) is restated next to it below.  Gradients are
torch autograd through the executed graph.  Writes only tests/golden/reference_graph_madnet_rs_64x128.npz:

    python tests/golden/make_reference_rs_golden.py

  rs<s>_<loss>_mad<k>_loss         module k's loss at scale s (s = 2, 3, 4; loss = reprojection | proxy), 64x128
  rs<s>_<loss>_mad<k>_grad:<var>   sub() of a module variable's gradient (k = 0, 2, 4; s = 2, 3)
  p100_rs3_<loss>_mad<k>_loss      module losses at 100x200, s = 3 (the centre crop of the first resize is active)
  left, right, proxy (64x128) and left100, right100, proxy100 (fp16-exact inputs); the weights are oracle.madnet.init_params(42)
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import tf1_shim  # noqa: E402
from oracle.run_reference_graph import REF, build, grads_of, mad_train_ops, sub  # noqa: E402

OUT = os.path.join(ROOT, 'tests', 'golden', 'reference_graph_madnet_rs_64x128.npz')
GRAD_VARS = lambda k: ('model/gc-read-pyramid/conv%d/weights' % (12 - 2 * k),
                       'model/G%d/fgc-volume-filtering-%d/disp-1/weights' % (6 - k, 6 - k),
                       'model/G%d/fgc-volume-filtering-%d/disp-6/biases' % (6 - k, 6 - k), 'model/context-7/biases')


def extend_shim(tf):
    """Comparison ops get_proxy_loss uses that the shim does not define (added here, so that the shim and the fixtures
    it writes stay as they are)."""
    for name, fn in (('logical_or', torch.logical_or), ('less_equal', torch.le), ('greater_equal', torch.ge)):
        if not hasattr(tf, name):
            setattr(tf, name, lambda a, b, fn=fn, name=name: tf1_shim._wrap(fn(tf1_shim._t(a), tf1_shim._t(b)), name))


def proxy_train_ops(tf, stereo_net, predictions, inputs, proxy, loss_factory, preprocessing, train_config, reprojection_scale):
    """Stereo_Continual_Adaptation.py:95-112: one (loss, variable list) per side output, proxy loss at 1/scale."""
    def scale_tensor(tensor, scale):                                   # :26-27
        return preprocessing.rescale_image(tensor, [tf.shape(tensor)[1] // scale, tf.shape(tensor)[2] // scale])
    preds = predictions[:-1]
    inputs_modules = {'left': scale_tensor(inputs['left'], reprojection_scale),
                      'right': scale_tensor(inputs['right'], reprojection_scale),
                      # the loss reads the target's shape only (valid_map's zeros_like, resize_to_prediction)
                      'target': scale_tensor(proxy, reprojection_scale) / reprojection_scale,
                      'proxy': scale_tensor(proxy, reprojection_scale) / reprojection_scale}
    assert len(preds) == len(train_config)
    ops = []
    for counter, p in enumerate(preds):
        multiplier = tf.cast(tf.shape(inputs['left'])[1] // tf.shape(p)[1], tf.float32)
        p = preprocessing.resize_to_prediction(p, inputs_modules['left']) * multiplier
        with tf.variable_scope('proxy_' + str(counter)):
            loss = loss_factory.get_proxy_loss('mean_l1', max_disp=192, weights=[0.1] * 10, reduced=True)([p], inputs_modules)
        var_accumulator = []
        for name in train_config[counter]:
            var_accumulator += stereo_net.get_variables(name)
        ops.append((loss, var_accumulator))
    return ops


def make_inputs(h, w, seed):
    from madstereo.synthetic import make_pair
    left, right, gt = make_pair(h, w, seed=seed)
    left = left.astype(np.float16).astype(np.float32); right = right.astype(np.float16).astype(np.float32)
    proxy = gt.astype(np.float16).astype(np.float32)
    proxy[:, ::7, ::5] = 0.0                         # holes, as in SGM proxies
    proxy[:, 3::11, 4::13] = 200.0                   # >= 192: invalid
    proxy[:, 5, :9] = 192.0
    return left, right, proxy


def run(h, w, seed, scales, grad_scales, prefix, out):
    from oracle.madnet import init_params
    left, right, proxy = make_inputs(h, w, seed)
    params = {k: np.asarray(v) for k, v in init_params(seed=42).items()}
    cfg = json.load(open(os.path.join(REF, 'block_config', 'MadNet_full.json')))
    tf, net, preds, full_loss, inputs, lf, pp = build('MADNet', 'MAD', left, right, params)
    extend_shim(tf)
    proxy_t = tf1_shim.TT(torch.as_tensor(proxy, dtype=torch.float32), 'input_reader/proxy')
    for s in scales:
        for kind in ('reprojection', 'proxy'):
            if kind == 'reprojection':
                ops = mad_train_ops(tf, net, preds, inputs, lf, pp, cfg, reprojection_scale=s)
            else:
                ops = proxy_train_ops(tf, net, preds, inputs, proxy_t, lf, pp, cfg, s)
            for k, (loss, var_list) in enumerate(ops):
                out['%srs%d_%s_mad%d_loss' % (prefix, s, kind, k)] = np.float32(float(loss))
                if s in grad_scales and k in (0, 2, 4):
                    gr = grads_of(loss, var_list)
                    for n in GRAD_VARS(k):
                        if gr.get(n) is not None:
                            out['%srs%d_%s_mad%d_grad:%s' % (prefix, s, kind, k, n)] = sub(gr[n])
    tag = '' if not prefix else prefix.rstrip('_')[1:]
    out['left' + tag] = left.astype(np.float16); out['right' + tag] = right.astype(np.float16)
    out['proxy' + tag] = proxy.astype(np.float16)


if __name__ == '__main__':
    torch.set_num_threads(1)
    sys.path.insert(0, os.path.join(ROOT, 'real-time-self-adaptive-deep-stereo_b200'))
    out = {}
    run(64, 128, 3, (2, 3, 4), (2, 3), '', out)
    run(100, 200, 11, (3,), (), 'p100_', out)
    np.savez_compressed(OUT, **out)
    print('wrote', OUT, '(%d arrays)' % len(out))
