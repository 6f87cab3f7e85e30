"""Run the reference's OWN graph-construction code over the eager TF shim (oracle/tf1_shim.py) -- TEST INFRASTRUCTURE.

Build container only (needs /root/reference; never imported by a test, bench.py or the product).  It imports, unmodified,
    Nets/__init__.py, Nets/Stereo_net.py, Nets/MadNet.py, Nets/DispNet.py, Nets/sharedLayers.py,
    Losses/loss_factory.py, Data_utils/preprocessing.py
with `tensorflow` replaced by the shim, builds the network exactly as Stereo_Online_Adaptation.py:54-65 does
(`tf.variable_scope('model')`, `split_layers=[None], sequence=True, train_portion='BEGIN', bulkhead=(mode=='MAD')`), the
full-resolution loss as :68-70, and the MAD / FULL train ops as :85-128 (the few lines of glue are restated here because
the driver script cannot be imported: it needs cv2 / matplotlib / a data reader); gradients are torch autograd through
the executed graph, restricted to the reference's own `stereo_net.get_variables(name)` lists.

    python -m oracle.run_reference_graph          # writes tests/golden/reference_graph_*.npz

tests/test_oracle_cpu.py then checks the oracle (oracle/madnet.py, oracle/dispnet.py, oracle/adaptation.py) and the host
mirror (Nets/, block_config) against these vectors.
"""
import importlib
import json
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = '/root/reference'
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'real-time-self-adaptive-deep-stereo_b200'))

from oracle import tf1_shim  # noqa: E402


def import_reference():
    """Install the shim as `tensorflow`, stub matplotlib (colour maps for summaries only) and import the reference."""
    tfm = tf1_shim.as_module()
    sys.modules['tensorflow'] = tfm
    mpl = types.ModuleType('matplotlib'); mpl.cm = types.ModuleType('matplotlib.cm')
    sys.modules.setdefault('matplotlib', mpl); sys.modules.setdefault('matplotlib.cm', mpl.cm)
    for k in [k for k in sys.modules if k.split('.')[0] in ('Nets', 'Losses', 'Data_utils', 'Sampler')]:
        del sys.modules[k]
    sys.path.insert(0, REF)
    try:
        nets = importlib.import_module('Nets')
        loss_factory = importlib.import_module('Losses.loss_factory')
        preprocessing = importlib.import_module('Data_utils.preprocessing')
    finally:
        sys.path.remove(REF)
    assert os.path.abspath(nets.__file__).startswith(REF), nets.__file__
    return tfm, nets, loss_factory, preprocessing


def build(model_name, mode, left, right, params, net_args=None):
    """Stereo_Online_Adaptation.py:54-70 (network + full-resolution loss).  `net_args` adds to / overrides the network
    arguments (e.g. MADNet's radius_d, stride, warping; left unset, the network's own defaults apply)."""
    tf1_shim.reset_graph(params)
    tf, nets, loss_factory, preprocessing = import_reference()
    left_t = tf1_shim.TT(torch.as_tensor(left, dtype=torch.float32), 'input_reader/left')
    right_t = tf1_shim.TT(torch.as_tensor(right, dtype=torch.float32), 'input_reader/right')
    inputs = {'left': left_t, 'right': right_t, 'target': None}
    with tf.variable_scope('model'):
        net_args = dict({'left_img': left_t, 'right_img': right_t, 'split_layers': [None], 'sequence': True,
                         'train_portion': 'BEGIN', 'bulkhead': mode == 'MAD'}, **(net_args or {}))
        stereo_net = nets.get_stereo_net(model_name, net_args)
        predictions = stereo_net.get_disparities()
    with tf.variable_scope('full_res_loss'):
        full_loss = loss_factory.get_reprojection_loss('mean_SSIM_l1', reduced=True)(predictions, inputs)
    return tf, stereo_net, predictions, full_loss, inputs, loss_factory, preprocessing


def mad_train_ops(tf, stereo_net, predictions, inputs, loss_factory, preprocessing, train_config, reprojection_scale=1):
    """Stereo_Online_Adaptation.py:87-118: one (loss, variable list) per side output."""
    def scale_tensor(tensor, scale):                                   # :22-23
        return preprocessing.rescale_image(tensor, [tf.shape(tensor)[1] // scale, tf.shape(tensor)[2] // scale])
    preds = predictions[:-1]
    inputs_modules = {'left': scale_tensor(inputs['left'], reprojection_scale),
                      'right': scale_tensor(inputs['right'], reprojection_scale), 'target': None}
    assert len(preds) == len(train_config)
    ops = []
    for counter, p in enumerate(preds):
        multiplier = tf.cast(tf.shape(inputs['left'])[1] // tf.shape(p)[1], tf.float32)
        p = preprocessing.resize_to_prediction(p, inputs_modules['left']) * multiplier
        with tf.variable_scope('reprojection_' + str(counter)):
            loss = loss_factory.get_reprojection_loss('mean_SSIM_l1', reduced=True)([p], inputs_modules)
        var_accumulator = []
        for name in train_config[counter]:
            var_accumulator += stereo_net.get_variables(name)
        ops.append((loss, var_accumulator))
    return ops


def sub(a, n=4096):
    """Deterministic subsample that keeps fixtures small: every k-th element of the flattened array (at most ~n)."""
    a = np.asarray(a).ravel()
    return a[::max(1, a.size // n)].copy()


def grads_of(loss, variables):
    uniq = []
    for v in variables:
        if all(v is not u for u in uniq):
            uniq.append(v)
    g = torch.autograd.grad(loss.t, [v.t for v in uniq], allow_unused=True, retain_graph=True)
    return {v.name[:-2]: (None if gi is None else gi.numpy().copy()) for v, gi in zip(uniq, g)}


def run_madnet(out_path, h=64, w=128):
    from madstereo.synthetic import make_pair
    from oracle.madnet import init_params
    left, right, _ = make_pair(h, w, seed=3)
    left = left.astype(np.float16).astype(np.float32); right = right.astype(np.float16).astype(np.float32)
    params = {k: np.asarray(v) for k, v in init_params(seed=42).items()}
    cfg = json.load(open(os.path.join(REF, 'block_config', 'MadNet_full.json')))
    out = {'left': left.astype(np.float16), 'right': right.astype(np.float16)}

    tf, net, preds, full_loss, inputs, lf, pp = build('MADNet', 'MAD', left, right, params)
    g = tf1_shim.graph()
    out['variable_names'] = np.array([n for n, _ in g.created])
    out['variable_shapes'] = np.array([json.dumps(list(s)) for _, s in g.created])
    out['layer_names'] = np.array(list(net.get_layers_names()))
    out['str_net'] = np.array(str(net))
    for i, d in enumerate(preds):
        out['disp%d' % i] = d.numpy()
    for k in ('left/conv4', 'right/conv12', 'fgc-volume-filtering-6/disp1', 'fgc-volume-filtering-4/disp3',
              'fgc-volume-filtering-2/disp6', 'context5', 'final_disp'):
        out['layer:' + k] = net[k].numpy()
    out['full_loss'] = np.float32(float(full_loss))
    # get_variables for every name the block configs use, and a few that show the prefix-regex behaviour
    probe = sorted({n for grp in cfg for n in grp} | {'left/conv1', 'right/conv1', 'final_disp', 'rescaled_prediction', 'context1'})
    out['get_variables'] = np.array(json.dumps({n: [v.name for v in net.get_variables(n)] for n in probe}))
    ops = mad_train_ops(tf, net, preds, inputs, lf, pp, cfg)
    for k, (loss, var_list) in enumerate(ops):
        out['mad%d_loss' % k] = np.float32(float(loss))
        gr = grads_of(loss, var_list)
        out['mad%d_vars' % k] = np.array(sorted(gr))
        out['mad%d_none' % k] = np.array(sorted(n for n, v in gr.items() if v is None))
        for n in ('model/gc-read-pyramid/conv%d/weights' % (12 - 2 * k), 'model/G%d/fgc-volume-filtering-%d/disp-1/weights' % (6 - k, 6 - k),
                  'model/G%d/fgc-volume-filtering-%d/disp-6/biases' % (6 - k, 6 - k)):
            if gr.get(n) is not None:
                out['mad%d_grad:%s' % (k, n)] = sub(gr[n])

    # FULL mode (:126-128): bulkhead off, minimize(full loss) over all trainable variables
    tf, net, preds, full_loss, inputs, lf, pp = build('MADNet', 'FULL', left, right, params)
    gr = grads_of(full_loss, tf.get_collection(tf.GraphKeys.TRAINABLE_VARIABLES))
    out['full_mode_loss'] = np.float32(float(full_loss))
    for n in ('model/gc-read-pyramid/conv1/weights', 'model/gc-read-pyramid/conv12/weights', 'model/G6/fgc-volume-filtering-6/disp-3/weights',
              'model/G3/fgc-volume-filtering-3/disp-1/weights', 'model/context-4/weights', 'model/context-7/biases'):
        out['full_grad:' + n] = sub(gr[n])
    np.savez_compressed(out_path, **out)
    print('wrote', out_path, '(%d arrays)' % len(out))


def run_dispnet(out_path, h=64, w=128):
    from madstereo.synthetic import make_pair
    from oracle.dispnet import init_params
    left, right, _ = make_pair(h, w, seed=5)
    left = left.astype(np.float16).astype(np.float32); right = right.astype(np.float16).astype(np.float32)
    params = {k: np.asarray(v) for k, v in init_params(seed=7).items()}
    out = {'left': left.astype(np.float16), 'right': right.astype(np.float16)}
    tf, net, preds, full_loss, inputs, lf, pp = build('Dispnet', 'FULL', left, right, params)
    g = tf1_shim.graph()
    out['variable_names'] = np.array([n for n, _ in g.created])
    out['variable_shapes'] = np.array([json.dumps(list(s)) for _, s in g.created])
    out['layer_names'] = np.array(list(net.get_layers_names()))
    for i, d in enumerate(preds):
        out['disp%d' % i] = d.numpy()
    out['full_loss'] = np.float32(float(full_loss))
    gr = grads_of(full_loss, tf.get_collection(tf.GraphKeys.TRAINABLE_VARIABLES))
    for n in ('model/conv1/weights', 'model/conv3/weights', 'model/up3/deconv/weights', 'model/up1/concat/weights', 'model/prediction/bias'):
        out['full_grad:' + n] = sub(gr[n])
    np.savez_compressed(out_path, **out)
    print('wrote', out_path, '(%d arrays)' % len(out))


def run_madnet_padded(out_path, h=100, w=200):
    """A size that is not a multiple of 64: exercises preprocessing.pad_image (REFLECT, :7-29) and the crop back to the
    input size in _make_disp / rescaled_prediction (MadNet.py:68-71,362-363).  Forward + losses only (small fixture)."""
    from madstereo.synthetic import make_pair
    from oracle.madnet import init_params
    left, right, _ = make_pair(h, w, seed=11)
    left = left.astype(np.float16).astype(np.float32); right = right.astype(np.float16).astype(np.float32)
    params = {k: np.asarray(v) for k, v in init_params(seed=42).items()}
    cfg = json.load(open(os.path.join(REF, 'block_config', 'MadNet_full.json')))
    out = {'left': left.astype(np.float16), 'right': right.astype(np.float16)}
    tf, net, preds, full_loss, inputs, lf, pp = build('MADNet', 'MAD', left, right, params)
    for i, d in enumerate(preds):
        out['disp%d' % i] = d.numpy().astype(np.float32)
    out['layer:final_disp'] = net['final_disp'].numpy()
    out['full_loss'] = np.float32(float(full_loss))
    for k, (loss, _vars) in enumerate(mad_train_ops(tf, net, preds, inputs, lf, pp, cfg)):
        out['mad%d_loss' % k] = np.float32(float(loss))
    np.savez_compressed(out_path, **out)
    print('wrote', out_path, '(%d arrays)' % len(out))


# MADNet at non-default correlation settings: (radius_d, stride, warping) -> fixture name
MADNET_VARIANTS = {(4, 2, False): 'reference_graph_madnet_r4s2_nowarp_64x128.npz',
                   (2, 3, True): 'reference_graph_madnet_r2s3_warp_64x128.npz'}
VARIANT_LAYERS = ('fgc-volume-filtering-6/disp1', 'fgc-volume-filtering-5/disp1', 'fgc-volume-filtering-4/disp3',
                  'fgc-volume-filtering-2/disp1', 'fgc-volume-filtering-2/disp6', 'context5', 'final_disp')
LEAKY_LAYERS = (['%s/conv%d' % (s, i) for s in ('left', 'right') for i in range(1, 13)] +
                ['fgc-volume-filtering-%d/disp%d' % (k, j) for k in (6, 5, 4, 3, 2) for j in range(1, 6)] +
                ['context%d' % j for j in range(1, 7)])
VARIANT_GRADS = ('model/gc-read-pyramid/conv1/weights', 'model/gc-read-pyramid/conv12/weights',
                 'model/G6/fgc-volume-filtering-6/disp-1/weights', 'model/G5/fgc-volume-filtering-5/disp-1/weights',
                 'model/G3/fgc-volume-filtering-3/disp-1/weights', 'model/G2/fgc-volume-filtering-2/disp-1/weights',
                 'model/G2/fgc-volume-filtering-2/disp-1/biases', 'model/context-4/weights')


def run_madnet_variant(out_path, radius_d, stride, warping, h=64, w=128):
    """The reference's Nets/MadNet.py with non-default radius_d / stride / warping: the estimators' input width follows
    the correlation's displacement count (len(range(-d, d+1, s))).  Disparities, layers, the MAD and FULL losses and a
    subsample of the FULL gradients.  `kink:<layer>` holds the sign (np.packbits of > 0) of every leaky-ReLU output of
    the reference's fp32 run: where a pre-activation lies within rounding of zero, the reference's side of the kink decides
    every gradient upstream of it, and the oracle can take the same side (MadNetOracle kink_signs)."""
    from madstereo.synthetic import make_pair
    from oracle.madnet import init_params
    left, right, _ = make_pair(h, w, seed=3)
    left = left.astype(np.float16).astype(np.float32); right = right.astype(np.float16).astype(np.float32)
    params = {k: np.asarray(v) for k, v in init_params(seed=42, radius_d=radius_d, stride=stride).items()}
    cfg = json.load(open(os.path.join(REF, 'block_config', 'MadNet_full.json')))
    args = {'radius_d': radius_d, 'stride': stride, 'warping': warping}
    out = {'left': left.astype(np.float16), 'right': right.astype(np.float16),
           'net_args': np.array(json.dumps(args))}
    tf, net, preds, full_loss, inputs, lf, pp = build('MADNet', 'MAD', left, right, params, args)
    g = tf1_shim.graph()
    out['variable_names'] = np.array([n for n, _ in g.created])
    out['variable_shapes'] = np.array([json.dumps(list(s)) for _, s in g.created])
    for i, d in enumerate(preds):
        out['disp%d' % i] = d.numpy()
    for k in VARIANT_LAYERS:
        out['layer:' + k] = net[k].numpy()
    for k in LEAKY_LAYERS:
        out['kink:' + k] = np.packbits(net[k].numpy() > 0)
    out['full_loss'] = np.float32(float(full_loss))
    for k, (loss, _vars) in enumerate(mad_train_ops(tf, net, preds, inputs, lf, pp, cfg)):
        out['mad%d_loss' % k] = np.float32(float(loss))
    tf, net, preds, full_loss, inputs, lf, pp = build('MADNet', 'FULL', left, right, params, args)
    gr = grads_of(full_loss, tf.get_collection(tf.GraphKeys.TRAINABLE_VARIABLES))
    out['full_mode_loss'] = np.float32(float(full_loss))
    for n in VARIANT_GRADS:
        out['full_grad:' + n] = sub(gr[n])
    np.savez_compressed(out_path, **out)
    print('wrote', out_path, '(%d arrays)' % len(out))


if __name__ == '__main__':
    torch.set_num_threads(1)
    gold = os.path.join(ROOT, 'tests', 'golden')
    run_madnet(os.path.join(gold, 'reference_graph_madnet_64x128.npz'))
    run_madnet_padded(os.path.join(gold, 'reference_graph_madnet_100x200.npz'))
    run_dispnet(os.path.join(gold, 'reference_graph_dispnet_64x128.npz'))
    for (d, s, warp), name in MADNET_VARIANTS.items():
        run_madnet_variant(os.path.join(gold, name), d, s, warp)
