"""Checkpoint import with the reference's matching rules, without TensorFlow.

Mirrors Data_utils/weights_utils.py of the reference: `get_var_to_restore_list` (:4-38: skip variables whose name
contains a `mask` entry, strip every `ignore_list` substring from the checkpoint key, prepend `prefix`, keep the key if
the result names a model variable) and `check_for_weights_or_restore_them` (:41-80: newest checkpoint of a log directory,
else the given initial weights, which may be a directory).  `tf.train.NewCheckpointReader` / `Saver.restore` are replaced
by madstereo.tf_checkpoint (TF "V2" bundles) and by `.npz` archives of name -> array.

`model` below is anything with `get_variable_names()` / `load_weights(dict)`: madstereo.adaptation.OnlineAdaptation.
"""
import os
import re

import numpy as np

from madstereo.tf_checkpoint import CheckpointReader, CheckpointError  # noqa: F401


def _open(ckpt_path):
    """-> (shape map, getter).  Accepts a TF V2 checkpoint prefix or an .npz archive."""
    if ckpt_path.endswith('.npz'):
        z = np.load(ckpt_path)
        return {k: list(z[k].shape) for k in z.files}, (lambda k: np.asarray(z[k]))
    r = CheckpointReader(ckpt_path)
    return r.get_variable_to_shape_map(), r.get_tensor


def get_var_to_restore_list(ckpt_path, mask=[], prefix="", ignore_list=[], variables=()):
    """{checkpoint key: model variable name} -- the reference returns the tf.Variable, here its name (without ':0')."""
    variables_dict = {}
    for name in variables:
        name = name[:-2] if name.endswith(':0') else name
        if not any(m in name for m in mask):
            variables_dict[name] = name
    var_to_shape_map, _get = _open(ckpt_path)
    var_to_restore = {}
    for key in var_to_shape_map:
        t_key = key
        for ig in ignore_list:
            t_key = t_key.replace(ig, '')
        if prefix + t_key in variables_dict:
            var_to_restore[key] = variables_dict[prefix + t_key]
    return var_to_restore


def load_weights(ckpt_path, variables, mask=[], prefix="", ignore_list=[]):
    """{model variable name: array} for every checkpoint entry that matches (what Saver.restore would assign)."""
    mapping = get_var_to_restore_list(ckpt_path, mask, prefix, ignore_list, variables)
    _shapes, get = _open(ckpt_path)
    return {var: get(key) for key, var in mapping.items()}


def load_adam_state(ckpt_path, trained_variables, beta1=0.9, beta2=0.999, prefix="", ignore_list=[]):
    """Adam optimizer state of the demo's graph (Demo/demo_model.py:163), as the demo's restore assigns it: a default
    tf.train.Saver() (Train.py) also saves `<var>/Adam` (m), `<var>/Adam_1` (v), `beta1_power` and `beta2_power`, and
    get_var_to_restore_list matches every global variable the checkpoint names.

    trained_variables: {variable name: shape} of the variables some train op trains (slots exist only for those).
    -> {'m': {var: array}, 'v': {var: array}, 'powers': (beta1_power, beta2_power) or None (nothing is trained),
        'found': number of matching checkpoint entries}.  Entries the checkpoint lacks start at zero / (beta1, beta2)."""
    names = list(trained_variables)
    wanted = [n + '/Adam' for n in names] + [n + '/Adam_1' for n in names]
    if names:
        wanted += ['beta1_power', 'beta2_power']
    mapping = get_var_to_restore_list(ckpt_path, [], prefix, ignore_list, wanted)
    _shapes, get = _open(ckpt_path)
    found = {var: np.asarray(get(key), dtype=np.float32) for key, var in mapping.items()}
    state = {'m': {}, 'v': {}, 'powers': None, 'found': len(found)}
    for n in names:
        shape = tuple(trained_variables[n])
        state['m'][n] = found[n + '/Adam'].reshape(shape) if n + '/Adam' in found else np.zeros(shape, np.float32)
        state['v'][n] = found[n + '/Adam_1'].reshape(shape) if n + '/Adam_1' in found else np.zeros(shape, np.float32)
    if names:
        state['powers'] = (float(found['beta1_power']) if 'beta1_power' in found else float(np.float32(beta1)),
                           float(found['beta2_power']) if 'beta2_power' in found else float(np.float32(beta2)))
    return state


def latest_checkpoint(logdir):
    """tf.train.latest_checkpoint: the prefix named by `<logdir>/checkpoint` (model_checkpoint_path: "...")."""
    state = os.path.join(logdir, 'checkpoint')
    if not os.path.exists(state):
        return None
    m = re.search(r'^model_checkpoint_path:\s*"(.*)"\s*$', open(state).read(), re.M)
    if not m:
        return None
    p = m.group(1)
    p = p if os.path.isabs(p) else os.path.join(logdir, p)
    return p if os.path.exists(p + '.index') else None


def check_for_weights_or_restore_them(logdir, model, initial_weights=None, prefix='', ignore_list=[]):
    """-> (restored?, step).  `model` replaces the reference's `session` argument."""
    names = model.get_variable_names()
    ckpt = latest_checkpoint(logdir) if logdir else None
    if ckpt:
        print('Found valid checkpoint file: {}'.format(ckpt))
        model.load_weights(load_weights(ckpt, names, [], prefix=""), strict=False)
        step = int(ckpt.split('-')[-1]) if ckpt.split('-')[-1].isdigit() else 0
        return True, step
    elif initial_weights is not None:
        if os.path.isdir(initial_weights):
            found = latest_checkpoint(initial_weights)
            if found is None:
                raise Exception('no usable checkpoint in directory {} (missing `checkpoint` state file or its .index)'.format(initial_weights))
            initial_weights = found
        w = load_weights(initial_weights, names, [], prefix=prefix, ignore_list=ignore_list)
        print('Found {} variables to restore in {}'.format(len(w), initial_weights))
        if len(w) > 0:
            model.load_weights(w, strict=False)
            return True, 0
        return False, 0
    else:
        print('Unable to restore any weight')
        return False, 0
