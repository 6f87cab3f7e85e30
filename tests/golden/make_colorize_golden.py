"""Golden colour maps from the REFERENCE's own preprocessing.colorize_img (Data_utils/preprocessing.py:91-117), executed
over the eager TF shim (oracle/tf1_shim.py) in the build container:

    python tests/golden/make_colorize_golden.py          # writes tests/golden/reference_colorize.npz

The shim lacks three ops colorize_img calls; they are supplied here: tf.reduce_min / tf.reduce_max over the whole tensor
and tf.round as torch.round (half to even, as tf.round).  matplotlib is not installed, so `cm.get_cmap` is replaced by a
colour map over an injected LUT: a seeded random one (the gather and the index, independent of any colour map) and the
repository's jet.  Every case keeps the index inside [0, 255]: out of range, the shim's gather would wrap where TF's GPU
gather writes zeros.  tests/test_summary_cpu.py checks tests/colorize_oracle.py against these outputs.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'real-time-self-adaptive-deep-stereo_b200'))

from oracle import tf1_shim  # noqa: E402
from oracle.run_reference_graph import import_reference  # noqa: E402
from madstereo.ops import colormap_lut  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'reference_colorize.npz')


def tie_values(n):
    """float32 v in (0, 1) whose float32 product v * 255 is exactly k + 0.5: rint must break the tie to even."""
    out = []
    for k in range(n):
        want = np.float32(k * 2 + 0.5)
        v = np.float32(want / np.float32(255))
        for cand in (v, np.nextafter(v, np.float32(1)), np.nextafter(v, np.float32(0))):
            if np.float32(cand * np.float32(255)) == want:
                out.append(cand)
                break
    return np.asarray(out, np.float32)


def cases():
    rng = np.random.default_rng(7)
    smooth = (rng.standard_normal((2, 6, 9, 1)) * 20 + 40).astype(np.float32)
    smooth[1, 2, 3, 0] = 150.0                                        # the batch maximum lives in image 1
    ties = tie_values(128)
    tie_map = np.concatenate([[0.0, 1.0], ties, np.full(16 * 9 - 2 - len(ties), 0.5, np.float32)]).astype(np.float32)
    tie_map = tie_map[:16 * 9].reshape(1, 16, 9, 1)
    return [('smooth_auto', smooth, None, None), ('smooth_given', smooth, float(np.floor(smooth.min())) - 1.5, 160.0),
            ('ties_auto', tie_map, None, None), ('ties_given', tie_map, 0.0, 1.0),
            ('one_frame', smooth[:1] * 0.5 - 3.0, None, None)]


def main():
    tf, _nets, _loss, preprocessing = import_reference()
    _t = tf1_shim._t
    tf.reduce_min = lambda x, *a, **k: tf1_shim.TT(torch.min(_t(x)), 'Min')
    tf.reduce_max = lambda x, *a, **k: tf1_shim.TT(torch.max(_t(x)), 'Max')
    tf.round = lambda x, *a, **k: tf1_shim.TT(torch.round(_t(x)), 'Round')
    luts = {'random': np.random.default_rng(11).uniform(0, 1, (256, 3)).astype(np.float32), 'jet': colormap_lut('jet')}
    data = {}
    for lut_name, lut in luts.items():
        rgba = np.concatenate([lut.astype(np.float64), np.ones((256, 1))], axis=1)
        preprocessing.cm.get_cmap = lambda name, rgba=rgba: (lambda idx: rgba[np.asarray(idx)])
        data['lut_' + lut_name] = lut
        for name, value, vmin, vmax in cases():
            tf1_shim.reset_graph()
            out = preprocessing.colorize_img(tf1_shim.TT(torch.from_numpy(value), 'value'), vmin=vmin, vmax=vmax, cmap='jet')
            key = '%s__%s' % (name, lut_name)
            data[key + '__value'] = value
            data[key + '__range'] = np.array([np.nan if vmin is None else vmin, np.nan if vmax is None else vmax], np.float32)
            data[key + '__out'] = out.t.detach().numpy().astype(np.float32)
    np.savez_compressed(OUT, **data)
    print('wrote', OUT, len(data), 'arrays')


if __name__ == '__main__':
    main()
