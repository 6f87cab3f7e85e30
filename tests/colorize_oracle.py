"""Host restatement of the summary images (TEST INFRASTRUCTURE): preprocessing.colorize_img and TF's ImageSummary
float -> uint8 normalization in numpy.

The reference computes the LUT index in float32 graph ops, so the index is restated with the same float32 operations, each
correctly rounded (numpy float32 arithmetic), and np.rint (half to even) for tf.round; anything it cannot decide that way
(the gather, the min / max, the normalization's comparisons) is exact.  tests/golden/make_colorize_golden.py pins this
restatement to the reference's own colorize_img.
"""
import numpy as np


def colorize_index(value, vmin=None, vmax=None):
    """LUT rows [B,H,W] of value [B,H,W,1]; 256 where TF's GPU gather reads outside the LUT (NaN included)."""
    v = np.asarray(value, dtype=np.float32)[..., 0]
    lo = np.float32(v.min() if vmin is None else vmin)
    hi = np.float32(v.max() if vmax is None else vmax)
    with np.errstate(invalid='ignore', divide='ignore'):
        x = np.rint((v - lo) / np.float32(hi - lo) * np.float32(255.0))
    ok = (x >= 0) & (x <= 255)
    return np.where(ok, np.nan_to_num(x), 256).astype(np.int64)


def colorize(value, lut, vmin=None, vmax=None):
    """colorize_img: float32 [B,H,W,3]; out-of-range / constant maps give 0."""
    table = np.concatenate([np.asarray(lut, np.float32), np.zeros((1, 3), np.float32)])
    return table[colorize_index(value, vmin, vmax)]


def summary_u8(colors):
    """ImageSummary's normalization of one float [H,W,3] image (the rule stated at csrc/summary.cu)."""
    c = np.asarray(colors, dtype=np.float32)
    finite = np.isfinite(c).all(axis=-1)
    lo = np.float32(c[finite].min()) if finite.any() else np.float32(np.inf)
    hi = np.float32(c[finite].max()) if finite.any() else np.float32(-np.inf)
    if lo < 0:
        m = max(abs(lo), abs(hi))
        scale, offset = (np.float32(0) if m < 1e-6 else np.float32(127) / m), np.float32(128)
    else:
        scale, offset = (np.float32(0) if hi < 1e-6 else np.float32(255) / hi), np.float32(0)
    with np.errstate(invalid='ignore'):
        out = np.trunc(np.where(finite[..., None], c, 0) * scale + offset).astype(np.uint8)
    out[~finite] = (255, 0, 0)
    return out


def summary_image(value, lut, vmin=None, vmax=None):
    """tf.summary.image(name, colorize_img(value, ...), max_outputs=1) pixels: image 0, normalized to uint8."""
    return summary_u8(colorize(value, lut, vmin, vmax)[0])
