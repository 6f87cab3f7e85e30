"""CPU oracle — TF1-semantics op restatements (TEST INFRASTRUCTURE, NOT PRODUCT CODE).

PARITY: TensorFlow 1.12 cannot be installed here and the reference ships no tests / golden vectors, so these
functions restate the documented TF 1.x behaviour of the ops the reference calls; each cites the reference call site it
follows (paths relative to /root/reference).  The restatement as a whole is pinned to the reference's own Python graph
code executed over oracle/tf1_shim.py (oracle/run_reference_graph.py -> tests/golden/reference_graph_*.npz); the
SAME-padding conv family, legacy resize and crop_or_pad kernels are shared with that shim and stay UNPINNED w.r.t.
TensorFlow's own kernels.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this package.  The product path (real-time-self-adaptive-deep-stereo_b200/) never does.

All tensors are NHWC torch tensors on any device (fp32 by default, fp64 for cross-checks); conv kernels are
HWIO [kh,kw,cin,cout] exactly like the reference's tf.get_variable shapes.
"""
import math

import torch
import torch.nn.functional as F


# --------------------------------------------------------------------------------------------
# padding helpers
# --------------------------------------------------------------------------------------------
def same_pad(in_size, k, stride=1, dilation=1):
    """TF 'SAME' padding for one spatial dim -> (out_size, pad_before, pad_after).

    out = ceil(in/s); pad_total = max((out-1)*s + k_eff - in, 0); before = total//2.
    (tf.nn.conv2d padding='SAME', Nets/sharedLayers.py:58; atrous: :72)
    """
    k_eff = (k - 1) * dilation + 1
    out = -(-in_size // stride)
    total = max((out - 1) * stride + k_eff - in_size, 0)
    return out, total // 2, total - total // 2


def _to_nchw(x):
    return x.permute(0, 3, 1, 2)


def _to_nhwc(x):
    return x.permute(0, 2, 3, 1)


def leaky(x, alpha):
    """tf.maximum(alpha*x, x)  (Nets/sharedLayers.py:54 default 0.1; Nets/MadNet.py:366-367 0.2)."""
    if alpha is None or alpha == 1.0:
        return x
    return torch.maximum(alpha * x, x)


def conv2d(x, w, b, stride=1, dilation=1, alpha=None):
    """act(conv2d_SAME(x, W, stride) + b)   — Nets/sharedLayers.py:54-63 (and :66-77 for dilation).

    x NHWC, w HWIO, b [cout]; alpha=None means linear activation (`lambda x: x`).
    """
    kh, kw, cin, cout = w.shape
    _, pt, pb = same_pad(x.shape[1], kh, stride, dilation)
    _, pl, pr = same_pad(x.shape[2], kw, stride, dilation)
    xn = F.pad(_to_nchw(x), (pl, pr, pt, pb))
    y = F.conv2d(xn, w.permute(3, 2, 0, 1).contiguous(), b, stride=stride, dilation=dilation)
    return leaky(_to_nhwc(y), alpha)


def conv2d_transpose(x, w, b, stride=2, alpha=None):
    """act(conv2d_transpose_SAME(x, W, out=in*stride) + b) — Nets/sharedLayers.py:80-92.

    w is [kh,kw,cout,cin] (TF transposed-conv filter = the forward conv's HWIO filter whose input
    is this op's output).  conv2d_transpose is the input-gradient of that forward SAME conv, i.e. a
    scatter with pad_before of the forward conv.
    """
    kh, kw, cout, cin = w.shape
    oh, ow = x.shape[1] * stride, x.shape[2] * stride
    _, pt, _ = same_pad(oh, kh, stride)
    _, pl, _ = same_pad(ow, kw, stride)
    # torch conv_transpose2d weight [cin, cout, kh, kw]; output size (in-1)*s - 2p + k (+ output_padding)
    wt = w.permute(3, 2, 0, 1).contiguous()
    full = F.conv_transpose2d(_to_nchw(x), wt, None, stride=stride)  # size (in-1)*s + k
    y = full[:, :, pt:pt + oh, pl:pl + ow]
    # rows beyond `full` can only be needed if pad_after < 0, which never happens for k>=s
    assert y.shape[2] == oh and y.shape[3] == ow
    y = y + b.view(1, -1, 1, 1)
    return leaky(_to_nhwc(y), alpha)


def pad_reflect_to_multiple(x, factor):
    """preprocessing.pad_image (Data_utils/preprocessing.py:7-29): REFLECT pad H,W up to a multiple."""
    h, w = x.shape[1], x.shape[2]
    nh = h if h % factor == 0 else (h // factor + 1) * factor
    nw = w if w % factor == 0 else (w // factor + 1) * factor
    pt, pb = (nh - h) // 2, (nh - h + 1) // 2
    pl, pr = (nw - w) // 2, (nw - w + 1) // 2
    if pt == pb == pl == pr == 0:
        return x
    return _to_nhwc(F.pad(_to_nchw(x), (pl, pr, pt, pb), mode='reflect'))


def crop_or_pad(x, th, tw):
    """tf.image.resize_image_with_crop_or_pad (Nets/MadNet.py:70,363): centred crop / zero pad."""
    h, w = x.shape[1], x.shape[2]
    if h > th:
        o = (h - th) // 2
        x = x[:, o:o + th]
    if w > tw:
        o = (w - tw) // 2
        x = x[:, :, o:o + tw]
    h, w = x.shape[1], x.shape[2]
    if h < th or w < tw:
        pt, pl = (th - h) // 2, (tw - w) // 2
        x = _to_nhwc(F.pad(_to_nchw(x), (pl, tw - w - pl, pt, th - h - pt)))
    return x


def _resize_axis_coeffs(in_size, out_size, dtype, device=None):
    # TF 1.x legacy bilinear (align_corners=False, no half-pixel centres):
    # scale = in/out (float32); src = dst*scale; lo=floor(src); hi=min(lo+1,in-1); lerp=src-lo
    scale = torch.tensor(in_size / out_size, dtype=torch.float32)
    dst = torch.arange(out_size, dtype=torch.float32)
    src = dst * scale
    lo = torch.floor(src)
    hi = torch.clamp(lo + 1, max=in_size - 1)
    lerp = (src - lo).to(dtype)
    return lo.long().to(device), hi.long().to(device), lerp.to(device)


def resize_bilinear(x, oh, ow):
    """tf.image.resize_images(x,[oh,ow]) TF-1.12 legacy bilinear (Nets/MadNet.py:69,274,...,362).

    Identity when sizes already match.  Differentiable (gather => scatter-add transpose).
    """
    h, w = x.shape[1], x.shape[2]
    if h == oh and w == ow:
        return x
    ylo, yhi, yl = _resize_axis_coeffs(h, oh, x.dtype, x.device)
    xlo, xhi, xl = _resize_axis_coeffs(w, ow, x.dtype, x.device)
    top = x[:, ylo]
    bot = x[:, yhi]
    xl = xl.view(1, 1, -1, 1)
    yl = yl.view(1, -1, 1, 1)
    tl, tr = top[:, :, xlo], top[:, :, xhi]
    bl, br = bot[:, :, xlo], bot[:, :, xhi]
    t = tl + (tr - tl) * xl
    bt = bl + (br - bl) * xl
    return t + (bt - t) * yl


def correlation(x, y, max_disp, stride=1):
    """sharedLayers.correlation_tf (Nets/sharedLayers.py:41-51).

    out[b,h,w,i] = mean_c x[b,h,w,c] * y[b,h,w+(i*stride-max_disp),c], zero outside.
    """
    w = x.shape[2]
    yp = _to_nhwc(F.pad(_to_nchw(y), (max_disp, max_disp, 0, 0)))
    outs = []
    for i in range(-max_disp, max_disp + 1, stride):
        shifted = yp[:, :, i + max_disp:i + max_disp + w]
        outs.append((shifted * x).mean(dim=-1, keepdim=True))
    return torch.cat(outs, dim=-1)


def linear_warp(feat, u):
    """MadNet._build_indeces + _linear_warping (Nets/MadNet.py:378-436).

    feat [B,h,w,C], u [B,h,w,1] = horizontal offset in pixels (cx = x + u); rows never move.
    Taps falling outside [0,w-1] get weight 0 (weights masked, indices clamped).
    """
    b, h, w, c = feat.shape
    xs = torch.arange(w, dtype=feat.dtype, device=feat.device).view(1, 1, w, 1)
    cx = xs + u
    x0 = torch.floor(cx)
    x1 = x0 + 1
    x0s = torch.clamp(x0, 0, w - 1)
    x1s = torch.clamp(x1, 0, w - 1)
    wt0 = (x1 - cx) * (x0 == x0s).to(feat.dtype)
    wt1 = (cx - x0) * (x1 == x1s).to(feat.dtype)
    i0 = x0s.long().expand(b, h, w, c)
    i1 = x1s.long().expand(b, h, w, c)
    im0 = torch.gather(feat, 2, i0)
    im1 = torch.gather(feat, 2, i1)
    return wt0 * im0 + wt1 * im1


def warp_image(img, disp):
    """preprocessing.warp_image + bilinear_sampler (Data_utils/preprocessing.py:121-230).

    Samples img at (x - disp, y) with CLAMPED indices and UNMASKED weights.  y is integral, so
    wt_y1 == 0 and only the row itself contributes.
    """
    b, h, w, c = img.shape
    xs = torch.arange(w, dtype=img.dtype, device=img.device).view(1, 1, w, 1)
    cx = xs - disp
    x0 = torch.floor(cx)
    x1 = x0 + 1
    wt0 = x1 - cx
    wt1 = cx - x0
    i0 = torch.clamp(x0, 0, w - 1).long().expand(b, h, w, c)
    i1 = torch.clamp(x1, 0, w - 1).long().expand(b, h, w, c)
    return wt0 * torch.gather(img, 2, i0) + wt1 * torch.gather(img, 2, i1)


def _avg_pool3_valid(x):
    return _to_nhwc(F.avg_pool2d(_to_nchw(x), 3, 1))


def ssim(x, y):
    """Losses/loss_factory.py:128-149 (3x3 VALID avg pools, C1=1e-4, C2=9e-4, clip((1-S)/2,0,1))."""
    c1, c2 = 0.01 ** 2, 0.03 ** 2
    mu_x = _avg_pool3_valid(x)
    mu_y = _avg_pool3_valid(y)
    sigma_x = _avg_pool3_valid(x ** 2) - mu_x ** 2
    sigma_y = _avg_pool3_valid(y ** 2) - mu_y ** 2
    sigma_xy = _avg_pool3_valid(x * y) - mu_x * mu_y
    n = (2 * mu_x * mu_y + c1) * (2 * sigma_xy + c2)
    d = (mu_x ** 2 + mu_y ** 2 + c1) * (sigma_x + sigma_y + c2)
    return torch.clamp((1 - n / d) / 2, 0, 1)


def mean_ssim_l1(x, y):
    """Losses/loss_factory.py:156-164, :28-38."""
    return 0.85 * ssim(x, y).mean() + 0.15 * (x - y).abs().mean()


def reprojection_loss(disp, left, right):
    """loss_factory.get_reprojection_loss('mean_SSIM_l1') single-scale (Losses/loss_factory.py:353-395).

    disp [B,H',W',1]; left/right [B,H,W,3] in 0..255.  Disparity is resized to the image size and
    multiplied by W_img/W_disp (=1 on the adaptation path).
    """
    left = left / 256.0
    right = right / 256.0
    scale = left.shape[2] / disp.shape[2]
    d = resize_bilinear(disp, left.shape[1], left.shape[2]) * scale
    return mean_ssim_l1(warp_image(right, d), left)


def momentum_update(w, g, m, lr, mu=0.9):
    """tf.train.MomentumOptimizer (Stereo_Online_Adaptation.py:85): m = mu*m + g ; w -= lr*m."""
    m_new = mu * m + g
    return w - lr * m_new, m_new


def xavier_uniform(rng, shape):
    """tf.contrib.layers.xavier_initializer (Nets/sharedLayers.py:4): U(-l,l), l=sqrt(6/(fan_in+fan_out))."""
    kh, kw, a, b = shape
    limit = math.sqrt(6.0 / (kh * kw * a + kh * kw * b))
    return rng.uniform(-limit, limit, size=shape).astype('float32')


def proxy_loss(disp, proxy, weight):
    """Losses/loss_factory.py:304-351 get_proxy_loss('mean_l1') for ONE prediction already at the proxy's resolution
    (resize_to_prediction is the identity, disparity_scale_factor 1): valid = !(proxy <= 0 | proxy >= 192);
    weight * sum(valid * |disp - proxy|) / sum(valid)   (:28-38 mean_l1).  No valid pixel: 0 (the reference gives nan)."""
    valid = (~((proxy <= 0) | (proxy >= 192))).to(disp.dtype)
    cnt = valid.sum()
    if float(cnt) == 0.0:
        return disp.sum() * 0.0
    return weight * (valid * (disp - proxy).abs()).sum() / cnt
