"""Python handle on the C++ engine (csrc/engine.cu) — torch CUDA tensors are memory containers only.

The engine replaces the single `sess.run(tf_fetches)` of the reference inner loop
(Stereo_Online_Adaptation.py:194-208): forward of the whole net, full-resolution reprojection loss, and the
selected train op (MAD module or FULL) with its momentum update, all as hand-written CUDA.
"""
import ctypes
from collections import OrderedDict, namedtuple
from ctypes import byref, c_float, c_int, c_size_t, c_void_p

import numpy as np
import torch

from ._lib import MadStereoError, check, lib

LayerInfo = namedtuple('LayerInfo', 'index name scope bias_name kh kw cin cout stride dilation transposed alpha')

MODE_NONE, MODE_MAD, MODE_FULL = 0, 1, 2


class _NullCtx(object):
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


_NULL_CTX = _NullCtx()


def _stream():
    return c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return c_void_p(t.data_ptr()) if t is not None else c_void_p(0)


class StereoEngine:
    def __init__(self, net_name, batch, height, width, radius_d=2, stride=1, warping=True, device=None):
        if not torch.cuda.is_available():
            raise MadStereoError('a CUDA device is required: libmadstereo has no CPU fallback')
        self.device = torch.device(device if device is not None else 'cuda:%d' % torch.cuda.current_device())
        self._lib = lib()
        self._dev_index = self.device.index if self.device.index is not None else torch.cuda.current_device()
        self.net_name, self.B, self.H, self.W = net_name, batch, height, width
        with self._on_device():
            self._h = self._lib.ms_engine_create(net_name.encode(), batch, height, width, radius_d, stride,
                                                 1 if warping else 0)
        if not self._h:
            raise MadStereoError('ms_engine_create: %s' % self._lib.ms_last_error().decode())
        self.layers = []
        n = self._lib.ms_engine_num_layers(self._h)
        for i in range(n):
            nm, sc, bn = (ctypes.create_string_buffer(128) for _ in range(3))
            dims = (c_int * 7)()
            alpha = c_float()
            check(self._lib.ms_engine_layer_info(self._h, i, nm, 128, sc, 128, bn, 128, dims, byref(alpha)), 'layer_info')
            self.layers.append(LayerInfo(i, nm.value.decode(), sc.value.decode(), bn.value.decode(), *list(dims),
                                         alpha.value))
        self.layer_by_name = {l.name: l for l in self.layers}
        self.n_groups = 0
        self.bound = False
        self._keep = []
        self.optimizer = 'momentum'
        self.resize_shape = None      # set_resize(): None = uint8 frames must be [B,H,W,3]; else (rh, rw), -1 = no rescale
        self._rs_stage = None
        self._rect = None             # set_rectification(): (left table, right table, scratch) the engine reads per frame
        self.reprojection_scale = 1
        self._rs_scratch = None       # set_reprojection_scale(): the loss-resolution buffers and tap tables

    def _on_device(self):
        """Context that makes this engine's GPU current -- a no-op object when it already is (the per-frame calls of a
        one-process-per-GPU run: entering torch.cuda.device() costs ~10 us of host time on the frame's critical path)."""
        if torch.cuda.current_device() == self._dev_index:
            return _NULL_CTX
        return torch.cuda.device(self.device)

    def __del__(self):
        try:
            if getattr(self, '_h', None):
                self._lib.ms_engine_destroy(self._h)
                self._h = None
        except Exception:
            pass

    # ---- construction ----------------------------------------------------------------------
    def set_groups(self, groups):
        """groups: list (one per MAD module) of lists of layer indices. Must be called before bind()."""
        arr = (c_int * len(self.layers))(*([-1] * len(self.layers)))
        for g, idxs in enumerate(groups):
            for i in idxs:
                if arr[i] != -1 and arr[i] != g:
                    raise MadStereoError('layer %s appears in two MAD groups: unsupported' % self.layers[i].name)
                arr[i] = g
        check(self._lib.ms_engine_set_groups(self._h, arr, len(self.layers), len(groups)), 'set_groups')
        self.n_groups = len(groups)

    def bind(self):
        npar, nws = c_size_t(), c_size_t()
        check(self._lib.ms_engine_sizes(self._h, byref(npar), byref(nws)), 'sizes')
        self.n_params = npar.value
        dev = self.device
        self.weights = torch.zeros(self.n_params, dtype=torch.float32, device=dev)
        self.grads = torch.zeros(self.n_params, dtype=torch.float32, device=dev)
        self.momentum = torch.zeros(self.n_params, dtype=torch.float32, device=dev)
        self.workspace = torch.empty(nws.value, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            check(self._lib.ms_engine_bind(self._h, _ptr(self.weights), _ptr(self.grads), _ptr(self.momentum),
                                           _ptr(self.workspace), nws.value, _stream()), 'bind')
        self.bound = True
        self.param_offsets = {}
        for l in self.layers:
            wo, bo = c_size_t(), c_size_t()
            check(self._lib.ms_engine_param_offsets(self._h, l.index, byref(wo), byref(bo)), 'param_offsets')
            self.param_offsets[l.index] = (wo.value, bo.value)
        self.group_ranges = []
        for g in range(self.n_groups):
            b, e = c_size_t(), c_size_t()
            check(self._lib.ms_engine_group_range(self._h, g, byref(b), byref(e)), 'group_range')
            self.group_ranges.append((b.value, e.value))

    def weight_shape(self, l):
        return (l.kh, l.kw, l.cout, l.cin) if l.transposed else (l.kh, l.kw, l.cin, l.cout)

    def param_views(self, arena=None):
        """OrderedDict TF-variable-name -> torch view (HWIO weights / [cout] bias) into an arena."""
        arena = self.weights if arena is None else arena
        out = OrderedDict()
        for l in self.layers:
            wo, bo = self.param_offsets[l.index]
            shp = self.weight_shape(l)
            out[l.scope + '/weights'] = arena[wo:wo + int(np.prod(shp))].view(*shp)
            out[l.scope + '/' + l.bias_name] = arena[bo:bo + l.cout]
        return out

    def load_params(self, params, strict=True):
        """strict=False: parameters absent from `params` keep their current values (tf.train.Saver with a partial
        var_list, Data_utils/weights_utils.py:27-37)."""
        views = self.param_views()
        for k, v in views.items():
            if k not in params:
                if strict:
                    raise MadStereoError('missing parameter %s' % k)
                continue
            v.copy_(torch.as_tensor(np.asarray(params[k]), dtype=torch.float32).to(self.device).reshape(v.shape))
        self.weights_changed()

    def export_params(self, arena=None):
        return OrderedDict((k, v.detach().cpu().numpy().copy()) for k, v in self.param_views(arena).items())

    # ---- per-frame calls ---------------------------------------------------------------------
    def set_input(self, left, right):
        """left/right: [B,H,W,3] float32 torch tensors (CUDA, or pinned/pageable CPU) or numpy arrays.  After set_resize(),
        uint8 frames [B,h,w,3] of any size are rescaled and centre-cropped / zero-padded to [B,H,W,3] on the device."""
        if self.resize_shape is not None and self._is_u8(left) and self._is_u8(right):
            self._set_input_resized(left, right)
            return
        if self._is_u8(left) and self._is_u8(right):
            l, r = self._as_u8(left), self._as_u8(right)
            self._keep = [l, r]
            with self._on_device():
                check(self._lib.ms_engine_set_input_u8(self._h, _ptr(l), _ptr(r), _stream()), 'set_input_u8')
            return
        l, r = self._as_f32(left), self._as_f32(right)
        self._keep = [l, r]
        with self._on_device():
            check(self._lib.ms_engine_set_input(self._h, _ptr(l), _ptr(r), _stream()), 'set_input')

    def set_resize(self, image_shape=(-1, -1)):
        """Accept uint8 frames of any size from now on, as the live demo feeds them (Demo/demo_model.py:80-86): a legacy
        bilinear rescale to image_shape = (rh, rw) (tf.image.resize_images, align_corners=False), then
        tf.image.resize_image_with_crop_or_pad to the engine's (H, W).  (-1, -1) skips the rescale; None turns the
        geometry off again (uint8 frames must then be exactly [B,H,W,3])."""
        if image_shape is not None:
            image_shape = tuple(int(v) for v in image_shape)
            if len(image_shape) != 2 or (min(image_shape) < 1 and image_shape != (-1, -1)):
                raise MadStereoError('set_resize: image_shape must be (height, width) or (-1, -1), got %r' % (image_shape,))
        elif self._rect is not None:
            raise MadStereoError('set_resize(None): turn rectification off first (set_rectification(None))')
        self.resize_shape = image_shape

    def set_rectification(self, map_left, map_right=None):
        """Rectify the uint8 camera frames of the set_resize() path on the device before they are rescaled: map_left /
        map_right are float32 [h,w,2] remap tables, map[y, x] = (src_x, src_y), as cv2.initUndistortRectifyMap(...,
        cv2.CV_32FC1) returns them stacked (madstereo.rectify builds them from a stereo calibration); frames must then be
        [B,h,w,3].  Bilinear, 0 outside the frame, rounded back to uint8 (what cv2.remap gives, up to OpenCV's 1/32-pixel
        fixed point).  None turns rectification off."""
        if map_left is None:
            with self._on_device():
                check(self._lib.ms_engine_set_rectification(self._h, c_void_p(0), c_void_p(0), 0, 0, c_void_p(0), 0),
                      'set_rectification')
            self._rect = None
            return
        if self.resize_shape is None:
            raise MadStereoError('set_rectification: rectification applies to the set_resize() input path; call set_resize first')
        maps = []
        for m in (map_left, map_right):
            if m is None:
                raise MadStereoError('set_rectification: each camera needs a table')
            m = torch.as_tensor(m)
            if m.dtype != torch.float32 or m.dim() != 3 or m.shape[2] != 2:
                raise MadStereoError('set_rectification: tables must be float32 [h,w,2], got %s %s' % (m.dtype, tuple(m.shape)))
            maps.append(m.to(self.device).contiguous())
        if maps[0].shape != maps[1].shape:
            raise MadStereoError('set_rectification: left %s and right %s tables differ in size'
                                 % (tuple(maps[0].shape), tuple(maps[1].shape)))
        h, w = int(maps[0].shape[0]), int(maps[0].shape[1])
        scratch = torch.empty(2 * self.B * h * w * 3, dtype=torch.uint8, device=self.device)
        with self._on_device():
            check(self._lib.ms_engine_set_rectification(self._h, _ptr(maps[0]), _ptr(maps[1]), h, w, _ptr(scratch),
                                                        scratch.numel()), 'set_rectification')
        self._rect = (maps[0], maps[1], scratch)      # the engine reads them on every frame

    def _u8_source(self, x):
        """uint8 [B,h,w,3] frame -> contiguous CUDA tensor on this engine's device (host frames are copied on the current
        stream into a staging buffer of the source size; pinned ones asynchronously)."""
        if isinstance(x, np.ndarray):
            x = torch.from_numpy(np.ascontiguousarray(x))
        if x.dim() != 4 or x.shape[0] != self.B or x.shape[3] != 3:
            raise MadStereoError('input shape %s is not [%d,h,w,3]' % (tuple(x.shape), self.B))
        if x.is_cuda and x.device != self.device:
            raise MadStereoError('input on %s, engine on %s' % (x.device, self.device))
        return x.contiguous()

    def _set_input_resized(self, left, right):
        l, r = self._u8_source(left), self._u8_source(right)
        if tuple(l.shape) != tuple(r.shape):
            raise MadStereoError('left %s and right %s frames differ in size' % (tuple(l.shape), tuple(r.shape)))
        h, w = int(l.shape[1]), int(l.shape[2])
        rh, rw = (h, w) if self.resize_shape == (-1, -1) else self.resize_shape
        self._keep_host = [l, r]              # a pinned source must outlive its asynchronous copy
        if not l.is_cuda or not r.is_cuda:
            shape = (2,) + tuple(l.shape)
            if self._rs_stage is None or tuple(self._rs_stage.shape) != shape:
                self._rs_stage = torch.empty(shape, dtype=torch.uint8, device=self.device)
            self._rs_stage[0].copy_(l, non_blocking=l.is_pinned())
            self._rs_stage[1].copy_(r, non_blocking=r.is_pinned())
            l, r = self._rs_stage[0], self._rs_stage[1]
        self._keep = [l, r]
        with self._on_device():
            check(self._lib.ms_engine_set_input_u8_resized(self._h, _ptr(l), _ptr(r), h, w, rh, rw, _stream()),
                  'set_input_u8_resized')

    def set_optimizer(self, kind, beta1=0.9, beta2=0.999, epsilon=1e-8):
        """'momentum' (tf.train.MomentumOptimizer, the default) or 'adam' (tf.train.AdamOptimizer, Demo/demo_model.py:163).
        Adam keeps its first moment in the momentum arena, its second moment in `adam_v` and the shared bias-correction
        powers [beta1_power, beta2_power] in `adam_powers` (start: beta1, beta2; advanced on the device by every update).
        Changing the optimizer drops the captured step graphs."""
        if not self.bound:
            raise MadStereoError('set_optimizer: bind() first')
        if kind == 'momentum':
            check(self._lib.ms_engine_set_optimizer(self._h, 0, 0.0, 0.0, 0.0, c_void_p(0), c_void_p(0)), 'set_optimizer')
        elif kind == 'adam':
            if getattr(self, 'adam_v', None) is None:
                self.adam_v = torch.zeros(self.n_params, dtype=torch.float32, device=self.device)
                self.adam_powers = torch.tensor([beta1, beta2], dtype=torch.float32, device=self.device)
            check(self._lib.ms_engine_set_optimizer(self._h, 1, beta1, beta2, epsilon, _ptr(self.adam_v),
                                                    _ptr(self.adam_powers)), 'set_optimizer')
            self.adam_betas = (float(beta1), float(beta2), float(epsilon))
        else:
            raise MadStereoError("set_optimizer: kind must be 'momentum' or 'adam', got %r" % (kind,))
        self.optimizer = kind

    @staticmethod
    def _is_u8(x):
        return (isinstance(x, np.ndarray) and x.dtype == np.uint8) or (torch.is_tensor(x) and x.dtype == torch.uint8)

    def _as_u8(self, x, c=3):
        if isinstance(x, np.ndarray):
            x = torch.from_numpy(np.ascontiguousarray(x))
        if not x.is_contiguous():
            x = x.contiguous()
        if tuple(x.shape) != (self.B, self.H, self.W, c):
            raise MadStereoError('input shape %s != %s' % (tuple(x.shape), (self.B, self.H, self.W, c)))
        return x

    def set_gt(self, gt):
        g = self._as_f32(gt, 1)
        self._keep_gt = g
        with self._on_device():
            check(self._lib.ms_engine_set_gt(self._h, _ptr(g), _stream()), 'set_gt')

    def set_proxy(self, proxy):
        """Proxy disparities [B,H,W,1] of the continual-adaptation variant (Stereo_Continual_Adaptation.py:54)."""
        g = self._as_f32(proxy, 1)
        self._keep_proxy = g
        with self._on_device():
            check(self._lib.ms_engine_set_proxy(self._h, _ptr(g), _stream()), 'set_proxy')

    def set_loss(self, kind, weight_full=0.01, weight_module=0.1):
        """kind: 'reprojection' (SSIM + L1, Stereo_Online_Adaptation.py) or 'proxy' (masked L1 to proxy labels)."""
        k = {'reprojection': 0, 'proxy': 1}[kind]
        check(self._lib.ms_engine_set_loss(self._h, k, weight_full, weight_module), 'set_loss')

    def set_reprojection_scale(self, scale):
        """Compute the MAD module losses at 1/scale resolution, as the reference's --reprojectionScale does: frames (or the
        proxy, divided by scale) and the module disparity resized to (H // scale, W // scale).  The disparity keeps its
        full-resolution units there, as in the reference.  The full-resolution loss, FULL and NONE are unchanged.  1 turns
        it off.  MADNet only; needs bind().  Changing the scale drops the captured step graphs."""
        scale = int(scale)
        if not self.bound:
            raise MadStereoError('set_reprojection_scale: bind() first')
        if scale == 1:
            check(self._lib.ms_engine_set_reprojection_scale(self._h, 1, c_void_p(0), 0), 'set_reprojection_scale')
            self.reprojection_scale, self._rs_scratch = 1, None
            return
        n = self._lib.ms_engine_reprojection_scratch_floats(self._h, scale)
        if n == 0:
            raise MadStereoError('set_reprojection_scale: %s' % self._lib.ms_last_error().decode())
        scratch = torch.empty(n, dtype=torch.float32, device=self.device)
        with self._on_device():
            check(self._lib.ms_engine_set_reprojection_scale(self._h, scale, _ptr(scratch), n), 'set_reprojection_scale')
        self.reprojection_scale, self._rs_scratch = scale, scratch

    def _as_f32(self, x, c=3):
        if isinstance(x, np.ndarray):
            x = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32))
        if x.dtype != torch.float32 or not x.is_contiguous():
            x = x.to(torch.float32).contiguous()
        if tuple(x.shape) != (self.B, self.H, self.W, c):
            raise MadStereoError('input shape %s != %s' % (tuple(x.shape), (self.B, self.H, self.W, c)))
        return x

    def forward(self, disp_mask=0b100000):
        with self._on_device():
            check(self._lib.ms_engine_forward(self._h, disp_mask, _stream()), 'forward')

    def loss(self, which, with_grad, slot, grad_scale=1.0):
        with self._on_device():
            check(self._lib.ms_engine_loss(self._h, which, 1 if with_grad else 0, slot, grad_scale, _stream()), 'loss')

    def backward(self, mode, group=0):
        with self._on_device():
            check(self._lib.ms_engine_backward(self._h, mode, group, _stream()), 'backward')

    def update(self, group, lr, mu=0.9, grad_scale=1.0):
        with self._on_device():
            check(self._lib.ms_engine_update(self._h, group, lr, mu, grad_scale, _stream()), 'update')

    def run(self, mode, group=0, disp_mask=0, with_update=True, lr=1e-4, mu=0.9, grad_scale=1.0):
        """One whole frame (forward, full-res loss, train op) — replayed as a single CUDA graph."""
        with self._on_device():
            check(self._lib.ms_engine_run(self._h, mode, group, disp_mask, int(with_update), lr, mu, grad_scale,
                                          _stream()), 'run')

    # ---- data parallel: gradient exchange over NVLink peer memory fused with the update (csrc/dp.cu) ----------
    def dp_setup(self, rank, world, process_group=None):
        """Allocate this rank's exchange buffer, all-gather the CUDA IPC handles through torch.distributed (plumbing
        only) and map every peer.  Afterwards run(..., with_update=2) performs all-reduce + momentum update in-graph."""
        import torch.distributed as dist
        mine = (ctypes.c_ubyte * 128)()
        with self._on_device():
            check(self._lib.ms_engine_dp_create(self._h, rank, world, mine), 'dp_create')
        gathered = [None] * world
        dist.all_gather_object(gathered, bytes(mine), group=process_group)
        blob = (ctypes.c_ubyte * (128 * world)).from_buffer_copy(b''.join(gathered))
        with self._on_device():
            check(self._lib.ms_engine_dp_connect(self._h, blob), 'dp_connect')
        dist.barrier(group=process_group)

    def dp_error(self):
        out = ctypes.c_uint(0)
        check(self._lib.ms_engine_dp_error(self._h, byref(out)), 'dp_error')
        return int(out.value)

    def weights_changed(self):
        """Call after writing the weight arena from outside (checkpoint load / reset)."""
        check(self._lib.ms_engine_weights_changed(self._h), 'weights_changed')

    def metrics(self):
        with self._on_device():
            check(self._lib.ms_engine_metrics(self._h, _stream()), 'metrics')

    def read_scalars(self):
        out = (c_float * 4)()
        with self._on_device():
            check(self._lib.ms_engine_read_scalars(self._h, out, _stream()), 'read_scalars')
        return list(out)

    # ---- profiling -----------------------------------------------------------------------------
    CATEGORIES = ('conv_fwd', 'conv_dgrad', 'conv_wgrad', 'corr_fwd', 'corr_bwd', 'loss', 'other')

    def profile(self, enable):
        """False/0 off; True/1 eager events; 2 = event nodes inside the replayed CUDA graph (in-graph kernel times)."""
        check(self._lib.ms_engine_profile(self._h, int(enable)), 'profile')

    def profile_event_overhead_us(self):
        return 1e3 * float(self._lib.ms_engine_profile_event_overhead_ms(self._h))

    def profile_layers(self):
        n = len(self.layers)
        ms = (ctypes.c_double * (3 * n))(); calls = (ctypes.c_longlong * (3 * n))()
        with self._on_device():
            check(self._lib.ms_engine_profile_layers(self._h, ms, calls), 'profile_layers')
        out = {}
        for d, name in enumerate(('fwd', 'dgrad', 'wgrad')):
            for i, l in enumerate(self.layers):
                if calls[d * n + i]:
                    out.setdefault(l.name, {})[name] = {'ms': ms[d * n + i], 'calls': calls[d * n + i]}
        return out

    def profile_read(self):
        ms, macs, byts = ((ctypes.c_double * 7)() for _ in range(3))
        calls = (ctypes.c_longlong * 7)()
        with self._on_device():
            check(self._lib.ms_engine_profile_read(self._h, ms, macs, byts, calls), 'profile_read')
        return {c: {'ms': ms[i], 'macs': macs[i], 'bytes': byts[i], 'calls': calls[i]}
                for i, c in enumerate(self.CATEGORIES)}

    def launch_count(self):
        return int(self._lib.ms_launch_count())

    # ---- introspection -------------------------------------------------------------------------
    def tensor_names(self):
        n = self._lib.ms_engine_num_tensors(self._h)
        out = []
        for i in range(n):
            b = ctypes.create_string_buffer(128)
            check(self._lib.ms_engine_tensor_name(self._h, i, b, 128), 'tensor_name')
            out.append(b.value.decode())
        return out

    def tensor_info(self, name):
        p = c_void_p()
        dims = (c_int * 5)()
        check(self._lib.ms_engine_tensor(self._h, name.encode(), byref(p), dims), 'tensor')
        return p.value, tuple(dims)

    FWD_KINDS = ('HEAD', 'ONE_CHANNEL', 'STEM', 'SMALL', 'BF', 'GEMM')
    DGRAD_KINDS = ('HEAD', 'BF', 'GEMM')
    WGRAD_KINDS = ('BF', 'STEM', 'HEAD', 'FP32')

    def layer_plan(self, i):
        """Layer i's planned kernels and views (after bind): {'fwd', 'dgrad', 'wgrad': kernel kind name, 'x', 'y', 'dpre',
        'dx': torch view [n,h,w,c] into the workspace, dx None when the layer has no input gradient}."""
        kinds = (c_int * 3)()
        ptrs = (c_void_p * 4)()
        dims = (c_int * 20)()
        check(self._lib.ms_engine_layer_plan(self._h, i, kinds, ptrs, dims), 'layer_plan')
        out = {'fwd': self.FWD_KINDS[kinds[0]], 'dgrad': self.DGRAD_KINDS[kinds[1]], 'wgrad': self.WGRAD_KINDS[kinds[2]]}
        for k, role in enumerate(('x', 'y', 'dpre', 'dx')):
            out[role] = self._view(ptrs[k], *dims[5 * k:5 * k + 5]) if ptrs[k] else None
        return out

    def tensor(self, name):
        """torch view [n,h,w,c] (strided) of an engine tensor inside the workspace."""
        p, (n, h, w, c, cs) = self.tensor_info(name)
        return self._view(p, n, h, w, c, cs)

    def _view(self, p, n, h, w, c, cs):
        base = self.workspace
        if self._rs_scratch is not None and 0 <= p - self._rs_scratch.data_ptr() < 4 * self._rs_scratch.numel():
            base = self._rs_scratch                   # rs_left / rs_right / rs_proxy / rs_disp
        off = (p - base.data_ptr()) // 4
        return base.as_strided((n, h, w, c), (h * w * cs, w * cs, cs, 1), off)
