"""DispNet-C on the H100 engine — host-side mirror of the reference class (Nets/DispNet.py:9-152).

Same construction API / argument validation (DispNet.py:23-37) / layer names (`conv1a`, `conv3/1`, `up5/deconv`, ...)
and `get_disparities()` ordering (5 side predictions, `prediction`, `rescaled_prediction`).  The graph itself
(:75-152) runs in libmadstereo (csrc/engine_dispnet.cu).  Only the correlation=True variant is built (the one the
adaptation drivers and block_config/dispnet_full.json use).
"""
from Nets import Stereo_net
from Nets.Stereo_net import LayerHandle, Variable
from madstereo.engine import StereoEngine

MAX_DISP = 40


class DispNet(Stereo_net.StereoNet):
    _valid_args = [
        ("left_img", "device buffer [B,H,W,3] for the left image batch"),
        ("right_img", "device buffer [B,H,W,3] for the right image batch"),
        ("correlation", "flag to enable the use of the correlation layer"),
    ] + Stereo_net.StereoNet._valid_args
    _netName = "Dispnet"

    def __init__(self, **kwargs):
        super(DispNet, self).__init__(**kwargs)

    def _validate_args(self, args):
        super(DispNet, self)._validate_args(args)
        if ("left_img" not in args) or ("right_img" not in args):
            raise Exception('Missing input op for left and right images')
        if "correlation" not in args:
            print('WARNING: Correlation unspecified, setting to True')
            args['correlation'] = True
        if not args['correlation']:
            raise Exception('correlation=False (plain DispNet-S) is not built in this engine')
        return args

    def _preprocess_inputs(self, args):
        self._left_input_batch = args['left_img']
        self._right_input_batch = args['right_img']
        shp = tuple(self._left_input_batch.shape)
        if len(shp) != 4 or shp[3] != 3 or tuple(self._right_input_batch.shape) != shp:
            raise Exception('left_img/right_img must be [B,H,W,3] buffers of equal shape')
        self._restore_shape = shp[1:3]
        self._padded_shape = tuple(-(-s // 64) * 64 for s in shp[1:3])     # pad_image(., 64), DispNet.py:59-73

    def _build_network(self, args):
        b, h, w, _ = tuple(self._left_input_batch.shape)
        self.bulkhead = False
        self.engine = eng = StereoEngine(self._netName, b, h, w, radius_d=MAX_DISP, stride=1, warping=False,
                                         device=getattr(self._left_input_batch, 'device', None))
        hp, wp = self._padded_shape
        self._vars_of_layer = {}
        all_vars = []

        def variables(l):
            vs = [Variable(l.scope + '/weights', eng, l.scope + '/weights'),
                  Variable(l.scope + '/' + l.bias_name, eng, l.scope + '/' + l.bias_name)]
            self._vars_of_layer[l.index] = vs
            all_vars.extend(vs)
            return vs

        L = eng.layer_by_name
        hh, ww = hp // 2, wp // 2
        self._add_to_layers('conv1a', LayerHandle(self, 'conv1a', (b, hh, ww, 64)), variables(L['conv1a']))
        self._add_to_layers('conv1b', LayerHandle(self, 'conv1b', (b, hh, ww, 64)), [])       # reuse scope: no vars
        hh, ww = hp // 4, wp // 4
        self._add_to_layers('conv2a', LayerHandle(self, 'conv2a', (b, hh, ww, 128)), variables(L['conv2a']))
        self._add_to_layers('conv2b', LayerHandle(self, 'conv2b', (b, hh, ww, 128)), [])
        self._add_to_layers('conv_redir', LayerHandle(self, 'conv_redir', (b, hh, ww, 64)), variables(L['conv_redir']))
        self._add_to_layers('corr', LayerHandle(self, 'corr', (b, hh, ww, 2 * MAX_DISP + 1)), [])
        for name in ('conv3', 'conv3/1', 'conv4', 'conv4/1', 'conv5', 'conv5/1', 'conv6', 'conv6/1'):
            l = L[name]
            if l.stride == 2:
                hh, ww = hh // 2, ww // 2
            self._add_to_layers(name, LayerHandle(self, name, (b, hh, ww, l.cout)), variables(l))
        for k, up in enumerate(('up5', 'up4', 'up3', 'up2', 'up1')):
            dec = L[up + '/deconv']
            self._add_to_layers(up + '/deconv', LayerHandle(self, up + '/deconv', (b, 2 * hh, 2 * ww, dec.cout)), variables(dec))
            self._add_to_layers(up + '/predict', LayerHandle(self, up + '/predict', (b, hh, ww, 1)), variables(L[up + '/predict']))
            self._disparities.append(LayerHandle(self, 'disparity_' + up, (b, h, w, 1), 'disp%d' % k))
            self._add_to_layers(up + '/up_predict', LayerHandle(self, up + '/up_predict', (b, 2 * hh, 2 * ww, 1)),
                                variables(L[up + '/up_predict']))
            self._add_to_layers(up + '/concat', LayerHandle(self, up + '/concat', (b, 2 * hh, 2 * ww, dec.cout)),
                                variables(L[up + '/concat']))
            hh, ww = 2 * hh, 2 * ww
        self._add_to_layers('prediction', LayerHandle(self, 'prediction', (b, hh, ww, 1)), variables(L['prediction']))
        self._disparities.append(LayerHandle(self, 'disparity_prediction', (b, h, w, 1), 'disp5'))
        resc = LayerHandle(self, 'rescaled_prediction', (b, h, w, 1), 'disp6')
        self._layers['rescaled_prediction'] = resc
        self._disparities.append(resc)
        self._all_variables = all_vars

    def layer_index_of_variable(self, var):
        for idx, vs in self._vars_of_layer.items():
            if any(v is var or v.name == var.name for v in vs):
                return idx
        raise KeyError(var.name)
