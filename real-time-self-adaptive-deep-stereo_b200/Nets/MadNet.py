"""MADNet on the H100 engine — host-side mirror of the reference class (Nets/MadNet.py:8-436).

Construction API, argument validation, layer names and `get_disparities()` ordering follow the reference;
the graph itself (pyramid :173-249, warp/correlation/estimator loop :251-351, context net :122-171, outputs
:68-71,:362-364) is executed by libmadstereo's C++ engine (csrc/engine.cu).
"""
from Nets import Stereo_net
from Nets.Stereo_net import LayerHandle, Variable
from madstereo.engine import StereoEngine


class MadNet(Stereo_net.StereoNet):
    _valid_args = [
        ("left_img", "device buffer [B,H,W,3] for the left image batch"),
        ("right_img", "device buffer [B,H,W,3] for the right image batch"),
        ("warping", "flag to enable warping"),
        ("context_net", "flag to enable context_net"),
        ("radius_d", "size f the patch using for correlation"),
        ("stride", "stride used for correlation"),
        ("bulkhead", "flag to stop gradient propagation among different resolution"),
    ] + Stereo_net.StereoNet._valid_args
    _netName = "MADNet"

    def __init__(self, **kwargs):
        super(MadNet, self).__init__(**kwargs)

    def _validate_args(self, args):
        super(MadNet, self)._validate_args(args)
        if ('left_img' not in args) or ('right_img' not in args):
            raise Exception('Missing input op for left and right images')
        if 'warping' not in args:
            print('WARNING: warping flag not setted, setting default True value')
            args['warping'] = True
        if 'context_net' not in args:
            print('WARNING: context_net flag not setted, setting default True value')
            args['context_net'] = True
        if 'radius_d' not in args:
            print('WARNING: radius_d not setted, setting default value 2')
            args['radius_d'] = 2
        if 'stride' not in args:
            print('WARNING: stride not setted, setting default value 1')
            args['stride'] = 1
        if 'bulkhead' not in args:
            args['bulkhead'] = False
        if not args['context_net']:
            # the reference's context_net=False branch references an undefined name (MadNet.py:360)
            raise Exception('context_net=False is broken in the reference (Nets/MadNet.py:360) and unsupported')
        return args

    def _preprocess_inputs(self, args):
        self._left_input_batch = args['left_img']
        self._right_input_batch = args['right_img']
        shp = tuple(self._left_input_batch.shape)
        if len(shp) != 4 or shp[3] != 3 or tuple(self._right_input_batch.shape) != shp:
            raise Exception('left_img/right_img must be [B,H,W,3] buffers of equal shape')
        self._restore_shape = shp[1:3]
        self._padded_shape = tuple(-(-s // 64) * 64 for s in shp[1:3])   # pad_image(.,64), MadNet.py:56-66

    def _build_network(self, args):
        b, h, w, _ = tuple(self._left_input_batch.shape)
        self.bulkhead = bool(args['bulkhead'])
        self.engine = eng = StereoEngine(self._netName, b, h, w, radius_d=args['radius_d'],
                                         stride=args['stride'], warping=bool(args['warping']),
                                         device=getattr(self._left_input_batch, 'device', None))
        hp, wp = self._padded_shape
        self._vars_of_layer = {}

        def variables(l):
            return [Variable(l.scope + '/weights', eng, l.scope + '/weights'),
                    Variable(l.scope + '/' + l.bias_name, eng, l.scope + '/' + l.bias_name)]

        all_vars = []
        pyr = [l for l in eng.layers if l.name.startswith('left/conv')]
        for prefix in ('left', 'right'):
            hh, ww = hp, wp
            for l in pyr:
                if l.stride == 2:
                    hh, ww = -(-hh // 2), -(-ww // 2)
                name = l.name.replace('left', prefix)
                vs = variables(l) if prefix == 'left' else []       # reuse scope matches no variable
                if prefix == 'left':
                    self._vars_of_layer[l.index] = vs
                    all_vars += vs
                self._add_to_layers(name, LayerHandle(self, name, (b, hh, ww, l.cout)), vs)
        for k in (6, 5, 4, 3, 2):
            hh, ww = hp // 2 ** k, wp // 2 ** k
            for j in range(1, 7):
                l = eng.layer_by_name['fgc-volume-filtering-%d/disp%d' % (k, j)]
                vs = variables(l)
                self._vars_of_layer[l.index] = vs
                all_vars += vs
                self._add_to_layers(l.name, LayerHandle(self, l.name, (b, hh, ww, l.cout)), vs)
            if k > 2:
                d = LayerHandle(self, 'disparity_%d' % k, (b, h, w, 1), 'disp%d' % (6 - k))
                self._disparities.append(d)
        for j in range(1, 8):
            l = eng.layer_by_name['context%d' % j]
            vs = variables(l)
            self._vars_of_layer[l.index] = vs
            all_vars += vs
            tname = l.name if j < 7 else 'final_disp'   # context7's own output is fused into final_disp
            self._add_to_layers(l.name, LayerHandle(self, l.name, (b, hp // 4, wp // 4, l.cout), tname), vs)
        # 'final_disp' is an add op directly under scope 'model' => prefix-matches every variable (Stereo_net.py:63-67)
        self._add_to_layers('final_disp', LayerHandle(self, 'final_disp', (b, hp // 4, wp // 4, 1)), list(all_vars))
        self._disparities.append(LayerHandle(self, 'disparity_2_context', (b, h, w, 1), 'disp4'))
        resc = LayerHandle(self, 'rescaled_prediction', (b, h, w, 1), 'disp5')
        self._layers['rescaled_prediction'] = resc          # set directly, no variables (MadNet.py:363)
        self._disparities.append(resc)
        self._all_variables = all_vars

    def layer_index_of_variable(self, var):
        for idx, vs in self._vars_of_layer.items():
            if any(v is var or v.name == var.name for v in vs):
                return idx
        raise KeyError(var.name)
