"""Host-side mirror of the reference's abstract StereoNet (Nets/Stereo_net.py:6-222).

Same construction protocol (_validate_args -> _preprocess_inputs -> _build_network), same public getters.
What differs by design: layers / disparities / variables are handles onto device buffers owned by the C++
engine (torch CUDA tensors used purely as containers) instead of TF graph nodes, and the graph itself is
executed by libmadstereo, not by a TF session.
"""
import abc
from collections import OrderedDict


class Variable(object):
    """Stand-in for a tf.Variable: name + views of weight / gradient / momentum inside the engine arenas."""

    def __init__(self, name, engine, key):
        self.name = name + ':0'
        self.op_name = name
        self._engine, self._key = engine, key

    @property
    def shape(self):
        return tuple(self.value().shape)

    def value(self):
        return self._engine.param_views()[self._key]

    def grad(self):
        return self._engine.param_views(self._engine.grads)[self._key]

    def momentum(self):
        return self._engine.param_views(self._engine.momentum)[self._key]

    def __repr__(self):
        return "<Variable '%s' shape=%s>" % (self.name, self.shape)


class LayerHandle(object):
    """Stand-in for a TF op output: lazily resolves to the engine tensor of that name."""

    def __init__(self, net, name, shape, tensor_name=None):
        self._net, self.name, self.shape = net, name, tuple(shape)
        self._tensor_name = tensor_name or name

    def get_shape(self):
        return self.shape

    def tensor(self):
        return self._net.engine.tensor(self._tensor_name)

    def numpy(self):
        return self.tensor().detach().cpu().numpy().copy()

    def __repr__(self):
        return "<Layer '%s' shape=%s>" % (self.name, self.shape)


def _accessor(attr, doc, as_list=False):
    """Build one of the trivial public getters of the reference class (Nets/Stereo_net.py:166-211)."""
    def get(self):
        value = getattr(self, attr)
        return list(value.keys()) if as_list else value
    get.__doc__ = doc
    return get


class StereoNet(object):
    """Base class of the two networks.  Construction protocol, printed banner, `WARNING:` lines for defaulted arguments,
    `str(net)` layout and the getter names are those of the reference (the drivers rely on them:
    Stereo_Online_Adaptation.py:62-65,114); the body is a table-driven restatement."""
    __metaclass__ = abc.ABCMeta

    _netName = "stereoNet"
    _ARG_DOC = OrderedDict([
        ("split_layer", "name of the layer where the network will be splitted"),
        ("sequence", "flag to use network on a video sequence instead of on single images"),
        ("train_portion", "one among 'BEGIN' or 'END' specify which portion of the network will be trained"),
        ("is_training", "boolean or placeholder to specify if the network is in train or inference mode"),
    ])
    _valid_args = list(_ARG_DOC.items())
    # (argument, value used when absent, message printed when absent) -- Nets/Stereo_net.py:131-163
    _COMMON_DEFAULTS = (
        ('split_layers', [None], 'WARNING: no split points selected, the network will flow without interruption'),
        ('train_portion', None, 'WARNING: train_portion not specified, using default END'),
        ('sequence', False, 'WARNING: sequence flag not setted, configuring the network for single image adaptation'),
        ('is_training', False, 'WARNING: flag for trainign not setted, using default False'),
    )
    _RULE = '=' * 50

    @classmethod
    def getPossibleArsg(cls):
        return cls._valid_args

    def __init__(self, **kwargs):
        self._layers, self._trainable_variables = OrderedDict(), OrderedDict()
        self._disparities, self._placeholders, self._layer_to_var = [], [], {}
        self.engine = None
        stages = ((self._validate_args, 'Args Validated, setting up graph'),
                  (self._preprocess_inputs, 'Meta op to preprocess data created'),
                  (self._build_network, 'Network ready'))
        for line in (self._RULE, 'Starting Creation of {}'.format(self._netName), self._RULE):
            print(line)
        args = kwargs
        for index, (stage, done) in enumerate(stages):
            result = stage(args)
            if index == 0:                      # _validate_args returns the completed argument dict
                args = result
            print(done)
        print(self._RULE)

    # -- helpers used by subclasses ---------------------------------------------------------------
    def _add_to_layers(self, name, handle, variables=()):
        """Register a layer and the variables created with it (the reference captures the variable list at creation time,
        Stereo_net.py:63-67).  With split_layers == [None] every variable is trainable (:73-76)."""
        owned = list(variables)
        self._layers[name] = handle
        self._layer_to_var[name] = owned
        if self._train_beginning or self._split_layers_list != [None]:
            self._trainable_variables.update((v, True) for v in owned)

    def __str__(self):
        tag = lambda layer: "Prediction Layer" if layer in self._disparities else "Layer"   # noqa: E731
        return "".join("{} {}: {}\n".format(tag(l), k, str(l.shape)) for k, l in self._layers.items())

    __repr__ = __str__

    def __getitem__(self, key):
        return self._layers[key]

    @abc.abstractmethod
    def _preprocess_inputs(self, args):
        """Subclasses bind the input buffers here."""

    @abc.abstractmethod
    def _build_network(self, args):
        """Subclasses create the engine and register layers / disparities here."""

    @abc.abstractmethod
    def _validate_args(self, args):
        """Common arguments; subclasses call this first, add their own defaults and return `args`."""
        for key, default, message in self._COMMON_DEFAULTS:
            if key in args:
                continue
            print(message)
            if key == 'train_portion':
                default = 'END' if args['split_layers'] != [None] else 'BEGIN'
            args[key] = default
        if args['train_portion'] not in ('BEGIN', 'END'):
            raise Exception('Invalid portion options {}'.format(args['train_portion']))
        if args['split_layers'] != [None]:
            raise Exception('split_layers other than [None] is not supported by the H100 engine '
                            '(the adaptation drivers always pass [None], Stereo_Online_Adaptation.py:57)')
        self._split_layers_list = args['split_layers']
        self._train_beginning = args['train_portion'] == 'BEGIN'
        self._sequence = args['sequence']
        self._isTraining = False

    # -- public API (Nets/Stereo_net.py:166-222) ----------------------------------------------------
    get_placeholders = _accessor('_placeholders', 'placeholders of split layers (always empty: sequence mode only)')
    get_all_layers = _accessor('_layers', 'OrderedDict layer name -> handle')
    get_disparities = _accessor('_disparities', 'disparity handles, coarse to fine, last = full resolution')
    get_trainable_variables = _accessor('_trainable_variables', 'list of trainable variables', as_list=True)

    def get_layers_names(self):
        return self._layers.keys()

    def get_placeholder(self, name):
        raise Exception('Unable to find placeholder for layer {}'.format(name + '_placeholder'))

    def get_variables(self, layer_name):
        """Variables created together with `layer_name`; a layer registered without variables yields []."""
        return self._layer_to_var.get(layer_name, []) if layer_name in self._layers else self._layer_to_var[layer_name]
