"""`caffe`-shaped shim for the MNC inference path.

Mirrors the slice of pycaffe the reference's callers use (caffe-mnc/python/caffe/_caffe.cpp:217-298,
pycaffe.py:62-108; tools/demo.py:126-129,70-90; lib/caffeWrapper/TesterWrapper.py:28-44):
``set_mode_gpu``, ``set_device``, ``TEST``, ``Net(prototxt, weights, phase)`` with ``.blobs``
(OrderedDict of Blob: ``.data`` fp32 numpy, ``.reshape(*dims)``, ``.shape/.num/.channels/...``) and
``.forward(**inputs)``, plus ``caffe.Layer`` -- the base class of Python layers
(python_layer.hpp:27-46: ``param_str_``, ``setup / reshape / forward``).

``Net`` does not interpret arbitrary graphs: it accepts the MNC 5-stage test graph
(models/VGG16/mnc_5stage/test.prototxt, checked layer by layer against caffe/mnc_graph.py) and runs
it on the fused engine.  CPU mode does not exist (the reference's MNC layers are
NOT_IMPLEMENTED on CPU too: roi_warping_layer.cpp:47)."""
from collections import OrderedDict

import numpy as np

TRAIN = 0
TEST = 1
_state = {"device": 0, "mode": "gpu"}


def set_mode_gpu():
    _state["mode"] = "gpu"


def set_mode_cpu():
    raise RuntimeError("mnc_b200 has no CPU path (neither does the reference: "
                       "roi_warping_layer.cpp:47, tools/demo.py:126)")


def set_device(device_id):
    import torch
    _state["device"] = int(device_id)
    torch.cuda.set_device(int(device_id))


class Blob(object):
    """Host-visible blob: fp32 numpy `data` (the pycaffe `.data` property is the host copy,
    _caffe.cpp:285), NCHW."""

    def __init__(self, *shape):
        self.data = np.zeros(shape if shape else (0,), dtype=np.float32)
        self.diff = None

    def reshape(self, *dims):
        dims = tuple(int(d) for d in dims)
        if self.data.shape != dims:
            self.data = np.zeros(dims, dtype=np.float32)

    @property
    def shape(self):
        return self.data.shape

    @property
    def count(self):
        return int(self.data.size)

    def _dim(self, i):
        return self.data.shape[i] if self.data.ndim > i else 1

    num = property(lambda self: self._dim(0))
    channels = property(lambda self: self._dim(1))
    height = property(lambda self: self._dim(2))
    width = property(lambda self: self._dim(3))


class _Phase(object):
    def __init__(self, v):
        self.v = v

    def __str__(self):
        return "TEST" if self.v == TEST else "TRAIN"

    def __eq__(self, o):
        return (o.v if isinstance(o, _Phase) else o) == self.v


class Layer(object):
    """Base class of Python layers (python_layer.hpp:17-52)."""

    def __init__(self, param_str="", phase=TEST):
        self.param_str_ = param_str
        self.phase = _Phase(phase)

    def setup(self, bottom, top):
        pass

    def reshape(self, bottom, top):
        pass

    def forward(self, bottom, top):
        pass

    def backward(self, top, propagate_down, bottom):
        raise NotImplementedError("inference path only")


from .net import Net  # noqa: E402
from . import layers  # noqa: E402,F401
