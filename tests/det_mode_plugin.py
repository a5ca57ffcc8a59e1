"""pytest plugin (-p det_mode_plugin): every api.KdTree is created with the deterministic map mode on, so existing tests run
unchanged against it (test_gpu_deterministic.py::test_reference_parity_holds_in_the_mode)."""
from fast_lio_b200 import api

_init = api.KdTree.__init__


def _init_det(self, *a, **kw):
    _init(self, *a, **kw)
    self.set_deterministic(True)


api.KdTree.__init__ = _init_det

