"""superpoint_graph_b200 — sm_90a (H100) implementation of the superpoint-graph learning hot path
(PointNet embedding + edge-conditioned convolution + GRU cell) behind the reference's own
`learning/pointnet`, `learning/ecc`, `learning/modules`, `learning/graphnet` operator API.

    from superpoint_graph_b200 import dropin; dropin.install()   # then run learning/main.py as is

The compute lives in libspg_b200.so (C-ABI: include/spg_b200.h); there is no CPU fallback.
"""
__version__ = "0.1.0"

from . import _lib  # noqa: F401


def library_path():
    return _lib.LIB_PATH
