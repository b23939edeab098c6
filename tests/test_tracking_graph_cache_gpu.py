"""GPU: a cached tracking graph is replayed only over the map it was captured for.  After a graph was built for a map,
tracking the same map with other colours must give the run of a freshly built graph, within test_tracking_gpu.py's
bounds (the backward's float atomics make two GPU runs differ in the last bits)."""
import numpy as np
import pytest

from test_tracking_gpu import _problem
from test_tracking_rule_gpu import N, _close, _track

pytestmark = pytest.mark.gpu


def test_cached_graph_is_not_replayed_with_other_colours(cuda_device):
    from splatam_b200 import mapping as M
    dev = cuda_device
    _, gauss, frame = _problem(dev)
    M._TRACK_GRAPHS.clear()
    try:
        warm = _track(gauss, frame, dev, N, True)
        assert len(M._TRACK_GRAPHS) == 1
        other = dict(gauss, rgb_colors=1 - gauss["rgb_colors"])
        after_warm = _track(other, frame, dev, N, True)
        M._TRACK_GRAPHS.clear()
        fresh = _track(other, frame, dev, N, True)
    finally:
        M._TRACK_GRAPHS.clear()
    assert not np.allclose(fresh[0][:8], warm[0][:8], rtol=1e-3)      # the colours change the losses
    _close(after_warm, fresh, N)
