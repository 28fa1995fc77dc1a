"""CPU-only: the splat backward workspace size (gf_splat_backward_workspace_bytes_ex) for flags 0 and
GF_BWD_DETERMINISTIC.  The layout is carved in one place on the host; these byte counts pin it, so that a change to
how the workspace is described or narrowed cannot move or resize a region unnoticed."""
import ctypes

import pytest

from gaussianformer_b200 import _lib
from gaussianformer_b200.csrc import build
from gaussianformer_b200.splat import _make_desc

# name: (G, N, C, H, W, D, variant, radii_axes, batch), plain bytes, deterministic bytes
CASES = {
    "cfg2": ((25601, 200 * 200 * 16, 18, 200, 200, 16, _lib.GF_SPLAT_BASE, 1, 1), 28195072, 61755136),
    "cfg4_prob_b2": ((6400, 200 * 200 * 16, 18, 200, 200, 16, _lib.GF_SPLAT_PROB, 1, 2), 38418176, 145402112),
    "ragged_fast": ((300, 37 * 21 * 6, 17, 37, 21, 6, _lib.GF_SPLAT_PROB, 3, 3), 578560, 8184064),
    "ragged_base_b3": ((513, 45 * 27 * 10, 16, 45, 27, 10, _lib.GF_SPLAT_BASE, 1, 3), 654848, 52098816),
}


@pytest.fixture(scope="module")
def L():
    build.build()
    return _lib.lib()


@pytest.mark.parametrize("name", list(CASES))
def test_backward_workspace_bytes(L, name):
    (G, N, C, H, W, D, variant, axes, B), plain, det = CASES[name]
    desc = _make_desc(G, N, C, H, W, D, variant, axes, 9, (-50.0, -50.0, -5.0), 0.5, 3.0, 1, B, 0)
    L.gf_debug_splat_backward_plan(-1, -1)   # the default slot budget
    assert L.gf_splat_backward_workspace_bytes_ex(ctypes.byref(desc), 0) == plain
    assert L.gf_splat_backward_workspace_bytes_ex(ctypes.byref(desc), _lib.GF_BWD_DETERMINISTIC) == det
