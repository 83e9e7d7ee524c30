"""The wide-route test seam without a device: B200_debug_wide is exported, and with it on every mxv / vxm / transpose still
refuses to run on the host."""
import pytest

import pygraphblas_b200 as gb
from pygraphblas_b200 import Matrix, Vector, lib


@pytest.mark.skipif(gb.have_device(), reason="only meaningful without a GPU")
def test_wide_switch_has_no_cpu_fallback():
    m = Matrix.from_lists([0, 1, 2], [1, 2, 0], [1, 2, 3])
    v = Vector.from_lists([0, 1, 2], [2, 3, 4])
    lib.B200_debug_wide(7)
    try:
        for call in (lambda: m.mxv(v), lambda: v.vxm(m), lambda: m.transpose()):
            with pytest.raises(gb.Panic, match="no CPU fallback"):
                call()
    finally:
        lib.B200_debug_wide(0)
