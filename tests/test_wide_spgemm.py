"""The wide route of the masked CSR x CSR methods of mxm without a device: with B200_debug_wide on, a masked product (with and
without a transposed B) still refuses to run on the host."""
import pytest

import pygraphblas_b200 as gb
from pygraphblas_b200 import Matrix, descriptor, lib


@pytest.mark.skipif(gb.have_device(), reason="only meaningful without a GPU")
def test_wide_switch_has_no_cpu_fallback_in_masked_mxm():
    A = Matrix.from_lists([0, 1, 2], [1, 2, 0], [1.0, 2.0, 3.0])
    M = Matrix.from_lists([0, 1, 2], [2, 0, 1], [True, True, True])
    lib.B200_debug_wide(7)
    try:
        for desc in (descriptor.S, descriptor.ST1, None, descriptor.T1):
            with pytest.raises(gb.Panic, match="no CPU fallback"):
                A.mxm(A, mask=M, semiring=gb.FP64.PLUS_TIMES, desc=desc)
    finally:
        lib.B200_debug_wide(0)
