"""The wide-route test seam without a device: with B200_debug_wide on, the calls that take the SpMM, dense-left and SDDMM routes
of mxm on a device still refuse to run on the host.  A dense form cannot be imported without a device, so the operands hold the
same tuples in CSR; GrB_mxm refuses before it picks a route."""
import numpy as np
import pytest

import pygraphblas_b200 as gb
from pygraphblas_b200 import Matrix, descriptor, lib


def full(rows, cols):
    I, J = np.nonzero(np.ones((rows, cols), bool))
    return Matrix.from_lists(I.tolist(), J.tolist(), [float(v) for v in range(rows * cols)], rows, cols)


@pytest.mark.skipif(gb.have_device(), reason="only meaningful without a GPU")
def test_wide_switch_has_no_cpu_fallback_in_mxm():
    A = Matrix.from_lists([0, 1, 2], [1, 2, 0], [1.0, 2.0, 3.0])
    X, Y, Xl = full(3, 2), full(3, 2), full(2, 3)
    with pytest.raises(gb.Panic, match="no CPU fallback"):
        Matrix.from_numpy(np.zeros((3, 2)))
    lib.B200_debug_wide(7)
    try:
        for call in (lambda: A.mxm(X), lambda: Xl.mxm(A), lambda: X.mxm(Y, mask=A, out=Matrix.sparse(gb.FP64, 3, 3), desc=descriptor.ST1)):
            with pytest.raises(gb.Panic, match="no CPU fallback"):
                call()
    finally:
        lib.B200_debug_wide(0)
