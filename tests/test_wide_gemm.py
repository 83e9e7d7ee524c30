"""The wide route of the unmasked and complemented-mask CSR x CSR bins of mxm without a device: the seam B200_debug_wide_gemm is
exported, and with it on, an unmasked product and a product under a complemented structural or valued mask still refuse to
run on the host."""
import pytest

import pygraphblas_b200 as gb
from pygraphblas_b200 import Matrix, descriptor, lib


def test_wide_gemm_seam_is_exported():
    assert callable(lib.B200_debug_wide_gemm)
    lib.B200_debug_wide_gemm(7, 100, 4096)
    lib.B200_debug_wide_gemm(0, 0, 0)


@pytest.mark.skipif(gb.have_device(), reason="only meaningful without a GPU")
def test_wide_gemm_switch_has_no_cpu_fallback():
    A = Matrix.from_lists([0, 1, 2], [1, 2, 0], [1.0, 2.0, 3.0])
    M = Matrix.from_lists([0, 1, 2], [2, 0, 1], [True, False, True])
    lib.B200_debug_wide_gemm(7, 0, 0)
    try:
        with pytest.raises(gb.Panic, match="no CPU fallback"):
            A.mxm(A, semiring=gb.FP64.PLUS_TIMES)
        for desc in (descriptor.SC, descriptor.C):
            with pytest.raises(gb.Panic, match="no CPU fallback"):
                A.mxm(A, mask=M, semiring=gb.FP64.PLUS_TIMES, desc=desc)
    finally:
        lib.B200_debug_wide_gemm(0, 0, 0)
