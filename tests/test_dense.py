"""CPU: the dense matrix import / export calls (B200_Matrix_import_dense / B200_Matrix_export_dense): declared and exported, every
argument error returned before the device check, GrB_PANIC without a device after it, and the argument handling of
Matrix.from_numpy / Matrix.to_numpy."""
import ctypes
import os

import numpy as np
import pytest

import pygraphblas_b200 as gb
from pygraphblas_b200 import Matrix, ffi, lib
from pygraphblas_b200.base import Panic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NULL = ffi.NULL
BIG = (1 << 31) - 1


def _import(nrows, ncols, x=True, present=None, where=0, handle=True):
    h = ffi.new("GrB_Matrix*") if handle else NULL
    buf = ffi.new("float[4]")
    return lib.B200_Matrix_import_dense(h, lib.GrB_FP32, nrows, ncols, ffi.cast("void*", buf) if x else NULL,
                                        present if present is not None else NULL, where), h


def _ok_or_panic(rc):
    # a valid call: GrB_PANIC without a device, success with one
    assert rc == (lib.GrB_SUCCESS if gb.have_device() else lib.GrB_PANIC)


def test_the_two_calls_are_declared_and_exported():
    with open(os.path.join(ROOT, "include", "b200grb.h")) as f:
        header = f.read()
    for name in ("B200_Matrix_import_dense", "B200_Matrix_export_dense"):
        assert f"GrB_Info {name}(" in header
        assert hasattr(lib, name)
        assert getattr(ctypes.CDLL(os.path.join(ROOT, "pygraphblas_b200", "libb200grb.so")), name) is not None


def test_import_null_arguments():
    assert _import(2, 2, handle=False)[0] == lib.GrB_NULL_POINTER
    assert _import(2, 2, x=False)[0] == lib.GrB_NULL_POINTER
    assert _import(0, 0, x=False)[0] == lib.GrB_NULL_POINTER


@pytest.mark.parametrize("where", [-1, 2, 3])
def test_import_where_outside_0_1(where):
    assert _import(2, 2, where=where)[0] == lib.GrB_INVALID_VALUE


@pytest.mark.parametrize("nrows,ncols", [(BIG + 1, 1), (1, BIG + 1), (1 << 16, 1 << 15), (BIG, 2), (46341, 46341)])
def test_import_beyond_the_dense_limit(nrows, ncols):
    assert _import(nrows, ncols)[0] == lib.GrB_INVALID_VALUE


def test_import_at_the_dense_limit_reaches_the_device_check():
    if gb.have_device():
        pytest.skip("with a device this would import 2^31-1 entries from a 4-entry buffer")
    for nrows, ncols in ((BIG, 1), (1, BIG), (46340, 46340)):
        assert _import(nrows, ncols)[0] == lib.GrB_PANIC


def test_import_valid_calls_panic_without_a_device():
    rc, h = _import(2, 2)
    _ok_or_panic(rc)
    if rc == lib.GrB_SUCCESS:
        lib.GrB_Matrix_free(h)
    else:
        assert h[0] == NULL
    if not gb.have_device():
        for nrows, ncols in ((0, 0), (0, 5), (5, 0)):
            assert _import(nrows, ncols)[0] == lib.GrB_PANIC


def test_export_validation_before_the_device_check():
    m = Matrix.sparse(gb.FP32, 3, 4)
    buf = np.zeros(12, np.float32)
    pres = np.zeros(12, np.uint8)
    x = ffi.cast("void*", buf.ctypes.data)
    p = ffi.cast("uint8_t*", pres.ctypes.data)
    assert lib.B200_Matrix_export_dense(NULL, x, p, 0) == lib.GrB_NULL_POINTER
    for where in (-1, 2):
        assert lib.B200_Matrix_export_dense(m._matrix[0], x, p, where) == lib.GrB_INVALID_VALUE
    for shape in ((BIG + 1, 1), (1 << 16, 1 << 15)):
        big = Matrix.sparse(gb.FP32, *shape)
        assert lib.B200_Matrix_export_dense(big._matrix[0], x, p, 0) == lib.GrB_INVALID_VALUE
    _ok_or_panic(lib.B200_Matrix_export_dense(m._matrix[0], x, p, 0))
    _ok_or_panic(lib.B200_Matrix_export_dense(m._matrix[0], NULL, NULL, 0))


def test_from_numpy_arguments():
    with pytest.raises(ValueError):
        Matrix.from_numpy(np.zeros(4, np.float32))
    with pytest.raises(ValueError):
        Matrix.from_numpy(np.zeros((2, 2, 2), np.float32))
    with pytest.raises(ValueError):
        Matrix.from_numpy(np.zeros((2, 3), np.float32), present=np.ones((3, 2), np.uint8))
    if gb.have_device():
        pytest.skip("the remaining calls import on a device (tests/test_dense_gpu.py)")
    # valid arguments of every kind reach the device check: a non-contiguous view, an explicit type, bool presence
    for x, kw in ((np.arange(6, dtype=np.int16).reshape(2, 3), {}),
                  (np.asfortranarray(np.ones((3, 2))), {}),
                  (np.arange(12.0).reshape(3, 4)[:, ::2], {"typ": gb.INT8}),
                  (np.zeros((2, 2), np.bool_), {"present": np.eye(2, dtype=np.bool_)})):
        with pytest.raises(Panic):
            Matrix.from_numpy(x, **kw)


def test_to_numpy_arguments():
    m = Matrix.sparse(gb.INT32, 2, 3)
    for out, pout in ((np.zeros((3, 2), np.int32), None), (np.zeros((2, 3), np.int64), None), (None, np.zeros((2, 3), np.int8)),
                      (np.zeros((3, 2), np.int32).T, None), (None, np.zeros(6, np.uint8))):
        with pytest.raises(ValueError):
            m.to_numpy(out=out, present_out=pout)
    if not gb.have_device():
        with pytest.raises(Panic):
            m.to_numpy()
