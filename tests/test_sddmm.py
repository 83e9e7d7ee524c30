"""CPU: GrB_mxm with two dense-form operands under a sparse mask (the sampled dense-dense product, DESIGN.md section 3.6).  The
call shape C<M> = X (+).(x) Y' keeps every argument check ahead of the device check and, without a device, ends in GrB_PANIC
(no CPU fallback).  Also the Python restatements the GPU module imports: the routing rule of GrB_mxm and the fold order of the
kernel (chunks of 64 in k order, the chunk partials folded pairwise in a fixed tree over chunk order)."""
import numpy as np
import pytest

import pygraphblas_b200 as gb
from pygraphblas_b200 import Matrix, descriptor, ffi, lib

NULL = ffi.NULL
SEG = 64        # restates SPMM_SEG (common.cuh)


# ------------------------------------------------------------------ restatements
def route(a_dense, b_dense, mask, mask_comp=False, mask_dense=False, positional=False, mask_nnz=0):
    """The route GrB_mxm takes for a builtin semiring on non-hypersparse operands, as far as the dense forms decide it."""
    if positional:
        return "positional"
    if a_dense and b_dense and mask and not mask_comp and not mask_dense and mask_nnz < (1 << 32):
        return "sddmm"
    return "other"


def tree_fold(partials, add):
    """The fold of spmm_combine_kernel over a list of (value, has) partials: pairwise, in place, in a fixed tree over the order."""
    p = list(partials)
    ns, w = len(p), 1
    while w < ns:
        for s in range(0, ns - w, 2 * w):
            (a, ha), (b, hb) = p[s], p[s + w]
            if hb:
                p[s] = (add(a, b) if ha else b, True)
        w *= 2
    return p[0] if p else (None, False)


def chunked_dot(x, y, add=np.add, mul=np.multiply, xp=None, yp=None):
    """(value, has) of one entry: k ascending in chunks of SEG, each chunk folded in order from its first present product, the
    partials through tree_fold.  x and y are 1-D arrays of the compute type; every operation rounds to that type."""
    d = len(x)
    parts = []
    for k0 in range(0, d, SEG):
        acc, has = None, False
        for k in range(k0, min(k0 + SEG, d)):
            if (xp is not None and not xp[k]) or (yp is not None and not yp[k]):
                continue
            z = mul(x[k], y[k])
            acc, has = (add(acc, z) if has else z), True
        parts.append((acc, has))
    return tree_fold(parts, add)


# ------------------------------------------------------------------ the restatements hold on their own
def test_routing_rule():
    assert route(True, True, True) == "sddmm"
    assert route(True, True, True, mask_nnz=(1 << 32) - 1) == "sddmm"
    for kw in ({"mask": False}, {"mask_comp": True}, {"mask_dense": True}, {"positional": True}, {"mask_nnz": 1 << 32}):
        args = {"a_dense": True, "b_dense": True, "mask": True, **kw}
        assert route(**args) != "sddmm", kw
    assert route(False, True, True) == "other" and route(True, False, True) == "other"


@pytest.mark.parametrize("ns", [1, 2, 3, 4, 5, 6, 7, 8, 9, 13, 16, 17])
def test_tree_fold_shape(ns):
    """On strings the fold shows its tree: complete groups of 2^l chunks, joined from the last group to the first."""
    got, has = tree_fold([(f"{i}", True) for i in range(ns)], lambda a, b: f"({a}{b})")
    assert has

    def full(lo, n):
        return f"{lo}" if n == 1 else f"({full(lo, n // 2)}{full(lo + n // 2, n // 2)})"

    groups, lo = [], 0
    for l in reversed(range(ns.bit_length())):
        if ns >> l & 1:
            groups.append(full(lo, 1 << l)); lo += 1 << l
    want = groups[-1]
    for g in reversed(groups[:-1]):
        want = f"({g}{want})"
    assert got == want


def test_tree_fold_skips_absent_partials():
    assert tree_fold([(None, False), (2, True), (None, False), (5, True)], lambda a, b: a + b) == (7, True)
    assert tree_fold([(None, False)] * 3, lambda a, b: a + b)[1] is False
    assert tree_fold([], lambda a, b: a + b) == (None, False)


def test_chunked_dot_is_left_to_right_up_to_one_chunk():
    rng = np.random.default_rng(1)
    for d in (1, 7, 63, 64):
        x, y = rng.random(d, dtype=np.float32), rng.random(d, dtype=np.float32)
        want = np.float32(x[0] * y[0])
        for k in range(1, d):
            want = np.float32(want + np.float32(x[k] * y[k]))
        got, has = chunked_dot(x, y)
        assert has and got.dtype == np.float32 and got == want
    x, y = rng.random(200), rng.random(200)
    got, _ = chunked_dot(x, y)
    assert abs(got - np.dot(x, y)) <= 1e-12 * np.dot(x, y)
    xp = np.zeros(200, bool)
    assert chunked_dot(x, y, xp=xp) == (None, False)
    xp[130] = True
    assert chunked_dot(x, y, xp=xp) == (x[130] * y[130], True)


# ------------------------------------------------------------------ the call shape without a device
@ffi.callback("void(void*, const void*, const void*)")
def _user_fn(z, x, y):
    pass


def _call(C, M, A, B, semiring=None, accum=NULL, desc=descriptor.ST1):
    return lib.GrB_mxm(C._matrix[0] if C is not None else NULL, M._matrix[0] if M is not None else NULL, accum,
                       semiring if semiring is not None else gb.FP32.PLUS_TIMES.get_op(),
                       A._matrix[0] if A is not None else NULL, B._matrix[0] if B is not None else NULL, desc.get_desc())


def test_every_check_comes_before_the_device_check():
    m, n, d = 5, 7, 3
    X = Matrix.from_lists([0, 4], [0, 2], [1.0, 2.0], m, d, gb.FP32)
    Y = Matrix.from_lists([0, 6], [1, 2], [1.0, 2.0], n, d, gb.FP32)
    M = Matrix.from_lists([0, 4], [0, 6], [True, True], m, n, gb.BOOL)
    C = Matrix.sparse(gb.FP32, m, n)
    assert _call(None, M, X, Y) == lib.GrB_NULL_POINTER
    assert _call(C, M, None, Y) == lib.GrB_NULL_POINTER
    assert _call(C, M, X, None) == lib.GrB_NULL_POINTER
    # dimensions: Y' under T1 must be d x n, C and M m x n
    assert _call(C, M, X, Y, desc=descriptor.S) == lib.GrB_DIMENSION_MISMATCH
    assert _call(Matrix.sparse(gb.FP32, m, d), M, X, Y) == lib.GrB_DIMENSION_MISMATCH
    assert _call(C, Matrix.sparse(gb.BOOL, n, m), X, Y) == lib.GrB_DIMENSION_MISMATCH
    # a user-defined multiply or accumulator, and a positional accumulator
    op = ffi.new("GrB_BinaryOp*")
    assert lib.GrB_BinaryOp_new(op, _user_fn, lib.GrB_FP32, lib.GrB_FP32, lib.GrB_FP32) == lib.GrB_SUCCESS
    sr = ffi.new("GrB_Semiring*")
    assert lib.GrB_Semiring_new(sr, lib.GrB_PLUS_MONOID_FP32, op[0]) == lib.GrB_SUCCESS
    try:
        assert _call(C, M, X, Y, semiring=sr[0]) == lib.GrB_INVALID_VALUE
        assert _call(C, M, X, Y, accum=op[0]) == lib.GrB_INVALID_VALUE
        assert _call(Matrix.sparse(gb.INT64, m, n), M, X, Y, accum=lib.GxB_FIRSTI_INT64) == lib.GrB_DOMAIN_MISMATCH
    finally:
        lib.GrB_Semiring_free(sr); lib.GrB_BinaryOp_free(op)
    assert C.nvals == 0


def test_the_valid_call_panics_without_a_device():
    if gb.have_device():
        pytest.skip("a GPU is present: the call computes (tests/test_sddmm_gpu.py)")
    X = Matrix.from_lists([0, 4], [0, 2], [1.0, 2.0], 5, 3, gb.FP32)
    Y = Matrix.from_lists([0, 6], [1, 2], [1.0, 2.0], 7, 3, gb.FP32)
    M = Matrix.from_lists([0, 4], [0, 6], [True, True], 5, 7, gb.BOOL)
    for desc in (descriptor.ST1, descriptor.T1):
        with pytest.raises(gb.base.Panic) as e:
            X.mxm(Y, mask=M, desc=desc, out=Matrix.sparse(gb.FP32, 5, 7))
        assert "no CPU fallback" in str(e.value)
    with pytest.raises(gb.base.Panic):
        Matrix.from_numpy(np.ones((5, 3), np.float32))      # a dense form exists only on a device
