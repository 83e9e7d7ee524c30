"""Positional operators and semirings (FIRSTI ... SECONDJ1, POSITIONI ... POSITIONJ1) without a GPU: the handles, what the
mirror makes of them, what every entry point refuses before it reads anything, and the model the GPU tests compare with."""
import numpy as np
import pytest

import pygraphblas_b200 as gb
from pygraphblas_b200 import ffi, lib
from pygraphblas_b200.base import NULL
import positional_model as pm

NAMES = ([f"GxB_{m}_{t}" for t in pm.TYPES for m in pm.POSITIONAL] +
         [f"GxB_{u}_{t}" for t in pm.TYPES for u in pm.UNARY] +
         [f"GxB_{a}_{m}_{t}" for t in pm.TYPES for a in pm.MONOIDS for m in pm.POSITIONAL])


def _ztype(handle):
    t = ffi.new("GrB_Type*")
    assert lib.GxB_BinaryOp_ztype(t, handle) == lib.GrB_SUCCESS
    return gb.types.from_handle(t[0]).name


def test_all_104_handles_are_exported_and_discovered_with_their_ztype():
    assert len(NAMES) == 104 and len(set(NAMES)) == 104
    for n in NAMES:
        assert hasattr(lib, n), n
    for t in pm.TYPES:
        T = gb.types.by_name(t)
        for m in pm.POSITIONAL:
            assert _ztype(getattr(T, m).get_op()) == t
            for a in pm.MONOIDS:
                s = getattr(T, f"{a}_{m}")
                assert s.name == f"{a}_{m}_{t}" and s.ztype.name == t
        for u in pm.UNARY:
            assert gb.ops.unaryops[f"{u}_{t}"].type == t
    assert "MIN_FIRSTI1_INT64" in gb.ops.semirings and "ANY_SECONDI_INT32" in gb.ops.semirings


def test_semiring_new_with_a_positional_multiply():
    h = ffi.new("GrB_Semiring*")
    assert lib.GrB_Semiring_new(h, lib.GrB_MIN_MONOID_INT64, lib.GxB_SECONDI_INT64) == lib.GrB_SUCCESS
    assert lib.GrB_Semiring_free(h) == lib.GrB_SUCCESS
    assert lib.GrB_Semiring_new(h, lib.GrB_PLUS_MONOID_INT32, lib.GxB_FIRSTJ1_INT32) == lib.GrB_SUCCESS
    assert lib.GrB_Semiring_free(h) == lib.GrB_SUCCESS
    assert lib.GrB_Semiring_new(h, lib.GrB_MIN_MONOID_INT32, lib.GxB_SECONDI_INT64) == lib.GrB_DOMAIN_MISMATCH
    assert lib.GrB_Semiring_new(h, lib.GrB_MIN_MONOID_FP64, lib.GxB_FIRSTI_INT64) == lib.GrB_DOMAIN_MISMATCH


def test_monoid_new_refuses_a_positional_operator():
    h = ffi.new("GrB_Monoid*")
    assert lib.GrB_Monoid_new_INT64(h, lib.GxB_FIRSTI_INT64, 0) == lib.GrB_DOMAIN_MISMATCH
    assert lib.GrB_Monoid_new_INT32(h, lib.GxB_SECONDJ1_INT32, 0) == lib.GrB_DOMAIN_MISMATCH


def _mat(typ=gb.INT64):
    return gb.Matrix.from_lists([0, 1, 2], [1, 2, 0], [5, 6, 7], 3, 3, typ)


def _vec(typ=gb.INT64):
    return gb.Vector.from_lists([0, 2], [3, 4], 3, typ)


def _refused(code, call, out, msg=None):
    before = out.to_lists()
    assert call() == code
    text = ffi.string(lib.B200_last_error()).decode()
    assert out.to_lists() == before
    if msg:
        assert msg in text


def test_positional_accumulators_are_refused_before_anything_is_read():
    A, B, C, u, w = _mat(), _mat(), _mat(), _vec(), _vec()
    acc = lib.GxB_FIRSTI_INT64
    DM = lib.GrB_DOMAIN_MISMATCH
    _refused(DM, lambda: lib.GrB_mxm(C._matrix[0], NULL, acc, lib.GxB_PLUS_TIMES_INT64, A._matrix[0], B._matrix[0], NULL), C)
    _refused(DM, lambda: lib.GrB_mxv(w._vector[0], NULL, acc, lib.GxB_PLUS_TIMES_INT64, A._matrix[0], u._vector[0], NULL), w)
    _refused(DM, lambda: lib.GrB_vxm(w._vector[0], NULL, acc, lib.GxB_MIN_SECONDI_INT64, u._vector[0], A._matrix[0], NULL), w)
    _refused(DM, lambda: lib.GrB_Matrix_apply(C._matrix[0], NULL, acc, lib.GrB_AINV_INT64, A._matrix[0], NULL), C)
    _refused(DM, lambda: lib.GrB_Vector_apply(w._vector[0], NULL, lib.GxB_SECONDJ1_INT32, lib.GxB_POSITIONI_INT64, u._vector[0], NULL), w)
    _refused(DM, lambda: lib.GrB_Matrix_eWiseAdd_BinaryOp(C._matrix[0], NULL, acc, lib.GrB_PLUS_INT64, A._matrix[0], B._matrix[0], NULL), C)
    _refused(DM, lambda: lib.GrB_transpose(C._matrix[0], NULL, acc, A._matrix[0], NULL), C)


@ffi.callback("void(void*, const void*, const void*)")
def _user_fn(z, x, y):
    pass


@pytest.mark.parametrize("mul", ["FIRSTI", "SECONDI1"])         # the count form and the inner form
def test_user_defined_monoid_or_accumulator_with_a_positional_semiring_is_refused(mul):
    """As for every other semiring: GrB_INVALID_VALUE before the device check and the hypersparse dispatch, output untouched."""
    op = ffi.new("GrB_BinaryOp*")
    assert lib.GrB_BinaryOp_new(op, _user_fn, lib.GrB_INT64, lib.GrB_INT64, lib.GrB_INT64) == lib.GrB_SUCCESS
    mon = ffi.new("GrB_Monoid*")
    assert lib.GrB_Monoid_new_INT64(mon, op[0], 0) == lib.GrB_SUCCESS
    user_sr = ffi.new("GrB_Semiring*")
    assert lib.GrB_Semiring_new(user_sr, mon[0], getattr(lib, f"GxB_{mul}_INT64")) == lib.GrB_SUCCESS
    builtin_sr = getattr(lib, f"GxB_PLUS_{mul}_INT64")
    big = 1 << 60
    A, B, C, u, w = _mat(), _mat(), _mat(), _vec(), _vec()
    H = gb.Matrix.from_lists([5, (1 << 40) + 5], [(1 << 31) + 3, 5], [1, 2], big, big, gb.INT64)
    HC = gb.Matrix.from_lists([5], [5], [9], big, big, gb.INT64)
    hu, hw = gb.Vector.from_lists([5], [1], big, gb.INT64), gb.Vector.from_lists([7], [3], big, gb.INT64)
    try:
        for sr, acc in [(user_sr[0], NULL), (builtin_sr, op[0])]:
            IV = lib.GrB_INVALID_VALUE
            _refused(IV, lambda: lib.GrB_mxv(w._vector[0], NULL, acc, sr, A._matrix[0], u._vector[0], NULL), w, "user-defined")
            _refused(IV, lambda: lib.GrB_vxm(w._vector[0], NULL, acc, sr, u._vector[0], A._matrix[0], NULL), w, "user-defined")
            _refused(IV, lambda: lib.GrB_mxm(C._matrix[0], NULL, acc, sr, A._matrix[0], B._matrix[0], NULL), C, "user-defined")
            _refused(IV, lambda: lib.GrB_mxm(HC._matrix[0], NULL, acc, sr, H._matrix[0], H._matrix[0], NULL), HC, "user-defined")
            _refused(IV, lambda: lib.GrB_mxv(hw._vector[0], NULL, acc, sr, H._matrix[0], hu._vector[0], NULL), hw, "user-defined")
            _refused(IV, lambda: lib.GrB_vxm(hw._vector[0], NULL, acc, sr, hu._vector[0], H._matrix[0], NULL), hw, "user-defined")
    finally:
        lib.GrB_Semiring_free(user_sr); lib.GrB_Monoid_free(mon); lib.GrB_BinaryOp_free(op)


@pytest.mark.parametrize("form", ["Matrix_eWiseAdd_BinaryOp", "Matrix_eWiseMult_BinaryOp", "Matrix_eWiseAdd_Semiring",
                                  "Matrix_eWiseMult_Semiring", "Vector_eWiseAdd_BinaryOp", "Vector_eWiseMult_BinaryOp",
                                  "Vector_eWiseAdd_Semiring", "Vector_eWiseMult_Semiring", "Matrix_kronecker_BinaryOp",
                                  "Matrix_reduce_BinaryOp"])
def test_operations_without_a_positional_form_refuse_it(form):
    A, B, C, u, v, w = _mat(), _mat(), _mat(), _vec(), _vec(), _vec()
    op = lib.GxB_MIN_FIRSTJ_INT64 if form.endswith("Semiring") else lib.GxB_SECONDI1_INT64
    f = getattr(lib, "GrB_" + form)
    if form == "Matrix_reduce_BinaryOp":
        call, out = (lambda: f(w._vector[0], NULL, NULL, op, A._matrix[0], NULL)), w
    elif form.startswith("Matrix"):
        call, out = (lambda: f(C._matrix[0], NULL, NULL, op, A._matrix[0], B._matrix[0], NULL)), C
    else:
        call, out = (lambda: f(w._vector[0], NULL, NULL, op, u._vector[0], v._vector[0], NULL)), w
    _refused(lib.GrB_INVALID_VALUE, call, out, f"positional operators are not supported by GrB_{form}")


def test_build_refuses_a_positional_dup():
    A = gb.Matrix.sparse(gb.INT64, 3, 3)
    I = ffi.new("GrB_Index[]", [0, 0]); X = ffi.new("int64_t[]", [1, 2])
    _refused(lib.GrB_INVALID_VALUE, lambda: lib.GrB_Matrix_build_INT64(A._matrix[0], I, I, X, 2, lib.GxB_FIRSTI_INT64), A,
             "positional operators are not supported by build")
    w = gb.Vector.sparse(gb.INT64, 3)
    _refused(lib.GrB_INVALID_VALUE, lambda: lib.GrB_Vector_build_INT64(w._vector[0], I, X, 2, lib.GxB_SECONDJ_INT64), w)


def test_positional_compute_panics_without_a_device():
    if gb.have_device():
        pytest.skip("a CUDA device is present: the GPU module computes these calls")
    A, B, C, u, w = _mat(gb.BOOL), _mat(gb.FP32), _mat(), _vec(), _vec()
    P = lib.GrB_PANIC
    assert lib.GrB_mxm(C._matrix[0], NULL, NULL, lib.GxB_ANY_SECONDI_INT64, A._matrix[0], B._matrix[0], NULL) == P
    assert lib.GrB_mxv(w._vector[0], NULL, NULL, lib.GxB_PLUS_FIRSTI_INT64, A._matrix[0], u._vector[0], NULL) == P
    assert lib.GrB_vxm(w._vector[0], NULL, NULL, lib.GxB_MIN_FIRSTJ_INT32, u._vector[0], A._matrix[0], NULL) == P
    assert lib.GrB_Matrix_apply(C._matrix[0], NULL, NULL, lib.GxB_POSITIONJ_INT64, A._matrix[0], NULL) == P
    assert lib.GrB_Vector_apply(w._vector[0], NULL, NULL, lib.GxB_POSITIONI1_INT32, u._vector[0], NULL) == P


# ------------------------------------------------------------------ the model, pinned
# A (4 x 5), by hand:          B (5 x 3):           u (5):
#   (0,1) (0,3)                  (1,0) (1,2)           u(1), u(3), u(4)
#   (1,0) (1,4)                  (3,1)
#   (2,1) (2,3) (2,4)            (4,0) (4,1) (4,2)
#   (3,2)                        (2,2)
A45 = {(0, 1): 1, (0, 3): 1, (1, 0): 1, (1, 4): 1, (2, 1): 1, (2, 3): 1, (2, 4): 1, (3, 2): 1}
B53 = {(1, 0): 1, (1, 2): 1, (3, 1): 1, (4, 0): 1, (4, 1): 1, (4, 2): 1, (2, 2): 1}
U5 = {1: 1, 3: 1, 4: 1}


def test_model_mxm_on_a_hand_worked_example():
    # products of C(i, j) by hand: inner indices k with A(i,k) and B(k,j)
    ks = {(0, 0): [1], (0, 2): [1], (0, 1): [3], (1, 0): [4], (1, 1): [4], (1, 2): [4],
          (2, 0): [1, 4], (2, 2): [1, 4], (2, 1): [3, 4], (3, 2): [2]}
    for mul, want in [("FIRSTI", lambda i, k, j: i), ("FIRSTJ", lambda i, k, j: k), ("SECONDI", lambda i, k, j: k),
                      ("SECONDJ1", lambda i, k, j: j + 1)]:
        T, _ = pm.product("PLUS", mul, "INT64", A45, B53)
        assert T == {e: sum(want(e[0], k, e[1]) for k in kk) for e, kk in ks.items()}, mul
    T, _ = pm.product("MIN", "SECONDI", "INT64", A45, B53)
    assert T[(2, 0)] == 1 and T[(2, 1)] == 3 and T[(3, 2)] == 2
    T, _ = pm.product("TIMES", "FIRSTI1", "INT32", A45, B53)
    assert T[(2, 1)] == 9 and T[(1, 1)] == 2


def test_model_mxv_and_vxm_on_a_hand_worked_example():
    # w = A u: row i gathers k in {1, 3, 4}
    w, _ = pm.mxv({}, "INT64", None, None, ("MIN", "SECONDI", "INT64"), A45, U5)
    assert w == {0: 1, 1: 4, 2: 1}
    w, _ = pm.mxv({}, "INT64", None, None, ("PLUS", "FIRSTI", "INT64"), A45, U5)
    assert w == {0: 0, 1: 1, 2: 6}                                   # count * i: 2*0, 1*1, 3*2
    w, _ = pm.mxv({}, "INT64", None, None, ("PLUS", "SECONDJ1", "INT64"), A45, U5)
    assert w == {0: 2, 1: 1, 2: 3}                                   # y at (k, 0): j = 0, + 1 per product
    w, _ = pm.mxv({}, "INT64", None, None, ("MAX", "FIRSTJ", "INT64"), A45, U5)
    assert w == {0: 3, 1: 4, 2: 4}
    # w' = u' A' (A' is 5 x 4): w(j) over k = rows of A' that u holds
    w, _ = pm.vxm({}, "INT64", None, None, ("PLUS", "FIRSTI", "INT64"), U5, A45, {"tran1": True})
    assert w == {0: 0, 1: 0, 2: 0}                                   # x at (0, k): i = 0
    w, _ = pm.vxm({}, "INT64", None, None, ("MIN", "SECONDJ", "INT64"), U5, A45, {"tran1": True})
    assert w == {0: 0, 1: 1, 2: 2}
    w, _ = pm.vxm({}, "INT64", None, None, ("MAX", "FIRSTJ1", "INT64"), U5, A45, {"tran1": True})
    assert w == {0: 4, 1: 5, 2: 5}


def test_model_apply_and_truncation():
    assert pm.apply("POSITIONJ1", "INT64", {(2, 7): 0}) == {(2, 7): 8}
    assert pm.apply("SECONDI", "INT64", {(2, 7): 0}, tran=True) == {(7, 2): 7}
    assert pm.apply_vector("POSITIONJ", "INT32", {5: 1}) == {5: 0}
    assert pm.apply_vector("FIRSTI1", "INT32", {5: 1}) == {5: 6}
    assert pm.trunc(2**31 + 3, "INT32") == -2147483645 and pm.trunc(2**40 + 5, "INT32") == 5
    assert pm.fold("PLUS", "INT32", [2**30] * 4) == 0 and pm.fold("TIMES", "INT32", [3] * 21) == pm.trunc(3**21, "INT32")


def _rand(rng, nrows, ncols, density):
    M = rng.random((nrows, ncols)) < density
    return {(int(i), int(j)): 1 for i, j in zip(*np.nonzero(M))}, M


def test_model_against_numpy_restatements():
    rng = np.random.default_rng(7)
    A, Ad = _rand(rng, 200, 300, 0.02)
    upres = rng.random(300) < 0.5
    u = {int(k): 1 for k in np.flatnonzero(upres)}
    hit = Ad & upres[None, :]
    rows = np.flatnonzero(hit.any(axis=1))
    # per-row min column index over present u
    w, _ = pm.mxv({}, "INT64", None, None, ("MIN", "SECONDI", "INT64"), A, u)
    assert w == {int(i): int(np.flatnonzero(hit[i]).min()) for i in rows}
    # count * i for PLUS_FIRSTI, and its INT32 wrap with indices shifted by 2^31 in the model's index
    w, _ = pm.mxv({}, "INT64", None, None, ("PLUS", "FIRSTI1", "INT64"), A, u)
    assert w == {int(i): int(hit[i].sum()) * (int(i) + 1) for i in rows}
    # mxm: C(i, j) = max k for MAX_SECONDI; count * j for PLUS_SECONDJ
    B, Bd = _rand(rng, 300, 50, 0.05)
    cnt = Ad.astype(np.int64) @ Bd.astype(np.int64)
    T, _ = pm.product("PLUS", "SECONDJ", "INT64", A, B)
    assert T == {(int(i), int(j)): int(cnt[i, j]) * int(j) for i, j in zip(*np.nonzero(cnt))}
    T, _ = pm.product("MAX", "SECONDI", "INT64", A, B)
    for (i, j), v in list(T.items())[:200]:
        assert v == int(np.flatnonzero(Ad[i] & Bd[:, j]).max())


def test_model_write_back_with_mask_and_accumulator():
    w, _ = pm.mxv({0: 10, 3: 4}, "INT64", {0: True, 2: False}, ("PLUS", "INT64"), ("MIN", "SECONDI", "INT64"), A45, U5,
                  {"replace": True})
    assert w == {0: 11}
    w, _ = pm.mxv({0: 10, 3: 4}, "INT64", {0: True}, None, ("MIN", "SECONDI", "INT64"), A45, U5,
                  {"mask_comp": True, "mask_struct": True})
    assert w == {0: 10, 1: 4, 2: 1}                                  # no accumulator: 3 is let through and T has nothing there
