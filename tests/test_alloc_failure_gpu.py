"""Device allocation failures: every compute entry point either succeeds or returns GrB_OUT_OF_MEMORY, frees what it
allocated, and leaves its operands (and the plans cached in them) usable.

B200_debug_fail_alloc(k) makes the k-th device allocation from now fail before it reaches the device.  For each entry
point the sweep injects k = 1, 2, ... on fresh operands until the call gets through, repeats the call on the same
objects without injection, compares the result with the clean one (itself checked against scipy / numpy), and frees
everything.  Afterwards the library holds exactly as many device blocks as after one clean round."""
import gc

import numpy as np
import pytest
import scipy.sparse as sp

import pygraphblas_b200 as gb
from pygraphblas_b200 import Matrix, Vector, BOOL, INT64, FP32, FP64, descriptor, lib
from pygraphblas_b200.generators import rmat_csr

pytestmark = pytest.mark.gpu
ffi = gb.ffi


def _snap(x):
    if isinstance(x, (Matrix, Vector)):
        return tuple(np.asarray(a) for a in x.to_arrays())
    return (np.asarray(x),)


def _same(a, b):
    return len(a) == len(b) and all(np.array_equal(p, q) for p, q in zip(a, b))


def _sweep(make, call, check=None):
    """Returns the number of allocation points the call went through."""
    def clean():
        ops = make()
        res = _snap(call(*ops))
        del ops
        gc.collect()
        return res

    ref = clean()
    if check is not None:
        check(ref)
    ref = clean()                           # warm-up round: scratch that stays between calls is in place
    live0 = lib.B200_debug_live_allocs()
    k = 0
    while True:
        k += 1
        assert k < 400, "the call never got through"
        ops = make()
        lib.B200_debug_fail_alloc(k)
        try:
            call(*ops)
            ok = True
        except gb.OutOfMemory:
            ok = False
        finally:
            lib.B200_debug_fail_alloc(0)
        assert _same(_snap(call(*ops)), ref), f"wrong result after the failure injected at allocation {k}"
        del ops
        gc.collect()
        if ok:
            break
    assert lib.B200_debug_live_allocs() == live0
    return k


def _rand_csr(rng, n, m, dens, dtype):
    S = sp.random(n, m, density=dens, format="csr", random_state=rng, dtype=np.float64)
    S.data = rng.integers(1, 9, S.nnz).astype(dtype)
    S.sort_indices()
    return S


def _mat(S, typ):
    return Matrix.from_csr(S.indptr, S.indices, S.data, S.shape[0], S.shape[1], typ)


def _mat_lists(S, typ):
    C = S.tocoo()
    return Matrix.from_lists(C.row.tolist(), C.col.tolist(), C.data.tolist(), S.shape[0], S.shape[1], typ)


def _close_vec(S, u):
    def check(ref):
        I, X = ref
        want = S @ u
        nz = np.diff(S.indptr) > 0
        assert np.array_equal(I, np.flatnonzero(nz)) and np.allclose(X, want[nz], rtol=1e-5)
    return check


def _vec_model(pres, vals):
    def check(ref):
        I, X = ref
        assert np.array_equal(I, np.flatnonzero(pres)) and np.array_equal(X, vals[pres])
    return check


def _same_csr(want):
    def check(ref):
        I, J, X = ref
        W = want.tocoo(); order = np.lexsort((W.col, W.row))
        assert np.array_equal(I, W.row[order]) and np.array_equal(J, W.col[order]) and np.array_equal(X, W.data[order])
    return check


@pytest.fixture(autouse=True)
def _injection_off():
    yield
    lib.B200_debug_fail_alloc(0)


@pytest.mark.parametrize("kind", ["tile", "run"])
def test_mxv_kernels(kind):
    rng = np.random.default_rng(3)
    S = _rand_csr(rng, 300 if kind == "tile" else 3000, 400 if kind == "tile" else 3000, 0.01, np.float32)
    u = rng.integers(1, 4, S.shape[1]).astype(np.float32)
    # u built on the host: its upload (vector_ensure_device, dense staging) runs under injection too
    k = _sweep(lambda: (_mat(S, FP32), Vector.from_lists(np.arange(len(u)), u, len(u), FP32)),
               lambda A, v: A.mxv(v, semiring=FP32.PLUS_TIMES), _close_vec(S.astype(np.float64), u.astype(np.float64)))
    assert k > (10 if kind != "tile" else 2)


def test_mxv_hot_table(monkeypatch, capfd):
    """The hot-table kernel: >= 2^20 entries and >= 2^16 columns.  Its plan builder is one more set of allocations on
    top of the run plan, so the sweep with it must go through more allocation points than the sweep without."""
    rng = np.random.default_rng(3)
    n, indptr, indices = rmat_csr(17)
    S = sp.csr_matrix((rng.integers(1, 5, len(indices)).astype(np.float32), indices, indptr), shape=(n, n))
    assert S.nnz >= 1 << 20 and S.shape[1] >= 1 << 16
    u = rng.integers(0, 4, n).astype(np.float32)
    make = lambda: (_mat(S, FP32), Vector.from_numpy(u))
    call = lambda A, v: A.mxv(v, semiring=FP32.PLUS_TIMES)
    A, v = make()
    lib.B200_set_burble(1)
    try:
        call(A, v)
    finally:
        lib.B200_set_burble(0)
    assert "hot-table" in capfd.readouterr().out
    del A, v
    k_hot = _sweep(make, call, _close_vec(S.astype(np.float64), u.astype(np.float64)))
    monkeypatch.setenv("B200GRB_SPMV_HOT", "0")
    try:
        lib.B200_reload_tunables()
        k_run = _sweep(make, call)
    finally:
        monkeypatch.delenv("B200GRB_SPMV_HOT")
        lib.B200_reload_tunables()
    assert k_hot > k_run + 3


def test_vxm_and_transpose():
    rng = np.random.default_rng(4)
    S = _rand_csr(rng, 2000, 1500, 0.01, np.float64)
    u = rng.integers(0, 4, S.shape[0]).astype(np.float64)
    _sweep(lambda: (_mat_lists(S, FP64), Vector.from_numpy(u)), lambda A, v: v.vxm(A, semiring=FP64.PLUS_TIMES),
           _close_vec(S.T.tocsr(), u))
    _sweep(lambda: (_mat_lists(S, FP64),), lambda A: A.transpose(), _same_csr(S.T.tocsr()))


@pytest.mark.parametrize("push", [False, True])
def test_masked_mxv_pull_push(push):
    rng = np.random.default_rng(5)
    n = 4000
    S = _rand_csr(rng, n, n, 0.002, np.float64)
    S.data[:] = 1
    mask = rng.random(n) < 0.5
    u = np.zeros(n, bool); u[rng.choice(n, 3 if push else 400, replace=False)] = True

    def make():
        A = _mat(S.astype(bool), BOOL)
        if push:
            Vector.from_numpy(np.ones(n, bool)).vxm(A, semiring=BOOL.LOR_LAND)      # the transpose the push path walks
        # u built on the host with few entries: uploaded by the scatter path of vector_ensure_device
        uf = np.flatnonzero(u)
        return A, Vector.from_lists(uf, [True] * len(uf), n, BOOL), Vector.from_numpy(mask, present=mask)

    def check(ref):
        I, X = ref
        want = (S @ u.astype(np.float64) > 0) & mask
        assert np.array_equal(I, np.flatnonzero(want))

    _sweep(make, lambda A, v, m: A.mxv(v, semiring=BOOL.LOR_LAND, mask=m, desc=descriptor.S), check)


def test_mxm_unmasked_all_bins():
    n, indptr, indices = rmat_csr(11, 16, seed=2)
    S = sp.csr_matrix((np.ones(len(indices), np.int64), indices, indptr), shape=(n, n))
    per_row = S @ np.diff(S.indptr)                  # multiplies per row of A @ A: the bins split at 128 and 2048
    assert ((per_row > 0) & (per_row <= 128)).any() and ((per_row > 128) & (per_row <= 2048)).any() and (per_row > 2048).any()
    _sweep(lambda: (_mat(S, INT64),), lambda A: A.mxm(A, semiring=INT64.PLUS_TIMES), _same_csr((S @ S).tocsr()))


@pytest.mark.parametrize("dot", [False, True])
def test_mxm_masked(dot):
    n, indptr, indices = rmat_csr(11, 16, seed=3)
    S = sp.csr_matrix((np.ones(len(indices), np.int64), indices, indptr), shape=(n, n))
    want = ((S @ (S.T if dot else S)).multiply(S)).tocsr()
    want.eliminate_zeros()
    _sweep(lambda: (_mat(S, INT64),),
           lambda A: A.mxm(A, mask=A, semiring=INT64.PLUS_PAIR, desc=descriptor.ST1 if dot else descriptor.S), _same_csr(want))


def test_vector_ops():
    rng = np.random.default_rng(6)
    n = 5000
    a = rng.integers(1, 9, n).astype(np.int64); pa = rng.random(n) < 0.6
    b = rng.integers(1, 9, n).astype(np.int64); pb = rng.random(n) < 0.6
    idx = rng.choice(n, 700, replace=False)
    mk = lambda: (Vector.from_lists(np.flatnonzero(pa), a[pa], n, INT64), Vector.from_numpy(b, present=pb))
    _sweep(mk, lambda u, v: u.eadd(v, INT64.PLUS), _vec_model(pa | pb, np.where(pa & pb, a + b, np.where(pa, a, b))))
    _sweep(mk, lambda u, v: u.apply(INT64.AINV), _vec_model(pa, -a))
    _sweep(mk, lambda u, v: u.extract(idx.tolist()), _vec_model(pa[idx], a[idx]))

    def reduced(ref):
        assert int(ref[0]) == int(a[pa].sum())
    _sweep(mk, lambda u, v: np.asarray(u.reduce_int()), reduced)

    def assign(u, v):
        u.assign(v.extract(idx.tolist()), index=idx.tolist())
        return u
    pres, vals = pa.copy(), a.copy()
    pres[idx], vals[idx] = pb[idx], b[idx]
    _sweep(mk, assign, _vec_model(pres, vals))


def test_matrix_ops():
    rng = np.random.default_rng(7)
    S = _rand_csr(rng, 300, 200, 0.05, np.int64)
    B = _rand_csr(rng, 6, 5, 0.4, np.int64)
    Il, Jl = [3, 1, 7, 100], [5, 0, 9]
    I = ffi.new("GrB_Index[]", Il); J = ffi.new("GrB_Index[]", Jl)
    D = S.toarray(); D[np.ix_(Il, Jl)] = 11                  # S has no stored zeros: its pattern is D's non-zeros

    def extract(A):
        C = Matrix.sparse(INT64, 4, 3)
        gb.base._check(lib.GrB_Matrix_extract(C._matrix[0], ffi.NULL, ffi.NULL, A._matrix[0], I, 4, J, 3, ffi.NULL))
        return C

    def assign(A):
        gb.base._check(lib.GrB_Matrix_assign_INT64(A._matrix[0], ffi.NULL, ffi.NULL, 11, I, 4, J, 3, ffi.NULL))
        return A

    def kron(A, Bm):
        C = Matrix.sparse(INT64, 300 * 6, 200 * 5)
        gb.base._check(lib.GrB_Matrix_kronecker_BinaryOp(C._matrix[0], ffi.NULL, ffi.NULL, INT64.TIMES.get_op(), A._matrix[0], Bm._matrix[0], ffi.NULL))
        return C

    _sweep(lambda: (_mat_lists(S, INT64),), lambda A: A.select(">", 4), _same_csr(sp.csr_matrix(S.multiply(S > 4))))
    _sweep(lambda: (_mat_lists(S, INT64),), extract, _same_csr(sp.csr_matrix(S[Il][:, Jl])))
    _sweep(lambda: (_mat_lists(S, INT64),), assign, _same_csr(sp.csr_matrix(D)))
    _sweep(lambda: (_mat_lists(S, INT64), _mat(B, INT64)), kron, _same_csr(sp.kron(S, B).tocsr()))
