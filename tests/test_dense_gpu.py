"""Dense-form matrices and GrB_mxm with a dense right operand (the SpMM path, DESIGN.md section 3.6), against the oracle on the
CSR equivalent of every dense operand: import / export round trips, a dense-form matrix in the other operations, the SpMM
kernel over semirings, types, k, row lengths on both sides of the split threshold, masks, accumulators, aliasing, value
edges and determinism, the CSR path for the same operands, and allocation failures."""
import gc

import numpy as np
import pytest
import scipy.sparse as sp

import pygraphblas_b200 as gb
from pygraphblas_b200 import Matrix, Vector, descriptor, ffi, lib
from pygraphblas_b200.generators import rmat_csr
from oracle import oracle as orc
import kernel_check as kc
import util
from test_alloc_failure_gpu import _sweep

pytestmark = pytest.mark.gpu

SEG = 64        # restates SPMM_SEG (spmm.cu): rows longer than this are folded in segments ("spmm-split")
NUM_FAST = ["FP32", "FP64", "INT32", "INT64", "UINT32", "UINT64"]
FAST = [(a, m, t) for t in NUM_FAST for a, m in (("PLUS", "TIMES"), ("MIN", "PLUS"), ("PLUS", "SECOND"), ("PLUS", "FIRST"),
                                                   ("PLUS", "PAIR"), ("MIN", "FIRST"), ("MIN", "SECOND"))] + \
       [("LOR", "LAND", "BOOL"), ("ANY", "PAIR", "BOOL"), ("LOR", "PAIR", "BOOL"), ("LOR", "SECOND", "BOOL"), ("LOR", "FIRST", "BOOL")]
RUNTIME = [(a, m, t) for t in util.ALL_T for (a, m, _) in util.semirings_for(t)
           if (a, m, t) not in FAST and not (a == "ANY" and m != "PAIR")]


def status(M):
    p = ffi.new("int*")
    assert lib.GxB_Matrix_Option_get(M._matrix[0], lib.GxB_SPARSITY_STATUS, p) == lib.GrB_SUCCESS
    return p[0]


def dense_x(rng, typ, n, k, density=None, values=None):
    x = util.rand_values(rng, typ, n * k).reshape(n, k) if values is None else values.reshape(n, k)
    pres = None if density is None else (rng.random((n, k)) < density).astype(np.uint8)
    return x, pres


def o_dense(typ, x, pres):
    I, J = np.nonzero(np.ones(x.shape, bool) if pres is None else pres.astype(bool))
    return orc.SpMat(typ, x.shape[0], x.shape[1], I, J, x[I, J])


def rand_csr(rng, typ, m, n, density, lens=None):
    if lens is None:
        S = sp.random(m, n, density=density, format="csr", random_state=rng)
    else:       # row i gets lens[i] distinct columns
        rows = np.repeat(np.arange(m), lens)
        cols = np.concatenate([rng.choice(n, L, replace=False) for L in lens]) if len(lens) else np.zeros(0, int)
        S = sp.csr_matrix((np.ones(len(rows)), (rows, cols)), shape=(m, n))
    S.sort_indices()
    S.data = util.rand_values(rng, typ, S.nnz)
    return S


def g_csr(typ, S):
    return Matrix.from_csr(S.indptr, S.indices, S.data, S.shape[0], S.shape[1], util.g_type(typ))


def g_dense(typ, x, pres):
    return Matrix.from_numpy(x, present=pres, typ=util.g_type(typ))


def keyed(M):
    I, J, X = M.to_arrays() if isinstance(M, Matrix) else (M.I, M.J, M.X)
    return np.asarray(I, np.int64) * M.ncols + np.asarray(J, np.int64), np.asarray(X)


def check(got, want, add, label):
    gI, gX = keyed(got)
    wI, wX = keyed(want)
    msg = kc.compare(gI, gX, wI, wX, want.type, add, label)
    assert msg is None, msg


def run_spmm(sr, A, X):
    C = Matrix.sparse(util.g_type(sr[2]), A.nrows, X.ncols)
    A.mxm(X, semiring=kc.semiring(*sr), out=C)
    return C, kc.last_kernel().split(";")


def expect_spmm(tokens, fast=None, write="dense", split=None):
    assert "spmm" in tokens, tokens
    if fast is not None:
        assert ("spmm-fast" if fast else "spmm-generic") in tokens, tokens
    assert f"write={write}" in tokens, tokens
    if split is not None:
        assert ("spmm-split" in tokens) == split, tokens


# ------------------------------------------------------------------ import / export
@pytest.mark.parametrize("typ", util.ALL_T)
def test_round_trip(typ):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(kc.seed_of("rt", typ))
    x = util.rand_edge_values(rng, typ, 7 * 5).reshape(7, 5)
    for pres in (None, (rng.random((7, 5)) < 0.5).astype(np.uint8)):
        M = g_dense(typ, x, pres)
        assert status(M) == (lib.GxB_FULL if pres is None else lib.GxB_BITMAP)
        gx, gp = M.to_numpy()
        want_p = np.ones((7, 5), np.uint8) if pres is None else pres
        assert np.array_equal(gp, want_p)
        assert np.array_equal(kc._bits(gx)[want_p == 1], kc._bits(x)[want_p == 1])
        assert M.nvals == int(want_p.sum())
        # where = 1: torch device tensors, through their raw bytes
        dx = torch.from_numpy(np.ascontiguousarray(x).view(np.uint8).reshape(-1).copy()).cuda()
        dp = torch.from_numpy(want_p.reshape(-1).copy()).cuda() if pres is not None else None
        h = ffi.new("GrB_Matrix*")
        gb.base._check(lib.B200_Matrix_import_dense(h, util.g_type(typ).gb_type, 7, 5, ffi.cast("void*", dx.data_ptr()),
                                                     ffi.cast("uint8_t*", dp.data_ptr()) if dp is not None else ffi.NULL, 1))
        M1 = Matrix(h)
        ox = torch.zeros_like(dx); op = torch.zeros(35, dtype=torch.uint8, device="cuda")
        gb.base._check(lib.B200_Matrix_export_dense(M1._matrix[0], ffi.cast("void*", ox.data_ptr()), ffi.cast("uint8_t*", op.data_ptr()), 1))
        assert np.array_equal(op.cpu().numpy().reshape(7, 5), want_p)
        got = ox.cpu().numpy().view(x.dtype).reshape(7, 5)
        assert np.array_equal(kc._bits(got)[want_p == 1], kc._bits(x)[want_p == 1])
        check(M1, o_dense(typ, x, want_p), "PLUS", f"{typ} where=1")
    # a CSR-built matrix exports the dense image of its tuples (zeros where absent) and stays CSR
    S = rand_csr(rng, typ, 9, 6, 0.3)
    C = g_csr(typ, S)
    cx, cp = C.to_numpy()
    rows = np.repeat(np.arange(9), np.diff(S.indptr))
    dense, pat = np.zeros((9, 6), x.dtype), np.zeros((9, 6), np.uint8)
    dense[rows, S.indices], pat[rows, S.indices] = S.data, 1
    assert np.array_equal(cp, pat) and np.array_equal(kc._bits(cx), kc._bits(dense))
    assert status(C) not in (lib.GxB_FULL, lib.GxB_BITMAP)


def test_empty_dense_shapes():
    for shape in ((0, 0), (0, 4), (4, 0)):
        M = Matrix.from_numpy(np.zeros(shape, np.float32))
        assert M.nvals == 0 and M.shape == shape
        x, p = M.to_numpy()
        assert x.shape == shape and p.shape == shape


def test_dense_form_in_other_operations():
    rng = np.random.default_rng(5)
    x, pres = dense_x(rng, "FP64", 12, 9, density=0.6)
    D = g_dense("FP64", x, pres)
    I, J = np.nonzero(pres)
    E = Matrix.from_lists(I, J, x[I, J], 12, 9, gb.FP64)
    assert D.nvals == E.nvals
    for a, b in zip(D.to_arrays(), E.to_arrays()):
        assert np.array_equal(a, b)
    assert D.get(int(I[0]), int(J[0])) == E.get(int(I[0]), int(J[0]))
    absent = np.argwhere(pres == 0)[0]
    assert D.get(int(absent[0]), int(absent[1])) is None
    assert status(D) == lib.GxB_BITMAP               # reading the tuples keeps the dense form
    assert D.eadd(E).iseq(E.eadd(E))
    assert D.transpose().iseq(E.transpose())
    u = Vector.from_lists(list(range(9)), util.rand_values(rng, "FP64", 9), 9, gb.FP64)
    assert D.mxv(u).iseq(E.mxv(u))
    B = Matrix.from_lists(*map(list, np.nonzero(np.ones((12, 9)))), [1.0] * 108, 12, 9, gb.FP64)
    assert B.eadd(B, mask=D).iseq(B.eadd(B, mask=E))
    Dd = D.dup()
    assert status(Dd) == lib.GxB_BITMAP and Dd.iseq(E)
    # every modification drops the dense form, and the next read reflects it
    D[0, 0] = 42.0
    assert status(D) not in (lib.GxB_FULL, lib.GxB_BITMAP)
    assert D.get(0, 0) == 42.0
    assert Dd.iseq(E)                                 # the copy keeps its own dense form
    F = g_dense("FP64", x, None)
    assert status(F) == lib.GxB_FULL
    del F[1, 1]
    assert F.nvals == 12 * 9 - 1 and status(F) not in (lib.GxB_FULL, lib.GxB_BITMAP)
    F.clear()
    assert F.nvals == 0


# ------------------------------------------------------------------ the SpMM path
def _semiring_case(sr, k, label, xtyp=None, atyp=None, xdens=None, rng=None):
    add, mul, typ = sr
    rng = rng or np.random.default_rng(kc.seed_of(label, sr, k))
    atyp, xtyp = atyp or typ, xtyp or typ
    S = rand_csr(rng, atyp, 40, 30, 0.15)
    S.data = kc.values(kc.seed_of(label, 1), atyp, S.nnz, kc.fp_pool_for(add, mul), 0) if atyp in util.FP_T else S.data
    x, pres = dense_x(rng, xtyp, 30, k, xdens)
    if xtyp in util.FP_T:
        x = kc.values(kc.seed_of(label, 2), xtyp, 30 * k, kc.fp_pool_for(add, mul), 1).reshape(30, k)
    C, tokens = run_spmm(sr, g_csr(atyp, S), g_dense(xtyp, x, pres))
    want = orc.mxm(orc.SpMat(C.type.name, 40, k), None, None, sr, kc.o_csr(atyp, S, S.data), o_dense(xtyp, x, pres))
    check(C, want, add, f"{label} {sr} k={k}")
    return tokens


@pytest.mark.parametrize("sr", FAST, ids=lambda s: "_".join(s))
def test_specialised_semirings(sr):
    for xdens in (None, 0.5):
        tokens = _semiring_case(sr, 8, "fast", xdens=xdens)
        expect_spmm(tokens, fast=True, split=False)


@pytest.mark.parametrize("sr", RUNTIME, ids=lambda s: "_".join(s))
def test_runtime_semirings(sr):
    tokens = _semiring_case(sr, 5, "runtime", xdens=0.7)
    expect_spmm(tokens, fast=False)


@pytest.mark.parametrize("atyp,xtyp,sr", [("INT8", "FP32", ("PLUS", "TIMES", "FP64")), ("BOOL", "INT16", ("MAX", "PLUS", "INT32")),
                                          ("FP64", "UINT8", ("MIN", "TIMES", "INT64")), ("UINT16", "BOOL", ("LOR", "LAND", "BOOL")),
                                          ("FP32", "FP32", ("LOR", "GT", "FP32")), ("INT64", "INT32", ("PLUS", "PAIR", "FP32"))])
def test_mixed_type_casts(atyp, xtyp, sr):
    tokens = _semiring_case(sr, 6, "cast", xtyp=xtyp, atyp=atyp, xdens=0.8)
    expect_spmm(tokens)


@pytest.mark.parametrize("k", [1, 2, 3, 4, 7, 8, 31, 32, 33, 64, 127, 128, 129, 256])
def test_every_k(k):
    for sr in (("PLUS", "TIMES", "FP32"), ("MIN", "PLUS", "INT32")):
        for xdens in (None, 0.6):
            expect_spmm(_semiring_case(sr, k, "k", xdens=xdens), fast=True)


@pytest.mark.parametrize("k", [1, 33])
def test_row_lengths_around_the_split(k):
    lens = [0, 1, 0, SEG - 1, SEG, SEG + 1, 2 * SEG, 2 * SEG + 1, 0, 3 * SEG - 1, 17, 5000]
    rng = np.random.default_rng(k)
    for sr, typ in ((("PLUS", "TIMES", "INT64"), "INT64"), (("PLUS", "TIMES", "FP32"), "FP32"), (("MAX", "PLUS", "FP64"), "FP64")):
        S = rand_csr(rng, typ, len(lens), 6000, None, lens=lens)
        x, pres = dense_x(rng, typ, 6000, k, 0.9)
        C, tokens = run_spmm(sr, g_csr(typ, S), g_dense(typ, x, pres))
        expect_spmm(tokens, split=True)
        check(C, orc.mxm(orc.SpMat(typ, len(lens), k), None, None, sr, kc.o_csr(typ, S, S.data), o_dense(typ, x, pres)), sr[0], f"lens {sr}")
    # rows all at the threshold: no split
    S = rand_csr(rng, "INT32", 20, 600, None, lens=[SEG] * 10 + [0] * 10)
    x, _ = dense_x(rng, "INT32", 600, k)
    C, tokens = run_spmm(("PLUS", "TIMES", "INT32"), g_csr("INT32", S), g_dense("INT32", x, None))
    expect_spmm(tokens, split=False)
    check(C, orc.mxm(orc.SpMat("INT32", 20, k), None, None, ("PLUS", "TIMES", "INT32"), kc.o_csr("INT32", S, S.data), o_dense("INT32", x, None)), "PLUS", "at SEG")


def test_single_long_row():
    rng = np.random.default_rng(11)
    S = rand_csr(rng, "FP32", 3, 200000, None, lens=[0, 150000, 3])
    x, _ = dense_x(rng, "FP32", 200000, 4)
    sr = ("PLUS", "TIMES", "FP32")
    C, tokens = run_spmm(sr, g_csr("FP32", S), g_dense("FP32", x, None))
    expect_spmm(tokens, split=True)
    check(C, orc.mxm(orc.SpMat("FP32", 3, 4), None, None, sr, kc.o_csr("FP32", S, S.data), o_dense("FP32", x, None)), "PLUS", "long row")


@pytest.mark.parametrize("a_dense", [False, True])
def test_transposed_a(a_dense):
    rng = np.random.default_rng(3)
    S = rand_csr(rng, "FP64", 30, 25, 0.2)
    x, pres = dense_x(rng, "FP64", 30, 7, 0.7)
    A = g_csr("FP64", S) if not a_dense else g_dense("FP64", S.toarray(), (S.toarray() != 0).astype(np.uint8))
    C = Matrix.sparse(gb.FP64, 25, 7)
    A.mxm(g_dense("FP64", x, pres), semiring=gb.FP64.PLUS_TIMES, out=C, desc=descriptor.T0)
    expect_spmm(kc.last_kernel().split(";"))
    oa = kc.o_csr("FP64", S, S.data) if not a_dense else o_dense("FP64", S.toarray(), (S.toarray() != 0).astype(np.uint8))
    check(C, orc.mxm(orc.SpMat("FP64", 25, 7), None, None, ("PLUS", "TIMES", "FP64"), oa, o_dense("FP64", x, pres), "T0"), "PLUS", "T0")


@pytest.mark.parametrize("desc", ["", "C", "R", "RC", "S", "SC", "RS", "RSC"])
@pytest.mark.parametrize("mask_kind", ["none", "dense", "dense-full", "csr"])
@pytest.mark.parametrize("c_kind", ["empty", "csr", "dense"])
def test_mask_accum_replace(desc, mask_kind, c_kind):
    if mask_kind == "none" and "S" in desc:
        pytest.skip("a structural flag without a mask is the no-mask case")
    rng = np.random.default_rng(kc.seed_of(desc, mask_kind, c_kind))
    m, n, k = 20, 15, 6
    S = rand_csr(rng, "INT32", m, n, 0.2)
    x, pres = dense_x(rng, "INT32", n, k, 0.8)
    mp = None if mask_kind == "dense-full" else (rng.random((m, k)) < 0.6).astype(np.uint8)
    mx = (rng.random((m, k)) < 0.5).astype(np.float32)           # mask values: true and false entries
    cx, cp = dense_x(rng, "INT64", m, k, 0.5)
    o_mask = None if mask_kind == "none" else o_dense("FP32", mx, mp)
    for accum in (None, ("PLUS", "INT64")):
        if c_kind == "empty":
            C, oc = Matrix.sparse(gb.INT64, m, k), orc.SpMat("INT64", m, k)
        elif c_kind == "dense":
            C, oc = g_dense("INT64", cx, cp), o_dense("INT64", cx, cp)
        else:
            I, J = np.nonzero(cp)
            C, oc = Matrix.from_lists(I, J, cx[I, J], m, k, gb.INT64), o_dense("INT64", cx, cp)
        M = None
        if mask_kind in ("dense", "dense-full"):
            M = g_dense("FP32", mx, mp)
        elif mask_kind == "csr":
            I, J = np.nonzero(mp)
            M = Matrix.from_lists(I, J, mx[I, J], m, k, gb.FP32)
            assert status(M) not in (lib.GxB_FULL, lib.GxB_BITMAP)
        d = getattr(descriptor, desc) if desc else None
        sr = ("PLUS", "TIMES", "INT32")
        A, X = g_csr("INT32", S), g_dense("INT32", x, pres)
        A.mxm(X, semiring=gb.INT32.PLUS_TIMES, out=C, mask=M, accum=util.g_accum(accum), desc=d)
        tokens = kc.last_kernel().split(";")
        want = orc.mxm(oc, o_mask, accum, sr, kc.o_csr("INT32", S, S.data), o_dense("INT32", x, pres), desc)
        check(C, want, "PLUS", f"{desc} {mask_kind} {c_kind} {accum}")
        if mask_kind == "none" and "C" in desc:
            continue                                   # C<!NULL>: the early exit, no product
        expect_spmm(tokens, write="csr" if mask_kind == "csr" else "dense")
        if mask_kind != "csr":
            assert status(C) in (lib.GxB_FULL, lib.GxB_BITMAP)


def test_aliasing():
    rng = np.random.default_rng(8)
    n = 24
    S = rand_csr(rng, "FP64", n, n, 0.2)
    x, pres = dense_x(rng, "FP64", n, n, 0.8)
    sr = ("PLUS", "TIMES", "FP64")
    want = orc.mxm(orc.SpMat("FP64", n, n), None, None, sr, kc.o_csr("FP64", S, S.data), o_dense("FP64", x, pres))
    # C aliases X: X = A X
    X = g_dense("FP64", x, pres)
    g_csr("FP64", S).mxm(X, semiring=gb.FP64.PLUS_TIMES, out=X)
    expect_spmm(kc.last_kernel().split(";"))
    check(X, want, "PLUS", "C is X")
    # C aliases A (A dense too): A = A X
    sd = S.toarray()
    A = g_dense("FP64", sd, (sd != 0).astype(np.uint8))
    A.mxm(g_dense("FP64", x, pres), semiring=gb.FP64.PLUS_TIMES, out=A)
    expect_spmm(kc.last_kernel().split(";"))
    want_a = orc.mxm(orc.SpMat("FP64", n, n), None, None, sr, o_dense("FP64", sd, (sd != 0).astype(np.uint8)), o_dense("FP64", x, pres))
    check(A, want_a, "PLUS", "C is A")
    # iterating X <- A X keeps the dense form
    X = g_dense("FP64", x, None)
    A = g_csr("FP64", S)
    for _ in range(3):
        A.mxm(X, semiring=gb.FP64.PLUS_TIMES, out=X)
    assert status(X) in (lib.GxB_FULL, lib.GxB_BITMAP)


@pytest.mark.parametrize("typ", util.ALL_T)
def test_value_edges_and_determinism(typ):
    rng = np.random.default_rng(kc.seed_of("edges", typ))
    for add, mul in (("MIN", "PLUS"), ("MAX", "TIMES"), ("PLUS", "TIMES")) if typ != "BOOL" else (("LOR", "LAND"), ("LAND", "LOR")):
        sr = (add, mul, typ)
        S = rand_csr(rng, typ, 30, 40, 0.2)
        S.data = kc.values(kc.seed_of(typ, add, 0), typ, S.nnz, "edge" if add != "PLUS" else kc.fp_pool_for(add, mul), 0)
        x = kc.values(kc.seed_of(typ, add, 1), typ, 40 * 9, "edge" if add != "PLUS" else kc.fp_pool_for(add, mul), 1).reshape(40, 9)
        C1, tokens = run_spmm(sr, g_csr(typ, S), g_dense(typ, x, None))
        C2, _ = run_spmm(sr, g_csr(typ, S), g_dense(typ, x, None))
        expect_spmm(tokens)
        a1, a2 = C1.to_numpy(), C2.to_numpy()
        assert np.array_equal(kc._bits(a1[0]), kc._bits(a2[0])) and np.array_equal(a1[1], a2[1])
        check(C1, orc.mxm(orc.SpMat(typ, 30, 9), None, None, sr, kc.o_csr(typ, S, S.data), o_dense(typ, x, None)), add, f"edges {sr}")


def test_csr_x_takes_the_old_path():
    rng = np.random.default_rng(4)
    S = rand_csr(rng, "FP32", 50, 40, 0.1)
    x, pres = dense_x(rng, "FP32", 40, 16, 0.5)
    I, J = np.nonzero(pres)
    Xc = Matrix.from_lists(I, J, x[I, J], 40, 16, gb.FP32)
    A = g_csr("FP32", S)
    Cs, tokens = run_spmm(("PLUS", "TIMES", "FP32"), A, g_dense("FP32", x, pres))
    expect_spmm(tokens)
    Cc = Matrix.sparse(gb.FP32, 50, 16)
    A.mxm(Xc, semiring=gb.FP32.PLUS_TIMES, out=Cc)
    tokens = kc.last_kernel().split(";")
    assert not any(t.startswith("spmm") for t in tokens) and not any(t.startswith("write=") for t in tokens), tokens
    assert any(t.startswith("esc-") or t == "spa" for t in tokens), tokens
    assert Cs.iseq(Cc)
    # transposed dense B falls back to the CSR path too
    Xt = g_dense("FP32", np.ascontiguousarray(x.T), np.ascontiguousarray(pres.T))
    Ct = Matrix.sparse(gb.FP32, 50, 16)
    A.mxm(Xt, semiring=gb.FP32.PLUS_TIMES, out=Ct, desc=descriptor.T1)
    assert not any(t.startswith("spmm") for t in kc.last_kernel().split(";"))
    assert Ct.iseq(Cc)


def test_rmat_s20_against_scipy():
    n, indptr, indices = rmat_csr(20, 16, 1)
    rng = np.random.default_rng(20)
    vals = (rng.random(len(indices), dtype=np.float32) + np.float32(0.5)).astype(np.float32)
    x = rng.random((n, 32), dtype=np.float32)
    A = Matrix.from_csr(indptr, indices, vals, n, n, gb.FP32)
    C, tokens = run_spmm(("PLUS", "TIMES", "FP32"), A, Matrix.from_numpy(x))
    expect_spmm(tokens, fast=True, split=True)
    got, pres = C.to_numpy()
    S = sp.csr_matrix((vals.astype(np.float64), indices, indptr), shape=(n, n))
    want = S @ x.astype(np.float64)
    nonempty = np.diff(indptr) > 0
    assert np.array_equal(pres.all(axis=1), nonempty) and not pres[~nonempty].any()
    err = np.abs(got - want) / np.maximum(np.abs(want), 1e-30)
    assert err[nonempty].max() <= 1e-6


# ------------------------------------------------------------------ allocation failures
def test_allocation_failures():
    rng = np.random.default_rng(9)
    S = rand_csr(rng, "FP32", 600, 300, 0.01, lens=[0] * 10 + [290] + [5] * 589)
    x, pres = dense_x(rng, "FP32", 300, 12, 0.7)
    mx, mp = dense_x(rng, "FP32", 600, 12, 0.5)
    _sweep(lambda: (), lambda: g_dense("FP32", x, pres))
    _sweep(lambda: (g_csr("FP32", S),), lambda A: A.to_numpy()[0])
    _sweep(lambda: (g_dense("FP32", x, pres),), lambda D: D.to_arrays()[2])                         # the CSR conversion
    _sweep(lambda: (g_csr("FP32", S), g_dense("FP32", x, pres)),
           lambda A, X: A.mxm(X, semiring=gb.FP32.PLUS_TIMES))
    _sweep(lambda: (g_csr("FP32", S), g_dense("FP32", x, pres), g_dense("FP32", mx, mp)),
           lambda A, X, M: A.mxm(X, semiring=gb.FP32.MIN_PLUS, out=g_dense("FP32", mx, None), mask=M, accum=gb.FP32.PLUS))
    _sweep(lambda: (g_csr("FP32", S), g_dense("FP32", x, pres), Matrix.from_lists(*np.nonzero(mp), mx[np.nonzero(mp)], 600, 12, gb.FP32)),
           lambda A, X, M: A.mxm(X, semiring=gb.FP32.PLUS_TIMES, mask=M))
    gc.collect()
