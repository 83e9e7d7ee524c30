"""GrB_mxm with a dense-form left operand, C = X (+).(x) op(B) (the left SpMM route, DESIGN.md section 3.6: C' = op(B)' (+).(x)' X' on
the SpMM kernel with the multiply's operands swapped), against the oracle on the CSR equivalent of every dense operand: semirings,
every mirrored multiply, casts, shapes around the transpose's tiles and its grid cap, the split, descriptors, masks, accumulators,
aliasing, two equivalent computations, a 16-source SSSP, the routes left unchanged, R-MAT s20 against scipy, value edges and
determinism, and allocation failures."""
import gc

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.csgraph as csgraph

import pygraphblas_b200 as gb
from pygraphblas_b200 import Matrix, Vector, descriptor, ffi, lib
from pygraphblas_b200.generators import rmat_csr
from pygraphblas_b200.ops import Semiring
from oracle import oracle as orc
import kernel_check as kc
import util
from test_alloc_failure_gpu import _sweep
from test_dense_gpu import FAST, RUNTIME, SEG, check, dense_x, g_csr, g_dense, o_dense, rand_csr, status

pytestmark = pytest.mark.gpu

# the multiply with its operands swapped (restates op_mirror, spmm.cu): mirror(y, x) = mul(x, y)
MIRROR = {"FIRST": "SECOND", "SECOND": "FIRST", "MINUS": "RMINUS", "RMINUS": "MINUS", "DIV": "RDIV", "RDIV": "DIV",
          "ISGT": "ISLT", "ISLT": "ISGT", "ISGE": "ISLE", "ISLE": "ISGE", "GT": "LT", "LT": "GT", "GE": "LE", "LE": "GE"}
CMP = ("GT", "LT", "GE", "LE")
DENSE = (lib.GxB_FULL, lib.GxB_BITMAP)


def new_semiring(add, mul, typ, ztyp):
    """A semiring through GrB_Semiring_new (for the multiplies that have no named builtin semiring)."""
    mon = getattr(lib, f"GrB_{add}_MONOID_{ztyp}")
    op = getattr(lib, f"GrB_{mul}_{typ}", None) or getattr(lib, f"GxB_{mul}_{typ}")
    h = ffi.new("GrB_Semiring*")
    gb.base._check(lib.GrB_Semiring_new(h, mon, op))
    return Semiring(add, mul, typ, h[0])


def tokens():
    return kc.last_kernel().split(";")


def expect_left(t, fast=None, write="dense", split=None, xtr=True, ttr=True):
    assert "spmm" in t and "spmm-left" in t, t
    if fast is not None:
        assert ("spmm-fast" if fast else "spmm-generic") in t, t
    assert f"write={write}" in t, t
    if split is not None:
        assert ("spmm-split" in t) == split, t
    if xtr is not None:
        assert ("x-transpose" in t) == xtr, t
    if ttr is not None:
        assert ("t-transpose" in t) == ttr, t


def not_left(t):
    assert "spmm-left" not in t and "x-transpose" not in t and "t-transpose" not in t, t


def run_left(sr, X, B, desc=None, semiring=None, ctyp=None):
    C = Matrix.sparse(util.g_type(ctyp or sr[2]), X.ncols if desc in ("T0", "T0T1") else X.nrows,
                      B.nrows if desc in ("T1", "T0T1") else B.ncols)
    X.mxm(B, semiring=semiring or kc.semiring(*sr), out=C, desc=getattr(descriptor, desc) if desc else None)
    return C, tokens()


def oracle_left(sr, C, ox, ob, desc=""):
    return orc.mxm(orc.SpMat(C.type.name, C.nrows, C.ncols), None, None, sr, ox, ob, desc)


def _semiring_case(sr, k, label, xtyp=None, btyp=None, xdens=None, n=30, m=40):
    add, mul, typ = sr
    rng = np.random.default_rng(kc.seed_of("left", label, sr, k))
    btyp, xtyp = btyp or typ, xtyp or typ
    S = rand_csr(rng, btyp, n, m, 0.15)
    if btyp in util.FP_T:
        S.data = kc.values(kc.seed_of(label, 1), btyp, S.nnz, kc.fp_pool_for(add, mul), 1)
    x, pres = dense_x(rng, xtyp, k, n, xdens)
    if xtyp in util.FP_T:
        x = kc.values(kc.seed_of(label, 2), xtyp, k * n, kc.fp_pool_for(add, mul), 0).reshape(k, n)
    C, t = run_left(sr, g_dense(xtyp, x, pres), g_csr(btyp, S))
    check(C, oracle_left(sr, C, o_dense(xtyp, x, pres), kc.o_csr(btyp, S, S.data)), add, f"{label} {sr} k={k}")
    return t


# ------------------------------------------------------------------ semirings
@pytest.mark.parametrize("sr", FAST, ids=lambda s: "_".join(s))
def test_specialised_semirings(sr):
    for xdens in (None, 0.5):
        expect_left(_semiring_case(sr, 8, "fast", xdens=xdens), fast=True, split=False)


@pytest.mark.parametrize("sr", RUNTIME, ids=lambda s: "_".join(s))
def test_runtime_semirings(sr):
    expect_left(_semiring_case(sr, 5, "runtime", xdens=0.7), fast=False)


@pytest.mark.parametrize("mul", sorted(MIRROR))
def test_mirrored_multiplies(mul):
    """Every output is one product X(r, i) (x) B(i, j) (one entry per column of B), on values where swapping x and y changes the
    answer: a multiply run without its mirror fails."""
    typ = "INT32" if mul in CMP else "FP64"
    ztyp = "BOOL" if mul in CMP else typ
    add = "LOR" if mul in CMP else "PLUS"
    rng = np.random.default_rng(kc.seed_of("mirror", mul))
    k, n, m = 9, 33, 70
    rows = np.sort(rng.integers(0, n, m))
    S = sp.csr_matrix((np.ones(m), (rows, np.arange(m))), shape=(n, m))
    S.sort_indices()
    pool = np.array([-2.0, -0.75, -0.25, 0.5, 1.0, 1.5, 3.0])
    S.data = (rng.integers(-3, 4, m) if typ == "INT32" else pool[rng.integers(0, len(pool), m)]).astype(orc.DTYPES[typ])
    x = (rng.integers(-3, 4, (k, n)) if typ == "INT32" else pool[rng.integers(0, len(pool), (k, n))]).astype(orc.DTYPES[typ])
    pres = (rng.random((k, n)) < 0.8).astype(np.uint8)
    sr = (add, mul, typ)
    C, t = run_left(sr, g_dense(typ, x, pres), g_csr(typ, S), semiring=new_semiring(add, mul, typ, ztyp), ctyp=ztyp)
    expect_left(t)
    ox, ob = o_dense(typ, x, pres), kc.o_csr(typ, S, S.data)
    want = oracle_left(sr, C, ox, ob)
    check(C, want, add, f"mirror {mul}")
    swapped = oracle_left((add, MIRROR[mul], typ), C, ox, ob)
    assert not np.array_equal(kc._bits(np.asarray(want.X)), kc._bits(np.asarray(swapped.X))), "inputs do not tell x from y"


def test_pow_takes_the_csr_path():
    rng = np.random.default_rng(12)
    S = rand_csr(rng, "FP64", 20, 25, 0.2)
    S.data = rng.choice([0.0, 1.0, 2.0, 3.0], S.nnz)
    x = rng.choice([0.5, 1.0, 2.0, -1.5], (6, 20))
    sr = ("PLUS", "POW", "FP64")
    C, t = run_left(sr, g_dense("FP64", x, None), g_csr("FP64", S), semiring=new_semiring("PLUS", "POW", "FP64", "FP64"))
    assert not any(s.startswith("spmm") for s in t), t
    check(C, oracle_left(sr, C, o_dense("FP64", x, None), kc.o_csr("FP64", S, S.data)), "PLUS", "pow")


@pytest.mark.parametrize("btyp,xtyp,sr", [("INT8", "FP32", ("PLUS", "TIMES", "FP64")), ("BOOL", "INT16", ("MAX", "PLUS", "INT32")),
                                          ("FP64", "UINT8", ("MIN", "TIMES", "INT64")), ("UINT16", "BOOL", ("LOR", "LAND", "BOOL")),
                                          ("FP32", "FP32", ("LOR", "GT", "FP32")), ("INT64", "INT32", ("PLUS", "PAIR", "FP32"))])
def test_mixed_type_casts(btyp, xtyp, sr):
    expect_left(_semiring_case(sr, 6, "cast", xtyp=xtyp, btyp=btyp, xdens=0.8))


# ------------------------------------------------------------------ shapes
@pytest.mark.parametrize("k", [1, 2, 3, 4, 7, 8, 31, 32, 33, 64, 127, 128, 129, 256])
def test_every_k(k):
    for sr in (("PLUS", "TIMES", "FP32"), ("MIN", "PLUS", "INT32")):
        for xdens in (None, 0.6):
            expect_left(_semiring_case(sr, k, "k", xdens=xdens), fast=True, xtr=k > 1)


@pytest.mark.parametrize("n,m", [(30, 1), (1, 40), (31, 33), (32, 32), (33, 31), (63, 65), (64, 64), (65, 95), (97, 1)])
def test_tile_edges(n, m):
    for k in (1, 5, 32, 33):
        for sr in (("PLUS", "TIMES", "FP64"), ("LOR", "LAND", "BOOL"), ("MAX", "PLUS", "INT16")):
            expect_left(_semiring_case(sr, k, "tiles", xdens=0.7, n=n, m=m), xtr=k > 1, ttr=m > 1)


@pytest.mark.parametrize("k,n,m", [(0, 5, 7), (4, 0, 7), (4, 5, 0), (0, 0, 0), (1, 0, 1)])
def test_empty_shapes(k, n, m):
    sr = ("PLUS", "TIMES", "FP32")
    x = np.zeros((k, n), np.float32)
    S = sp.csr_matrix((n, m), dtype=np.float32)
    X = Matrix.from_numpy(x)
    C, t = run_left(sr, X, g_csr("FP32", S))
    if status(X) in DENSE:
        assert "spmm-left" in t, t
    assert C.shape == (k, m) and C.nvals == 0


def test_transpose_grid_cap():
    """More 32 x 32 tiles than the capped grid has CTAs (16 per SM), in both transposes."""
    rng = np.random.default_rng(13)
    k, n, m = 33, 70000, 70000                   # X' and T' have 2 x 2188 tiles each
    sr = ("PLUS", "TIMES", "FP32")
    rows, cols = rng.integers(0, n, 150000), rng.integers(0, m, 150000)
    S = sp.csr_matrix((np.ones(len(rows), np.float32), (rows, cols)), shape=(n, m))
    S.sum_duplicates()
    S.data = util.rand_values(rng, "FP32", S.nnz)
    x, pres = dense_x(rng, "FP32", k, n, 0.9)
    C, t = run_left(sr, g_dense("FP32", x, pres), g_csr("FP32", S))
    expect_left(t)
    check(C, oracle_left(sr, C, o_dense("FP32", x, pres), kc.o_csr("FP32", S, S.data)), "PLUS", "grid cap")


# ------------------------------------------------------------------ the split (rows of op(B)' = columns of B)
@pytest.mark.parametrize("k", [1, 33])
def test_column_lengths_around_the_split(k):
    lens = [0, 1, 0, SEG - 1, SEG, SEG + 1, 2 * SEG, 2 * SEG + 1, 0, 3 * SEG - 1, 17, 5000]
    rng = np.random.default_rng(k)
    for sr, typ in ((("PLUS", "TIMES", "INT64"), "INT64"), (("PLUS", "TIMES", "FP32"), "FP32"), (("MAX", "PLUS", "FP64"), "FP64")):
        St = rand_csr(rng, typ, len(lens), 6000, None, lens=lens)      # B' has the row lengths: B's columns
        S = St.T.tocsr(); S.sort_indices()
        x, pres = dense_x(rng, typ, k, 6000, 0.9)
        C, t = run_left(sr, g_dense(typ, x, pres), g_csr(typ, S))
        expect_left(t, split=True, xtr=k > 1)
        check(C, oracle_left(sr, C, o_dense(typ, x, pres), kc.o_csr(typ, S, S.data)), sr[0], f"lens {sr}")
    # columns all at the threshold: no split
    St = rand_csr(rng, "INT32", 20, 600, None, lens=[SEG] * 10 + [0] * 10)
    S = St.T.tocsr(); S.sort_indices()
    x, _ = dense_x(rng, "INT32", k, 600)
    sr = ("PLUS", "TIMES", "INT32")
    C, t = run_left(sr, g_dense("INT32", x, None), g_csr("INT32", S))
    expect_left(t, split=False, xtr=k > 1)
    check(C, oracle_left(sr, C, o_dense("INT32", x, None), kc.o_csr("INT32", S, S.data)), "PLUS", "at SEG")


def test_single_long_column():
    rng = np.random.default_rng(11)
    S = rand_csr(rng, "FP32", 3, 200000, None, lens=[0, 150000, 3]).T.tocsr()
    S.sort_indices()
    x, _ = dense_x(rng, "FP32", 4, 200000)
    sr = ("PLUS", "TIMES", "FP32")
    C, t = run_left(sr, g_dense("FP32", x, None), g_csr("FP32", S))
    expect_left(t, split=True)
    check(C, oracle_left(sr, C, o_dense("FP32", x, None), kc.o_csr("FP32", S, S.data)), "PLUS", "long column")


# ------------------------------------------------------------------ descriptors
@pytest.mark.parametrize("desc", ["T0", "T1", "T0T1"])
@pytest.mark.parametrize("k", [1, 6, 40])
def test_transposed_operands(desc, k):
    rng = np.random.default_rng(kc.seed_of("desc", desc, k))
    n, m = 35, 27
    sr = ("PLUS", "TIMES", "FP64")
    S = rand_csr(rng, "FP64", m, n, 0.2) if "T1" in desc else rand_csr(rng, "FP64", n, m, 0.2)
    x, pres = dense_x(rng, "FP64", n, k, 0.7) if "T0" in desc else dense_x(rng, "FP64", k, n, 0.7)
    B = g_csr("FP64", S)
    C, t = run_left(sr, g_dense("FP64", x, pres), B, desc=desc)
    expect_left(t, xtr=k > 1 and "T0" not in desc)
    check(C, oracle_left(sr, C, o_dense("FP64", x, pres), kc.o_csr("FP64", S, S.data), desc), "PLUS", desc)


# ------------------------------------------------------------------ mask, accumulator, replace
@pytest.mark.parametrize("desc", ["", "C", "R", "RC", "S", "SC", "RS", "RSC"])
@pytest.mark.parametrize("mask_kind", ["none", "dense", "dense-full", "csr"])
@pytest.mark.parametrize("c_kind", ["empty", "csr", "dense"])
def test_mask_accum_replace(desc, mask_kind, c_kind):
    if mask_kind == "none" and "S" in desc:
        pytest.skip("a structural flag without a mask is the no-mask case")
    rng = np.random.default_rng(kc.seed_of("left", desc, mask_kind, c_kind))
    k, n, m = 6, 15, 20
    S = rand_csr(rng, "INT32", n, m, 0.2)
    x, pres = dense_x(rng, "INT32", k, n, 0.8)
    mp = None if mask_kind == "dense-full" else (rng.random((k, m)) < 0.6).astype(np.uint8)
    mx = (rng.random((k, m)) < 0.5).astype(np.float32)
    cx, cp = dense_x(rng, "INT64", k, m, 0.5)
    o_mask = None if mask_kind == "none" else o_dense("FP32", mx, mp)
    for accum in (None, ("PLUS", "INT64")):
        if c_kind == "empty":
            C, oc = Matrix.sparse(gb.INT64, k, m), orc.SpMat("INT64", k, m)
        elif c_kind == "dense":
            C, oc = g_dense("INT64", cx, cp), o_dense("INT64", cx, cp)
        else:
            I, J = np.nonzero(cp)
            C, oc = Matrix.from_lists(I, J, cx[I, J], k, m, gb.INT64), o_dense("INT64", cx, cp)
        M = None
        if mask_kind in ("dense", "dense-full"):
            M = g_dense("FP32", mx, mp)
        elif mask_kind == "csr":
            I, J = np.nonzero(mp)
            M = Matrix.from_lists(I, J, mx[I, J], k, m, gb.FP32)
        d = getattr(descriptor, desc) if desc else None
        sr = ("PLUS", "TIMES", "INT32")
        g_dense("INT32", x, pres).mxm(g_csr("INT32", S), semiring=gb.INT32.PLUS_TIMES, out=C, mask=M, accum=util.g_accum(accum), desc=d)
        t = tokens()
        want = orc.mxm(oc, o_mask, accum, sr, o_dense("INT32", x, pres), kc.o_csr("INT32", S, S.data), desc)
        check(C, want, "PLUS", f"{desc} {mask_kind} {c_kind} {accum}")
        if mask_kind == "none" and "C" in desc:
            continue                                   # C<!NULL>: the early exit, no product
        expect_left(t, write="csr" if mask_kind == "csr" else "dense")
        if mask_kind != "csr":
            assert status(C) in DENSE


# ------------------------------------------------------------------ aliasing
def test_aliasing():
    rng = np.random.default_rng(8)
    n, k = 24, 5
    S = rand_csr(rng, "FP64", n, n, 0.2)
    sr = ("PLUS", "TIMES", "FP64")
    ob = kc.o_csr("FP64", S, S.data)
    # C is X: X <- X A, three times, stays a dense form
    x, pres = dense_x(rng, "FP64", k, n, 0.8)
    X, ox = g_dense("FP64", x, pres), o_dense("FP64", x, pres)
    A = g_csr("FP64", S)
    for it in range(3):
        X.mxm(A, semiring=gb.FP64.PLUS_TIMES, out=X)
        expect_left(tokens())
        assert status(X) in DENSE
        ox = orc.mxm(orc.SpMat("FP64", k, n), None, None, sr, ox, ob)
        check(X, ox, "PLUS", f"C is X, step {it}")
    # C is B: B <- X B (square)
    x, pres = dense_x(rng, "FP64", n, n, 0.7)
    B = g_csr("FP64", S)
    g_dense("FP64", x, pres).mxm(B, semiring=gb.FP64.PLUS_TIMES, out=B)
    expect_left(tokens())
    check(B, orc.mxm(orc.SpMat("FP64", n, n), None, None, sr, o_dense("FP64", x, pres), ob), "PLUS", "C is B")


# ------------------------------------------------------------------ equivalences
@pytest.mark.parametrize("sr", [("PLUS", "TIMES", "FP32"), ("MIN", "FIRST", "FP32"), ("MAX", "PLUS", "FP64"), ("PLUS", "MINUS", "FP64"),
                                ("PLUS", "SECOND", "INT64")], ids=lambda s: "_".join(s))
def test_equivalent_computations(sr):
    """X (+).(x) A, bit for bit, equals (A' (+).(x)' X')' on the right route and k GrB_vxm calls (quarter values: exact sums)."""
    add, mul, typ = sr
    rng = np.random.default_rng(kc.seed_of("equiv", sr))
    k, n, m = 37, 300, 260
    dt = np.dtype(orc.DTYPES[typ])
    S = rand_csr(rng, typ, n, m, 0.05, lens=list(rng.integers(0, 150, n)))
    S.data = (rng.integers(-4, 5, S.nnz) / (4.0 if typ in util.FP_T else 1.0)).astype(dt)
    x = (rng.integers(-4, 5, (k, n)) / (4.0 if typ in util.FP_T else 1.0)).astype(dt)
    pres = (rng.random((k, n)) < 0.7).astype(np.uint8)
    C, t = run_left(sr, g_dense(typ, x, pres), g_csr(typ, S))
    expect_left(t)
    got, gp = C.to_numpy()
    got = np.where(gp.astype(bool), got, dt.type(0))
    # the right route under the mirrored multiply, on X' = (X')' stored n x k, then transposed
    A = g_csr(typ, S)
    R = Matrix.sparse(util.g_type(typ), m, k)
    A.mxm(g_dense(typ, np.ascontiguousarray(x.T), np.ascontiguousarray(pres.T)), semiring=kc.semiring(add, MIRROR.get(mul, mul), typ),
          out=R, desc=descriptor.T0)
    t = tokens()
    assert "spmm" in t and "spmm-left" not in t, t
    rv, rp = R.to_numpy()
    assert np.array_equal(rp.T, gp)
    assert np.array_equal(kc._bits(np.where(rp.astype(bool), rv, dt.type(0)).T), kc._bits(got))
    # k vxm calls, one per row of X
    for r in range(k):
        u = Vector.from_numpy(np.ascontiguousarray(x[r]), present=np.ascontiguousarray(pres[r]))
        w = Vector.sparse(util.g_type(typ), m)
        u.vxm(A, semiring=kc.semiring(*sr), out=w)
        wv, wp = w.to_numpy()
        assert np.array_equal(wp, gp[r]), r
        assert np.array_equal(kc._bits(np.where(wp.astype(bool), wv, dt.type(0))), kc._bits(got[r])), r


# ------------------------------------------------------------------ end to end: 16-source SSSP
def test_multi_source_sssp():
    n, indptr, indices = rmat_csr(14, 16, 3)
    rng = np.random.default_rng(14)
    w = rng.integers(1, 10, len(indices)).astype(np.float64)
    A = Matrix.from_csr(indptr, indices, w, n, n, gb.FP64)
    sources = rng.choice(n, 16, replace=False)
    d0, p0 = np.zeros((16, n)), np.zeros((16, n), np.uint8)
    p0[np.arange(16), sources] = 1
    D = Matrix.from_numpy(d0, present=p0)
    prev = D.to_numpy()
    for it in range(n):
        D.mxm(A, semiring=gb.FP64.MIN_PLUS, accum=gb.FP64.MIN, out=D)
        expect_left(tokens(), fast=True)
        assert status(D) in DENSE
        cur = D.to_numpy()
        if np.array_equal(cur[1], prev[1]) and np.array_equal(cur[0][cur[1] == 1], prev[0][prev[1] == 1]):
            break
        prev = cur
    dist = csgraph.dijkstra(sp.csr_matrix((w, indices, indptr), shape=(n, n)), directed=True, indices=sources)
    got, pres = D.to_numpy()
    assert np.array_equal(pres.astype(bool), np.isfinite(dist))
    assert np.array_equal(got[pres == 1], dist[pres == 1])


# ------------------------------------------------------------------ routes left unchanged
def test_unchanged_routes():
    rng = np.random.default_rng(15)
    S = rand_csr(rng, "INT64", 20, 30, 0.2)
    x, pres = dense_x(rng, "INT64", 7, 20, 0.8)
    I, J = np.nonzero(pres)
    Xc = Matrix.from_lists(I, J, x[I, J], 7, 20, gb.INT64)
    # dense A with dense B: the right route
    sd = S.toarray()
    C = Matrix.sparse(gb.INT64, 7, 30)
    g_dense("INT64", x, pres).mxm(g_dense("INT64", sd, (sd != 0).astype(np.uint8)), semiring=gb.INT64.PLUS_TIMES, out=C)
    t = tokens()
    assert "spmm" in t, t
    not_left(t)
    # a positional semiring with a dense left operand: the positional rewrite, same result as with a CSR left operand
    for s in (gb.INT64.MIN_FIRSTJ, gb.INT64.MIN_SECONDJ):
        C1 = g_dense("INT64", x, pres).mxm(g_csr("INT64", S), semiring=s, out=Matrix.sparse(gb.INT64, 7, 30))
        t = tokens()
        assert any(e.startswith("positional=") for e in t), t
        not_left(t)
        assert C1.iseq(Xc.mxm(g_csr("INT64", S), semiring=s, out=Matrix.sparse(gb.INT64, 7, 30)))
    # k * m > 2^31 - 1: the CSR path (its product rows stay in the small bin)
    m = (1 << 30) + 1
    bi = np.array([0, 3, 3, 50, 99]); bj = np.array([0, 5, m - 1, 1 << 29, m - 1])
    bv = np.array([2, 3, 4, 5, 6], np.int64)
    B = Matrix.from_lists(bi, bj, bv, 100, m, gb.INT64)
    x2 = rng.integers(-5, 6, (2, 100)).astype(np.int64)
    C = Matrix.sparse(gb.INT64, 2, m)
    Matrix.from_numpy(x2).mxm(B, semiring=gb.INT64.PLUS_TIMES, out=C)
    t = tokens()
    assert not any(e.startswith("spmm") for e in t), t
    want = {}
    for i, j, v in zip(bi, bj, bv):
        for r in range(2):
            want[(r, int(j))] = want.get((r, int(j)), 0) + int(x2[r, i]) * int(v)
    gI, gJ, gX = C.to_arrays()
    assert sorted(zip(map(int, gI), map(int, gJ), map(int, gX))) == sorted((r, j, v) for (r, j), v in want.items())


# ------------------------------------------------------------------ R-MAT s20 against scipy
def test_rmat_s20_against_scipy():
    n, indptr, indices = rmat_csr(20, 16, 1)
    rng = np.random.default_rng(20)
    vals = (rng.random(len(indices), dtype=np.float32) + np.float32(0.5)).astype(np.float32)
    x = rng.random((32, n), dtype=np.float32)
    A = Matrix.from_csr(indptr, indices, vals, n, n, gb.FP32)
    C, t = run_left(("PLUS", "TIMES", "FP32"), Matrix.from_numpy(x), A)
    expect_left(t, fast=True, split=True)
    got, pres = C.to_numpy()
    St = sp.csr_matrix((vals.astype(np.float64), indices, indptr), shape=(n, n)).T.tocsr()
    want = (St @ x.T.astype(np.float64)).T
    nonempty = np.bincount(indices, minlength=n) > 0          # the non-empty columns of A
    assert np.array_equal(pres.all(axis=0), nonempty) and not pres[:, ~nonempty].any()
    err = np.abs(got - want) / np.maximum(np.abs(want), 1e-30)
    assert err[:, nonempty].max() <= 1e-6


# ------------------------------------------------------------------ value edges and determinism
@pytest.mark.parametrize("typ", util.ALL_T)
def test_value_edges_and_determinism(typ):
    rng = np.random.default_rng(kc.seed_of("left-edges", typ))
    for add, mul in (("MIN", "PLUS"), ("MAX", "TIMES"), ("PLUS", "TIMES")) if typ != "BOOL" else (("LOR", "LAND"), ("LAND", "LOR")):
        sr = (add, mul, typ)
        S = rand_csr(rng, typ, 40, 30, 0.2)
        S.data = kc.values(kc.seed_of(typ, add, 1), typ, S.nnz, "edge" if add != "PLUS" else kc.fp_pool_for(add, mul), 1)
        x = kc.values(kc.seed_of(typ, add, 0), typ, 9 * 40, "edge" if add != "PLUS" else kc.fp_pool_for(add, mul), 0).reshape(9, 40)
        C1, t = run_left(sr, g_dense(typ, x, None), g_csr(typ, S))
        C2, _ = run_left(sr, g_dense(typ, x, None), g_csr(typ, S))
        expect_left(t)
        a1, a2 = C1.to_numpy(), C2.to_numpy()
        assert np.array_equal(kc._bits(a1[0]), kc._bits(a2[0])) and np.array_equal(a1[1], a2[1])
        check(C1, oracle_left(sr, C1, o_dense(typ, x, None), kc.o_csr(typ, S, S.data)), add, f"edges {sr}")


# ------------------------------------------------------------------ allocation failures
def test_allocation_failures():
    rng = np.random.default_rng(9)
    S = rand_csr(rng, "FP32", 600, 300, None, lens=[0] * 10 + [290] + [5] * 589).T.tocsr()
    S.sort_indices()
    x, pres = dense_x(rng, "FP32", 12, 300, 0.7)
    mx, mp = dense_x(rng, "FP32", 12, 600, 0.5)
    _sweep(lambda: (g_dense("FP32", x, pres), g_csr("FP32", S)),
           lambda X, B: X.mxm(B, semiring=gb.FP32.PLUS_TIMES))
    _sweep(lambda: (g_dense("FP32", x, pres), g_csr("FP32", S), g_dense("FP32", mx, mp)),
           lambda X, B, M: X.mxm(B, semiring=gb.FP32.MIN_PLUS, out=g_dense("FP32", mx, None), mask=M, accum=gb.FP32.PLUS))
    _sweep(lambda: (g_dense("FP32", x, pres), g_csr("FP32", S), Matrix.from_lists(*np.nonzero(mp), mx[np.nonzero(mp)], 12, 600, gb.FP32)),
           lambda X, B, M: X.mxm(B, semiring=gb.FP32.PLUS_TIMES, mask=M))
    _sweep(lambda: (g_dense("FP32", np.ascontiguousarray(x.T), np.ascontiguousarray(pres.T)), g_csr("FP32", S)),
           lambda X, B: X.mxm(B, semiring=gb.FP32.PLUS_TIMES, out=Matrix.sparse(gb.FP32, 12, 600), desc=descriptor.T0))
    gc.collect()
