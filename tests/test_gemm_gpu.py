"""GrB_mxm with two full dense-form operands, the tiled semiring GEMM (DESIGN.md section 3.6, "Two full dense operands"): the
same bits as the SpMM route on the same values (A given an all-ones presence array takes that route), the FP fold order
against its restatement at the value edges, every type against the oracle, the four descriptor forms, masks, accumulators
and replace, the routes left alone, aliasing, sizes, determinism, allocation failures, and all-pairs shortest paths,
transitive closure and a GNN layer end to end."""
import gc

import numpy as np
import pytest
import scipy.sparse as sp
from scipy.sparse import csgraph

import pygraphblas_b200 as gb
from pygraphblas_b200 import Matrix, descriptor, ffi, lib
from pygraphblas_b200.generators import rmat_csr
from oracle import oracle as orc
import kernel_check as kc
import util
from test_alloc_failure_gpu import _sweep
from test_dense_gpu import FAST, RUNTIME, check, g_csr, g_dense, o_dense, rand_csr, status
from test_gemm import route
from test_sddmm import SEG, tree_fold

pytestmark = pytest.mark.gpu

DENSE = (lib.GxB_FULL, lib.GxB_BITMAP)
KS = (1, 2, 63, 64, 65, 127, 128, 129, 192, 1000, 4097)
EDGES = (1, 7, 127, 129, 300)


def tokens():
    return kc.last_kernel().split(";")


def expect_gemm(t, fast=None, tree=None, write="dense"):
    assert "gemm" in t and not any(e.startswith(("spmm", "sddmm")) for e in t), t
    if fast is not None:
        assert ("gemm-fast" if fast else "gemm-generic") in t, t
    if tree is not None:
        assert ("gemm-tree" in t) == tree, t
    assert f"write={write}" in t, t


def vals(rng, typ, shape, fp_random=True):
    """Values of typ; FP ones uniform in [-0.25, 0.75), so every FP sum depends on its order."""
    n = int(np.prod(shape))
    if typ in util.FP_T and fp_random:
        return (rng.random(n) - 0.25).astype(orc.DTYPES[typ]).reshape(shape)
    return util.rand_values(rng, typ, n).reshape(shape)


def mxm(sr, A, B, desc="", mask=None, C=None, accum=None, ctyp=None, shape=None):
    if C is None:
        C = Matrix.sparse(util.g_type(ctyp or orc.semiring_ztype(sr)), *shape)
    A.mxm(B, semiring=kc.semiring(*sr), mask=mask, out=C, accum=util.g_accum(accum), desc=util.g_desc(desc))
    return C, tokens()


def dense_bits(C):
    x, p = C.to_numpy()
    return kc._bits(x), p


def same_as_spmm(sr, m, k, n, label, atyp=None, btyp=None, a=None, b=None):
    """C = A (+).(x) B on the GEMM and on the SpMM route (A with an all-ones presence array): the same bits, the same presence."""
    add, mul, typ = sr
    rng = np.random.default_rng(kc.seed_of("gemm", label, sr, m, k, n))
    atyp, btyp = atyp or typ, btyp or typ
    a = vals(rng, atyp, (m, k)) if a is None else a
    b = vals(rng, btyp, (k, n)) if b is None else b
    C1, t1 = mxm(sr, g_dense(atyp, a, None), g_dense(btyp, b, None), shape=(m, n))
    expect_gemm(t1, tree=k > SEG)
    C2, t2 = mxm(sr, g_dense(atyp, a, np.ones((m, k), np.uint8)), g_dense(btyp, b, None), shape=(m, n))
    assert "spmm" in t2 and "gemm" not in t2, t2
    (x1, p1), (x2, p2) = dense_bits(C1), dense_bits(C2)
    assert np.array_equal(p1, p2), f"{label} {sr}: presence differs"
    assert np.array_equal(x1, x2), f"{label} {sr} m={m} k={k} n={n}: {int((x1 != x2).sum())} values differ"
    assert status(C1) == (lib.GxB_FULL if k > 0 else lib.GxB_BITMAP)
    return t1, a, b, C1


# ------------------------------------------------------------------ the same bits as the SpMM route
@pytest.mark.parametrize("sr", FAST, ids=lambda s: "_".join(s))
def test_specialised_semirings(sr):
    for m, k, n in ((7, 1, 129), (129, 65, 7), (127, 64, 300), (1, 129, 1)):
        t, *_ = same_as_spmm(sr, m, k, n, "fast")
        expect_gemm(t, fast=True)


@pytest.mark.parametrize("k", KS)
def test_k_on_both_sides_of_the_chunk(k):
    for sr in (("PLUS", "TIMES", "FP32"), ("PLUS", "TIMES", "FP64"), ("MIN", "PLUS", "INT64"), ("LOR", "LAND", "BOOL")):
        t, *_ = same_as_spmm(sr, 129, k, 127 if k < 1000 else 65, "k")
        expect_gemm(t, fast=True, tree=k > SEG)


@pytest.mark.parametrize("m", EDGES)
def test_edges_of_the_tiles(m):
    for n in EDGES:
        same_as_spmm(("PLUS", "TIMES", "FP32"), m, 70, n, "edges")
    same_as_spmm(("MIN", "PLUS", "UINT32"), m, 3, 300, "edges")


@pytest.mark.parametrize("sr", RUNTIME[::3], ids=lambda s: "_".join(s))
def test_runtime_semirings(sr):
    for k in (5, 70):
        t, *_ = same_as_spmm(sr, 37, k, 66, "runtime")
        expect_gemm(t, fast=False)


@pytest.mark.parametrize("atyp,btyp,sr", [("INT8", "FP32", ("PLUS", "TIMES", "FP64")), ("BOOL", "INT16", ("MAX", "PLUS", "INT32")),
                                          ("FP64", "UINT8", ("MIN", "TIMES", "INT64")), ("UINT16", "BOOL", ("LOR", "LAND", "BOOL")),
                                          ("FP32", "FP32", ("LOR", "GT", "FP32")), ("INT64", "INT32", ("PLUS", "PAIR", "FP32"))])
def test_mixed_type_casts(atyp, btyp, sr):
    for k in (6, 100):
        same_as_spmm(sr, 20, k, 33, "cast", atyp=atyp, btyp=btyp)


# ------------------------------------------------------------------ FP order: the restatement, vectorised over outputs
def chunked_gemm(a, b, add, mul):
    """T = a (+).(x) b in the fold order of the kernel: k ascending in chunks of SEG, each folded left to right from its first
    product, the chunk partials through tree_fold.  Every operation rounds to the arrays' type."""
    k = a.shape[1]
    parts = []
    with np.errstate(all="ignore"):
        for k0 in range(0, k, SEG):
            acc = mul(a[:, k0, None], b[None, k0, :])
            for kk in range(k0 + 1, min(k0 + SEG, k)):
                acc = add(acc, mul(a[:, kk, None], b[None, kk, :]))
            parts.append((acc, True))
        return tree_fold(parts, lambda x, y: add(x, y))[0]


NP_OPS = {"PLUS": np.add, "TIMES": np.multiply, "MIN": np.fmin, "MAX": np.fmax}


@pytest.mark.parametrize("typ", util.FP_T)
@pytest.mark.parametrize("add,mul", [("MIN", "PLUS"), ("MAX", "TIMES"), ("PLUS", "TIMES")])
def test_fp_order_at_the_value_edges(typ, add, mul):
    m, k, n = 33, 200, 40
    rng = np.random.default_rng(kc.seed_of("gemm-order", typ, add, mul))
    dt = orc.DTYPES[typ]
    a = util.rand_edge_values(rng, typ, m * k, 0.3).reshape(m, k)
    b = util.rand_edge_values(rng, typ, k * n, 0.3).reshape(k, n)
    for desc in ("", "T0T1"):
        A = g_dense(typ, a if desc == "" else np.ascontiguousarray(a.T), None)
        B = g_dense(typ, b if desc == "" else np.ascontiguousarray(b.T), None)
        C, t = mxm((add, mul, typ), A, B, desc, shape=(m, n))
        expect_gemm(t, fast=(add, mul, typ) in FAST, tree=True)
        got, pres = C.to_numpy()
        assert pres.all()
        want = chunked_gemm(a.astype(dt), b.astype(dt), NP_OPS[add], NP_OPS[mul]).astype(dt)
        keys = np.arange(m * n)
        msg = kc.compare(keys, got.reshape(-1), keys, want.reshape(-1), typ, add, f"{typ} {add}.{mul} {desc}")
        assert msg is None, msg


# ------------------------------------------------------------------ every type at its edges, against the oracle
@pytest.mark.parametrize("typ", util.ALL_T)
def test_value_edges_against_the_oracle(typ):
    m, k, n = 20, 9, 18
    srs = (("MIN", "PLUS"), ("MAX", "TIMES"), ("PLUS", "TIMES"), ("TIMES", "PLUS")) if typ != "BOOL" else (("LOR", "LAND"), ("LAND", "LOR"))
    for add, mul in srs:
        sr = (add, mul, typ)
        pool = "edge" if add in ("MIN", "MAX") else kc.fp_pool_for(add, mul)
        a = kc.values(kc.seed_of("gemm-edges", typ, add, 0), typ, m * k, pool, 0).reshape(m, k)
        b = kc.values(kc.seed_of("gemm-edges", typ, add, 1), typ, k * n, pool, 1).reshape(k, n)
        C1, t = mxm(sr, g_dense(typ, a, None), g_dense(typ, b, None), shape=(m, n))
        C2, _ = mxm(sr, g_dense(typ, a, None), g_dense(typ, b, None), shape=(m, n))
        expect_gemm(t, fast=None)
        assert all(np.array_equal(kc._bits(np.asarray(x)), kc._bits(np.asarray(y))) for x, y in zip(C1.to_arrays(), C2.to_arrays()))
        want = orc.mxm(orc.SpMat(typ, m, n), None, None, sr, o_dense(typ, a, None), o_dense(typ, b, None), "")
        check(C1, want, add, f"edges {sr}")


# ------------------------------------------------------------------ descriptors
@pytest.mark.parametrize("desc", ["", "T0", "T1", "T0T1"])
def test_descriptors(desc):
    m, k, n = 45, 150, 70
    rng = np.random.default_rng(kc.seed_of("gemm-desc", desc))
    tr = np.ascontiguousarray
    for sr in (("PLUS", "TIMES", "INT32"), ("MIN", "PLUS", "FP32"), ("MAX", "TIMES", "FP64"), ("PLUS", "TIMES", "UINT8"),
               ("LOR", "LAND", "BOOL"), ("PLUS", "MINUS", "INT64")):
        typ = sr[2]
        a, b = vals(rng, typ, (m, k)), vals(rng, typ, (k, n))
        ga = a if "T0" not in desc else tr(a.T)
        gb_ = b if "T1" not in desc else tr(b.T)
        C, t = mxm(sr, g_dense(typ, ga, None), g_dense(typ, gb_, None), desc, shape=(m, n))
        expect_gemm(t, tree=True)
        want = orc.mxm(orc.SpMat(typ, m, n), None, None, sr, o_dense(typ, ga, None), o_dense(typ, gb_, None), desc)
        check(C, want, sr[0], f"{desc} {sr}")
    # FP PLUS under every form: the chunked order, and the same bits whatever the layout
    a, b = vals(rng, "FP32", (m, k)), vals(rng, "FP32", (k, n))
    C, t = mxm(("PLUS", "TIMES", "FP32"), g_dense("FP32", a if "T0" not in desc else tr(a.T), None),
               g_dense("FP32", b if "T1" not in desc else tr(b.T), None), desc, shape=(m, n))
    expect_gemm(t, fast=True, tree=True)
    assert np.array_equal(kc._bits(C.to_numpy()[0]), kc._bits(chunked_gemm(a, b, np.add, np.multiply)))


# ------------------------------------------------------------------ masks, accumulators, replace
MASKS = ["none", "dense", "dense-full", "csr"]


@pytest.mark.parametrize("desc", ["", "C", "R", "RC", "S", "SC", "RS", "RSC"])
@pytest.mark.parametrize("mask", MASKS)
@pytest.mark.parametrize("c_kind", ["empty", "csr", "dense"])
def test_masks_accumulators_replace(desc, mask, c_kind):
    rng = np.random.default_rng(kc.seed_of("gemm-mask", desc, mask, c_kind))
    m, k, n = 30, 70, 27
    sr = ("PLUS", "TIMES", "INT32")
    a, b = vals(rng, "INT32", (m, k)), vals(rng, "INT32", (k, n))
    mv = util.rand_values(rng, "FP32", m * n).reshape(m, n)
    mv[rng.random((m, n)) < 0.3] = 0
    mp = (rng.random((m, n)) < 0.6).astype(np.uint8)
    cx = util.rand_values(rng, "INT64", m * n).reshape(m, n)
    cp = (rng.random((m, n)) < 0.5).astype(np.uint8)
    for accum in (None, ("PLUS", "INT64")):
        if mask == "none":
            M, om = None, None
        elif mask == "dense":
            M, om = g_dense("FP32", mv, mp), o_dense("FP32", mv, mp)
        elif mask == "dense-full":
            M, om = g_dense("FP32", mv, None), o_dense("FP32", mv, None)
        else:
            I, J = np.nonzero(mp)
            M, om = Matrix.from_lists(I, J, mv[I, J], m, n, gb.FP32), orc.SpMat("FP32", m, n, I, J, mv[I, J])
        if c_kind == "empty":
            C, oc = Matrix.sparse(gb.INT64, m, n), orc.SpMat("INT64", m, n)
        elif c_kind == "dense":
            C, oc = g_dense("INT64", cx, cp), o_dense("INT64", cx, cp)
        else:
            I, J = np.nonzero(cp)
            C, oc = Matrix.from_lists(I, J, cx[I, J], m, n, gb.INT64), o_dense("INT64", cx, cp)
        C, t = mxm(sr, g_dense("INT32", a, None), g_dense("INT32", b, None), desc, mask=M, C=C, accum=accum)
        if M is None and "C" in desc:
            assert "gemm" not in t, t                                   # C<!NULL>: no product
        elif mask == "csr" and "C" not in desc:
            assert "sddmm" in t, t                                      # a sparse mask keeps the SDDMM
        else:
            expect_gemm(t, fast=True, tree=True, write="csr" if mask == "csr" else "dense")
            if mask != "csr":
                assert status(C) in DENSE
        want = orc.mxm(oc, om, accum, sr, o_dense("INT32", a, None), o_dense("INT32", b, None), desc)
        check(C, want, "PLUS", f"{desc} {mask} {c_kind} {accum}")


# ------------------------------------------------------------------ routes left alone
def test_routes_left_alone():
    rng = np.random.default_rng(21)
    m, k, n = 9, 12, 11
    sr = ("PLUS", "TIMES", "INT64")
    a, b = vals(rng, "INT64", (m, k)), vals(rng, "INT64", (k, n))
    ones = lambda s: np.ones(s, np.uint8)
    oa, ob = o_dense("INT64", a, None), o_dense("INT64", b, None)
    want = orc.mxm(orc.SpMat("INT64", m, n), None, None, sr, oa, ob, "")
    for A, B in ((g_dense("INT64", a, ones((m, k))), g_dense("INT64", b, None)),
                 (g_dense("INT64", a, None), g_dense("INT64", b, ones((k, n)))),
                 (g_dense("INT64", a, ones((m, k))), g_dense("INT64", b, ones((k, n))))):
        C, t = mxm(sr, A, B, shape=(m, n))
        assert "spmm" in t and "gemm" not in t, t                       # presence on either operand
        check(C, want, "PLUS", "presence")
    S = rand_csr(rng, "BOOL", m, n, 0.4)
    C, t = mxm(sr, g_dense("INT64", a, None), g_dense("INT64", b, None), mask=g_csr("BOOL", S), shape=(m, n))
    assert "sddmm" in t and "gemm" not in t, t                          # a sparse, not complemented mask
    C, t = mxm(("MIN", "FIRSTJ", "INT64"), g_dense("INT64", a, None), g_dense("INT64", b, None), shape=(m, n))
    assert any(e.startswith("positional=") for e in t) and "gemm" not in t, t
    Bc = Matrix.from_lists(*np.nonzero(b), b[np.nonzero(b)], k, n, gb.INT64)
    C, t = mxm(sr, g_dense("INT64", a, None), Bc, shape=(m, n))
    assert "spmm-left" in t and "gemm" not in t, t                      # a CSR operand
    check(C, want, "PLUS", "csr B")
    assert route(True, True, False) == "gemm" and route(True, True, False, a_pres=True) == "other"
    assert route(True, True, True) == "sddmm" and route(True, True, True, mask_comp=True) == "gemm"


# ------------------------------------------------------------------ aliasing
def test_aliasing():
    rng = np.random.default_rng(22)
    n, sr = 70, ("PLUS", "TIMES", "FP64")
    x, y = vals(rng, "FP64", (n, n)), vals(rng, "FP64", (n, n))
    ox, oy = o_dense("FP64", x, None), o_dense("FP64", y, None)
    acc = ("PLUS", "FP64")
    for alias in ("A", "B"):
        X, Y = g_dense("FP64", x, None), g_dense("FP64", y, None)
        C = X if alias == "A" else Y
        C, t = mxm(sr, X, Y, C=C, accum=acc)
        expect_gemm(t, fast=True, tree=True)
        want = chunked_gemm(x, y, np.add, np.multiply) + (x if alias == "A" else y)
        assert np.array_equal(kc._bits(C.to_numpy()[0]), kc._bits(want))
    # A is B: X X and X X'
    for desc in ("", "T1"):
        X = g_dense("FP64", x, None)
        C, t = mxm(sr, X, X, desc, shape=(n, n))
        expect_gemm(t, fast=True)
        assert np.array_equal(kc._bits(C.to_numpy()[0]), kc._bits(chunked_gemm(x, x if desc == "" else np.ascontiguousarray(x.T), np.add, np.multiply)))
    # D <- min(D, D min.+ D), in place
    d = rng.integers(0, 50, (n, n)).astype(np.float64)
    D = g_dense("FP64", d, None)
    for _ in range(3):
        D, t = mxm(("MIN", "PLUS", "FP64"), D, D, C=D, accum=("MIN", "FP64"))
        expect_gemm(t, fast=True)
        d = np.minimum(d, (d[:, :, None] + d[None, :, :]).min(axis=1))
    assert np.array_equal(D.to_numpy()[0], d) and status(D) == lib.GxB_FULL


# ------------------------------------------------------------------ sizes
def test_sizes():
    rng = np.random.default_rng(23)
    # a long m with n = 1: more tiles than one grid dimension holds
    m = (1 << 24) + 3
    a = rng.integers(-3, 4, (m, 3)).astype(np.int32)
    b = rng.integers(-3, 4, (3, 1)).astype(np.int32)
    C, t = mxm(("PLUS", "TIMES", "INT32"), g_dense("INT32", a, None), g_dense("INT32", b, None), shape=(m, 1))
    expect_gemm(t, fast=True, tree=False)
    got, pres = C.to_numpy()
    assert pres.all() and np.array_equal(got, a @ b)
    del a, C, got, pres
    # k = 0: no entries
    for sr in (("PLUS", "TIMES", "FP32"), ("MIN", "PLUS", "INT64")):
        C, t = mxm(sr, Matrix.from_numpy(np.zeros((5, 0), orc.DTYPES[sr[2]])), Matrix.from_numpy(np.zeros((0, 7), orc.DTYPES[sr[2]])),
                   shape=(5, 7))
        assert "gemm" in t and C.nvals == 0 and C.shape == (5, 7)
    # m or n of 1, and empty dimensions
    for m, k, n in ((1, 100, 50), (50, 100, 1), (1, 1, 1)):
        same_as_spmm(("PLUS", "TIMES", "FP32"), m, k, n, "sizes")
    for m, k, n in ((0, 5, 4), (4, 5, 0)):
        C, t = mxm(("PLUS", "TIMES", "FP32"), Matrix.from_numpy(np.ones((m, k), np.float32)), Matrix.from_numpy(np.ones((k, n), np.float32)),
                   shape=(m, n))
        assert "gemm" in t and C.nvals == 0
    flops, nout = ffi.new("uint64_t*"), ffi.new("uint64_t*")
    mxm(("PLUS", "TIMES", "FP32"), Matrix.from_numpy(np.ones((6, 70), np.float32)), Matrix.from_numpy(np.ones((70, 5), np.float32)), shape=(6, 5))
    lib.B200_last_mxm_stats(flops, nout)
    assert flops[0] == 6 * 70 * 5


def test_determinism():
    rng = np.random.default_rng(24)
    a, b = vals(rng, "FP32", (300, 1000)), vals(rng, "FP32", (1000, 129))
    got = [dense_bits(mxm(("PLUS", "TIMES", "FP32"), g_dense("FP32", a, None), g_dense("FP32", b, None), shape=(300, 129))[0])[0]
           for _ in range(2)]
    assert np.array_equal(got[0], got[1])


# ------------------------------------------------------------------ allocation failures
def test_allocation_failures():
    rng = np.random.default_rng(25)
    m, k, n = 40, 30, 50
    a, b = vals(rng, "FP32", (m, k)), vals(rng, "FP32", (k, n))
    mv = (rng.random((m, n)) < 0.5).astype(np.float32)
    _sweep(lambda: (g_dense("FP32", a, None), g_dense("FP32", b, None)),
           lambda A, B: A.mxm(B, semiring=gb.FP32.MIN_PLUS, out=Matrix.sparse(gb.FP32, m, n)))
    _sweep(lambda: (g_dense("FP32", a, None), g_dense("FP32", b, None), g_dense("FP32", mv, None)),
           lambda A, B, M: A.mxm(B, semiring=gb.FP32.PLUS_TIMES, mask=M, out=g_dense("FP32", mv, None), accum=gb.FP32.PLUS))
    a2, b2 = vals(rng, "INT64", (m, 200)), vals(rng, "INT8", (n, 200))
    _sweep(lambda: (g_dense("INT64", a2, None), g_dense("INT8", b2, None)),
           lambda A, B: A.mxm(B, semiring=gb.INT64.PLUS_TIMES, desc=descriptor.T1, out=Matrix.sparse(gb.INT64, m, n)))
    gc.collect()


# ------------------------------------------------------------------ end to end
def test_all_pairs_shortest_paths():
    n, indptr, indices = rmat_csr(10, 8, seed=3)
    rng = np.random.default_rng(26)
    w = rng.integers(1, 20, len(indices)).astype(np.float64)
    G = sp.csr_matrix((w, indices, indptr), shape=(n, n))
    G.sum_duplicates()
    d = np.full((n, n), np.inf)
    d[G.nonzero()] = G.data
    np.fill_diagonal(d, 0.0)
    D = Matrix.from_numpy(d)
    steps = 0
    while (1 << steps) < n:
        D.mxm(D, semiring=gb.FP64.MIN_PLUS, out=D, accum=gb.FP64.MIN)
        expect_gemm(tokens(), fast=True, tree=True)
        steps += 1
    want = csgraph.shortest_path(G, method="D", directed=True)
    got, pres = D.to_numpy()
    assert pres.all() and np.array_equal(got, want)


def test_transitive_closure():
    n, indptr, indices = rmat_csr(10, 4, seed=4)
    G = sp.csr_matrix((np.ones(len(indices), bool), indices, indptr), shape=(n, n))
    r = G.toarray() | np.eye(n, dtype=bool)
    R = Matrix.from_numpy(r)
    for _ in range(10):
        R.mxm(R, semiring=gb.BOOL.LOR_LAND, out=R, accum=gb.BOOL.LOR)
        expect_gemm(tokens(), fast=True, tree=True)
    want = np.isfinite(csgraph.shortest_path(G.astype(np.float64), unweighted=True, directed=True))
    assert np.array_equal(R.to_numpy()[0], want)


def test_gnn_layer():
    """(A H) W and A (H W): the feature transform on the GEMM, the aggregation on the SpMM kernel."""
    n, indptr, indices = rmat_csr(12, 8, seed=5)
    rng = np.random.default_rng(27)
    d, f = 64, 48
    av = (rng.random(len(indices)) + 0.1).astype(np.float32)
    h = (rng.random((n, d)) + 0.1).astype(np.float32)
    wt = (rng.random((d, f)) + 0.1).astype(np.float32)
    A = Matrix.from_csr(indptr, indices, av, n, n, gb.FP32)
    A64 = sp.csr_matrix((av.astype(np.float64), indices, indptr), shape=(n, n))
    want = A64 @ (h.astype(np.float64) @ wt.astype(np.float64))
    rows = np.diff(indptr) > 0
    HW = Matrix.sparse(gb.FP32, n, f)
    Matrix.from_numpy(h).mxm(Matrix.from_numpy(wt), semiring=gb.FP32.PLUS_TIMES, out=HW)
    expect_gemm(tokens(), fast=True, tree=False)
    out = A.mxm(HW, semiring=gb.FP32.PLUS_TIMES, out=Matrix.sparse(gb.FP32, n, f))
    assert "spmm" in tokens()
    got, pres = out.to_numpy()
    assert np.array_equal(pres.all(axis=1), rows)
    assert (np.abs(got[rows] - want[rows]) / want[rows]).max() <= 1e-6
    ah = A.mxm(Matrix.from_numpy(h), semiring=gb.FP32.PLUS_TIMES, out=Matrix.sparse(gb.FP32, n, d)).to_numpy()[0]
    AH = Matrix.from_numpy(ah)
    out = AH.mxm(Matrix.from_numpy(wt), semiring=gb.FP32.PLUS_TIMES, out=Matrix.sparse(gb.FP32, n, f))
    expect_gemm(tokens(), fast=True, tree=False)
    got = out.to_numpy()[0]
    assert (np.abs(got[rows] - want[rows]) / want[rows]).max() <= 1e-6
