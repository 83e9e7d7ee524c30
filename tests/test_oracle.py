"""CPU tests that PIN THE ORACLE: against every golden vector the reference's tests hold for
the mxm/mxv/vxm path, against an independent pure-Python model, against scipy, and against
the known karate-club triangle count."""
import numpy as np
import pytest
import scipy.sparse as sp

from oracle import oracle as orc
from oracle import pymodel
import util


def test_oracle_matches_reference_goldens(goldens):
    assert len(goldens["cases"]) >= 30
    for case in goldens["cases"]:
        res = util.oracle_run(case)
        ok = util.same_mat(res, case["expect"]) if case["op"] == "mxm" else util.same_vec(res, case["expect"])
        assert ok, f"{case['id']} ({case['source']}): got {res}, expected {case['expect']}"


def _dict(d):
    if "nrows" in d:
        return {(i, j): orc.DTYPES[d["type"]](x) for i, j, x in zip(d["I"], d["J"], d["X"])}
    return {(i, 0): orc.DTYPES[d["type"]](x) for i, x in zip(d["I"], d["X"])}


@pytest.mark.parametrize("seed", range(40))
def test_oracle_matches_python_model(seed):
    rng = np.random.default_rng(seed)
    typ = util.ALL_T[seed % len(util.ALL_T)]
    m, k, n = rng.integers(1, 9, 3)
    A = util.rand_mat(rng, typ, int(k) if seed % 3 == 1 else int(m), int(m) if seed % 3 == 1 else int(k), 0.4)
    B = util.rand_mat(rng, rng.choice(util.ALL_T), int(k), int(n), 0.4)
    desc = "T0" if seed % 3 == 1 else ""
    extra = ["", "C", "R", "RC", "S", "RSC", "SC", "RS"][seed % 8]
    desc = extra + desc
    ctype = rng.choice(util.ALL_T)
    C = util.rand_mat(rng, ctype, int(m), int(n), 0.3)
    M = util.rand_mat(rng, rng.choice(util.ALL_T), int(m), int(n), 0.5) if seed % 2 == 0 else None
    srs = util.semirings_for(typ)
    sr = srs[seed % len(srs)]
    ztype = orc.semiring_ztype(sr)
    accum = None
    if seed % 4 >= 2:
        accum = (["PLUS", "MIN", "MAX", "SECOND", "FIRST", "TIMES"][seed % 6], ctype)
    f = orc.parse_desc(desc)
    expect = pymodel.mxm(_dict(C), ctype, _dict(M) if M else None, M["type"] if M else None, accum, sr,
                         _dict(A), A["type"], _dict(B), B["type"], f)
    got = orc.mxm(util.o_mat(C), util.o_mat(M) if M else None, accum, sr, util.o_mat(A), util.o_mat(B), desc).todict()
    assert set(got) == set(expect), (seed, sr, desc, got, expect)
    for kk in got:
        assert got[kk] == expect[kk].item(), (seed, sr, desc, kk, got[kk], expect[kk])


@pytest.mark.parametrize("desc", ["C", "RC", "SC", "RSC"])
def test_oracle_complemented_null_mask(desc):
    """C<!NULL>: nothing is let through; REPLACE clears C (both restatements agree, C API 1.3 section 4.3)."""
    rng = np.random.default_rng(5)
    A, B, C = util.rand_mat(rng, "INT32", 6, 6, 0.5), util.rand_mat(rng, "INT32", 6, 6, 0.5), util.rand_mat(rng, "INT32", 6, 6, 0.4)
    sr = ("PLUS", "TIMES", "INT32")
    for accum in (None, ("PLUS", "INT32")):
        got = orc.mxm(util.o_mat(C), None, accum, sr, util.o_mat(A), util.o_mat(B), desc).todict()
        expect = pymodel.mxm(_dict(C), "INT32", None, None, accum, sr, _dict(A), "INT32", _dict(B), "INT32", orc.parse_desc(desc))
        assert set(got) == set(expect) == (set() if "R" in desc else set(_dict(C)))
        assert all(got[k] == _dict(C)[k] for k in got)


def test_oracle_plus_times_matches_scipy():
    # BASELINE.json configs[0]: 1024 x 1024 random 1% CSR, PLUS_TIMES_FP64 mxv
    A = sp.random(1024, 1024, density=0.01, format="csr", dtype=np.float64, random_state=0)
    A.sort_indices()
    u = np.random.default_rng(0).random(1024)
    coo = A.tocoo()
    Ao = orc.SpMat("FP64", 1024, 1024, coo.row, coo.col, coo.data)
    uo = orc.SpVec("FP64", 1024, np.arange(1024), u)
    w = orc.mxv(orc.SpVec("FP64", 1024), None, None, ("PLUS", "TIMES", "FP64"), Ao, uo)
    ref = A @ u
    nz = np.diff(A.indptr) > 0
    assert np.array_equal(w.I, np.nonzero(nz)[0])
    assert np.allclose(w.X, ref[nz], rtol=1e-12, atol=0)
    # SpGEMM against scipy too
    B = sp.random(300, 200, density=0.03, format="csr", dtype=np.float64, random_state=1)
    Cs = (A[:200, :300] @ B).tocoo()
    a2 = A[:200, :300].tocoo()
    b2 = B.tocoo()
    Co = orc.mxm(orc.SpMat("FP64", 200, 200), None, None, ("PLUS", "TIMES", "FP64"),
                 orc.SpMat("FP64", 200, 300, a2.row, a2.col, a2.data), orc.SpMat("FP64", 300, 200, b2.row, b2.col, b2.data))
    ref = sp.csr_matrix(Cs).todok()
    assert Co.nvals == len(ref)
    for (i, j), x in Co.todict().items():
        assert abs(ref[i, j] - x) <= 1e-12 * abs(x)


def test_oracle_karate_triangles(goldens):
    import networkx as nx
    G = nx.karate_club_graph()
    n = G.number_of_nodes()
    rows, cols = [], []
    for a, b in G.edges():
        lo, hi = min(a, b), max(a, b)
        rows.append(hi); cols.append(lo)            # strict lower triangle L
    L = orc.SpMat("INT64", n, n, rows, cols, np.ones(len(rows), np.int64))
    # demo/Triangle-Counting.ipynb:581-582: L.mxm(L, mask=L) with PLUS_PAIR, then reduce
    C = orc.mxm(orc.SpMat("INT64", n, n), L, None, ("PLUS", "PAIR", "INT64"), L, L, "")
    assert int(C.X.sum()) == goldens["known_answers"]["karate_triangles"]["value"] == 45
    # dot form C<L> = L * L' (descriptor ST1, demo/TriangleCentrality.ipynb:596) counts the same triangles
    C2 = orc.mxm(orc.SpMat("INT64", n, n), L, None, ("PLUS", "PAIR", "INT64"), L, L, "ST1")
    assert int(C2.X.sum()) == 45


def test_fast_kernels_match_oracle():
    """The typed OpenMP kernels used as the bench CPU baseline agree with the generic oracle."""
    import ctypes
    from pygraphblas_b200.generators import rmat_csr
    L = orc.lib()
    n, indptr, indices = rmat_csr(10, 8, seed=5)
    nnz = len(indices)
    rng = np.random.default_rng(3)
    vals = (rng.random(nnz, dtype=np.float32) + 0.5).astype(np.float32)
    u = rng.random(n, dtype=np.float32)
    w = np.zeros(n, np.float32); pres = np.zeros(n, np.uint8)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    L.fast_spmv_plus_times_f32(ctypes.c_int64(n), p(indptr), p(indices), p(vals), p(u), p(w), p(pres))
    rows = np.repeat(np.arange(n), np.diff(indptr))
    Ao = orc.SpMat("FP32", n, n, rows, indices, vals)
    wo = orc.mxv(orc.SpVec("FP32", n), None, None, ("PLUS", "TIMES", "FP32"), Ao, orc.SpVec("FP32", n, np.arange(n), u))
    assert np.array_equal(np.nonzero(pres)[0], wo.I)
    assert np.allclose(w[pres != 0], wo.X, rtol=1e-5)
    # the partitioned / first-touch variant of the same kernel (bench.py reports the faster of the two)
    L.fast_spmv_plan_f32.restype = ctypes.c_void_p
    for nt in (1, 3, 8):
        plan = ctypes.c_void_p(L.fast_spmv_plan_f32(ctypes.c_int64(n), p(indptr), p(indices), p(vals), ctypes.c_int(nt)))
        w2 = np.full(n, -1, np.float32); pres2 = np.full(n, 9, np.uint8)
        L.fast_spmv_plan_run_f32(plan, p(u), p(w2), p(pres2))
        L.fast_spmv_plan_free_f32(plan)
        assert np.array_equal(pres2, pres) and np.allclose(w2, w, rtol=1e-6, atol=0), nt
    # masked plus_pair (triangle kernel), both formulations
    Ls = sp.tril(sp.csr_matrix((np.ones(nnz), indices, indptr), shape=(n, n)) + sp.csr_matrix((np.ones(nnz), indices, indptr), shape=(n, n)).T, -1).tocsr()
    Ls.sort_indices()
    lp, lj = Ls.indptr.astype(np.int64), Ls.indices.astype(np.uint32)
    cval = np.zeros(len(lj), np.int64); chas = np.zeros(len(lj), np.uint8)
    L.fast_masked_saxpy_plus_pair_i64(ctypes.c_int64(n), ctypes.c_int64(n), p(lp), p(lj), p(lp), p(lj), p(lp), p(lj), p(cval), p(chas))
    lrows = np.repeat(np.arange(n), np.diff(lp))
    Lo = orc.SpMat("INT64", n, n, lrows, lj, np.ones(len(lj), np.int64))
    Co = orc.mxm(orc.SpMat("INT64", n, n), Lo, None, ("PLUS", "PAIR", "INT64"), Lo, Lo, "S")
    assert int(cval.sum()) == int(Co.X.sum())
    assert int(chas.sum()) == Co.nvals
    cval2 = np.zeros(len(lj), np.int64); chas2 = np.zeros(len(lj), np.uint8)
    L.fast_masked_dot_plus_pair_i64(ctypes.c_int64(n), p(lp), p(lj), p(lp), p(lj), p(lp), p(lj), p(cval2), p(chas2))
    Cd = orc.mxm(orc.SpMat("INT64", n, n), Lo, None, ("PLUS", "PAIR", "INT64"), Lo, Lo, "ST1")
    assert int(cval2.sum()) == int(Cd.X.sum()) and int(chas2.sum()) == Cd.nvals


# ------------------------------------------------------------------ the oracle at the edges of each type
def _dot(sr, a, b, atype=None, btype=None, ctype=None):
    """C(0,0) of the 1 x n times n x 1 product under semiring sr, or None when it has no entry."""
    atype, btype = atype or sr[2], btype or sr[2]
    n = len(a)
    A = orc.SpMat(atype, 1, n, np.zeros(n), np.arange(n), np.asarray(a, orc.DTYPES[atype]))
    B = orc.SpMat(btype, n, 1, np.arange(n), np.zeros(n), np.asarray(b, orc.DTYPES[btype]))
    C = orc.mxm(orc.SpMat(ctype or orc.semiring_ztype(sr), 1, 1), None, None, sr, A, B)
    return C.X[0] if C.nvals else None


def _bits(x):
    return np.asarray(x).view(np.uint64 if np.asarray(x).dtype.itemsize == 8 else np.uint32).item()


def test_oracle_integers_wrap():
    assert _dot(("PLUS", "TIMES", "INT8"), [127, 1], [2, 1]) == -1               # 254 -> -2, then + 1
    assert _dot(("PLUS", "FIRST", "INT8"), [127, 1], [0, 0]) == -128
    assert _dot(("TIMES", "SECOND", "INT16"), [1, 1], [256, 256]) == 0          # 2^16 wraps to 0
    assert _dot(("PLUS", "MINUS", "INT32"), [-2**31], [1]) == 2**31 - 1
    assert _dot(("PLUS", "TIMES", "UINT64"), [2**63, 2**63], [1, 1]) == 0
    assert _dot(("MAX", "FIRST", "UINT64"), [2**63, 1], [0, 0]) == 2**63          # unsigned order
    assert _dot(("MIN", "SECOND", "UINT64"), [0, 0], [2**64 - 1, 2**63]) == 2**63
    assert _dot(("BXNOR", "BXNOR", "UINT8"), [0], [0]) == 255


def test_oracle_integer_division_rules():
    div = lambda t, x, y: _dot(("PLUS", "DIV", t), [x], [y])
    assert div("INT32", -2**31, -1) == -2**31                                    # INT_MIN / -1 wraps
    assert div("INT8", -128, -1) == -128
    assert div("INT32", 5, 0) == 2**31 - 1 and div("INT32", -5, 0) == -2**31 and div("INT32", 0, 0) == 0
    assert div("UINT8", 5, 0) == 255 and div("UINT8", 0, 0) == 0
    assert div("INT16", -7, 2) == -3                                               # truncation toward zero
    assert _dot(("PLUS", "RDIV", "INT64"), [-1], [-2**63]) == -2**63


def test_oracle_float_to_integer_casts_saturate():
    # operands cast to the multiply's type: NaN -> 0, out of range -> the nearest end, fractions truncate
    a = np.array([np.nan, 1e10, -1e10, 3.7, -3.7, np.inf, -np.inf], np.float64)
    for k, want in enumerate([0, 127, -128, 3, -3, 127, -128]):
        assert _dot(("PLUS", "FIRST", "INT8"), [a[k]], [1], atype="FP64") == want, a[k]
    for k, want in enumerate([0, 10**10, 0, 3, 0, 2**64 - 1, 0]):
        assert _dot(("PLUS", "FIRST", "UINT64"), [a[k]], [1], atype="FP64") == want, a[k]
    # the write-back cast of the result: FP32 result into an INT16 output
    assert _dot(("PLUS", "TIMES", "FP32"), [np.inf], [1], ctype="INT16") == 2**15 - 1
    assert _dot(("PLUS", "TIMES", "FP32"), [np.nan], [1], ctype="INT16") == 0
    assert _dot(("PLUS", "TIMES", "FP32"), [-1e30], [1], ctype="UINT32") == 0
    assert _dot(("PLUS", "TIMES", "FP64"), [1e300], [1], ctype="UINT64") == 2**64 - 1


def test_oracle_fp_min_max_ignore_nan_and_keep_signs():
    nan, inf = np.nan, np.inf
    assert _dot(("MIN", "FIRST", "FP32"), [nan, 2.0], [0, 0]) == 2.0
    assert _dot(("MIN", "FIRST", "FP32"), [2.0, nan], [0, 0]) == 2.0
    assert np.isnan(_dot(("MIN", "FIRST", "FP32"), [nan], [0]))                   # a sole NaN product stays NaN (an entry)
    assert np.isnan(_dot(("MIN", "PLUS", "FP32"), [inf], [-inf]))                 # +Inf + -Inf = NaN, not +Inf
    assert _dot(("MAX", "FIRST", "FP64"), [-inf, nan], [0, 0]) == -inf
    assert np.isnan(_dot(("MAX", "TIMES", "FP64"), [0.0], [inf]))
    m = _dot(("PLUS", "FIRST", "FP32"), [-0.0], [1])                              # a sole -0.0 keeps its sign
    assert _bits(m) == _bits(np.float32(-0.0))
    assert _bits(_dot(("PLUS", "FIRST", "FP64"), [-0.0, 0.0], [1, 1])) == 0       # -0 + +0 = +0
    tiny = np.finfo(np.float32).smallest_subnormal
    assert _dot(("PLUS", "TIMES", "FP32"), [tiny, tiny], [1, 2]) == np.float32(3) * tiny      # subnormals are kept
    assert _dot(("PLUS", "DIV", "FP64"), [1.0, -1.0], [0.0, 0.0]) is not None and np.isnan(_dot(("PLUS", "DIV", "FP64"), [1.0, -1.0], [0.0, 0.0]))


def test_edge_value_pools():
    for t in util.ALL_T:
        pool = util.edge_values(t)
        assert pool.dtype == orc.DTYPES[t] and len(np.unique(pool.view(f"u{pool.dtype.itemsize}") if t != "BOOL" else pool)) == len(pool)
    f32 = util.edge_values("FP32")
    assert np.isnan(f32).sum() == 1 and (f32 == np.inf).sum() == 1 and np.signbit(f32[f32 == 0]).sum() == 1
    sub = f32[(f32 != 0) & (np.abs(f32) < np.finfo(np.float32).tiny)]
    assert len(sub) == 4 and np.abs(sub).min() == np.finfo(np.float32).smallest_subnormal
    assert set(util.edge_values("UINT64").tolist()) == {0, 1, 2, 2**63 - 1, 2**63, 2**64 - 2, 2**64 - 1}
    assert util.edge_values("INT16").min() == -2**15
    rng = np.random.default_rng(0)
    v = util.rand_edge_values(rng, "INT32", 4000, 0.5)
    assert 600 < (np.abs(v.astype(np.int64)) > 5).sum() < 1200                   # half from the pool, 4 of its 9 values are large
