"""GPU parity tests: the CUDA path (through the C ABI and the host-side mirror) against the
reference's golden vectors and against the CPU oracle on the same seeded inputs.
Bit-exact for BOOL / integer types and for MIN/MAX; FP PLUS within 1e-6 relative
(BASELINE.json north_star tolerance) -- the random FP inputs are multiples of 1/4 so that
most FP cases are in fact exact."""
import numpy as np
import pytest
import scipy.sparse as sp

import pygraphblas_b200 as gb
from pygraphblas_b200 import Matrix, Vector, INT64, FP32, FP64, BOOL, UINT8, descriptor, Accum
from oracle import oracle as orc
import util

pytestmark = pytest.mark.gpu
RTOL = 1e-6


def _check(case, got):
    exp = util.oracle_run(case)
    if case["op"] == "mxm":
        assert got.type == exp.type and np.array_equal(got.I, exp.I) and np.array_equal(got.J, exp.J), (case, got, exp)
    else:
        assert got.type == exp.type and np.array_equal(got.I, exp.I), (case, got, exp)
    if got.type in ("FP32", "FP64"):
        assert np.allclose(got.X, exp.X, rtol=RTOL, atol=0, equal_nan=True), (case, got, exp)
    else:
        assert np.array_equal(got.X, exp.X), (case, got, exp)


def test_device_present():
    assert gb.have_device(), "the gpu tests must run on the CUDA path"
    before = gb.lib.B200_kernel_launches()
    Matrix.from_lists([0], [0], [1]).mxv(Vector.from_lists([0], [1]))
    assert gb.lib.B200_kernel_launches() > before


def test_reference_goldens(goldens):
    for case in goldens["cases"]:
        if case["id"] == "test_mxm_imatmul_alias":
            case = dict(case); case["C"] = case["A"]        # C aliases A
        if case["id"] in ("test_RCT0", "test_RC"):
            case = dict(case); case["w"] = case["u"]        # out aliases the input vector
        got = util.product_run(case)
        ok = util.same_mat(got, case["expect"]) if case["op"] == "mxm" else util.same_vec(got, case["expect"])
        assert ok, f"{case['id']} ({case['source']}): got {got}, expected {case['expect']}"


def test_reference_api_forms():
    """The call forms of tests/test_matrix.py:249-306 and tests/test_vector.py:298-315."""
    m = Matrix.from_lists([0, 1, 2], [1, 2, 0], [1, 2, 3])
    n = Matrix.from_lists([0, 1, 2], [1, 2, 0], [2, 3, 4])
    r = Matrix.from_lists([0, 1, 2], [2, 0, 1], [3, 8, 6])
    o = m.mxm(n)
    assert o.nrows == 3 and o.ncols == 3 and o.nvals == 3 and o.iseq(r) and r.iseq(m @ n)
    with INT64.PLUS_PLUS:
        assert (m @ n).iseq(Matrix.from_lists([0, 1, 2], [2, 0, 1], [4, 6, 5]))
    with BOOL.LOR_LAND:
        assert (m @ n).iseq(Matrix.from_lists([0, 1, 2], [2, 0, 1], [True, True, True]))
    with descriptor.T0:
        assert (m @ n).iseq(m.mxm(n, desc=descriptor.T0))
    assert m.min_plus(n).iseq(Matrix.from_lists([0, 1, 2], [2, 0, 1], [4, 6, 5]))
    o = m.dup()
    with Accum(INT64.min):
        o @= n
    assert o.to_lists() == [[0, 0, 1, 1, 2, 2], [1, 2, 0, 2, 0, 1], [1, 3, 8, 2, 3, 6]]
    m @= n
    assert r.iseq(m)
    assert m.mxm(n, semiring=BOOL.LOR_LAND).iseq(Matrix.from_lists([0, 1, 2], [0, 1, 2], [True, True, True]))
    assert m.mxm(n, cast=FP32).type is FP32
    # mxv / vxm
    m = Matrix.from_lists([0, 1, 2, 3], [1, 2, 0, 1], [1, 2, 3, 4])
    v = Vector.from_lists([0, 1, 2], [2, 3, 4])
    o = m.mxv(v)
    assert o.iseq(Vector.from_lists([0, 1, 2, 3], [3, 8, 6, 12])) and o.iseq(m @ v)
    assert o.iseq(m.transpose().mxv(v, desc=descriptor.T0))
    m = Matrix.from_lists([0, 1, 2, 0], [1, 2, 0, 3], [1, 2, 3, 4])
    o = v.vxm(m)
    assert o.iseq(Vector.from_lists([0, 1, 2, 3], [12, 2, 6, 8])) and (v @ m).iseq(o)
    assert v.vxm(m, mask=Vector.from_lists([1], [True], size=4)).iseq(Vector.from_lists([1], [2], size=4))
    assert v.vxm(m.transpose(), desc=descriptor.T1).iseq(o)
    # promotion of the output type (tests/test_matrix.py:1017-1028)
    a = Matrix.from_lists([0, 1], [0, 1], [4, 2], typ=FP32)
    assert (a @ Matrix.from_lists([0, 1], [0, 1], [4, 2], typ=FP64)).type is FP64
    assert (a @ Matrix.from_lists([0, 1], [0, 1], [4, 2], typ=UINT8)).type is FP32
    # dense UINT8 power (tests/test_matrix.py:858-864)
    d = Matrix.from_lists(np.repeat(np.arange(10), 10), np.tile(np.arange(10), 10), np.ones(100), typ=UINT8)
    assert (d @ d).iseq(d ** 2) and set((d ** 3).to_arrays()[2].tolist()) == {100}


@pytest.mark.parametrize("seed", range(120))
def test_random_mxv_vxm_against_oracle(seed):
    rng = np.random.default_rng(1000 + seed)
    typ = util.ALL_T[seed % len(util.ALL_T)]
    m, n = int(rng.integers(1, 70)), int(rng.integers(1, 70))
    if seed % 10 == 9:
        m, n = int(rng.integers(2000, 6000)), int(rng.integers(2000, 6000))      # several SpMV tiles
    dens = [0.0, 0.05, 0.3, 1.0][seed % 4] if max(m, n) < 100 else 0.002
    op = "mxv" if seed % 2 == 0 else "vxm"
    desc = util.DESCS_M[seed % len(util.DESCS_M)]
    A = util.rand_mat(rng, typ, m, n, dens)
    tran = ("T0" in desc) if op == "mxv" else ("T1" in desc)
    # mxv: A'(out x in); vxm: u'A' -> out = ncols(A')
    rows, cols = (n, m) if tran else (m, n)
    in_n, out_n = (cols, rows) if op == "mxv" else (rows, cols)
    u = util.rand_vec(rng, rng.choice(util.ALL_T), in_n, [1.0, 0.5, 0.1][seed % 3])
    wtype = rng.choice(util.ALL_T)
    w = util.rand_vec(rng, wtype, out_n, 0.4)
    mask = util.rand_vec(rng, rng.choice(util.ALL_T), out_n, 0.5) if seed % 3 != 0 else None
    srs = util.semirings_for(typ)
    sr = srs[(seed // 2) % len(srs)]
    accum = (["PLUS", "MIN", "MAX", "SECOND", "TIMES"][seed % 5], wtype) if seed % 4 >= 2 else None
    case = {"op": op, "A": A, "u": u, "w": w, "mask": mask, "accum": accum, "semiring": list(sr), "desc": desc}
    _check(case, util.product_run(case))


@pytest.mark.parametrize("op", ["mxv", "vxm", "mxm"])
@pytest.mark.parametrize("desc", ["C", "RC", "SC", "RSC"])
@pytest.mark.parametrize("acc", [None, "PLUS"])
def test_complemented_null_mask(op, desc, acc):
    """C<!NULL> / w<!NULL>: the complement of "no mask" lets nothing through -- the output keeps its entries, or is
    cleared under GrB_REPLACE (C API 1.3 section 4.3; SuiteSparse's quick-mask exit), for every entry point."""
    rng = np.random.default_rng(77)
    A = util.rand_mat(rng, "INT64", 9, 9, 0.4)
    accum = (acc, "INT64") if acc else None
    if op == "mxm":
        case = {"op": "mxm", "A": A, "B": util.rand_mat(rng, "INT64", 9, 9, 0.4), "C": util.rand_mat(rng, "INT64", 9, 9, 0.3),
                "mask": None, "accum": accum, "semiring": ["PLUS", "TIMES", "INT64"], "desc": desc}
    else:
        case = {"op": op, "A": A, "u": util.rand_vec(rng, "INT64", 9, 0.7), "w": util.rand_vec(rng, "INT64", 9, 0.5),
                "mask": None, "accum": accum, "semiring": ["PLUS", "TIMES", "INT64"], "desc": desc}
    got = util.product_run(case)
    _check(case, got)
    before = case["C"] if op == "mxm" else case["w"]
    assert len(got.I) == (0 if "R" in desc else len(before["I"]))


@pytest.mark.parametrize("seed", range(120))
def test_random_mxm_against_oracle(seed):
    rng = np.random.default_rng(5000 + seed)
    typ = util.ALL_T[seed % len(util.ALL_T)]
    m, k, n = (int(x) for x in rng.integers(1, 40, 3))
    if seed % 10 == 9:
        m, k, n = 300, 400, 350
    dens = [0.0, 0.1, 0.4, 1.0][seed % 4] if seed % 10 != 9 else 0.02
    desc = util.DESCS_M[seed % len(util.DESCS_M)]
    A = util.rand_mat(rng, typ, k if "T0" in desc else m, m if "T0" in desc else k, dens)
    B = util.rand_mat(rng, rng.choice(util.ALL_T), n if "T1" in desc else k, k if "T1" in desc else n, dens)
    ctype = rng.choice(util.ALL_T)
    C = util.rand_mat(rng, ctype, m, n, [0.0, 0.3][seed % 2])
    M = util.rand_mat(rng, rng.choice(util.ALL_T), m, n, 0.5) if seed % 3 != 0 else None
    srs = util.semirings_for(typ)
    sr = srs[(seed // 2) % len(srs)]
    accum = (["PLUS", "MIN", "MAX", "SECOND", "TIMES"][seed % 5], ctype) if seed % 4 >= 2 else None
    case = {"op": "mxm", "A": A, "B": B, "C": C, "mask": M, "accum": accum, "semiring": list(sr), "desc": desc}
    _check(case, util.product_run(case))


def test_config1_plumbing_1024_fp64():
    """BASELINE.json configs[0]: 1024 x 1024 random 1% CSR, Matrix.mxv PLUS_TIMES_FP64."""
    A = sp.random(1024, 1024, density=0.01, format="csr", dtype=np.float64, random_state=0)
    A.sort_indices()
    u = np.random.default_rng(0).random(1024)
    w = Matrix.from_scipy(A).mxv(Vector.from_numpy(u))
    x, p = w.to_numpy()
    ref = A @ u
    nz = np.diff(A.indptr) > 0
    assert np.array_equal(p != 0, nz)
    assert np.allclose(x[nz], ref[nz], rtol=1e-12, atol=0)


def _rmat(scale, ef=16, seed=1):
    from pygraphblas_b200.generators import rmat_csr
    return rmat_csr(scale, ef, seed)


def test_rmat_spmv_fp32_against_cpu_port():
    """R-MAT scale 16 PLUS_TIMES_FP32 SpMV (configs[1] shape) vs the OpenMP port of the oracle."""
    import ctypes
    n, indptr, indices = _rmat(16)
    rng = np.random.default_rng(2)
    vals = (rng.random(len(indices), dtype=np.float32) + 0.5).astype(np.float32)
    u = rng.random(n, dtype=np.float32)
    A = Matrix.from_csr(indptr, indices, vals, n, n, FP32)
    w = A.mxv(Vector.from_numpy(u), semiring=FP32.PLUS_TIMES)
    x, p = w.to_numpy()
    L = orc.lib()
    ref = np.zeros(n, np.float32); rp = np.zeros(n, np.uint8)
    ptr = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    L.fast_spmv_plus_times_f32(ctypes.c_int64(n), ptr(indptr), ptr(indices), ptr(vals), ptr(u), ptr(ref), ptr(rp))
    assert np.array_equal(p, rp)
    assert np.allclose(x[p != 0], ref[p != 0], rtol=2e-5, atol=0)     # fp32 sums of up to ~10^4 terms in different orders
    # exact cross-check in float64 accumulate: relative error of the GPU result vs an fp64 reference
    ref64 = sp.csr_matrix((vals.astype(np.float64), indices, indptr), shape=(n, n)) @ u.astype(np.float64)
    assert np.max(np.abs(x[p != 0] - ref64[p != 0]) / ref64[p != 0]) < 1e-5
    # vxm / T0 on the same graph: w = A'u
    wt = A.mxv(Vector.from_numpy(u), semiring=FP32.PLUS_TIMES, desc=descriptor.T0)
    xt, pt = wt.to_numpy()
    reft = sp.csr_matrix((vals.astype(np.float64), indices, indptr), shape=(n, n)).T @ u.astype(np.float64)
    assert np.allclose(xt[pt != 0], reft[pt != 0], rtol=1e-5)


def test_rmat_bfs_levels_match_scipy():
    """configs[2] shape: LOR_LAND BOOL mxv with complemented mask + replace, iterated to a full BFS."""
    from scipy.sparse.csgraph import breadth_first_order
    n, indptr, indices = _rmat(14)
    At = sp.csr_matrix((np.ones(len(indices), np.bool_), indices, indptr), shape=(n, n))
    A = Matrix.from_csr(indptr, indices, None, n, n, BOOL)
    src = int(np.argmax(np.diff(indptr)))
    # pull BFS along in-edges of A': next = A' q  (vxm form, demo/Introduction-to-GraphBLAS-with-Python.ipynb:4311)
    level = np.full(n, -1, np.int64); level[src] = 0
    q = Vector.sparse(BOOL, n); q[src] = True
    visited = Vector.sparse(BOOL, n); visited[src] = True
    depth = 0
    while q.nvals:
        depth += 1
        q = q.vxm(A, semiring=BOOL.LOR_LAND, mask=visited, desc=descriptor.RC)
        I, _ = q.to_arrays()
        if not len(I):
            break
        level[I.astype(np.int64)] = depth
        for i in I.tolist()[:0]:
            pass
        xv, pv = visited.to_numpy()
        pv[I.astype(np.int64)] = 1; xv[I.astype(np.int64)] = True
        visited = Vector.from_numpy(xv, present=pv, typ=BOOL)
    order, pred = breadth_first_order(At, src, directed=True, return_predecessors=True)
    ref = np.full(n, -1, np.int64); ref[src] = 0
    for node in order[1:]:
        ref[node] = ref[pred[node]] + 1
    assert np.array_equal(level, ref)


PULL_CASES = [("LOR", "LAND", "BOOL"), ("LAND", "LOR", "BOOL"), ("ANY", "PAIR", "BOOL"), ("LOR", "GT", "INT32"), ("LAND", "EQ", "FP32"),
              ("LOR", "FIRST", "BOOL"), ("ANY", "PAIR", "INT64"), ("LAND", "SECOND", "BOOL")]


@pytest.mark.parametrize("k", range(len(PULL_CASES) * 3))
def test_masked_pull_hub_rows_against_oracle(k):
    """The masked saturating-monoid kernel pair: batches of short rows, rows over 4096 entries (CTA-per-row
    kernel), empty rows, sparse and dense u, every mask flavour."""
    sr = PULL_CASES[k % len(PULL_CASES)]
    rng = np.random.default_rng(7000 + k)
    n = 9000
    typ = sr[2]
    hubs = rng.choice(n, 3, replace=False)
    I = [np.full(d, h) for h, d in zip(hubs, (8500, 5000, 4097))]
    J = [rng.choice(n, len(x), replace=False) for x in I]
    short_rows = rng.choice(n, 5000, replace=False)
    deg = rng.integers(1, 40, len(short_rows))
    I.append(np.repeat(short_rows, deg)); J.append(rng.integers(0, n, int(deg.sum())))
    I, J = np.concatenate(I), np.concatenate(J)
    key = np.unique(I.astype(np.int64) * n + J)
    I, J = np.divmod(key, n)
    A = {"type": typ, "nrows": n, "ncols": n, "I": I.tolist(), "J": J.tolist(), "X": util.rand_values(rng, typ, len(I)).tolist()}
    u = util.rand_vec(rng, typ, n, [0.001, 0.05, 1.0][k % 3])
    desc = ["RC", "C", "S", "", "RSC", "SC"][k % 6]
    mask = util.rand_vec(rng, ["BOOL", "UINT8", "FP32"][k % 3], n, 0.5)
    w = util.rand_vec(rng, "BOOL" if sr[0] != "ANY" else typ, n, 0.3)
    case = {"op": "mxv" if k % 2 == 0 else "vxm", "A": A, "u": u, "w": w, "mask": mask, "accum": None, "semiring": list(sr), "desc": desc}
    if case["op"] == "vxm":
        case["A"] = dict(A, I=A["J"], J=A["I"])
    _check(case, util.product_run(case))


@pytest.mark.parametrize("k", range(1, len(PULL_CASES) * 3, 2))
def test_masked_push_forced_against_oracle(k, monkeypatch):
    """The same cases in their vxm form with the push kernel forced for every frontier size (the other
    orientation of A is in HBM for vxm, so push is available): idempotent stores must reproduce the fold."""
    monkeypatch.setenv("B200GRB_FORCE_PUSH", "1")
    gb.lib.B200_reload_tunables()
    try:
        test_masked_pull_hub_rows_against_oracle(k)
    finally:
        monkeypatch.delenv("B200GRB_FORCE_PUSH")
        gb.lib.B200_reload_tunables()


def test_rmat_triangle_count_masked_mxm():
    """configs[3] shape: C<L> = L (+.pair) L on the strict lower triangle of A + A' (masked hash SpGEMM),
    and the masked-dot form C<L> = L L' (descriptor ST1); both against the CPU port and scipy."""
    n, indptr, indices = _rmat(13)
    S = sp.csr_matrix((np.ones(len(indices)), indices, indptr), shape=(n, n))
    Ls = sp.tril(S + S.T, -1).tocsr(); Ls.sort_indices(); Ls.data[:] = 1
    tri_ref = int((Ls @ Ls).multiply(Ls).sum())
    L = Matrix.from_csr(Ls.indptr, Ls.indices, np.ones(Ls.nnz, np.int64), n, n, INT64)
    C = L.mxm(L, mask=L, semiring=INT64.PLUS_PAIR, desc=descriptor.S)
    assert int(C.to_arrays()[2].sum()) == tri_ref
    C2 = L.mxm(L, mask=L, semiring=INT64.PLUS_PAIR, desc=descriptor.ST1)
    ref2 = int((Ls @ Ls.T).multiply(Ls).sum())
    assert int(C2.to_arrays()[2].sum()) == ref2
    # valued mask gives the same answer here (all mask values are 1)
    C3 = L.mxm(L, mask=L, semiring=INT64.PLUS_PAIR)
    assert C3.iseq(C)


def test_rmat_masked_mxm_large_ST1_and_valued_mask():
    """Above 2^18 entries C<M> = A*B' runs through the cached transpose + chunked masked hash kernels."""
    n, indptr, indices = _rmat(15)
    S = sp.csr_matrix((np.ones(len(indices)), indices, indptr), shape=(n, n))
    Ls = sp.tril(S + S.T, -1).tocsr(); Ls.sort_indices(); Ls.data[:] = 1
    assert Ls.nnz >= 1 << 18
    rng = np.random.default_rng(9)
    lv = rng.integers(1, 4, Ls.nnz).astype(np.int64)
    L = Matrix.from_csr(Ls.indptr, Ls.indices, lv, n, n, INT64)
    Lw = sp.csr_matrix((lv.astype(np.float64), Ls.indices, Ls.indptr), shape=(n, n))
    C = L.mxm(L, mask=L, semiring=INT64.PLUS_TIMES, desc=descriptor.ST1)
    R = (Lw @ Lw.T).multiply(Ls).tocsr(); R.sort_indices(); R.eliminate_zeros()
    Ap, Aj, Ax = C.to_csr()
    assert np.array_equal(Ap, R.indptr) and np.array_equal(Aj, R.indices) and np.array_equal(Ax, R.data.astype(np.int64))
    # valued mask: entries with value 0 mask nothing in
    mv = (rng.integers(0, 2, Ls.nnz)).astype(np.int64)
    Mk = Matrix.from_csr(Ls.indptr, Ls.indices, mv, n, n, INT64)
    C2 = L.mxm(L, mask=Mk, semiring=INT64.PLUS_TIMES)
    Mp = sp.csr_matrix((mv.astype(np.float64), Ls.indices.copy(), Ls.indptr.copy()), shape=(n, n)); Mp.eliminate_zeros()
    R2 = (Lw @ Lw).multiply(Mp > 0).tocsr(); R2.sort_indices(); R2.eliminate_zeros()
    Bp, Bj, Bx = C2.to_csr()
    assert np.array_equal(Bp, R2.indptr) and np.array_equal(Bj, R2.indices) and np.array_equal(Bx, R2.data.astype(np.int64))


@pytest.mark.parametrize("mode", [{}, {"B200GRB_SPMV_HOT": "64"}, {"B200GRB_SPMV_HOT": "0"}])
def test_large_spmv_all_kernel_variants(mode):
    """Large dense-u SpMV through every kernel variant (hot-table run kernel with TMA-staged runs at two table
    sizes, plain run kernel): exact against the oracle on small-integer data, for specialised and
    run-time semirings."""
    import os
    old = {k: os.environ.get(k) for k in ("B200GRB_SPMV_HOT",)}
    os.environ.update(mode)
    gb.lib.B200_reload_tunables()                 # the switches are read at GrB_init and on request only
    try:
        _large_spmv_body()
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
        gb.lib.B200_reload_tunables()


def _large_spmv_body():
    n, indptr, indices = _rmat(17)
    assert len(indices) >= 1 << 20
    rng = np.random.default_rng(11)
    for typ, sr_names in ((FP32, ["PLUS_TIMES", "MIN_PLUS", "MAX_MIN"]), (INT64, ["PLUS_TIMES", "MIN_FIRST"]), (FP64, ["PLUS_SECOND"])):
        vals = rng.integers(1, 9, len(indices)).astype(typ.dtype)
        u = rng.integers(0, 9, n).astype(typ.dtype)
        A = Matrix.from_csr(indptr, indices, vals, n, n, typ)
        rows = np.repeat(np.arange(n), np.diff(indptr))
        for name in sr_names:
            w = A.mxv(Vector.from_numpy(u), semiring=getattr(typ, name))
            x, p = w.to_numpy()
            add, mul = name.split("_")
            ref = orc.mxv(orc.SpVec(typ.name, n), None, None, (add, mul, typ.name), orc.SpMat(typ.name, n, n, rows, indices, vals),
                          orc.SpVec(typ.name, n, np.arange(n), u))
            assert np.array_equal(np.nonzero(p)[0], ref.I), name
            assert np.array_equal(x[p != 0], ref.X), name      # small integers: exact in every type


@pytest.mark.parametrize("dens", [0.0005, 0.03, 0.6])
def test_large_spmv_sparse_u(dens):
    """Sparse u on a large matrix (run kernel with presence bytes), specialised and run-time semirings, mxv and
    vxm, with and without accumulator; exact against the oracle on small-integer data."""
    n, indptr, indices = _rmat(16)
    rng = np.random.default_rng(12)
    rows = np.repeat(np.arange(n), np.diff(indptr))
    for typ, sr_names in ((FP32, ["PLUS_TIMES", "MIN_PLUS", "MAX_SECOND"]), (INT64, ["PLUS_PAIR", "MIN_FIRST", "TIMES_MAX"]), (BOOL, ["LOR_LAND", "LXOR_LOR"])):
        vals = rng.integers(1, 4, len(indices)).astype(typ.dtype)
        ui = np.sort(rng.choice(n, max(1, int(n * dens)), replace=False))
        ux = rng.integers(0, 3, len(ui)).astype(typ.dtype)
        A = Matrix.from_csr(indptr, indices, vals, n, n, typ)
        oA = orc.SpMat(typ.name, n, n, rows, indices, vals)
        for k, name in enumerate(sr_names):
            add, mul = name.split("_")
            u = Vector.from_lists(ui.tolist(), ux.tolist(), n, typ)
            ou = orc.SpVec(typ.name, n, ui, ux)
            if k % 2 == 0:
                w = A.mxv(u, semiring=getattr(typ, name))
                ref = orc.mxv(orc.SpVec(typ.name, n), None, None, (add, mul, typ.name), oA, ou)
            else:
                w0i = np.sort(rng.choice(n, n // 3, replace=False)); w0x = rng.integers(0, 5, len(w0i)).astype(typ.dtype)
                w = Vector.from_lists(w0i.tolist(), w0x.tolist(), n, typ)
                acc = "LOR" if typ is BOOL else "PLUS"
                u.vxm(A, out=w, accum=getattr(typ, acc), semiring=getattr(typ, name))
                ref = orc.vxm(orc.SpVec(typ.name, n, w0i, w0x), None, (acc, typ.name), (add, mul, typ.name), ou, oA)
            I, X = w.to_arrays()
            assert np.array_equal(I, ref.I), (name, dens)
            assert np.array_equal(X, ref.X), (name, dens)


def test_rmat_unmasked_spgemm_matches_scipy():
    """configs[3] secondary: unmasked A (+.second) A, all three row bins (ESC / ESC / dense accumulator)."""
    n, indptr, indices = _rmat(12)
    rng = np.random.default_rng(4)
    vals = rng.integers(1, 5, len(indices)).astype(np.float32)
    A = Matrix.from_csr(indptr, indices, vals, n, n, FP32)
    C = A.mxm(A, semiring=FP32.PLUS_TIMES)
    S = sp.csr_matrix((vals.astype(np.float64), indices, indptr), shape=(n, n))
    R = (S @ S).tocsr(); R.sort_indices()
    Ap, Aj, Ax = C.to_csr()
    assert np.array_equal(Ap, R.indptr) and np.array_equal(Aj, R.indices)
    assert np.allclose(Ax, R.data, rtol=1e-6)
    C2 = A.mxm(A, semiring=FP32.PLUS_SECOND)
    P = sp.csr_matrix((np.ones(len(indices)), indices, indptr), shape=(n, n))
    R2 = (P @ S).tocsr(); R2.sort_indices()
    assert np.allclose(C2.to_csr()[2], R2.data, rtol=1e-6)


@pytest.mark.parametrize("typ,sr", [(FP32, "PLUS_TIMES"), (FP64, "PLUS_SECOND"), (INT64, "PLUS_TIMES"), (FP32, "MIN_PLUS"), (BOOL, "LOR_LAND"), (UINT8, "MAX_FIRST")])
def test_unmasked_spgemm_esc_equals_model_and_scipy(typ, sr):
    """The expand-sort-compress numeric kernels (small bin: a warp per row, medium bin: a CTA per row) against the oracle --
    pattern and every value, bit for bit (quarter-valued inputs: every fold order gives the same sum) -- and, for PLUS_TIMES,
    against scipy.  The graph has rows in all three bins."""
    n, indptr, indices = _rmat(12)
    rng = np.random.default_rng(8)
    if typ in (FP32, FP64):
        vals = (rng.integers(1, 9, len(indices)) / 4.0).astype(typ.dtype)
    elif typ is BOOL:
        vals = np.ones(len(indices), np.bool_)
    else:
        vals = rng.integers(1, 4, len(indices)).astype(typ.dtype)
    A = Matrix.from_csr(indptr, indices, vals, n, n, typ)
    C = A.mxm(A, semiring=getattr(typ, sr))
    assert {"esc-small", "esc-medium", "spa"} <= set(gb.ffi.string(gb.lib.B200_debug_last_kernel()).decode().split(";"))
    rows = np.repeat(np.arange(n), np.diff(indptr))
    Ao = orc.SpMat(typ.name, n, n, rows, indices, vals)
    ref = orc.mxm(orc.SpMat(typ.name, n, n), None, None, (*sr.split("_"), typ.name), Ao, Ao, "")
    ci, cj, cx = C.to_arrays()
    assert np.array_equal(ci, ref.I) and np.array_equal(cj, ref.J)
    assert cx.dtype == ref.X.dtype and np.array_equal(cx.view(np.uint8), ref.X.view(np.uint8))
    if sr == "PLUS_TIMES":
        S = sp.csr_matrix((vals.astype(np.float64), indices, indptr), shape=(n, n))
        R = (S @ S).tocsr(); R.sort_indices()
        Cp, Cj, Cx = C.to_csr()
        assert np.array_equal(Cp, R.indptr) and np.array_equal(Cj, R.indices) and np.array_equal(Cx.astype(np.float64), R.data)


def test_sssp_min_plus_matches_scipy():
    """configs[4] shape: MIN_PLUS_FP32 sweeps with accum MIN, output aliasing the input, T0."""
    from scipy.sparse.csgraph import shortest_path
    n, indptr, indices = _rmat(11, 8, seed=3)
    rng = np.random.default_rng(3)
    wts = (1.0 - rng.random(len(indices), dtype=np.float32)).astype(np.float32)
    A = Matrix.from_csr(indptr, indices, wts, n, n, FP32)
    src = int(np.argmax(np.diff(indptr)))
    d0 = np.full(n, np.inf, np.float32); d0[src] = 0
    v = Vector.from_numpy(d0)
    for _ in range(n):
        before = v.to_numpy()[0].copy()
        A.mxv(v, out=v, accum=FP32.MIN, semiring=FP32.MIN_PLUS, desc=descriptor.T0)
        if np.array_equal(before, v.to_numpy()[0]):
            break
    ref = shortest_path(sp.csr_matrix((wts.astype(np.float64), indices, indptr), shape=(n, n)), directed=True, indices=src)
    got = v.to_numpy()[0].astype(np.float64)
    fin = np.isfinite(ref)
    assert np.array_equal(np.isfinite(got), fin)
    assert np.allclose(got[fin], ref[fin], rtol=1e-5)


def test_hot_calls_from_a_thread_pool():
    """SURVEY.md 8(b) threading: the reference drives `lib` from a ThreadPool (demo/dnn/challenge.py:48-51); calls
    on distinct objects from distinct host threads must give the oracle's results."""
    from concurrent.futures import ThreadPoolExecutor

    def work(seed):
        rng = np.random.default_rng(9000 + seed)
        typ = util.ALL_T[seed % len(util.ALL_T)]
        A = util.rand_mat(rng, typ, 40, 30, 0.2)
        u = util.rand_vec(rng, typ, 30, 0.7)
        w = util.rand_vec(rng, typ, 40, 0.3)
        sr = util.semirings_for(typ)[seed % 5]
        case = {"op": "mxv", "A": A, "u": u, "w": w, "mask": None, "accum": None, "semiring": list(sr), "desc": ""}
        _check(case, util.product_run(case))
        B = util.rand_mat(rng, typ, 30, 20, 0.2)
        case = {"op": "mxm", "A": A, "B": B, "C": util.rand_mat(rng, typ, 40, 20, 0.1), "mask": None, "accum": None, "semiring": list(sr), "desc": ""}
        _check(case, util.product_run(case))
        return seed

    with ThreadPoolExecutor(8) as ex:
        assert sorted(ex.map(work, range(48))) == list(range(48))


@pytest.mark.parametrize("seed", range(8))
def test_hypersparse_operands_compute_in_their_compact_space(seed):
    """Unsized objects are 2^60 x 2^60 like the reference's (matrix.py:167-170); their mxv / vxm / mxm must give what the
    same tuples give in a small sized space (ids spread over the 2^60 range), for masks / accumulators / descriptors."""
    rng = np.random.default_rng(4000 + seed)
    n = 24
    big = np.sort(rng.choice(1 << 59, size=n, replace=False).astype(np.uint64)) + np.uint64(1 << 33)     # the big id of small id k
    typ = ["INT64", "FP64", "BOOL", "UINT8"][seed % 4]
    A = util.rand_mat(rng, typ, n, n, 0.3)
    B = util.rand_mat(rng, typ, n, n, 0.3)
    u = util.rand_vec(rng, typ, n, 0.6)
    w = util.rand_vec(rng, typ, n, 0.4)
    M = util.rand_mat(rng, "BOOL", n, n, 0.5)
    m = util.rand_vec(rng, "BOOL", n, 0.5)
    desc = ["", "T0", "RC", "S", "T1", "RSC", "T0T1", "C"][seed]
    srs = util.semirings_for(typ)
    sr = srs[seed % len(srs)]
    accum = ("PLUS" if typ != "BOOL" else "LOR", typ) if seed % 2 else None
    T = gb.types.by_name(typ)

    def big_mat(d):
        return Matrix.from_lists(big[np.array(d["I"], np.int64)] if d["I"] else [], big[np.array(d["J"], np.int64)] if d["J"] else [], d["X"],
                                 1 << 60, 1 << 60, gb.types.by_name(d["type"]))

    def big_vec(d):
        return Vector.from_lists(big[np.array(d["I"], np.int64)] if d["I"] else [], d["X"], 1 << 60, gb.types.by_name(d["type"]))

    gsr, gacc, gdesc = util.g_semiring(sr), util.g_accum(accum), util.g_desc(desc)
    use_mask = seed % 3 != 0
    # mxv / vxm
    for op in ("mxv", "vxm"):
        case = {"op": op, "A": A, "u": u, "w": w, "mask": m if use_mask else None, "accum": accum, "semiring": list(sr), "desc": desc}
        small = util.product_run(case)
        Ab, ub, wb, mb = big_mat(A), big_vec(u), big_vec(w), (big_vec(m) if use_mask else None)
        out = Ab.mxv(ub, semiring=gsr, out=wb, mask=mb, accum=gacc, desc=gdesc) if op == "mxv" else ub.vxm(Ab, semiring=gsr, out=wb, mask=mb, accum=gacc, desc=gdesc)
        assert out.size == 1 << 60
        I, X = out.to_arrays()
        assert np.array_equal(I, big[np.asarray(small.I, np.int64)]) and np.array_equal(X, small.X), (op, desc)
    # mxm
    case = {"op": "mxm", "A": A, "B": B, "C": util.rand_mat(rng, typ, n, n, 0.2), "mask": M if use_mask else None, "accum": accum, "semiring": list(sr), "desc": desc}
    small = util.product_run(case)
    Cb = big_mat(case["C"])
    out = big_mat(A).mxm(big_mat(B), semiring=gsr, out=Cb, mask=big_mat(M) if use_mask else None, accum=gacc, desc=gdesc)
    I, J, X = out.to_arrays()
    assert np.array_equal(I, big[np.asarray(small.I, np.int64)]) and np.array_equal(J, big[np.asarray(small.J, np.int64)]) and np.array_equal(X, small.X), desc
