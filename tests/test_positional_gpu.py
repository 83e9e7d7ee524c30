"""Positional semirings and operators on the device, against the model of tests/positional_model.py: every semiring on mxm /
mxv / vxm, the call forms around the product, every kernel path a positional call is rewritten onto, INT32 wrap-around,
hypersparse operands (original indices, not compact ranks), apply, and BFS with a parent tree."""
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.csgraph as csgraph

import pygraphblas_b200 as gb
from pygraphblas_b200 import Matrix, Vector, descriptor, ffi, lib
import positional_model as pm
import util
from kernel_check import entries, record_kernels, seed_of, tunables
from test_value_edges_gpu import GEMM, SPMV, gemm_patterns, spmv_pattern

pytestmark = pytest.mark.gpu

REACHED = set()
OPERAND_T = ["BOOL", "INT8", "UINT16", "FP32", "FP64"]
SEMIRINGS = [(a, m, t) for t in pm.TYPES for a in pm.MONOIDS for m in pm.POSITIONAL]


def _kernels():
    return record_kernels(REACHED)


def _sr(add, mul, typ):
    return getattr(util.g_type(typ), f"{add}_{mul}")


def mat_of(d, typ, nrows, ncols):
    I, J = zip(*sorted(d)) if d else ((), ())
    return Matrix.from_lists(list(I), list(J), [d[e] for e in sorted(d)], nrows, ncols, util.g_type(typ))


def vec_of(d, typ, n):
    I = sorted(d)
    return Vector.from_lists(I, [d[k] for k in I], n, util.g_type(typ))


def dict_m(M):
    I, J, X = M.to_lists()
    return {(int(i), int(j)): x for i, j, x in zip(I, J, X)}


def dict_v(v):
    I, X = v.to_lists()
    return {int(i): x for i, x in zip(I, X)}


def rand_d(rng, shape, density, typ):
    n = int(np.prod(shape))
    flat = rng.choice(n, size=int(n * density), replace=False)
    vals = util.rand_values(rng, typ, len(flat)).tolist()
    if len(shape) == 1:
        return {int(k): v for k, v in zip(flat, vals)}
    return {(int(f // shape[1]), int(f % shape[1])): v for f, v in zip(flat, vals)}


def check(got, want, cands, add, label):
    if add == "ANY" and cands is not None:
        assert set(got) == set(want), label
        bad = [k for k, v in got.items() if int(v) not in cands[k]]
        assert not bad, f"{label}: ANY value not a valid index at {bad[:5]}"
    else:
        got = {k: int(v) for k, v in got.items()}
        want = {k: int(v) for k, v in want.items()}
        assert got == want, f"{label}: {[(k, got.get(k), want.get(k)) for k in set(got) ^ set(want) or [k for k in got if got[k] != want[k]]][:5]}"


# ------------------------------------------------------------------ every semiring, operands of every kind of type
@pytest.mark.parametrize("sr", SEMIRINGS, ids=["_".join(s) for s in SEMIRINGS])
def test_semiring_on_mxm_mxv_vxm(sr):
    add, mul, typ = sr
    rng = np.random.default_rng(seed_of(*sr))
    ta, tb = OPERAND_T[rng.integers(0, 5)], OPERAND_T[rng.integers(0, 5)]
    A, B = rand_d(rng, (23, 31), 0.15, ta), rand_d(rng, (31, 17), 0.15, tb)
    u, v = rand_d(rng, (31,), 0.5, tb), rand_d(rng, (23,), 0.5, tb)
    s = _sr(*sr)
    C = mat_of(A, ta, 23, 31).mxm(mat_of(B, tb, 31, 17), semiring=s)
    assert C.type.name == typ
    assert "positional=" in ";".join(_kernels())
    want, cands = pm.mxm({}, typ, None, None, sr, A, B)
    check(dict_m(C), want, cands, add, f"mxm {sr}")
    w = mat_of(A, ta, 23, 31).mxv(vec_of(u, tb, 31), semiring=s)
    assert w.type.name == typ
    want, cands = pm.mxv({}, typ, None, None, sr, A, u)
    check(dict_v(w), want, cands, add, f"mxv {sr}")
    w = vec_of(v, tb, 23).vxm(mat_of(A, ta, 23, 31), semiring=s)
    assert w.type.name == typ
    want, cands = pm.vxm({}, typ, None, None, sr, v, A)
    check(dict_v(w), want, cands, add, f"vxm {sr}")


# ------------------------------------------------------------------ call forms around the product
FORMS = ["", "T0", "T1", "T0T1", "S", "C", "SC", "R", "RSC", "RC"]
FORM_SR = [("MIN", "SECONDI", "INT64"), ("PLUS", "FIRSTI1", "INT32"), ("TIMES", "SECONDJ", "INT64"), ("MAX", "FIRSTJ1", "INT32")]


def _desc(form):
    return dict(replace="R" in form, mask_comp="C" in form, mask_struct="S" in form, tran0="T0" in form, tran1="T1" in form)


@pytest.mark.parametrize("sr", FORM_SR, ids=["_".join(s) for s in FORM_SR])
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("accum", [None, ("PLUS", "INT64")])
def test_call_forms(sr, form, masked, accum):
    add, mul, typ = sr
    rng = np.random.default_rng(seed_of(sr, form, masked, accum))
    d = _desc(form)
    g_desc = getattr(descriptor, form) if form else None
    gacc = util.g_accum(accum)
    n = 19
    A, B = rand_d(rng, (n, n), 0.2, "FP32"), rand_d(rng, (n, n), 0.2, "UINT16")
    M = rand_d(rng, (n, n), 0.4, "INT8") if masked else None
    C0 = rand_d(rng, (n, n), 0.3, "INT64")
    out = mat_of(C0, "INT64", n, n)
    mat_of(A, "FP32", n, n).mxm(mat_of(B, "UINT16", n, n), semiring=_sr(*sr), out=out, mask=mat_of(M, "INT8", n, n) if masked else None,
                               accum=gacc, desc=g_desc)
    want, _ = pm.mxm(C0, "INT64", M, accum, sr, A, B, d)
    check(dict_m(out), want, None, add, f"mxm {form}")
    u, m, w0 = rand_d(rng, (n,), 0.6, "BOOL"), rand_d(rng, (n,), 0.5, "FP64") if masked else None, rand_d(rng, (n,), 0.4, "INT64")
    for vxm in (False, True):
        w = vec_of(w0, "INT64", n)
        gm = vec_of(m, "FP64", n) if masked else None
        if vxm:
            vec_of(u, "BOOL", n).vxm(mat_of(A, "FP32", n, n), semiring=_sr(*sr), out=w, mask=gm, accum=gacc, desc=g_desc)
            want, _ = pm.vxm(w0, "INT64", m, accum, sr, u, A, d)
        else:
            mat_of(A, "FP32", n, n).mxv(vec_of(u, "BOOL", n), semiring=_sr(*sr), out=w, mask=gm, accum=gacc, desc=g_desc)
            want, _ = pm.mxv(w0, "INT64", m, accum, sr, A, u, d)
        check(dict_v(w), want, None, add, f"{'vxm' if vxm else 'mxv'} {form}")


@pytest.mark.parametrize("sr", FORM_SR, ids=["_".join(s) for s in FORM_SR])
def test_complemented_null_mask_and_aliasing(sr):
    add, mul, typ = sr
    rng = np.random.default_rng(seed_of("alias", sr))
    n = 21
    A, u = rand_d(rng, (n, n), 0.2, "INT64"), rand_d(rng, (n,), 0.5, "INT64")
    # C<!NULL>: nothing is let through; under REPLACE the output is cleared
    w = vec_of(u, "INT64", n)
    mat_of(A, "INT64", n, n).mxv(vec_of(u, "INT64", n), semiring=_sr(*sr), out=w, desc=descriptor.C)
    assert dict_v(w) == u
    mat_of(A, "INT64", n, n).mxv(vec_of(u, "INT64", n), semiring=_sr(*sr), out=w, desc=descriptor.RC)
    assert dict_v(w) == {}
    # w = A w, C = C C, w<w> += w A
    w = vec_of(u, "INT64", n)
    mat_of(A, "INT64", n, n).mxv(w, semiring=_sr(*sr), out=w)
    check(dict_v(w), pm.mxv({}, "INT64", None, None, sr, A, u)[0], None, add, "mxv aliased")
    C = mat_of(A, "INT64", n, n)
    C.mxm(C, semiring=_sr(*sr), out=C)
    check(dict_m(C), pm.mxm({}, "INT64", None, None, sr, A, A)[0], None, add, "mxm aliased")
    w = vec_of(u, "INT64", n)
    w.vxm(mat_of(A, "INT64", n, n), semiring=_sr(*sr), out=w, mask=w, accum=util.g_accum(("PLUS", "INT64")))
    check(dict_v(w), pm.vxm(u, "INT64", u, ("PLUS", "INT64"), sr, u, A)[0], None, add, "vxm aliased")


# ------------------------------------------------------------------ every kernel path a positional call is rewritten onto
# (positional semiring, what it runs on): inner form -> (+).SECOND on mxv / (+).FIRST on vxm; count form -> (+).PAIR
SPMV_SR = {"tile-8": [("MIN", "SECONDI", "INT64"), ("PLUS", "FIRSTI", "INT32"), ("ANY", "FIRSTJ1", "INT64")],
           "run": [("MIN", "SECONDI", "INT64"), ("TIMES", "SECONDJ1", "INT32"), ("MAX", "FIRSTI", "INT64")],
           "run-sparse-u": [("PLUS", "FIRSTJ", "INT64"), ("PLUS", "FIRSTI", "INT64")],
           "hot": [("MIN", "SECONDI", "INT64"), ("PLUS", "FIRSTI", "INT64")],
           "pull": [("ANY", "SECONDI", "INT64"), ("ANY", "FIRSTI1", "INT32")],
           "push": [("ANY", "SECONDI", "INT64"), ("ANY", "FIRSTI", "INT64")]}


def _np_mxv(S, upres, mp, sr, off_mxv=True):
    """w = S u with a positional semiring, restated with numpy (rows of S gather the present u)."""
    add, mul, typ = sr
    H = S.multiply(sp.csr_matrix(upres[None, :].astype(np.int8))).tocsr() if not upres.all() else S.tocsr()
    H.eliminate_zeros(); H.sort_indices()
    out = {}
    base, off = (mul[:-1], 1) if mul.endswith("1") else (mul, 0)
    for i in range(H.shape[0]):
        ks = H.indices[H.indptr[i]:H.indptr[i + 1]]
        if len(ks) == 0 or (mp is not None and not mp[i]):
            continue
        vals = {"FIRSTI": [i] * len(ks), "FIRSTJ": ks, "SECONDI": ks, "SECONDJ": [0] * len(ks)}[base]
        out[i] = pm.fold(add if add != "ANY" else "MIN", typ, [int(x) + off for x in vals])
    return out


@pytest.mark.parametrize("path", list(SPMV_SR))
def test_spmv_paths(path):
    cfg = SPMV[path]
    S = spmv_pattern(cfg["shape"])
    nrows, ncols = S.shape
    A = Matrix.from_csr(S.indptr, S.indices, np.ones(S.nnz, np.int64), nrows, ncols, gb.INT64)   # push: A's type = operand type
    rng = np.random.default_rng(seed_of("spmv", path))
    upres = rng.random(ncols) < (0.02 if path == "push" else 0.6) if cfg.get("sparse_u") else np.ones(ncols, bool)
    u = Vector.from_numpy(np.ones(ncols, np.int64), present=upres if cfg.get("sparse_u") else None, typ=gb.INT64)
    mp = rng.random(nrows) < 0.7 if cfg.get("mask") else None
    mask = Vector.from_numpy(np.ones(nrows, bool), present=mp) if mp is not None else None
    if path == "push":
        Vector.from_numpy(np.ones(nrows, np.int64), typ=gb.INT64).vxm(A, semiring=gb.INT64.ANY_FIRST)   # builds A's transpose
    with tunables(**cfg["env"]):
        for sr in SPMV_SR[path]:
            w = A.mxv(u, semiring=_sr(*sr), mask=mask, desc=descriptor.S if mask is not None else None)
            ks = _kernels()
            form = "positional=inner" if sr[1].rstrip("1") in ("FIRSTJ", "SECONDI") else "positional=count"
            assert form in ks, (path, sr, ks)
            # the count form runs (+).PAIR, which reads no u: nothing for the hot table to serve
            want_k = "run" if path == "hot" and form == "positional=count" else cfg["kernel"]
            assert want_k in entries(ks), (path, sr, ks)
            REACHED.add(f"{path}: {want_k}")
            want = _np_mxv(S, upres, mp, sr)
            got = dict_v(w)
            if sr[0] == "ANY":
                assert set(got) == set(want), (path, sr)
                H = S.tocsr()
                base, off = (sr[1][:-1], 1) if sr[1].endswith("1") else (sr[1], 0)
                for i in list(got)[:2000]:
                    ks_i = H.indices[H.indptr[i]:H.indptr[i + 1]]
                    valid = {int(k) + off for k in ks_i if upres[k]} if base in ("SECONDI", "FIRSTJ") else {i + off}
                    assert int(got[i]) in valid, (path, sr, i)
            else:
                check(got, want, None, sr[0], f"{path} {sr}")


GEMM_SR = [("MIN", "SECONDI", "INT64"), ("PLUS", "FIRSTI1", "INT32"), ("MAX", "SECONDJ", "INT64"), ("TIMES", "FIRSTJ", "INT32")]


@pytest.mark.parametrize("path", list(GEMM))
def test_spgemm_paths(path):
    env, want_k = GEMM[path]
    SA, SB, SM, desc = gemm_patterns(path)
    Bt = SB.T.tocsr() if "T1" in desc else SB
    nrows, ncols = SA.shape[0], Bt.shape[1]
    A = Matrix.from_csr(SA.indptr, SA.indices, np.ones(SA.nnz, np.int8), *SA.shape, gb.INT8)
    B = Matrix.from_csr(SB.indptr, SB.indices, np.ones(SB.nnz, bool), *SB.shape, gb.BOOL)
    M = Matrix.from_csr(SM.indptr, SM.indices, None, *SM.shape) if SM is not None else None
    Ad = {(int(i), int(j)): 1 for i, j in zip(*SA.nonzero())}
    Bd = {(int(i), int(j)): 1 for i, j in zip(*SB.nonzero())}
    Md = {(int(i), int(j)): True for i, j in zip(*SM.nonzero())} if SM is not None else None
    with tunables(**env):
        for sr in GEMM_SR:
            C = Matrix.sparse(util.g_type(sr[2]), nrows, ncols)
            A.mxm(B, semiring=_sr(*sr), out=C, mask=M, desc=getattr(descriptor, desc) if desc else None)
            ks = _kernels()
            form = "positional=inner" if sr[1].rstrip("1") in ("FIRSTJ", "SECONDI") else "positional=count"
            assert form in ks and all(k in ks for k in want_k), (path, sr, ks)
            want, _ = pm.mxm({}, sr[2], Md, None, sr, Ad, Bd, _desc(desc))
            check(dict_m(C), want, None, sr[0], f"{path} {sr}")


# The inner form of mxm gives op(B)'s entries their row index when B has fewer entries than A: its row in B, in B's cached
# transpose (T1), or its column in B itself under the dot method (T1 + mask, which pairs rows of A with rows of B).
INNER_B = {"plain": ("", False, None), "T1": ("T1", False, None), "T1-dot": ("ST1", True, "dot"), "T0T1": ("T0T1", False, None),
           "T1-masked": ("RST1", True, None)}


@pytest.mark.parametrize("case", list(INNER_B) + ["hyper-T1", "hyper-dot"])
def test_mxm_inner_form_on_the_sparser_operand_b(case):
    hyper = case.startswith("hyper")
    form, masked, want_k = INNER_B["T1-dot" if case == "hyper-dot" else "T1" if hyper else case]
    rng = np.random.default_rng(seed_of("inner-B", case))
    n = 37
    A, B = rand_d(rng, (n, n), 0.3, "FP32"), rand_d(rng, (n, n), 0.05, "INT8")
    M = rand_d(rng, (n, n), 0.5, "BOOL") if masked else None
    dim = n
    if hyper:      # original indices beyond 2^31 in every index space (both cases are T1: B's columns are the inner space)
        dim = BIG
        sh = lambda d, r, c: {(i * r + 5, j * c + 3): v for (i, j), v in d.items()} if d is not None else None
        A, B, M = sh(A, 1 << 40, 1 << 31), sh(B, 1 << 40, 1 << 31), sh(M, 1 << 40, 1 << 40)
    for sr in [("MIN", "SECONDI", "INT64"), ("PLUS", "FIRSTJ1", "INT32"), ("MAX", "SECONDI1", "INT32")]:
        C = Matrix.sparse(util.g_type(sr[2]), dim, dim)
        mat_of(A, "FP32", dim, dim).mxm(mat_of(B, "INT8", dim, dim), semiring=_sr(*sr), out=C,
                                        mask=mat_of(M, "BOOL", dim, dim) if masked else None, desc=getattr(descriptor, form) if form else None)
        ks = _kernels()
        assert "positional=inner" in ks and "positional-operand=B" in ks, (case, sr, ks)
        if want_k:
            assert want_k in ks, (case, sr, ks)
        want, _ = pm.mxm({}, sr[2], M, None, sr, A, B, _desc(form))
        check(dict_m(C), want, None, sr[0], f"{case} {sr}")


# ------------------------------------------------------------------ INT32 wrap-around
def test_int32_wrap_around():
    # row i = 70000 of a 70001 x 2^15 matrix with 2^15 entries: PLUS_FIRSTI = 70000 * 32768 > 2^31, TIMES_FIRSTI1 = 70001^32768
    n, k = 70001, 1 << 15
    A = Matrix.from_lists([n - 1] * k, list(range(k)), [1] * k, n, k, gb.BOOL)
    u = Vector.from_numpy(np.ones(k, bool), typ=gb.BOOL)
    for add, mul in [("PLUS", "FIRSTI"), ("TIMES", "FIRSTI1"), ("PLUS", "SECONDI1")]:
        for typ in pm.TYPES:
            w = A.mxv(u, semiring=_sr(add, mul, typ))
            base, off = (mul[:-1], 1) if mul.endswith("1") else (mul, 0)
            vals = [n - 1 + off] * k if base == "FIRSTI" else [j + off for j in range(k)]
            assert dict_v(w) == {n - 1: pm.fold(add, typ, vals)}, (add, mul, typ)


# ------------------------------------------------------------------ hypersparse operands: original indices
BIG = 1 << 60
IDX = [5, (1 << 31) + 3, (1 << 40) + 5]


@pytest.mark.parametrize("typ", pm.TYPES)
def test_hypersparse_operands_give_original_indices(typ):
    A = {(IDX[0], IDX[1]): 1, (IDX[2], IDX[1]): 1, (IDX[2], IDX[2]): 1, (IDX[1], IDX[0]): 1}
    u = {IDX[1]: 1, IDX[2]: 1}
    gA, gu = mat_of(A, "INT64", BIG, BIG), vec_of(u, "INT64", BIG)
    for add, mul in [("MIN", "SECONDI"), ("PLUS", "FIRSTI1"), ("MAX", "FIRSTJ"), ("PLUS", "SECONDJ1")]:
        sr = (add, mul, typ)
        w = gA.mxv(gu, semiring=_sr(*sr))
        check(dict_v(w), pm.mxv({}, typ, None, None, sr, A, u)[0], None, add, f"hyper mxv {sr}")
        w = gu.vxm(gA, semiring=_sr(*sr))
        check(dict_v(w), pm.vxm({}, typ, None, None, sr, u, A)[0], None, add, f"hyper vxm {sr}")
        C = gA.mxm(gA, semiring=_sr(*sr))
        check(dict_m(C), pm.mxm({}, typ, None, None, sr, A, A)[0], None, add, f"hyper mxm {sr}")
    got = dict_v(gA.mxv(gu, semiring=_sr("MIN", "SECONDI", typ)))
    assert got[IDX[2]] == pm.trunc(IDX[1], typ) and got[IDX[0]] == pm.trunc(IDX[1], typ)


# ------------------------------------------------------------------ apply
@pytest.mark.parametrize("typ", pm.TYPES)
@pytest.mark.parametrize("tran", [False, True])
def test_apply_on_matrices_and_vectors(typ, tran):
    rng = np.random.default_rng(seed_of("apply", typ, tran))
    A = rand_d(rng, (13, 29), 0.3, "FP64")
    gA = mat_of(A, "FP64", 13, 29)
    shape = (29, 13) if tran else (13, 29)
    for op in pm.UNARY:
        out = Matrix.sparse(util.g_type(typ), *shape)
        gA.apply(getattr(util.g_type(typ), op), out=out, desc=descriptor.T0 if tran else None)
        assert dict_m(out) == pm.apply(op, typ, A, tran), op
    for op in pm.POSITIONAL:
        T = util.g_type(typ)
        out = Matrix.sparse(T, *shape)
        gA.apply_first(gb.Scalar.from_value(3.5), getattr(T, op), out=out, desc=descriptor.T0 if tran else None)
        assert dict_m(out) == pm.apply(op, typ, A, tran), op
        out = Matrix.sparse(T, *shape)
        gA.apply_second(getattr(T, op), 7, out=out, desc=descriptor.T0 if tran else None)
        assert dict_m(out) == pm.apply(op, typ, A, tran), op
    u = rand_d(rng, (29,), 0.5, "UINT16")
    gu = vec_of(u, "UINT16", 29)
    for op in pm.UNARY + pm.POSITIONAL:
        T = util.g_type(typ)
        w = Vector.sparse(T, 29)
        if op in pm.UNARY:
            gu.apply(getattr(T, op), out=w)
        else:
            gu.apply_second(getattr(T, op), 1, out=w)
        assert dict_v(w) == pm.apply_vector(op, typ, u), op


def test_apply_with_mask_and_accumulator():
    rng = np.random.default_rng(5)
    A, C0, M = rand_d(rng, (11, 11), 0.4, "INT64"), rand_d(rng, (11, 11), 0.4, "INT64"), rand_d(rng, (11, 11), 0.5, "BOOL")
    out = mat_of(C0, "INT64", 11, 11)
    mat_of(A, "INT64", 11, 11).apply(gb.INT64.POSITIONJ1, out=out, mask=mat_of(M, "BOOL", 11, 11), accum=gb.INT64.PLUS)
    T = pm.apply("POSITIONJ1", "INT64", A)
    assert {k: int(v) for k, v in dict_m(out).items()} == {k: int(v) for k, v in pm.writeback(C0, "INT64", M, ("PLUS", "INT64"), T, "INT64", {}).items()}


# ------------------------------------------------------------------ BFS with a parent tree: q'<!pi> = q' ANY.SECONDI A
def test_bfs_with_parents_on_rmat():
    from pygraphblas_b200.generators import rmat_csr
    n, indptr, indices = rmat_csr(16)
    S = sp.csr_matrix((np.ones(len(indices), bool), indices, indptr), shape=(n, n))
    S.sort_indices()
    A = Matrix.from_csr(S.indptr, S.indices, np.ones(S.nnz, bool), n, n, gb.BOOL)
    src = int(np.argmax(np.diff(S.indptr)))
    parent = Vector.from_lists([src], [src], n, gb.INT64)
    q = Vector.from_lists([src], [src], n, gb.INT64)
    sr = gb.INT64.ANY_SECONDI
    # vxm: y at (k, j) of A, SECONDI = k, the vertex the edge k -> j leaves from
    while q.nvals:
        q = q.vxm(A, semiring=sr, mask=parent, desc=descriptor.RSC)
        _kernels()
        parent.eadd(q, gb.INT64.FIRST, out=parent)
    level = csgraph.shortest_path(S, unweighted=True, indices=src)
    P = dict_v(parent)
    reached = {int(v) for v in np.flatnonzero(np.isfinite(level))}
    assert set(P) == reached
    for v, p in P.items():
        if v == src:
            assert p == src
            continue
        assert S[p, v], (v, p)
        assert level[p] == level[v] - 1, (v, p, level[p], level[v])


# ------------------------------------------------------------------ allocation failures on the new paths
ALLOC_CASES = ["mxv-inner", "mxv-count", "vxm-inner", "vxm-count", "mxm-inner", "mxm-count", "mxm-masked", "apply", "vector-apply",
               "hyper-mxv", "hyper-mxm"]


@pytest.mark.parametrize("case", ALLOC_CASES)
def test_allocation_failure(case):
    """A failure injected at every device allocation of a positional call: GrB_OUT_OF_MEMORY or success, nothing leaked,
    and the operands give the clean result afterwards (test_alloc_failure_gpu's sweep)."""
    from test_alloc_failure_gpu import _sweep
    rng = np.random.default_rng(seed_of("alloc", case))
    n = BIG if case.startswith("hyper") else 300
    A, B = rand_d(rng, (300, 300), 0.03, "FP32"), rand_d(rng, (300, 300), 0.03, "INT8")
    if case.startswith("hyper"):
        A = {(i * (1 << 40) + 5, j * (1 << 31) + 3): v for (i, j), v in A.items()}
        B = {(i * (1 << 31) + 3, j + 7): v for (i, j), v in B.items()}
    u = {k: v for (k, _), v in list(B.items())[:150]}
    make = {
        "mxv-inner": lambda: (mat_of(A, "FP32", n, n), vec_of(u, "INT8", n)),
        "mxv-count": lambda: (mat_of(A, "FP32", n, n), vec_of(u, "INT8", n)),
        "vxm-inner": lambda: (vec_of(u, "INT8", n), mat_of(A, "FP32", n, n)),
        "vxm-count": lambda: (vec_of(u, "INT8", n), mat_of(A, "FP32", n, n)),
        "mxm-inner": lambda: (mat_of(A, "FP32", n, n), mat_of(B, "INT8", n, n)),
        "mxm-count": lambda: (mat_of(A, "FP32", n, n), mat_of(B, "INT8", n, n)),
        "mxm-masked": lambda: (mat_of(A, "FP32", n, n), mat_of(B, "INT8", n, n), mat_of(A, "FP32", n, n)),
        "apply": lambda: (mat_of(A, "FP32", n, n),),
        "vector-apply": lambda: (vec_of(u, "INT8", n),),
        "hyper-mxv": lambda: (mat_of(A, "FP32", n, n), vec_of(u, "INT8", n)),
        "hyper-mxm": lambda: (mat_of(A, "FP32", n, n), mat_of(B, "INT8", n, n)),
    }[case]
    call = {
        "mxv-inner": lambda A, u: A.mxv(u, semiring=INT_SR_INNER),
        "mxv-count": lambda A, u: A.mxv(u, semiring=INT_SR_COUNT),
        "vxm-inner": lambda u, A: u.vxm(A, semiring=INT_SR_INNER),
        "vxm-count": lambda u, A: u.vxm(A, semiring=gb.INT64.TIMES_SECONDJ1),
        "mxm-inner": lambda A, B: A.mxm(B, semiring=INT_SR_INNER),
        "mxm-count": lambda A, B: A.mxm(B, semiring=INT_SR_COUNT),
        "mxm-masked": lambda A, B, M: A.mxm(B, semiring=gb.INT32.MAX_SECONDJ, mask=M),
        "apply": lambda A: A.apply(gb.INT64.POSITIONJ1, out=Matrix.sparse(gb.INT64, n, n), desc=descriptor.T0),
        "vector-apply": lambda u: u.apply(gb.INT32.POSITIONI, out=Vector.sparse(gb.INT32, n)),
        "hyper-mxv": lambda A, u: A.mxv(u, semiring=INT_SR_COUNT),
        "hyper-mxm": lambda A, B: A.mxm(B, semiring=INT_SR_INNER),
    }[case]
    assert _sweep(make, call) >= 1


INT_SR_INNER = gb.INT64.MIN_SECONDI1
INT_SR_COUNT = gb.INT64.PLUS_FIRSTI


# ------------------------------------------------------------------ ledger
def test_every_rewritten_path_was_reached(request):
    """Runs last in the module: every SpMV / SpGEMM path above was entered by a positional call, in both forms."""
    selected = {i.name.split("[")[0] for i in request.session.items if i.module.__name__ == __name__}
    if not {"test_spmv_paths", "test_spgemm_paths"} <= selected:
        pytest.skip("the path tests were not selected")
    want = {"positional=inner", "positional=count", "run", "run (sparse u)", "run+hot-table (TMA-staged)", "pull", "push"}
    want |= {k for _, ks in GEMM.values() for k in ks}
    missing = want - REACHED
    assert not missing, f"never reached: {sorted(missing)}"
    assert "tile-8: run" in REACHED          # the small matrix runs on the run kernel too
