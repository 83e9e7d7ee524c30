"""GrB_mxm with two dense-form operands under a sparse mask, C<M> = X (+).(x) Y' (the sampled dense-dense product, DESIGN.md
section 3.6), against the oracle on the CSR equivalent of every dense operand: semirings, types, d on both sides of the chunk
length, presence arrays, structural and valued masks of every shape, the four descriptor forms, accumulators, replace, aliasing,
casts, value edges, independence from the mask, the routes left alone, R-MAT s16 and a GNN layer against scipy, allocation
failures, and the SASS of the kernels."""
import gc
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import scipy.sparse as sp

import pygraphblas_b200 as gb
from pygraphblas_b200 import Matrix, descriptor, lib
from pygraphblas_b200.generators import rmat_csr
from oracle import oracle as orc
import kernel_check as kc
import util
from test_alloc_failure_gpu import _sweep
from test_dense_gpu import FAST, RUNTIME, check, g_csr, g_dense, o_dense, rand_csr, status
from test_sddmm import SEG, chunked_dot, route

pytestmark = pytest.mark.gpu

DENSE = (lib.GxB_FULL, lib.GxB_BITMAP)


def tokens():
    return kc.last_kernel().split(";")


def expect_sddmm(t, fast=None, pattern=None, xtr=False, ytr=False):
    assert "sddmm" in t and not any(e.startswith("spmm") for e in t), t
    if fast is not None:
        assert ("sddmm-fast" if fast else "sddmm-generic") in t, t
    if pattern is not None:
        assert f"pattern={pattern}" in t, t
    assert ("x-transpose" in t) == xtr and ("y-transpose" in t) == ytr, t


def operand(rng, typ, rows, d, density=None, pool=None, side=0, seed=0):
    x = kc.values(seed, typ, rows * d, pool, side) if pool and typ in util.FP_T else util.rand_values(rng, typ, rows * d)
    x = x.reshape(rows, d)
    pres = None if density is None else (rng.random((rows, d)) < density).astype(np.uint8)
    return x, pres


def mask_csr(rng, typ, m, n, density=0.2, lens=None, zeros=False):
    S = rand_csr(rng, typ, m, n, density, lens=lens)
    if zeros and S.nnz:                                  # explicit zeros / false: entries a valued mask switches off
        S.data[rng.random(S.nnz) < 0.4] = 0
    return S


def run(sr, X, Y, M, desc="ST1", C=None, accum=None, ctyp=None):
    C = C if C is not None else Matrix.sparse(util.g_type(ctyp or orc.semiring_ztype(sr)), M.nrows, M.ncols)
    X.mxm(Y, semiring=kc.semiring(*sr), mask=M, out=C, accum=util.g_accum(accum), desc=getattr(descriptor, desc))
    return C, tokens()


def want_of(sr, ox, oy, om, m, n, desc="ST1", oc=None, accum=None, ctyp=None):
    oc = oc if oc is not None else orc.SpMat(ctyp or orc.semiring_ztype(sr), m, n)
    return orc.mxm(oc, om, accum, sr, ox, oy, desc)


def case(sr, d, label, m=37, n=29, xdens=None, ydens=None, mtyp="BOOL", desc="ST1", xtyp=None, ytyp=None, pool=True, zeros=False):
    add, mul, typ = sr
    rng = np.random.default_rng(kc.seed_of("sddmm", label, sr, d))
    xtyp, ytyp = xtyp or typ, ytyp or typ
    p = kc.fp_pool_for(add, mul) if pool else None
    x, xp = operand(rng, xtyp, m, d, xdens, p, 0, kc.seed_of(label, 1, d))
    y, yp = operand(rng, ytyp, n, d, ydens, p, 1, kc.seed_of(label, 2, d))
    S = mask_csr(rng, mtyp, m, n, 0.25, zeros=zeros)
    if "T1" not in desc:                                 # Y given d x n
        y, yp = np.ascontiguousarray(y.T), None if yp is None else np.ascontiguousarray(yp.T)
    C, t = run(sr, g_dense(xtyp, x, xp), g_dense(ytyp, y, yp), g_csr(mtyp, S), desc)
    want = want_of(sr, o_dense(xtyp, x, xp), o_dense(ytyp, y, yp), kc.o_csr(mtyp, S, S.data), m, n, desc)
    check(C, want, add, f"{label} {sr} d={d}")
    return t


# ------------------------------------------------------------------ semirings, d up to one chunk: the oracle's fold, bit for bit
DS = (1, 3, 4, 7, 32, 33, 64)


@pytest.mark.parametrize("sr", FAST, ids=lambda s: "_".join(s))
def test_specialised_semirings(sr):
    for d in DS:
        expect_sddmm(case(sr, d, "fast"), fast=True, pattern="mask")
    expect_sddmm(case(sr, 8, "fast-pres", xdens=0.5, ydens=0.6), fast=True, pattern="compact")


@pytest.mark.parametrize("sr", RUNTIME[::2], ids=lambda s: "_".join(s))
def test_runtime_semirings(sr):
    for d in DS:
        expect_sddmm(case(sr, d, "runtime", xdens=0.7 if d % 2 else None), fast=False)


def test_the_lists_cover_every_type():
    assert {t for _, _, t in FAST + RUNTIME[::2]} == set(util.ALL_T)


# ------------------------------------------------------------------ d beyond one chunk: chunks of SEG, partials in the fixed tree
@pytest.mark.parametrize("d", [65, 128, 200])
def test_long_rows_exact_types(d):
    assert d > SEG
    for sr in (("PLUS", "TIMES", "INT32"), ("PLUS", "TIMES", "UINT8"), ("MIN", "PLUS", "INT64"), ("LOR", "LAND", "BOOL"),
               ("PLUS", "TIMES", "FP32"), ("PLUS", "TIMES", "FP64"), ("MAX", "PLUS", "FP32"), ("PLUS", "PAIR", "INT16")):
        expect_sddmm(case(sr, d, "long", pool=False))                       # rand_values: quarters, every sum exact
        expect_sddmm(case(sr, d, "long-pres", xdens=0.3, ydens=0.9, pool=False), pattern="compact")


@pytest.mark.parametrize("d", [65, 128, 200])
@pytest.mark.parametrize("typ", ["FP32", "FP64"])
def test_long_rows_random_fp(typ, d):
    rng = np.random.default_rng(kc.seed_of("long-fp", typ, d))
    m, n = 12, 10
    dt = np.dtype(orc.DTYPES[typ])
    x, y = (rng.random((m, d)) - 0.25).astype(dt), (rng.random((n, d)) - 0.25).astype(dt)
    xp = (rng.random((m, d)) < 0.9).astype(np.uint8)
    S = mask_csr(rng, "BOOL", m, n, 0.4)
    for pres in (None, xp):
        C, t = run(("PLUS", "TIMES", typ), g_dense(typ, x, pres), g_dense(typ, y, None), g_csr("BOOL", S))
        expect_sddmm(t, fast=True, pattern="mask" if pres is None else "compact")
        I, J, V = C.to_arrays()
        assert len(I) == S.nnz
        for i, j, v in zip(I, J, V):
            want, has = chunked_dot(x[i], y[j], xp=None if pres is None else pres[i])
            assert has and kc._bits(np.asarray([v]))[0] == kc._bits(np.asarray([want], dt))[0], (i, j, v, want)
            keep = np.ones(d, bool) if pres is None else pres[i].astype(bool)
            ref = np.dot(x[i].astype(np.float64)[keep], y[j].astype(np.float64)[keep])
            scale = np.dot(np.abs(x[i].astype(np.float64))[keep], np.abs(y[j].astype(np.float64))[keep])
            assert abs(float(v) - ref) <= 1e-6 * scale


# ------------------------------------------------------------------ presence
@pytest.mark.parametrize("xdens", [None, 0.0, 0.3, 0.9])
@pytest.mark.parametrize("ydens", [None, 0.0, 0.3, 0.9])
def test_presence(xdens, ydens):
    for sr, d in ((("PLUS", "TIMES", "FP64"), 5), (("MIN", "PLUS", "INT32"), 70), (("PLUS", "PAIR", "INT64"), 9)):
        t = case(sr, d, "presence", xdens=xdens, ydens=ydens)
        expect_sddmm(t, pattern="mask" if xdens is None and ydens is None else "compact")


def test_all_absent_operand_gives_an_empty_result():
    rng = np.random.default_rng(3)
    x, y = util.rand_values(rng, "FP32", 20 * 6).reshape(20, 6), util.rand_values(rng, "FP32", 15 * 6).reshape(15, 6)
    S = mask_csr(rng, "BOOL", 20, 15, 0.3)
    C, t = run(("PLUS", "TIMES", "FP32"), g_dense("FP32", x, np.zeros((20, 6), np.uint8)), g_dense("FP32", y, None), g_csr("BOOL", S))
    expect_sddmm(t, pattern="compact")
    assert C.nvals == 0


# ------------------------------------------------------------------ masks
@pytest.mark.parametrize("mtyp", util.ALL_T)
def test_valued_masks_of_every_type(mtyp):
    for desc in ("T1", "ST1"):
        t = case(("PLUS", "TIMES", "INT32"), 6, f"valued {desc}", mtyp=mtyp, desc=desc, zeros=True)
        expect_sddmm(t, fast=True, pattern="mask" if desc == "ST1" else "compact")
    expect_sddmm(case(("MAX", "PLUS", "FP32"), 40, "valued-pres", mtyp=mtyp, desc="T1", zeros=True, xdens=0.5), pattern="compact")


def _mask_shape_case(lens, m, n, d, label, sr=("PLUS", "TIMES", "FP64")):
    rng = np.random.default_rng(kc.seed_of("mask-shape", label))
    typ = sr[2]
    x, _ = operand(rng, typ, m, d)
    y, _ = operand(rng, typ, n, d)
    S = mask_csr(rng, "INT8", m, n, lens=lens, zeros=True)
    for desc in ("ST1", "T1"):
        C, t = run(sr, g_dense(typ, x, None), g_dense(typ, y, None), g_csr("INT8", S), desc)
        expect_sddmm(t)
        check(C, want_of(sr, o_dense(typ, x, None), o_dense(typ, y, None), kc.o_csr("INT8", S, S.data), m, n, desc), sr[0], label)
    return S


def test_mask_shapes():
    n = 70
    assert _mask_shape_case([0] * 9, 9, n, 5, "empty mask").nnz == 0
    _mask_shape_case([0, 3, 0, 0, n, 0, 1, 0, 0], 9, n, 5, "empty rows, one full row")
    _mask_shape_case([0] * 8 + [n], 9, n, 5, "only the last row, every column")
    S = _mask_shape_case([1, 2, 3, 5, 7, 11, 13, 0, 3], 9, n, 33, "primes")
    assert S.nnz % 32 and S.nnz % 4


def test_row_changes_on_every_lane():
    """Rows of 33 entries: over 32 consecutive rows the row change falls on every lane position of a warp."""
    n, d = 40, 4
    lens = [33] * 32 + [1, 0, 2]
    S = _mask_shape_case(lens, len(lens), n, d, "lanes", sr=("PLUS", "TIMES", "INT64"))
    starts = np.cumsum([0] + lens[:32]) % 32
    assert set(starts.tolist()) == set(range(32)) and S.nnz % 4


def test_last_row_and_column():
    rng = np.random.default_rng(5)
    m, n, d = 50, 45, 7
    x, _ = operand(rng, "FP32", m, d)
    y, _ = operand(rng, "FP32", n, d)
    M = Matrix.from_lists([0, m - 1, m - 1], [n - 1, 0, n - 1], [True] * 3, m, n, gb.BOOL)
    C, t = run(("PLUS", "TIMES", "FP32"), g_dense("FP32", x, None), g_dense("FP32", y, None), M)
    expect_sddmm(t, pattern="mask")
    I, J, V = C.to_arrays()
    assert list(zip(I, J)) == [(0, n - 1), (m - 1, 0), (m - 1, n - 1)]
    assert np.array_equal(V, [chunked_dot(x[i], y[j])[0] for i, j in zip(I, J)])


# ------------------------------------------------------------------ descriptors: one kernel behind the four forms
@pytest.mark.parametrize("d", [1, 6, 40])
@pytest.mark.parametrize("xdens", [None, 0.7])
def test_four_descriptor_forms_give_the_same_bits(d, xdens):
    rng = np.random.default_rng(kc.seed_of("desc", d, xdens))
    m, n = 23, 31                                        # m, n, d pairwise different
    sr = ("PLUS", "TIMES", "FP32")
    x, xp = operand(rng, "FP32", m, d, xdens)
    y, yp = operand(rng, "FP32", n, d, xdens)
    x, y = (x + rng.random((m, d))).astype(np.float32), (y + rng.random((n, d))).astype(np.float32)   # order-sensitive sums
    S = mask_csr(rng, "BOOL", m, n, 0.3)
    tr = lambda a: None if a is None else np.ascontiguousarray(a.T)
    forms = {"ST1": (x, xp, y, yp), "S": (x, xp, tr(y), tr(yp)), "ST0T1": (tr(x), tr(xp), y, yp), "ST0": (tr(x), tr(xp), tr(y), tr(yp))}
    ref = None
    for desc, (a, ap, b, bp) in forms.items():
        C, t = run(sr, g_dense("FP32", a, ap), g_dense("FP32", b, bp), g_csr("BOOL", S), desc)
        expect_sddmm(t, fast=True, pattern="mask" if xdens is None else "compact",
                     xtr="T0" in desc and d > 1, ytr="T1" not in desc and d > 1)
        got = tuple(kc._bits(np.asarray(a_)) for a_ in C.to_arrays())
        if ref is None:
            ref = got
            check(C, want_of(sr, o_dense("FP32", a, ap), o_dense("FP32", b, bp), kc.o_csr("BOOL", S, S.data), m, n, desc), "PLUS", desc)
        assert all(np.array_equal(p, q) for p, q in zip(got, ref)), desc


def test_pair_needs_no_transpose():
    """PLUS.PAIR over full operands reads neither: d on every edge, no transpose built whatever the descriptor."""
    rng = np.random.default_rng(6)
    m, n, d = 12, 9, 70
    S = mask_csr(rng, "BOOL", m, n, 0.5)
    C, t = run(("PLUS", "PAIR", "INT32"), Matrix.from_numpy(np.ones((d, m), np.int32)), Matrix.from_numpy(np.ones((d, n), np.int32)),
               g_csr("BOOL", S), "ST0")
    expect_sddmm(t, fast=True, pattern="mask")
    assert C.nvals == S.nnz and set(C.to_arrays()[2].tolist()) == {d}


# ------------------------------------------------------------------ accumulators, replace, C of every kind
@pytest.mark.parametrize("desc", ["T1", "RT1", "ST1", "RST1"])
@pytest.mark.parametrize("c_kind", ["empty", "csr", "dense"])
def test_accum_replace(desc, c_kind):
    rng = np.random.default_rng(kc.seed_of("sddmm-accum", desc, c_kind))
    m, n, d = 14, 17, 6
    sr = ("PLUS", "TIMES", "INT32")
    x, xp = operand(rng, "INT32", m, d, 0.8)
    y, yp = operand(rng, "INT32", n, d)
    S = mask_csr(rng, "FP32", m, n, 0.4, zeros=True)
    cx = util.rand_values(rng, "INT64", m * n).reshape(m, n)
    cp = (rng.random((m, n)) < 0.5).astype(np.uint8)
    for accum in (None, ("PLUS", "INT64"), ("MIN", "INT64")):
        if c_kind == "empty":
            C, oc = Matrix.sparse(gb.INT64, m, n), orc.SpMat("INT64", m, n)
        elif c_kind == "dense":
            C, oc = g_dense("INT64", cx, cp), o_dense("INT64", cx, cp)
        else:
            I, J = np.nonzero(cp)
            C, oc = Matrix.from_lists(I, J, cx[I, J], m, n, gb.INT64), o_dense("INT64", cx, cp)
        C, t = run(sr, g_dense("INT32", x, xp), g_dense("INT32", y, yp), g_csr("FP32", S), desc, C=C, accum=accum)
        expect_sddmm(t, pattern="compact")
        want = want_of(sr, o_dense("INT32", x, xp), o_dense("INT32", y, yp), kc.o_csr("FP32", S, S.data), m, n, desc, oc=oc, accum=accum)
        check(C, want, "PLUS", f"{desc} {c_kind} {accum}")


def test_aliasing():
    rng = np.random.default_rng(8)
    n, sr = 16, ("PLUS", "TIMES", "FP64")
    x, xp = operand(rng, "FP64", n, n, 0.8)
    y, _ = operand(rng, "FP64", n, n)
    S = mask_csr(rng, "FP64", n, n, 0.3)
    ox, oy, om = o_dense("FP64", x, xp), o_dense("FP64", y, None), kc.o_csr("FP64", S, S.data)
    for alias in ("A", "B", "M"):
        X, Y, M = g_dense("FP64", x, xp), g_dense("FP64", y, None), g_csr("FP64", S)
        C = {"A": X, "B": Y, "M": M}[alias]
        oc = {"A": ox, "B": oy, "M": om}[alias]
        C, t = run(sr, X, Y, M, "T1", C=C, accum=("PLUS", "FP64"))
        expect_sddmm(t)
        check(C, want_of(sr, ox, oy, om, n, n, "T1", oc=oc, accum=("PLUS", "FP64")), "PLUS", f"C is {alias}")
        assert status(C) not in DENSE


@pytest.mark.parametrize("xtyp,ytyp,sr", [("INT8", "FP32", ("PLUS", "TIMES", "FP64")), ("BOOL", "INT16", ("MAX", "PLUS", "INT32")),
                                          ("FP64", "UINT8", ("MIN", "TIMES", "INT64")), ("UINT16", "BOOL", ("LOR", "LAND", "BOOL")),
                                          ("FP32", "FP32", ("LOR", "GT", "FP32")), ("INT64", "INT32", ("PLUS", "PAIR", "FP32"))])
def test_mixed_type_casts(xtyp, ytyp, sr):
    for desc in ("ST1", "S"):
        expect_sddmm(case(sr, 6, "cast", xtyp=xtyp, ytyp=ytyp, xdens=0.8, desc=desc), pattern="compact",
                     ytr=desc == "S" and sr[1] != "PAIR")


@pytest.mark.parametrize("typ", util.ALL_T)
def test_value_edges_and_determinism(typ):
    rng = np.random.default_rng(kc.seed_of("sddmm-edges", typ))
    m, n, d = 20, 18, 9
    srs = (("MIN", "PLUS"), ("MAX", "TIMES"), ("PLUS", "TIMES"), ("TIMES", "PLUS")) if typ != "BOOL" else (("LOR", "LAND"), ("LAND", "LOR"))
    for add, mul in srs:
        sr = (add, mul, typ)
        pool = "edge" if add in ("MIN", "MAX") else kc.fp_pool_for(add, mul)
        x = kc.values(kc.seed_of(typ, add, 0), typ, m * d, pool, 0).reshape(m, d)
        y = kc.values(kc.seed_of(typ, add, 1), typ, n * d, pool, 1).reshape(n, d)
        xp = (rng.random((m, d)) < 0.5).astype(np.uint8)      # short folds: a sole NaN or -0.0 must survive
        S = mask_csr(rng, "BOOL", m, n, 0.5)
        C1, t = run(sr, g_dense(typ, x, xp), g_dense(typ, y, None), g_csr("BOOL", S))
        C2, _ = run(sr, g_dense(typ, x, xp), g_dense(typ, y, None), g_csr("BOOL", S))
        expect_sddmm(t, pattern="compact")
        assert all(np.array_equal(kc._bits(np.asarray(a)), kc._bits(np.asarray(b))) for a, b in zip(C1.to_arrays(), C2.to_arrays()))
        check(C1, want_of(sr, o_dense(typ, x, xp), o_dense(typ, y, None), kc.o_csr("BOOL", S, S.data), m, n), add, f"edges {sr}")


# ------------------------------------------------------------------ T(i, j) does not depend on M
@pytest.mark.parametrize("d", [5, 32, 150])
def test_independence_from_the_mask(d):
    rng = np.random.default_rng(d)
    m, n = 40, 300
    x, y = rng.random((m, d), dtype=np.float32), rng.random((n, d), dtype=np.float32)
    X, Y = Matrix.from_numpy(x), Matrix.from_numpy(y)
    i, j = 17, 123
    long_row = np.sort(rng.choice(n, 200, replace=False))
    long_row = np.unique(np.append(long_row, j))
    # alone; inside a long row; in the last, partly filled warp of a mask with many entries before it
    many = sp.random(m, n, density=0.3, format="csr", random_state=rng)
    many = sp.csr_matrix(sp.vstack([many[:m - 1], sp.csr_matrix((1, n))]))
    masks = [Matrix.from_lists([i], [j], [True], m, n, gb.BOOL),
             Matrix.from_lists([i] * len(long_row), long_row, [True] * len(long_row), m, n, gb.BOOL)]
    I, J = many.nonzero()
    masks.append(Matrix.from_lists(list(I) + [m - 1], list(J) + [j], [True] * (len(I) + 1), m, n, gb.BOOL))
    got = []
    for k, M in enumerate(masks):
        C, t = run(("PLUS", "TIMES", "FP32"), X, Y, M)
        expect_sddmm(t, fast=True, pattern="mask")
        got.append(C.get(i if k < 2 else m - 1, j))
    want0, _ = chunked_dot(x[i], y[j])
    want2, _ = chunked_dot(x[m - 1], y[j])
    assert np.float32(got[0]) == want0 and np.float32(got[1]) == want0 and np.float32(got[2]) == want2


# ------------------------------------------------------------------ routes left alone
def test_other_routes_are_unchanged():
    rng = np.random.default_rng(15)
    m, n, d = 9, 11, 6
    sr = ("PLUS", "TIMES", "INT64")
    x, xp = operand(rng, "INT64", m, d, 0.8)
    y, yp = operand(rng, "INT64", n, d, 0.8)
    S = mask_csr(rng, "BOOL", m, n, 0.4)
    ox, oy, om = o_dense("INT64", x, xp), o_dense("INT64", y, yp), kc.o_csr("BOOL", S, S.data)
    yt, ytp = np.ascontiguousarray(y.T), np.ascontiguousarray(yp.T)
    oyt = o_dense("INT64", yt, ytp)
    Ic, Jc = np.nonzero(yp)
    Ycsr = Matrix.from_lists(Ic, Jc, y[Ic, Jc], n, d, gb.INT64)
    mdense = S.toarray().astype(bool)

    def go(X, Y, M, desc, o_x, o_y, o_m):
        C = Matrix.sparse(gb.INT64, m, n)
        X.mxm(Y, semiring=gb.INT64.PLUS_TIMES, mask=M, out=C, desc=getattr(descriptor, desc) if desc else None)
        t = tokens()
        assert "sddmm" not in t, t
        check(C, orc.mxm(orc.SpMat("INT64", m, n), o_m, None, sr, o_x, o_y, desc), "PLUS", f"route {desc} {o_m is not None}")
        return t

    X = g_dense("INT64", x, xp)
    assert "spmm" in go(X, g_dense("INT64", yt, ytp), None, "", ox, oyt, None)                      # no mask
    assert "spmm" in go(X, g_dense("INT64", yt, ytp), g_csr("BOOL", S), "C", ox, oyt, om)          # complemented mask
    go(X, g_dense("INT64", y, yp), g_csr("BOOL", S), "CT1", ox, oy, om)
    t = go(X, g_dense("INT64", yt, ytp), g_dense("BOOL", mdense, mdense.astype(np.uint8)), "", ox, oyt,
           o_dense("BOOL", mdense, mdense.astype(np.uint8)))                                       # dense-form mask
    assert "spmm" in t and "write=dense" in t, t
    assert "spmm-left" in go(X, Ycsr, g_csr("BOOL", S), "T1", ox, oy, om)                          # one CSR operand
    # a positional semiring: the positional rewrite
    C = Matrix.sparse(gb.INT64, m, n)
    X.mxm(g_dense("INT64", y, yp), semiring=gb.INT64.MIN_FIRSTJ, mask=g_csr("BOOL", S), out=C, desc=descriptor.ST1)
    t = tokens()
    assert any(e.startswith("positional=") for e in t) and "sddmm" not in t, t
    Xc = Matrix.from_lists(*np.nonzero(xp), x[np.nonzero(xp)], m, d, gb.INT64)
    assert C.iseq(Xc.mxm(Ycsr, semiring=gb.INT64.MIN_FIRSTJ, mask=g_csr("BOOL", S), out=Matrix.sparse(gb.INT64, m, n), desc=descriptor.ST1))
    # the restated rule agrees with what was seen
    assert route(True, True, True, mask_nnz=S.nnz) == "sddmm" and route(True, True, False) == "other"
    assert route(True, True, True, mask_comp=True) == "other" and route(True, True, True, mask_dense=True) == "other"
    assert route(True, False, True) == "other" and route(True, True, True, positional=True) == "positional"


def test_empty_shapes():
    for m, n, d in ((5, 7, 0), (0, 7, 3), (5, 0, 3), (0, 0, 0)):
        X, Y = Matrix.from_numpy(np.zeros((m, d), np.float32)), Matrix.from_numpy(np.zeros((n, d), np.float32))
        M = Matrix.from_lists([0], [0], [True], m, n, gb.BOOL) if m and n else Matrix.sparse(gb.BOOL, m, n)
        C = Matrix.sparse(gb.FP32, m, n)
        X.mxm(Y, semiring=gb.FP32.PLUS_TIMES, mask=M, out=C, desc=descriptor.ST1)
        if status(X) in DENSE and status(Y) in DENSE:
            assert "sddmm" in tokens()
        assert C.nvals == 0 and C.shape == (m, n)


# ------------------------------------------------------------------ at scale, against scipy
def _edge_dots(x, y, rows, cols, chunk=1 << 20):
    out = np.empty(len(rows))
    for s in range(0, len(rows), chunk):
        out[s:s + chunk] = np.einsum("ij,ij->i", x[rows[s:s + chunk]].astype(np.float64), y[cols[s:s + chunk]].astype(np.float64))
    return out


def test_rmat_s16_against_scipy():
    n, indptr, indices = rmat_csr(16, 16, 1)
    rng = np.random.default_rng(16)
    d = 32
    x, y = rng.random((n, d), dtype=np.float32), rng.random((n, d), dtype=np.float32)
    M = Matrix.from_csr(indptr, indices, np.ones(len(indices), np.bool_), n, n, gb.BOOL)
    C, t = run(("PLUS", "TIMES", "FP32"), Matrix.from_numpy(x), Matrix.from_numpy(y), M)
    expect_sddmm(t, fast=True, pattern="mask")
    I, J, V = C.to_arrays()
    rows = np.repeat(np.arange(n), np.diff(indptr))
    assert np.array_equal(I, rows) and np.array_equal(J, indices)
    want = _edge_dots(x, y, rows, indices)
    assert (np.abs(V - want) / want).max() <= 1e-6
    flops, nout = gb.ffi.new("uint64_t*"), gb.ffi.new("uint64_t*")
    lib.B200_last_mxm_stats(flops, nout)
    assert flops[0] == len(indices) * d and nout[0] == len(indices)


def test_gnn_layer_scores_then_aggregation():
    """S<A> = H (+).(x) H' on the new route, then S (+).(x) H on the SpMM kernel; S stays on the device in between."""
    n, indptr, indices = rmat_csr(14, 16, 2)
    rng = np.random.default_rng(14)
    d = 32
    h = rng.random((n, d), dtype=np.float32)
    A = Matrix.from_csr(indptr, indices, np.ones(len(indices), np.float32), n, n, gb.FP32)
    H = Matrix.from_numpy(h)
    S = Matrix.sparse(gb.FP32, n, n)
    H.mxm(H, semiring=gb.FP32.PLUS_TIMES, mask=A, desc=descriptor.ST1, out=S)
    expect_sddmm(tokens(), fast=True, pattern="mask")
    out = Matrix.sparse(gb.FP32, n, d)
    S.mxm(H, semiring=gb.FP32.PLUS_TIMES, out=out)
    assert "spmm" in tokens()
    rows = np.repeat(np.arange(n), np.diff(indptr))
    S64 = sp.csr_matrix((_edge_dots(h, h, rows, indices), indices, indptr), shape=(n, n))
    want = S64 @ h.astype(np.float64)
    got, pres = out.to_numpy()
    nonempty = np.diff(indptr) > 0
    assert np.array_equal(pres.all(axis=1), nonempty) and not pres[~nonempty].any()
    assert (np.abs(got[nonempty] - want[nonempty]) / want[nonempty]).max() <= 4e-6


# ------------------------------------------------------------------ allocation failures
def test_allocation_failures():
    rng = np.random.default_rng(9)
    m, n, d = 60, 50, 12
    x, xp = operand(rng, "FP32", m, d, 0.7)
    y, _ = operand(rng, "FP32", n, d)
    S = mask_csr(rng, "FP32", m, n, 0.2, zeros=True)
    xt, xtp, yt = np.ascontiguousarray(x.T), np.ascontiguousarray(xp.T), np.ascontiguousarray(y.T)
    out = lambda: Matrix.sparse(gb.FP32, m, n)
    _sweep(lambda: (g_dense("FP32", x, None), g_dense("FP32", y, None), g_csr("FP32", S)),
           lambda X, Y, M: X.mxm(Y, semiring=gb.FP32.PLUS_TIMES, mask=M, desc=descriptor.ST1, out=out()))
    _sweep(lambda: (g_dense("FP32", x, xp), g_dense("FP32", y, None), g_csr("FP32", S)),
           lambda X, Y, M: X.mxm(Y, semiring=gb.FP32.MIN_PLUS, mask=M, desc=descriptor.T1, out=out(), accum=gb.FP32.PLUS))
    _sweep(lambda: (g_dense("FP32", xt, xtp), g_dense("FP32", yt, None), g_csr("FP32", S)),
           lambda X, Y, M: X.mxm(Y, semiring=gb.FP32.PLUS_TIMES, mask=M, desc=descriptor.T0, out=out()))
    _sweep(lambda: (g_dense("INT8", x.astype(np.int8), None), g_dense("FP32", yt, None), g_csr("FP32", S)),
           lambda X, Y, M: X.mxm(Y, semiring=gb.FP64.PLUS_TIMES, mask=M, desc=descriptor.S, out=Matrix.sparse(gb.FP64, m, n)))
    gc.collect()


# ------------------------------------------------------------------ the SASS of the kernels
def test_no_local_memory_in_the_kernels():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    libpath = os.path.join(root, "pygraphblas_b200", "libb200grb.so")
    if not os.path.exists(exe):
        pytest.skip("cuobjdump is not available")
    text = subprocess.run([exe, "-sass", libpath], capture_output=True, text=True, timeout=600).stdout
    name, seen, bad = None, set(), []
    for line in text.splitlines():
        f = re.search(r"Function : (\S+)", line)
        if f:
            name = f.group(1)
            continue
        if name and "sddmm" in name:
            seen.add(name)
            if re.search(r"\b(LDL|STL)\b", line):
                bad.append(f"{name}: {line.strip()}")
    assert len([s for s in seen if "sddmm_kernel" in s]) == 47 + 21      # the specialised semirings and the run-time domains
    assert not bad, "\n".join(bad[:10])
