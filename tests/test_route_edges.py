"""CPU: the checks of tests/test_route_edges_gpu.py can fail.  The exact-sum helper agrees with fractions.Fraction; the fold orders
restated there equal the oracle on dyadic values and tell orders apart on general values; and results mutated the ways a kernel
goes subtly wrong (a fused multiply-add fold, subnormals flushed to zero, neighbouring segments folded in the other order, an error
one ulp beyond the bound) are rejected by check_fp, the comparison the GPU module applies to every FP sum."""
from fractions import Fraction

import numpy as np
import pytest

from oracle import oracle as orc
import util
from kernel_check import _bits, o_csr, seed_of
from test_dense_gpu import o_dense
from test_sddmm import SEG, chunked_dot, tree_fold
from test_value_edges_gpu import _general_values
from test_route_edges_gpu import (SPLIT_LENS, check_fp, exact_sums, lens_csr, left_order, ltr_fold, products, sddmm_order,
                                  spmm_order, two_product, with_data)

FP_T = util.FP_T


def _fraction_sums(keys, a, b):
    out = {}
    for k, x, y in zip(np.asarray(keys).tolist(), np.asarray(a, np.float64).tolist(), np.asarray(b, np.float64).tolist()):
        out[k] = out.get(k, Fraction(0)) + Fraction(x) * Fraction(y)
    return np.array(sorted(out)), np.array([float(out[k]) for k in sorted(out)])


# ------------------------------------------------------------------ the exact sums
@pytest.mark.parametrize("scale", ["normal", "subnormal"])
@pytest.mark.parametrize("typ", FP_T)
def test_exact_sums_agree_with_fractions(typ, scale):
    rng = np.random.default_rng(seed_of("exact", typ, scale))
    n = 3000
    keys = rng.integers(0, 60, n)
    a, b = _general_values(rng, typ, n, "normal"), _general_values(rng, typ, n, scale)
    uk, got = exact_sums(keys, a, b, typ)
    wk, want = _fraction_sums(keys, a, b)
    assert np.array_equal(uk, wk)
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64))
    if scale == "subnormal":
        assert (np.abs(want) < np.finfo(orc.DTYPES[typ]).tiny).any()


def test_two_product_is_exact():
    rng = np.random.default_rng(3)
    a, b = rng.standard_normal(2000) * 2.0 ** rng.integers(-300, 300, 2000), rng.standard_normal(2000)
    p, e = two_product(a, b)
    for x, y, pp, ee in zip(a.tolist(), b.tolist(), p.tolist(), e.tolist()):
        assert Fraction(pp) + Fraction(ee) == Fraction(x) * Fraction(y)


# ------------------------------------------------------------------ the restated orders
def _dyadic(rng, typ, n):
    return util.rand_values(rng, typ, n)


@pytest.mark.parametrize("typ", FP_T)
def test_orders_equal_the_oracle_on_dyadic_values(typ):
    """Every fold order gives the same bits on multiples of 1/4: the restatements agree with orc.mxm."""
    rng = np.random.default_rng(5)
    S = lens_csr(SPLIT_LENS, 400, 2)
    av = _dyadic(rng, typ, S.nnz)
    x = _dyadic(rng, typ, 400 * 7).reshape(400, 7)
    xp = (rng.random((400, 7)) < 0.7).astype(np.uint8)
    sr = ("PLUS", "TIMES", typ)
    oa, ox = o_csr(typ, S, av), o_dense(typ, x, xp)
    ref = orc.mxm(orc.SpMat(typ, S.shape[0], 7), None, None, sr, oa, ox)
    k, v = spmm_order(with_data(S, av), x, xp, typ)
    assert np.array_equal(k, ref.I.astype(np.int64) * 7 + ref.J.astype(np.int64)) and np.array_equal(_bits(v), _bits(ref.X))
    # the left route: X (7 x 400) times S' (400 x 10)
    B = S.T.tocsr(); B.sort_indices()
    xl, xlp = np.ascontiguousarray(x.T), np.ascontiguousarray(xp.T)
    ref = orc.mxm(orc.SpMat(typ, 7, B.shape[1]), None, None, sr, o_dense(typ, xl, xlp), o_csr(typ, B, B.data.astype(orc.DTYPES[typ])))
    k, v = left_order(xl, xlp, B, typ)
    assert np.array_equal(k, ref.I.astype(np.int64) * B.shape[1] + ref.J.astype(np.int64)) and np.array_equal(_bits(v), _bits(ref.X))
    # SDDMM at d = 130 under a full mask, and the Gustavson fold of esc
    xs, ys = _dyadic(rng, typ, 5 * 130).reshape(5, 130), _dyadic(rng, typ, 4 * 130).reshape(4, 130)
    ref = orc.mxm(orc.SpMat(typ, 5, 4), None, None, sr, o_dense(typ, xs, None), o_dense(typ, ys, None), "T1")
    k, v = sddmm_order(xs, None, ys, None, np.arange(20), 4, typ)
    assert np.array_equal(k, ref.I.astype(np.int64) * 4 + ref.J.astype(np.int64)) and np.array_equal(_bits(v), _bits(ref.X))
    keys, a, b, n = products(oa, ox, "")
    k, v = ltr_fold(keys, a, b, typ)
    ref = orc.mxm(orc.SpMat(typ, S.shape[0], 7), None, None, sr, oa, ox)
    assert np.array_equal(k, ref.I.astype(np.int64) * 7 + ref.J.astype(np.int64)) and np.array_equal(_bits(v), _bits(ref.X))


# ------------------------------------------------------------------ a crafted long row and its mutations
LONG = 4 * SEG                          # four segments: the tree ((s0 s1) (s2 s3)) differs from every other bracketing


def _long_row(typ, scale, seed):
    """One row of LONG entries (and a short one) times a dense X of one column: (S with values, x, products, restated order)."""
    rng = np.random.default_rng(seed)
    S = lens_csr([LONG, 5], LONG + 10, seed)
    av = _general_values(rng, typ, S.nnz, "normal")
    x = _general_values(rng, typ, LONG + 10, scale).reshape(-1, 1)
    Sv = with_data(S, av)
    keys, a, b, _ = products(o_csr(typ, S, av), o_dense(typ, x, None), "")
    return Sv, x, (keys, a, b), spmm_order(Sv, x, None, typ)


def _first(pred, typ, scale):
    """The first seed whose long row makes pred true (the mutation changes the result), so every case below tests something."""
    for seed in range(200):
        r = _long_row(typ, scale, seed)
        if pred(*r):
            return r
    raise AssertionError("no seed separates the mutation from the documented order")


def _rejected(got, prods, typ, ordered):
    keys, a, b = prods
    with pytest.raises(AssertionError):
        check_fp(np.unique(keys), got, keys, a, b, typ, "mutated", ordered)


@pytest.mark.parametrize("scale", ["normal", "subnormal"])
@pytest.mark.parametrize("typ", FP_T)
def test_the_documented_order_passes(typ, scale):
    Sv, x, (keys, a, b), ordered = _long_row(typ, scale, 0)
    assert check_fp(ordered[0], ordered[1], keys, a, b, typ, "order", ordered) <= 4 * LONG
    assert check_fp(ordered[0], ordered[1], keys, a, b, typ, "bound only") >= 0


@pytest.mark.parametrize("typ", FP_T)
def test_order_differs_from_a_plain_left_to_right_fold(typ):
    def differs(Sv, x, prods, ordered):
        return not np.array_equal(_bits(ltr_fold(*prods, typ)[1]), _bits(ordered[1]))
    Sv, x, prods, ordered = _first(differs, typ, "normal")
    _rejected(ltr_fold(*prods, typ)[1], prods, typ, ordered)


def _round(fr, dt):
    """A Fraction correctly rounded to dt (ties to even)."""
    c = dt.type(float(fr))                   # float(Fraction) is correctly rounded to float64; FP32 can be one ulp off after it
    cands = [c, np.nextafter(c, dt.type(np.inf)), np.nextafter(c, dt.type(-np.inf))]
    return min(cands, key=lambda v: (abs(Fraction(float(v)) - fr), int(_bits(np.asarray([v]))[0]) & 1))


def _fma_fold(Sv, x, typ):
    """The documented order with every multiply-add contracted: inside a segment acc = fma(a, x, acc), the exact a x + acc rounded
    once per step to typ; the segment partials through tree_fold as before."""
    dt = np.dtype(orc.DTYPES[typ])
    out = []
    for r in range(Sv.shape[0]):
        idx = np.arange(Sv.indptr[r], Sv.indptr[r + 1])
        segs = [idx] if len(idx) <= SEG else [idx[s:s + SEG] for s in range(0, len(idx), SEG)]
        parts = []
        for seg in segs:
            acc = None
            for e in seg:
                p = Fraction(float(Sv.data[e])) * Fraction(float(x[Sv.indices[e], 0]))
                acc = _round(p if acc is None else Fraction(float(acc)) + p, dt)
            parts.append((acc, acc is not None))
        out.append(tree_fold(parts, lambda p, q: dt.type(p + q))[0])
    return np.asarray(out, dt)


@pytest.mark.parametrize("typ", FP_T)
def test_fused_multiply_add_fold_is_rejected(typ):
    def differs(Sv, x, prods, ordered):
        return not np.array_equal(_bits(_fma_fold(Sv, x, typ)), _bits(ordered[1]))
    Sv, x, prods, ordered = _first(differs, typ, "normal")
    _rejected(_fma_fold(Sv, x, typ), prods, typ, ordered)


def _ftz(v):
    dt = np.asarray(v).dtype
    return dt.type(0) if v != 0 and abs(v) < np.finfo(dt).tiny else v


def _flushed(Sv, x, typ):
    dt = orc.DTYPES[typ]
    k, v = [], []
    for r in range(Sv.shape[0]):
        cols = Sv.indices[Sv.indptr[r]:Sv.indptr[r + 1]]
        val, has = chunked_dot(np.asarray(Sv.data[Sv.indptr[r]:Sv.indptr[r + 1]], dt), x[cols, 0].astype(dt),
                               add=lambda p, q: _ftz(np.add(p, q)), mul=lambda p, q: _ftz(np.multiply(p, q)))
        if has:
            k.append(r); v.append(val)
    return np.asarray(v, dt)


@pytest.mark.parametrize("typ", FP_T)
def test_flush_to_zero_is_rejected(typ):
    def differs(Sv, x, prods, ordered):
        return not np.array_equal(_bits(_flushed(Sv, x, typ)), _bits(ordered[1]))
    Sv, x, prods, ordered = _first(differs, typ, "subnormal")
    _rejected(_flushed(Sv, x, typ), prods, typ, ordered)


def _swapped_segments(Sv, x, typ):
    """The long row with its second and third segments exchanged: the same partials, folded as ((s0 s2) (s1 s3))."""
    dt = orc.DTYPES[typ]
    out = []
    for r in range(Sv.shape[0]):
        idx = np.arange(Sv.indptr[r], Sv.indptr[r + 1])
        if len(idx) > 3 * SEG:
            idx = np.concatenate([idx[:SEG], idx[2 * SEG:3 * SEG], idx[SEG:2 * SEG], idx[3 * SEG:]])
        out.append(chunked_dot(np.asarray(Sv.data[idx], dt), x[Sv.indices[idx], 0].astype(dt))[0])
    return np.asarray(out, dt)


@pytest.mark.parametrize("typ", FP_T)
def test_neighbouring_segment_order_is_rejected(typ):
    def differs(Sv, x, prods, ordered):
        return not np.array_equal(_bits(_swapped_segments(Sv, x, typ)), _bits(ordered[1]))
    Sv, x, prods, ordered = _first(differs, typ, "normal")
    _rejected(_swapped_segments(Sv, x, typ), prods, typ, ordered)
    # the tree itself: four partials join as ((s0 s1) (s2 s3))
    assert tree_fold([(f"{i}", True) for i in range(4)], lambda p, q: f"({p}{q})")[0] == "((01)(23))"


@pytest.mark.parametrize("scale", ["normal", "subnormal"])
@pytest.mark.parametrize("typ", FP_T)
def test_one_ulp_beyond_the_bound_is_rejected(typ, scale):
    """The routes held to the bound only (spa, spa-split): a result just inside the bound passes, one ulp beyond it does not."""
    dt = orc.DTYPES[typ]
    Sv, x, (keys, a, b), ordered = _long_row(typ, scale, 1)
    hp = np.float64 if typ == "FP32" else np.longdouble
    uk, inv = np.unique(keys, return_inverse=True)
    prod = a.astype(hp) * b.astype(hp)
    exact = np.zeros(len(uk), hp); np.add.at(exact, inv, prod)
    mag = np.zeros(len(uk), hp); np.add.at(mag, inv, np.abs(prod))
    n = np.bincount(inv).astype(np.float64) + 1
    u = float(np.finfo(dt).eps) / 2
    bound = (n * u / (1 - n * u)).astype(hp) * mag + n.astype(hp) * (hp(np.finfo(dt).smallest_subnormal) / 2)
    inside = (exact + bound).astype(dt)
    while (np.abs(inside.astype(hp) - exact) > bound).any():
        bad = np.abs(inside.astype(hp) - exact) > bound
        inside[bad] = np.nextafter(inside[bad], exact[bad].astype(dt))
    check_fp(uk, inside, keys, a, b, typ, "inside")
    beyond = inside.copy()
    while not (np.abs(beyond.astype(hp) - exact) > bound).all():
        ok = np.abs(beyond.astype(hp) - exact) <= bound
        beyond[ok] = np.nextafter(beyond[ok], dt(np.inf))
    assert (util.ulps(beyond, inside) <= 1).all()
    for i in range(len(uk)):
        one = inside.copy()
        one[i] = beyond[i]
        with pytest.raises(AssertionError):
            check_fp(uk, one, keys, a, b, typ, "beyond")
