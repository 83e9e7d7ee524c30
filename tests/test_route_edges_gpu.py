"""The mxm routes added after tests/test_value_edges_gpu.py, against the oracle at the edges of each type and their FP sums against an
exact reference: SpMM with a dense right operand and with a dense left operand (spmm.cu), the sampled dense-dense product
(sddmm.cu), mxm under a complemented mask (the esc / spa / spa-split bins of spgemm.cu) and hypersparse operands (hyper.cu).

Each entry of ROUTES forces one route through the operands' form and shape and the descriptor, and asserts it through
B200_debug_last_kernel.  Every route gets four checks:

* The edge table: every (add, mul) of test_value_edges_gpu.semirings() on all 11 types (the left route also every multiply that
  op_mirror swaps), with kernel_check's value pools, against the oracle through kernel_check.compare: BOOL and integer results bit
  for bit, NaN matches NaN, +-0 match under MIN / MAX, an ANY value must be one of the entry's products.
* Mixed types: the MIXED rows of test_value_edges_gpu, plus a mirrored multiply and casts that saturate into C.
* FP PLUS_TIMES at general values (random mantissas, exponents over 2^+-6, also scaled into the subnormal range), against the
  exact sum of each entry's products (FP32: products exact in float64, math.fsum; FP64: TwoProduct by Veltkamp's split, then
  math.fsum; fractions.Fraction where a product is too small for the split).  Every route stays within check_bound's gamma_n
  bound.  The routes whose fold order is documented equal a Python restatement of it bit for bit: SpMM right and left (left to
  right up to SPMM_SEG entries of the sparse operand's row, tree_fold over the segments, products with an absent dense entry
  skipped) and SDDMM (chunked_dot).  esc-small and esc-medium fold the products of a column in their Gustavson position order,
  from the first product on (spgemm.cu's compress step): that is the oracle's left-to-right fold over k, so they are held to
  that order bit for bit as well.  Hypersparse results equal the same tuples computed in a small sized space, bit for bit.
  Routes without atomics (spmm, sddmm, esc, and the hypersparse calls that land on them) give the same bits on a second run; spa
  and spa-split combine with atomics and are held to the bound only.
* A ledger: test_every_route_was_reached.

The largest error against the exact reference, in ulps of the rounded exact sum, is kept per route in MAX_ULP and printed by the
ledger."""
import functools
import math
from fractions import Fraction

import numpy as np
import pytest
import scipy.sparse as sp

from pygraphblas_b200 import Matrix, Vector, descriptor
from oracle import oracle as orc
import util
from kernel_check import (_bits, compare, entries, full_count, o_csr, products_by_entry, record_kernels, seed_of, semiring,
                          values, vec_products)
from test_value_edges_gpu import MIXED, _expand, _general_values, check_bound, semirings
from test_sddmm import SEG, chunked_dot
from test_dense_gpu import FAST, g_dense, o_dense
from test_dense_left_gpu import new_semiring
from test_complement_mxm_gpu import MEDIUM, blocked_pattern, mask_shapes, mask_vals, product_pattern, route as comp_route

pytestmark = pytest.mark.gpu

ALL_T, FP_T = util.ALL_T, util.FP_T
REACHED = set()
MAX_ULP = {}


def _kernels():
    return record_kernels(REACHED)


# ------------------------------------------------------------------ exact sums and the documented fold orders (pure numpy)
def _veltkamp(a):
    c = a * 134217729.0                         # 2^27 + 1
    hi = c - (c - a)
    return hi, a - hi


def two_product(a, b):
    """(p, e) with p + e == a * b exactly, p = fl(a * b), for float64 a, b whose product neither overflows nor comes near the
    subnormal range (|a b| >= 2^-969, |a|, |b| < 2^995)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    p = a * b
    ah, al = _veltkamp(a)
    bh, bl = _veltkamp(b)
    e = ((ah * bh - p) + ah * bl + al * bh) + al * bl
    return p, e


def exact_sums(keys, a, b, typ):
    """The sum of the products a * b of each key, correctly rounded to float64: (sorted unique keys, sums).  FP32 products are exact
    in float64; FP64 products are split into p + e by two_product, or summed as Fractions where a product is too small for the
    split."""
    keys = np.asarray(keys, np.int64)
    order = np.argsort(keys, kind="stable")
    keys, a64, b64 = keys[order], np.asarray(a, np.float64)[order], np.asarray(b, np.float64)[order]
    uk, start = np.unique(keys, return_index=True)
    bounds = list(start) + [len(keys)]
    if typ == "FP32":
        terms, small = [a64 * b64], np.zeros(len(keys), bool)
    else:
        p, e = two_product(a64, b64)
        terms, small = [p, e], (np.abs(p) < 2.0 ** -969) & (a64 != 0) & (b64 != 0)
    out = np.empty(len(uk))
    for g in range(len(uk)):
        lo, hi = bounds[g], bounds[g + 1]
        if small[lo:hi].any():
            out[g] = float(sum((Fraction(float(x)) * Fraction(float(y)) for x, y in zip(a64[lo:hi], b64[lo:hi])), Fraction(0)))
        else:
            out[g] = math.fsum(np.concatenate([t[lo:hi] for t in terms]).tolist())
    return uk, out


def max_ulp(got, exact, typ):
    """The largest distance of got from the exact sums rounded to typ, in ulps (FP32 rounds through float64: it can differ from
    the correctly rounded FP32 value only on a double-rounding tie, enough for an ulp count)."""
    want = np.asarray(exact).astype(orc.DTYPES[typ])
    return float(util.ulps(np.asarray(got, orc.DTYPES[typ]), want).max()) if len(want) else 0.0


def ltr_fold(keys, a, b, typ):
    """The left-to-right fold of each key's products in the order given (the oracle's Gustavson order, esc's position order),
    from the first product on, every operation rounded to typ.  Returns (sorted unique keys, values)."""
    dt = orc.DTYPES[typ]
    keys = np.asarray(keys, np.int64)
    order = np.argsort(keys, kind="stable")
    k, z = keys[order], (np.asarray(a, dt) * np.asarray(b, dt))[order]
    uk, start, cnt = np.unique(k, return_index=True, return_counts=True)
    acc = z[start].copy()
    for t in range(1, int(cnt.max()) if len(cnt) else 0):
        g = np.flatnonzero(cnt > t)
        acc[g] = (acc[g] + z[start[g] + t]).astype(dt)
    return uk, acc


def spmm_order(S, x, xp, typ):
    """T = S (+).(x) X (S CSR m x n with its values, X n x k dense, xp its presence or None) in the SpMM kernel's order: row r's
    entries in column order, cut into segments of SEG entries when the row is longer than SEG, each segment folded left to right
    from its first present product, the partials through tree_fold.  Returns (keys r * k + j, values) of the present results."""
    dt = orc.DTYPES[typ]
    m, k = S.shape[0], x.shape[1]
    keys, vals = [], []
    for r in range(m):
        cols = S.indices[S.indptr[r]:S.indptr[r + 1]]
        av = np.asarray(S.data[S.indptr[r]:S.indptr[r + 1]], dt)
        for j in range(k):
            v, has = chunked_dot(av, x[cols, j].astype(dt), yp=None if xp is None else xp[cols, j])
            if has:
                keys.append(r * k + j); vals.append(v)
    return np.asarray(keys, np.int64), np.asarray(vals, dt)


def left_order(x, xp, S, typ):
    """T = X (+).(x) S (X k x n dense, S CSR n x m): the left route runs T' = S' (+).(x)' X' on the SpMM kernel, so T(r, c) folds the
    entries of column c of S in row order, in segments of SEG entries."""
    St = S.T.tocsr()
    St.sort_indices()
    kT, vT = spmm_order(St, np.ascontiguousarray(x.T), None if xp is None else np.ascontiguousarray(xp.T), typ)
    m, k = St.shape[0], x.shape[0]
    c, r = np.divmod(kT, k)
    keys = r * m + c
    o = np.argsort(keys)
    return keys[o], vT[o]


def sddmm_order(x, xp, y, yp, mkeys, n, typ):
    """T<M>(i, j) = chunked_dot(X(i, :), Y(j, :)) at the mask positions mkeys = i * n + j (X m x d, Y n x d)."""
    dt = orc.DTYPES[typ]
    keys, vals = [], []
    for key in np.asarray(mkeys, np.int64):
        i, j = divmod(int(key), n)
        v, has = chunked_dot(x[i].astype(dt), y[j].astype(dt), xp=None if xp is None else xp[i], yp=None if yp is None else yp[j])
        if has:
            keys.append(key); vals.append(v)
    return np.asarray(keys, np.int64), np.asarray(vals, dt)


def check_fp(gK, gX, keys, a, b, typ, label, ordered=None):
    """The FP check of every route: presence and check_bound's gamma_n bound against the products (keys, a, b), and, when the
    route's order is documented, the bits of `ordered` = (keys, values) of its restatement.  Returns the largest ulp error
    against the exact sum."""
    check_bound(gK, gX, keys, a, b, typ, label)
    gX = np.asarray(gX, orc.DTYPES[typ])
    if ordered is not None:
        oK, oX = ordered
        assert np.array_equal(np.asarray(gK, np.int64), oK), f"{label}: presence differs from the restated order"
        bad = np.flatnonzero(_bits(gX) != _bits(np.asarray(oX, gX.dtype)))
        assert len(bad) == 0, (f"{label}: {len(bad)} of {len(oK)} values differ from the documented fold order, e.g. got "
                               f"{gX[bad[:3]].tolist()}, order {np.asarray(oX)[bad[:3]].tolist()}")
    _, exact = exact_sums(keys, a, b, typ)
    return max_ulp(gX, exact, typ)


# ------------------------------------------------------------------ operands
def lens_csr(lens, ncols, seed):
    """A sorted CSR pattern whose row r has lens[r] distinct random columns."""
    rng = np.random.default_rng(seed)
    cols = [np.sort(rng.choice(ncols, int(L), replace=False)) for L in lens]
    indptr = np.r_[0, np.cumsum(lens)].astype(np.int64)
    S = sp.csr_matrix((np.ones(int(indptr[-1])), np.concatenate(cols).astype(np.int32) if cols else np.zeros(0, np.int32), indptr),
                      shape=(len(lens), ncols))
    S.sort_indices()
    return S


def with_data(S, v):
    T = S.copy()
    T.data = np.asarray(v)
    return T


def private_columns(S):
    """S with one more column per row: row k gets column S.ncols + k, which no other row has.  As the right operand of A B, each
    entry A(i, k) then reaches one output column, (i, S.ncols + k), with exactly one product."""
    T = sp.hstack([S, sp.identity(S.shape[0], format="csr")], format="csr")
    T.sort_indices()
    return T


def partial_mask(SA, SB, seed):
    """A mask over A B that holds a random half of every row's product columns and as many columns without a product: the
    complement blocks part of every row and leaves the rest."""
    P = product_pattern(SA, SB)
    rng = np.random.default_rng(seed)
    rows = []
    for i in range(P.shape[0]):
        pc = P.indices[P.indptr[i]:P.indptr[i + 1]]
        miss = np.setdiff1d(np.arange(P.shape[1]), pc)
        rows.append(np.union1d(rng.choice(pc, len(pc) // 2, replace=False), rng.choice(miss, min(len(miss), len(pc) // 2), replace=False)))
    return lens_csr_of(rows, P.shape[1])


def lens_csr_of(rows, ncols):
    lens = [len(r) for r in rows]
    S = sp.csr_matrix((np.ones(sum(lens)), np.concatenate(rows).astype(np.int32), np.r_[0, np.cumsum(lens)]), shape=(len(rows), ncols))
    S.sort_indices()
    return S


def lone_products(SA, SB):
    """The output keys i * ncols + j of the rows above MEDIUM products (the spa and spa-split rows) that exactly one product
    reaches: there the accumulator's start value meets a single product."""
    n = SB.shape[1]
    Ar = np.repeat(np.arange(SA.shape[0], dtype=np.int64), np.diff(SA.indptr))
    keys, _, _ = _expand(Ar, SA.indices.astype(np.int64), np.ones(SA.nnz), SB.indptr, SB.indices, np.ones(SB.nnz), n)
    uk, cnt = np.unique(keys, return_counts=True)
    f = np.bincount(Ar, weights=np.diff(SB.indptr)[SA.indices], minlength=SA.shape[0])
    return uk[(cnt == 1) & (f[uk // n] > MEDIUM)]


SPLIT_LENS = [0, 1, SEG - 1, SEG, SEG + 1, 2 * SEG, 2 * SEG + 1, 3 * SEG - 1, 3 * SEG + 5, 17]
HOLE_ROW = 8                        # its second segment (entries SEG .. 2 SEG - 1) has every X entry absent


# Each route: operand forms (("csr", pattern) or ("dense", rows, cols, presence or None)), the mask (None, ("csr", pattern, mask
# type or None for structural), ("dense", presence, type)), the descriptor, and the seam tokens it must show.
@functools.lru_cache(maxsize=None)
def route_operands(name):
    rng = np.random.default_rng(seed_of("route", name))
    pres = lambda r, c, d: (rng.random((r, c)) < d).astype(np.uint8)
    if name == "spmm-k1-dense-mask":
        S = lens_csr(rng.integers(0, SEG + 1, 40), 300, 1)
        return dict(A=("csr", S), B=("dense", 300, 1, None), M=("dense", pres(40, 1, 0.7), "FP32"), desc="")
    if name == "spmm-split-k33":
        S = lens_csr(SPLIT_LENS, 400, 2)
        xp = pres(400, 33, 0.7)
        hole = S.indices[S.indptr[HOLE_ROW] + SEG:S.indptr[HOLE_ROW] + 2 * SEG]
        xp[hole, :] = 0
        return dict(A=("csr", S), B=("dense", 400, 33, xp), M=None, desc="")
    if name == "spmm-split-csr-mask":
        S = lens_csr(SPLIT_LENS, 400, 3)
        return dict(A=("csr", S), B=("dense", 400, 33, None), M=("csr", lens_csr(rng.integers(0, 34, 10), 33, 4), "BOOL"), desc="")
    if name == "left":               # X 9 x 400 with presence, B 400 x 10 whose columns straddle SEG
        B = lens_csr(SPLIT_LENS, 400, 5).T.tocsr()
        B.sort_indices()
        return dict(A=("dense", 9, 400, pres(9, 400, 0.8)), B=("csr", B), M=None, desc="")
    if name == "left-k1-csr-mask":
        B = lens_csr(SPLIT_LENS, 400, 6).T.tocsr()
        B.sort_indices()
        return dict(A=("dense", 1, 400, None), B=("csr", B), M=("csr", lens_csr([7], 10, 7), "INT8"), desc="")
    if name == "left-T0-m1":          # X given n x k (INP0 = TRAN), B one column of 3 SEG + 5 entries
        B = lens_csr([3 * SEG + 5], 250, 8).T.tocsr()
        B.sort_indices()
        return dict(A=("dense", 250, 5, pres(250, 5, 0.7)), B=("csr", B), M=None, desc="T0")
    if name == "sddmm-d33":
        return dict(A=("dense", 37, 33, None), B=("dense", 29, 33, None), M=("csr", lens_csr(rng.integers(0, 12, 37), 29, 9), None),
                    desc="ST1")
    if name == "sddmm-d130-pres":
        return dict(A=("dense", 23, 130, pres(23, 130, 0.7)), B=("dense", 19, 130, pres(19, 130, 0.85)),
                    M=("csr", lens_csr(rng.integers(0, 10, 23), 19, 10), "INT8"), desc="T1")
    if name == "sddmm-y-transpose":  # Y given d x n (no INP1 = TRAN): the kernel reads its dense transpose
        return dict(A=("dense", 31, 40, None), B=("dense", 40, 27, pres(40, 27, 0.9)),
                    M=("csr", lens_csr(rng.integers(0, 9, 31), 27, 11), None), desc="S")
    if name in ("comp-bins-struct", "comp-bins-valued"):
        # B rows of 3 entries over 64 shared columns and one private column: row r of A has 4 lens[r] products, about lens[r] / 21
        # per shared column and one in each private column it reaches; 4, 80, 128 | 132, 1200, 2048 | 2052, 3600 products:
        # esc-small, esc-medium and spa rows.  mask_shapes' pattern covers none of row 4, all of rows 5 and 6, part of row 7 (spa)
        SA = lens_csr([1, 20, 32, 33, 300, 512, 513, 900], 1000, 12)
        SB = private_columns(lens_csr([3] * 1000, 64, 13))
        return dict(A=("csr", SA), B=("csr", SB), M=("csr", mask_shapes(SA, SB, 14), None if name.endswith("struct") else "INT8"),
                    desc="SC" if name.endswith("struct") else "C")
    if name in ("comp-split", "comp-split-valued"):
        # B rows of 512 entries over 2048 shared columns and one private column: row 0 of A has 513 x 513 = 263169 > SPLIT_FLOPS
        # products (spa-split), about 128 per shared column and one in each of its 513 private columns; row 1 has 3 x 513 = 1539
        # (esc-medium).  The mask blocks part of both rows
        SA = lens_csr([513, 3], 513, 15)
        SB = private_columns(lens_csr([512] * 513, 2048, 16))
        valued = name.endswith("valued")
        return dict(A=("csr", SA), B=("csr", SB), M=("csr", partial_mask(SA, SB, 17), "INT8" if valued else None),
                    desc="C" if valued else "SC")
    raise KeyError(name)


ROUTES = {
    # name: (the tokens the seam must show, the fold order of its FP sums)
    "spmm-k1-dense-mask": (["spmm", "write=dense"], "spmm"),
    "spmm-split-k33": (["spmm", "spmm-split", "write=dense"], "spmm"),
    "spmm-split-csr-mask": (["spmm", "spmm-split", "write=csr"], "spmm"),
    "left": (["spmm", "spmm-left", "x-transpose", "t-transpose", "spmm-split", "write=dense"], "left"),
    "left-k1-csr-mask": (["spmm", "spmm-left", "t-transpose", "spmm-split", "write=csr"], "left"),
    "left-T0-m1": (["spmm", "spmm-left", "spmm-split", "write=dense"], "left"),
    "sddmm-d33": (["sddmm", "pattern=mask"], "sddmm"),
    "sddmm-d130-pres": (["sddmm", "pattern=compact"], "sddmm"),
    "sddmm-y-transpose": (["sddmm"], "sddmm"),
    "comp-bins-struct": (None, "esc"),
    "comp-bins-valued": (None, "esc"),
    "comp-split": (None, "esc"),
    "comp-split-valued": (None, "esc"),
}
ABSENT = {"spmm-k1-dense-mask": ["spmm-split", "spmm-left"], "spmm-split-k33": ["spmm-left"], "left-k1-csr-mask": ["x-transpose"],
          "left-T0-m1": ["x-transpose", "t-transpose"], "sddmm-d33": ["x-transpose", "y-transpose"]}
FAST_SET = set(FAST)


def expect_route(name, t, sr, SA=None, SB=None, blocks=True, homogeneous=True):
    want, _ = ROUTES[name]
    if want is None:                 # the complemented bins, by the product count of each row
        assert entries(t) == comp_route(SA, SB, blocks), (name, sr, t)
        return
    for tok in want:
        assert tok in t, (name, sr, tok, t)
    for tok in ABSENT.get(name, []):
        assert tok not in t, (name, sr, tok, t)
    kind = "sddmm" if name.startswith("sddmm") else "spmm"
    assert (f"{kind}-fast" in t) != (f"{kind}-generic" in t), (name, sr, t)
    if homogeneous:
        assert (f"{kind}-fast" in t) == (tuple(sr) in FAST_SET), (name, sr, t)
    if name == "sddmm-y-transpose":
        assert "y-transpose" in t, (name, sr, t)             # Y has absent entries: transposed even when the multiply ignores it


def _size(spec):
    return spec[1].nnz if spec[0] == "csr" else spec[1] * spec[2]


def _dev(spec, typ, v):
    if spec[0] == "csr":
        S = spec[1]
        return Matrix.from_csr(S.indptr, S.indices, v, *S.shape, util.g_type(typ))
    return g_dense(typ, np.asarray(v).reshape(spec[1], spec[2]), spec[3])


def _orc(spec, typ, v):
    if spec[0] == "csr":
        return o_csr(typ, spec[1], np.asarray(v))
    return o_dense(typ, np.asarray(v).reshape(spec[1], spec[2]), spec[3])


def _mask(ops, seed):
    M = ops["M"]
    if M is None:
        return None, None, None
    if M[0] == "dense":
        mp, mt = M[1], M[2]
        mv = mask_vals(mt, mp.size, seed).reshape(mp.shape)
        return g_dense(mt, mv, mp), o_dense(mt, mv, mp), None
    S, mt = M[1], M[2]
    mv = np.ones(S.nnz, bool) if mt is None else mask_vals(mt, S.nnz, seed)
    mt = mt or "BOOL"
    return Matrix.from_csr(S.indptr, S.indices, mv, *S.shape, util.g_type(mt)), o_csr(mt, S, mv), mv


def _eff(o, tran):
    """An oracle matrix as a CSR (indptr, indices, values) of op(o), its values in their CSR order."""
    I, J, X = np.asarray(o.I, np.int64), np.asarray(o.J, np.int64), np.asarray(o.X)
    nr, nc = o.nrows, o.ncols
    if tran:
        I, J, nr, nc = J, I, nc, nr
    order = np.lexsort((J, I))
    I, J, X = I[order], J[order], X[order]
    return np.r_[0, np.cumsum(np.bincount(I, minlength=nr))].astype(np.int64), J, X, nr, nc


def products(oa, ob, desc):
    """(keys i * ncols + j, a, b) of every product of op(A) op(B), in Gustavson order, and ncols."""
    Ap, Ac, Av, m, _ = _eff(oa, "T0" in desc)
    Bp, Bc, Bv, _, n = _eff(ob, "T1" in desc)
    Ar = np.repeat(np.arange(m, dtype=np.int64), np.diff(Ap))
    keys, a, b = _expand(Ar, Ac, Av, Bp, Bc, Bv, n)
    return keys, a, b, n


def any_candidates(oa, ob, desc, mul):
    Ap, Ac, Av, m, _ = _eff(oa, "T0" in desc)
    Bp, Bc, Bv, _, n = _eff(ob, "T1" in desc)
    return products_by_entry(np.repeat(np.arange(m, dtype=np.int64), np.diff(Ap)), Ac, Av, Bp, Bc, Bv, n, mul)


def keyed(C):
    I, J, X = C.to_arrays()
    return np.asarray(I, np.int64) * C.ncols + np.asarray(J, np.int64), X


def _blocks(ops, mv):
    M = ops["M"]
    return len(blocked_pattern(M[1], mv, M[2] is None or "S" in ops["desc"])) > 0


def left_extras(typ):
    """The multiplies op_mirror swaps that semirings() leaves out: the comparisons (LOR monoid) and the IS* operators."""
    if typ == "BOOL":
        return [("LOR", m, typ) for m in ("GT", "LT", "GE", "LE")]
    return [("LOR", m, typ) for m in ("GT", "LT", "GE", "LE")] + [("PLUS", m, typ) for m in ("ISGT", "ISLT", "ISGE", "ISLE")]


def _sr_handle(sr):
    if sr[1] in ("GT", "LT", "GE", "LE", "ISGT", "ISLT", "ISGE", "ISLE"):
        return new_semiring(sr[0], sr[1], sr[2], orc.semiring_ztype(sr))
    return semiring(*sr)


# ------------------------------------------------------------------ 1. the edge table
def run_route_edges(name, typ):
    ops = route_operands(name)
    desc = ops["desc"]
    groups = semirings(typ)
    if name.startswith("left"):
        groups = groups + [("edge", left_extras(typ))]
    comp = ops["A"][0] == "csr" and ops["B"][0] == "csr"
    if comp:
        lone = lone_products(ops["A"][1], ops["B"][1])
        assert len(lone) > 0, name
    errors, calls = [], 0
    for pool, srs in groups:
        seed = seed_of(name, typ, pool)
        av = values(seed, typ, _size(ops["A"]), pool, 0)
        bv = values(seed + 1, typ, _size(ops["B"]), pool, 1)
        A, B = _dev(ops["A"], typ, av), _dev(ops["B"], typ, bv)
        oa, ob = _orc(ops["A"], typ, av), _orc(ops["B"], typ, bv)
        M, Mo, mv = _mask(ops, seed + 2)
        for sr in srs:
            zt = orc.semiring_ztype(sr)
            m = oa.ncols if "T0" in desc else oa.nrows
            n = ob.nrows if "T1" in desc else ob.ncols
            C = Matrix.sparse(util.g_type(zt), m, n)
            A.mxm(B, semiring=_sr_handle(sr), out=C, mask=M, desc=getattr(descriptor, desc) if desc else None)
            t = _kernels()
            calls += 1
            if ops["A"][0] == "csr" and ops["B"][0] == "csr":
                expect_route(name, t, sr, ops["A"][1], ops["B"][1], _blocks(ops, mv))
            else:
                expect_route(name, t, sr)
            gK, gX = keyed(C)
            ref = orc.mxm(orc.SpMat(zt, m, n), Mo, None, sr, oa, ob, desc)
            rK = ref.I.astype(np.int64) * n + ref.J.astype(np.int64)
            cands = any_candidates(oa, ob, desc, sr[1]) if sr[0] == "ANY" else None
            if comp:
                _lone_specials(name, sr, lone, oa, ob, desc, rK)
            e = compare(gK, gX, rK, ref.X, zt, sr[0], f"{name} {'_'.join(sr)}", cands)
            if e:
                errors.append(e)
    assert calls > 0
    assert not errors, f"{len(errors)} of {calls} calls differ on {name}:\n" + "\n".join(errors[:40])


def _lone_specials(name, sr, lone, oa, ob, desc, rK):
    """In the spa / spa-split rows, some entry the mask lets through has a single product, and for FP MIN / MAX / PLUS with the
    TIMES multiply, that sole product is NaN (MIN / MAX) or -0.0 (PLUS) somewhere: the accumulator's start value (accum_init)
    decides such an entry on its own."""
    kept = np.intersect1d(lone, rK)
    assert len(kept) > 0, (name, sr, "no single-product entry of a spa / spa-split row survives the mask")
    if sr[2] not in FP_T or sr[1] != "TIMES" or sr[0] not in ("MIN", "MAX", "PLUS"):
        return
    keys, a, b, _ = products(oa, ob, desc)
    sel = np.isin(keys, kept)
    with np.errstate(all="ignore"):
        z = a[sel] * b[sel]
    if sr[0] == "PLUS":
        assert ((z == 0) & np.signbit(z)).any(), (name, sr, "no -0.0 as the sole product of an entry")
    else:
        assert np.isnan(z).any(), (name, sr, "no NaN as the sole product of an entry")


@pytest.mark.parametrize("typ", ALL_T)
@pytest.mark.parametrize("name", list(ROUTES))
def test_route_edges(name, typ):
    run_route_edges(name, typ)


# ------------------------------------------------------------------ hypersparse operands
HYPER = 1 << 60
HYPER_IDS = np.array([0, 1, 7, (1 << 31) + 1, (1 << 31) + 2, (1 << 31) + 5, (1 << 40) + 3, HYPER - 2, HYPER - 1], np.uint64)


@functools.lru_cache(maxsize=None)
def hyper_operands(form):
    """Tuples over HYPER_IDS (ids 0, just above 2^31 and 2^60 - 1 included).  mxv / vxm: A 9 x 9 dense-ish, u sparse; mxm: A and B,
    and for "mxm-comp" a complemented mask."""
    rng = np.random.default_rng(seed_of("hyper", form))
    ni = len(HYPER_IDS)

    def pattern(nr, nc, d):
        P = rng.random((nr, nc)) < d
        P[0, 0] = P[-1, -1] = P[-1, 0] = True
        return np.nonzero(P)

    out = dict(A=pattern(ni, ni, 0.7))
    if form in ("mxv", "vxm"):
        out["u"] = np.flatnonzero(rng.random(ni) < 0.8)
    else:
        out["B"] = pattern(ni, ni, 0.6)
        if form == "mxm-comp":
            out["M"] = pattern(ni, ni, 0.3)
    return out


def _hyper_call(form, typ, sr, av, bv, mv, big, accum=None, ctyp=None, c_init=None):
    """The call in the 2^60 space (big) or in the 9-id space; returns (keys as (i, j) rank pairs, values, tokens).  c_init: the
    entries w / C holds before the call, (ranks, values) for a vector, (row ranks, column ranks, values) for a matrix."""
    ops = hyper_operands(form)
    ids = HYPER_IDS if big else np.arange(len(HYPER_IDS), dtype=np.uint64)
    dim = HYPER if big else len(HYPER_IDS)
    gt = util.g_type(typ)
    zt = ctyp or orc.semiring_ztype(sr)
    ai, aj = ops["A"]
    A = Matrix.from_lists(ids[ai], ids[aj], av, dim, dim, gt)
    s = _sr_handle(sr)
    acc = util.g_accum(accum)
    if form in ("mxv", "vxm"):
        u = Vector.from_lists(ids[ops["u"]], bv, dim, gt)
        w = Vector.sparse(util.g_type(zt), dim) if c_init is None else Vector.from_lists(ids[c_init[0]], c_init[1], dim, util.g_type(zt))
        (A.mxv(u, semiring=s, out=w, accum=acc) if form == "mxv" else u.vxm(A, semiring=s, out=w, accum=acc))
        t = _kernels()
        I, X = w.to_arrays()
        return np.searchsorted(ids, np.asarray(I, np.uint64)).astype(np.int64), X, t
    bi, bj = ops["B"]
    B = Matrix.from_lists(ids[bi], ids[bj], bv, dim, dim, gt)
    M = None
    if "M" in ops:
        mi, mj = ops["M"]
        M = Matrix.from_lists(ids[mi], ids[mj], mv, dim, dim, util.g_type("BOOL"))
    C = (Matrix.sparse(util.g_type(zt), dim, dim) if c_init is None else
         Matrix.from_lists(ids[c_init[0]], ids[c_init[1]], c_init[2], dim, dim, util.g_type(zt)))
    A.mxm(B, semiring=s, out=C, mask=M, accum=acc, desc=descriptor.C if M is not None else None)
    t = _kernels()
    I, J, X = C.to_arrays()
    n = len(HYPER_IDS)
    return (np.searchsorted(ids, np.asarray(I, np.uint64)).astype(np.int64) * n +
            np.searchsorted(ids, np.asarray(J, np.uint64)).astype(np.int64)), X, t


def _hyper_oracle(form, typ, sr, av, bv, mv):
    ops = hyper_operands(form)
    n = len(HYPER_IDS)
    zt = orc.semiring_ztype(sr)
    ai, aj = ops["A"]
    oa = orc.SpMat(typ, n, n, ai, aj, av)
    if form in ("mxv", "vxm"):
        ou = orc.SpVec(typ, n, ops["u"], bv)
        if form == "mxv":
            ref = orc.mxv(orc.SpVec(zt, n), None, None, sr, oa, ou)
        else:
            ref = orc.vxm(orc.SpVec(zt, n), None, None, sr, ou, oa)
        return ref.I.astype(np.int64), ref.X, oa, ou
    bi, bj = ops["B"]
    ob = orc.SpMat(typ, n, n, bi, bj, bv)
    om = None
    if "M" in ops:
        mi, mj = ops["M"]
        om = orc.SpMat("BOOL", n, n, mi, mj, mv)
    ref = orc.mxm(orc.SpMat(zt, n, n), om, None, sr, oa, ob, "C" if om is not None else "")
    return ref.I.astype(np.int64) * n + ref.J.astype(np.int64), ref.X, oa, ob


HYPER_FORMS = ["mxv", "vxm", "mxm", "mxm-comp"]


def _hyper_expect(form, t):
    e = entries(t)
    if form == "mxm-comp":
        assert any(k.startswith("esc-") for k in e), t
    elif form == "mxm":
        assert any(k.startswith("esc-") or k == "spa" for k in e), t
    else:
        assert any(k.startswith("run") for k in e), t
    REACHED.add(f"hyper-{form}")


def _hyper_values(form, typ, pool, seed):
    ops = hyper_operands(form)
    av = values(seed, typ, len(ops["A"][0]), pool, 0)
    bv = values(seed + 1, typ, len(ops["u"]) if "u" in ops else len(ops["B"][0]), pool, 1)
    mv = mask_vals("BOOL", len(ops["M"][0]), seed + 2) if "M" in ops else None
    return av, bv, mv


@pytest.mark.parametrize("typ", ALL_T)
@pytest.mark.parametrize("form", HYPER_FORMS)
def test_hyper_edges(form, typ):
    """The edge table on 2^60-dimensional objects: against the oracle on the compact tuples, and bit for bit against the same
    tuples in a 9 x 9 space."""
    errors, calls = [], 0
    for pool, srs in semirings(typ):
        av, bv, mv = _hyper_values(form, typ, pool, seed_of("hyper", form, typ, pool))
        for sr in srs:
            gK, gX, t = _hyper_call(form, typ, sr, av, bv, mv, True)
            _hyper_expect(form, t)
            sK, sX, _ = _hyper_call(form, typ, sr, av, bv, mv, False)
            calls += 1
            label = f"hyper {form} {'_'.join(sr)}"
            assert np.array_equal(gK, sK) and np.array_equal(_bits(np.asarray(gX)), _bits(np.asarray(sX))), \
                f"{label}: the 2^60 space and the small space differ"
            rK, rX, oa, ob = _hyper_oracle(form, typ, sr, av, bv, mv)
            cands = None
            if sr[0] == "ANY":
                n = len(HYPER_IDS)
                if form in ("mxv", "vxm"):
                    S = sp.csr_matrix((np.ones(len(oa.I), bool), (oa.I.astype(np.int64), oa.J.astype(np.int64))), shape=(n, n))
                    upres = np.zeros(n, bool); upres[ob.I.astype(np.int64)] = True
                    uv = np.zeros(n, orc.DTYPES[typ]); uv[ob.I.astype(np.int64)] = ob.X
                    cands = vec_products(uv, upres, S, np.asarray(oa.X), sr[1], form == "vxm")
                else:
                    cands = any_candidates(oa, ob, "", sr[1])
            e = compare(gK, gX, rK, rX, orc.semiring_ztype(sr), sr[0], label, cands)
            if e:
                errors.append(e)
    assert not errors, f"{len(errors)} of {calls} calls differ:\n" + "\n".join(errors[:40])


# ------------------------------------------------------------------ 2. mixed types
# MIXED of test_value_edges_gpu, and for the routes: a multiply op_mirror swaps on operands cast from FP64 edge values into a
# saturating INT32 (NaN -> 0, +-Inf -> the ends), the result cast into INT8 (wrap-around); an INT64 RMINUS into UINT8 under MIN
ROUTE_MIXED = MIXED + [
    ("FP64", ("MAX", "DIV", "INT32"), "INT8", None),
    ("INT64", ("MIN", "RMINUS", "INT16"), "UINT8", ("PLUS", "INT32")),
]
MIXED_ROUTES = ["spmm-split-k33", "spmm-split-csr-mask", "left", "left-T0-m1", "sddmm-d130-pres", "sddmm-y-transpose",
                "comp-bins-valued", "comp-split", "comp-split-valued"]


@pytest.mark.parametrize("case", range(len(ROUTE_MIXED)))
@pytest.mark.parametrize("name", MIXED_ROUTES)
def test_mixed_types(name, case):
    otyp, sr, ctyp, acc = ROUTE_MIXED[case]
    ops = route_operands(name)
    desc = ops["desc"]
    rng = np.random.default_rng(seed_of("mixed", name, case))
    av = util.rand_edge_values(rng, otyp, _size(ops["A"]), 0.5)
    bv = util.rand_edge_values(rng, otyp, _size(ops["B"]), 0.5)
    A, B = _dev(ops["A"], otyp, av), _dev(ops["B"], otyp, bv)
    oa, ob = _orc(ops["A"], otyp, av), _orc(ops["B"], otyp, bv)
    M, Mo, mv = _mask(ops, seed_of("mixed-m", name, case))
    m = oa.ncols if "T0" in desc else oa.nrows
    n = ob.nrows if "T1" in desc else ob.ncols
    Sc = lens_csr(rng.integers(0, min(n, 7) + 1, m), n, seed_of("mixed-c", name, case))
    cv = util.rand_edge_values(rng, ctyp, Sc.nnz, 0.5)
    C = Matrix.from_csr(Sc.indptr, Sc.indices, cv, m, n, util.g_type(ctyp))
    A.mxm(B, semiring=semiring(*sr), out=C, mask=M, accum=util.g_accum(acc), desc=getattr(descriptor, desc) if desc else None)
    t = _kernels()
    if ops["A"][0] == "csr" and ops["B"][0] == "csr":
        expect_route(name, t, sr, ops["A"][1], ops["B"][1], _blocks(ops, mv))
    else:
        expect_route(name, t, sr, homogeneous=False)
    gK, gX = keyed(C)
    ref = orc.mxm(o_csr(ctyp, Sc, cv), Mo, acc, sr, oa, ob, desc)
    e = compare(gK, gX, ref.I.astype(np.int64) * n + ref.J.astype(np.int64), ref.X, ctyp, sr[0], f"{name} {ROUTE_MIXED[case]}")
    assert e is None, e


@pytest.mark.parametrize("case", range(len(ROUTE_MIXED)))
@pytest.mark.parametrize("form", ["mxv", "mxm-comp"])
def test_hyper_mixed_types(form, case):
    otyp, sr, ctyp, acc = ROUTE_MIXED[case]
    rng = np.random.default_rng(seed_of("hyper-mixed", form, case))
    ops = hyper_operands(form)
    av = util.rand_edge_values(rng, otyp, len(ops["A"][0]), 0.5)
    bv = util.rand_edge_values(rng, otyp, len(ops["u"]) if "u" in ops else len(ops["B"][0]), 0.5)
    mv = mask_vals("BOOL", len(ops["M"][0]), 3) if "M" in ops else None
    n = len(HYPER_IDS)
    # w / C starts with entries of its own type, edge values included, which the accumulator (when the row has one) combines
    if form == "mxv":
        ci = np.flatnonzero(rng.random(n) < 0.5)
        c_init = (ci, util.rand_edge_values(rng, ctyp, len(ci), 0.5))
    else:
        ci, cj = np.nonzero(rng.random((n, n)) < 0.4)
        c_init = (ci, cj, util.rand_edge_values(rng, ctyp, len(ci), 0.5))
    gK, gX, t = _hyper_call(form, otyp, sr, av, bv, mv, True, accum=acc, ctyp=ctyp, c_init=c_init)
    _hyper_expect(form, t)
    sK, sX, _ = _hyper_call(form, otyp, sr, av, bv, mv, False, accum=acc, ctyp=ctyp, c_init=c_init)
    assert np.array_equal(gK, sK) and np.array_equal(_bits(np.asarray(gX)), _bits(np.asarray(sX)))
    ai, aj = ops["A"]
    oa = orc.SpMat(otyp, n, n, ai, aj, av)
    if form == "mxv":
        ref = orc.mxv(orc.SpVec(ctyp, n, *c_init), None, acc, sr, oa, orc.SpVec(otyp, n, ops["u"], bv))
        rK = ref.I.astype(np.int64)
    else:
        ob = orc.SpMat(otyp, n, n, *ops["B"], bv)
        om = orc.SpMat("BOOL", n, n, *ops["M"], mv)
        ref = orc.mxm(orc.SpMat(ctyp, n, n, *c_init), om, acc, sr, oa, ob, "C")
        rK = ref.I.astype(np.int64) * n + ref.J.astype(np.int64)
    e = compare(gK, gX, rK, ref.X, ctyp, sr[0], f"hyper {form} {ROUTE_MIXED[case]}")
    assert e is None, e


# ------------------------------------------------------------------ 3. FP sums at general values
def _record_ulp(name, typ, scale, u):
    k = (name, typ, scale)
    MAX_ULP[k] = max(MAX_ULP.get(k, 0.0), u)


def _order(name, ops, oa, ob, keys, a, b, typ, av, bv):
    kind = ROUTES[name][1]
    if kind == "spmm":
        S = with_data(ops["A"][1], av)
        B = ops["B"]
        return spmm_order(S, np.asarray(bv).reshape(B[1], B[2]), B[3], typ)
    if kind == "left":
        X = ops["A"]
        x, xp = np.asarray(av).reshape(X[1], X[2]), X[3]
        if "T0" in ops["desc"]:
            x, xp = np.ascontiguousarray(x.T), None if xp is None else np.ascontiguousarray(xp.T)
        return left_order(x, xp, with_data(ops["B"][1], bv), typ)
    if kind == "sddmm":
        X, Y = ops["A"], ops["B"]
        x, xp = np.asarray(av).reshape(X[1], X[2]), X[3]
        y, yp = np.asarray(bv).reshape(Y[1], Y[2]), Y[3]
        if "T1" not in ops["desc"]:
            y, yp = np.ascontiguousarray(y.T), None if yp is None else np.ascontiguousarray(yp.T)
        return sddmm_order(x, xp, y, yp, np.unique(keys), y.shape[0], typ)
    return None


@pytest.mark.parametrize("scale", ["normal", "subnormal"])
@pytest.mark.parametrize("typ", FP_T)
@pytest.mark.parametrize("name", list(ROUTES))
def test_fp_sums(name, typ, scale):
    ops = route_operands(name)
    desc = ops["desc"]
    rng = np.random.default_rng(seed_of("fp", name, typ, scale))
    av = _general_values(rng, typ, _size(ops["A"]), "normal")
    bv = _general_values(rng, typ, _size(ops["B"]), scale)
    A, B = _dev(ops["A"], typ, av), _dev(ops["B"], typ, bv)
    oa, ob = _orc(ops["A"], typ, av), _orc(ops["B"], typ, bv)
    M, Mo, mv = _mask(ops, seed_of("fp-m", name))
    m = oa.ncols if "T0" in desc else oa.nrows
    n = ob.nrows if "T1" in desc else ob.ncols
    sr = ("PLUS", "TIMES", typ)
    runs = []
    for _ in range(2):
        C = Matrix.sparse(util.g_type(typ), m, n)
        A.mxm(B, semiring=semiring(*sr), out=C, mask=M, desc=getattr(descriptor, desc) if desc else None)
        t = _kernels()
        runs.append(keyed(C))
    if ops["A"][0] == "csr" and ops["B"][0] == "csr":
        expect_route(name, t, sr, ops["A"][1], ops["B"][1], _blocks(ops, mv))
    else:
        expect_route(name, t, sr)
    (gK, gX), (gK2, gX2) = runs
    # the products of the positions the mask lets through (the oracle's presence, which the edge table holds the route to)
    keys, a, b, _ = products(oa, ob, desc)
    ref = orc.mxm(orc.SpMat(typ, m, n), Mo, None, sr, oa, ob, desc)
    keep = np.isin(keys, ref.I.astype(np.int64) * n + ref.J.astype(np.int64))
    keys, a, b = keys[keep], a[keep], b[keep]
    kind = ROUTES[name][1]
    ordered = _order(name, ops, oa, ob, keys, a, b, typ, av, bv)
    if ordered is not None:             # the restatement computes every position; the mask keeps some
        sel = np.isin(ordered[0], keys)
        ordered = ordered[0][sel], ordered[1][sel]
    label = f"{name} {typ} {scale}"
    if kind == "esc":
        # esc-small / esc-medium rows: the oracle's left-to-right fold, bit for bit; spa / spa-split rows: the bound only
        SA, SB = ops["A"][1], ops["B"][1]
        f = np.bincount(np.repeat(np.arange(SA.shape[0]), np.diff(SA.indptr)), weights=np.diff(SB.indptr)[SA.indices],
                        minlength=SA.shape[0])
        esc_rows = np.flatnonzero((f > 0) & (f <= 2048))
        lk, lv = ltr_fold(keys, a, b, typ)
        sel = np.isin(lk // n, esc_rows)
        gsel = np.isin(gK // n, esc_rows)
        assert np.array_equal(gK[gsel], lk[sel]), f"{label}: esc presence"
        bad = np.flatnonzero(_bits(np.asarray(gX)[gsel]) != _bits(lv[sel]))
        assert len(bad) == 0, f"{label}: {len(bad)} esc values differ from the oracle's left-to-right fold"
        assert len(esc_rows) > 0
        # the spa / spa-split rows combine with atomics: only the esc rows must give the same bits twice
        assert np.array_equal(gK, gK2) and np.array_equal(_bits(np.asarray(gX)[gsel]), _bits(np.asarray(gX2)[gsel])), \
            f"{label}: two runs differ on the esc rows"
    else:
        assert np.array_equal(gK, gK2) and np.array_equal(_bits(np.asarray(gX)), _bits(np.asarray(gX2))), f"{label}: two runs differ"
    u = check_fp(gK, gX, keys, a, b, typ, label, ordered)
    _record_ulp(name, typ, scale, u)


@pytest.mark.parametrize("scale", ["normal", "subnormal"])
@pytest.mark.parametrize("typ", FP_T)
@pytest.mark.parametrize("form", HYPER_FORMS)
def test_hyper_fp_sums(form, typ, scale):
    rng = np.random.default_rng(seed_of("hyper-fp", form, typ, scale))
    ops = hyper_operands(form)
    av = _general_values(rng, typ, len(ops["A"][0]), "normal")
    bv = _general_values(rng, typ, len(ops["u"]) if "u" in ops else len(ops["B"][0]), scale)
    mv = mask_vals("BOOL", len(ops["M"][0]), 5) if "M" in ops else None
    sr = ("PLUS", "TIMES", typ)
    gK, gX, t = _hyper_call(form, typ, sr, av, bv, mv, True)
    _hyper_expect(form, t)
    sK, sX, _ = _hyper_call(form, typ, sr, av, bv, mv, False)
    label = f"hyper {form} {typ} {scale}"
    assert np.array_equal(gK, sK) and np.array_equal(_bits(np.asarray(gX)), _bits(np.asarray(sX))), f"{label}: spaces differ"
    rK, _, oa, ob = _hyper_oracle(form, typ, sr, av, bv, mv)
    n = len(HYPER_IDS)
    if form in ("mxv", "vxm"):
        ai, aj = oa.I.astype(np.int64), oa.J.astype(np.int64)
        uv = np.zeros(n, orc.DTYPES[typ]); upres = np.zeros(n, bool)
        uv[ob.I.astype(np.int64)] = ob.X; upres[ob.I.astype(np.int64)] = True
        k_in, k_out = (aj, ai) if form == "mxv" else (ai, aj)
        keep = upres[k_in]
        keys, a, b = k_out[keep], np.asarray(oa.X)[keep], uv[k_in[keep]]
    else:
        keys, a, b, _ = products(oa, ob, "")
        keys, a, b = keys[np.isin(keys, rK)], a[np.isin(keys, rK)], b[np.isin(keys, rK)]
    u = check_fp(gK, gX, keys, a, b, typ, label)
    _record_ulp(f"hyper-{form}", typ, scale, u)


# ------------------------------------------------------------------ 4. every route of the table was reached
ALL_ROUTES = {"spmm-fast", "spmm-generic", "spmm-split", "spmm-left", "x-transpose", "t-transpose", "write=dense", "write=csr",
              "sddmm-fast", "sddmm-generic", "y-transpose", "pattern=mask", "pattern=compact",
              "esc-small", "esc-medium", "spa", "spa-split"} | {f"hyper-{f}" for f in HYPER_FORMS}


def test_every_route_was_reached(request):
    mine = [it for it in request.session.items if it.module is request.module and it is not request.node]
    if len(mine) < full_count(request.module, request.node.originalname):
        pytest.skip("only part of the module was selected")
    missing = ALL_ROUTES - REACHED
    assert not missing, f"routes no case reached: {sorted(missing)}"
    worst = {}
    for (name, typ, scale), u in MAX_ULP.items():
        worst[(name, typ)] = max(worst.get((name, typ), 0.0), u)
    print("\nlargest error against the exact sum, in ulps (normal and subnormal scale):")
    for (name, typ), u in sorted(worst.items()):
        print(f"  {name:24s} {typ}: {u:g}")
