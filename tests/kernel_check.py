"""Helpers shared by the GPU modules that force one mxv / vxm / mxm kernel path at a time and compare it with the oracle:
the kernel-path seam, the tunables switch, the value pools, the comparison rules and the ANY candidates."""
import contextlib
import functools
import os
import zlib

import numpy as np

import pygraphblas_b200 as gb
from pygraphblas_b200 import ffi, lib
from pygraphblas_b200.ops import Semiring
from oracle import oracle as orc
import util

FP_T = util.FP_T


def seed_of(*parts, bits=16):
    """A seed from a description of the case that is the same in every process (hash() of a string is not)."""
    return zlib.crc32(repr(parts).encode()) & ((1 << bits) - 1)


# ------------------------------------------------------------------ value pools
def fp_pools(typ):
    dt = orc.DTYPES[typ]
    tiny = np.finfo(dt).smallest_subnormal
    specials = [np.nan, np.inf, -np.inf, 0.0, -0.0]
    return {
        # the whole edge pool: MIN / MAX / ANY folds are order-independent whatever the values
        "edge": (None, None),
        # dyadic values: every product is a multiple of 1/4 no larger than 4, every sum of them is exact
        "dyadic": (specials + [0.5, -0.5, 1.0, -1.0, 2.0, -2.0],) * 2,
        # products of magnitude <= 2: no entry has enough factors to overflow, so TIMES folds are exact in any order
        "unit": (specials + [1.0, -1.0],) * 2,
        # subnormal sums: A small integers, B multiples of the smallest subnormal (fixed-point arithmetic, exact)
        "subnormal": ([np.inf, 0.0, -0.0, 1.0, -1.0, 2.0, -2.0], [np.nan, 0.0, -0.0] + [k * tiny for k in (1, -1, 2, -2, 3, -3)]),
    }


def fp_pool_for(add, mul):
    """The pool whose folds are exact in any order under the monoid add (FP operands)."""
    if add in ("MIN", "MAX", "ANY"):
        return "edge"
    return "dyadic" if add == "PLUS" else "unit"


def values(seed, typ, n, pool, side):
    """n values of typ: for FP from side 0 (A) or 1 (B, u) of the named pool, else (and for the edge pool) util.rand_edge_values."""
    rng = np.random.default_rng(seed)
    dt = orc.DTYPES[typ]
    if typ in FP_T:
        p = fp_pools(typ)[pool][side]
        if p is not None:
            return np.asarray(p, dt)[rng.integers(0, len(p), n)]
    return util.rand_edge_values(rng, typ, n, 0.5)


# ------------------------------------------------------------------ semirings
@functools.lru_cache(maxsize=None)
def semiring(add, mul, typ):
    t = util.g_type(typ)
    s = getattr(t, f"{add}_{mul}", None)
    if s is not None:
        return s
    mon = getattr(t, f"{add}_MONOID", None) or getattr(t, "LXNOR_MONOID")
    h = ffi.new("GrB_Semiring*")
    gb.base._check(lib.GrB_Semiring_new(h, mon.get_op(), getattr(t, mul).get_op()))
    return Semiring(add, mul, typ, h[0])


def spmv_specialised(add, mul, typ):
    """Restates spmv_is_fast: the semirings with compile-time specialised SpMV kernels."""
    if typ == "BOOL":
        return (add == "LOR" and mul in ("LAND", "PAIR", "SECOND", "FIRST")) or (add == "ANY" and mul == "PAIR")
    if typ in ("FP32", "FP64", "INT32", "INT64", "UINT32", "UINT64"):
        return (add == "PLUS" and mul in ("TIMES", "SECOND", "FIRST", "PAIR")) or (add == "MIN" and mul in ("PLUS", "FIRST", "SECOND"))
    return False


# ------------------------------------------------------------------ the kernel-path seam
def last_kernel():
    return ffi.string(lib.B200_debug_last_kernel()).decode()


def record_kernels(reached):
    """The tokens of B200_debug_last_kernel, also added to the set `reached`."""
    k = last_kernel().split(";")
    reached.update(k)
    return k


def entries(tokens):
    """The kernel entries of a seam reading, without the "key=value" variant tokens."""
    return [k for k in tokens if "=" not in k]


@contextlib.contextmanager
def tunables(**env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update({k: str(v) for k, v in env.items()})
    lib.B200_reload_tunables()
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
        lib.B200_reload_tunables()


# ------------------------------------------------------------------ comparison
def _bits(x):
    x = np.ascontiguousarray(x)
    return x.view(f"u{x.dtype.itemsize}") if x.dtype != np.bool_ else x


def compare(gI, gX, want_I, want_X, typ, add, label, candidates=None):
    """None when the result matches the oracle's, else a description.  Presence must be identical.  Values: bit-exact,
    except that any NaN matches any NaN, +0 matches -0 under MIN / MAX, and an ANY value must be one of the entry's
    products (`candidates`, from products_by_entry / vec_products)."""
    gI, want_I = np.asarray(gI, np.int64), np.asarray(want_I, np.int64)
    if not np.array_equal(gI, want_I):
        extra, miss = np.setdiff1d(gI, want_I), np.setdiff1d(want_I, gI)
        return f"{label}: presence differs (extra {extra[:5].tolist()}, missing {miss[:5].tolist()})"
    gX, want_X = np.asarray(gX), np.asarray(want_X)
    if add == "ANY" and candidates is not None:
        pairs, nan_keys = candidates
        gnan = np.isnan(gX) if gX.dtype.kind == "f" else np.zeros(len(gX), bool)
        bad = [k for k, (i, b, n) in enumerate(zip(gI.tolist(), _bits(gX).tolist(), gnan.tolist()))
               if not (i in nan_keys if n else (i, b) in pairs)]
        return f"{label}: ANY value not among the entry's products at {gI[bad[:5]].tolist()}: {gX[bad[:5]].tolist()}" if bad else None
    ok = _bits(gX) == _bits(want_X)
    if gX.dtype.kind == "f":
        ok |= np.isnan(gX) & np.isnan(want_X)
        if add in ("MIN", "MAX"):
            ok |= (gX == 0) & (want_X == 0)
    if ok.all():
        return None
    bad = np.flatnonzero(~ok)[:5]
    return f"{label}: {int((~ok).sum())} values differ, e.g. at {gI[bad].tolist()}: got {gX[bad].tolist()}, oracle {want_X[bad].tolist()}"


def _candidates(keys, prod):
    """The values an ANY fold may return: {(entry key, bit pattern)} and the keys that have a NaN product."""
    keys = np.asarray(keys, np.int64)
    nan = np.isnan(prod) if prod.dtype.kind == "f" else np.zeros(len(prod), bool)
    return set(zip(keys[~nan].tolist(), _bits(prod)[~nan].tolist())), set(keys[nan].tolist())


def _mul(mul, a, b):
    with np.errstate(all="ignore"):
        if mul == "FIRST":
            return a
        if mul == "SECOND":
            return b
        if a.dtype == np.bool_:
            return a & b
        return a * b


def products_by_entry(Ar, Ac, Av, Bp, Bc, Bv, ncols, mul):
    """The products of A (COO) times B (CSR), keyed by i * ncols + j: the values an ANY fold may return."""
    lens = (Bp[Ac + 1] - Bp[Ac]).astype(np.int64)
    rows = np.repeat(Ar, lens)
    starts = np.repeat(Bp[Ac].astype(np.int64) - np.concatenate(([0], np.cumsum(lens)[:-1])), lens)
    pos = np.arange(int(lens.sum())) + starts
    prod = _mul(mul, np.repeat(Av, lens), Bv[pos])
    return _candidates(rows.astype(np.int64) * ncols + Bc[pos].astype(np.int64), prod)


def vec_products(uv, upres, S, av, mul, vxm):
    """The products of A u (mxv: mul(A(i,k), u(k))) or u' A (vxm: mul(u(k), A(k,j))), keyed by output index."""
    C = S.tocoo()
    rows, cols = C.row.astype(np.int64), C.col.astype(np.int64)
    order = np.lexsort((cols, rows))
    rows, cols = rows[order], cols[order]
    a = np.asarray(av)                    # CSR order == row-major order
    k = rows if vxm else cols
    keep = upres[k]
    if vxm:
        prod, out_idx = _mul(mul, uv[rows[keep]], a[keep]), cols[keep]
    else:
        prod, out_idx = _mul(mul, a[keep], uv[cols[keep]]), rows[keep]
    return _candidates(out_idx, prod)


# ------------------------------------------------------------------ operands
def o_csr(typ, S, vals):
    """An oracle matrix straight from a sorted CSR pattern (no re-sort)."""
    m = orc.SpMat.__new__(orc.SpMat)
    m.type, m.nrows, m.ncols = typ, S.shape[0], S.shape[1]
    m.I = np.repeat(np.arange(S.shape[0], dtype=np.uint64), np.diff(S.indptr))
    m.J = S.indices.astype(np.uint64)
    m.X = np.ascontiguousarray(vals)
    return m
