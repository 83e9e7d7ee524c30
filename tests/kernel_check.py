"""Helpers shared by the GPU modules that force one mxv / vxm / mxm kernel path at a time and compare it with the oracle:
the kernel-path seam, the tunables switch, the value pools, the comparison rules and the ANY candidates."""
import contextlib
import functools
import os
import zlib

import numpy as np
import scipy.sparse as sp

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


# ------------------------------------------------------------------ the hot-table SpMV, restated (spmv_run.cu / spmv_run.cuh)
HOT_EXT = 1 << 17
HOT_T = ("BOOL", "INT32", "INT64", "UINT32", "UINT64", "FP32", "FP64")      # the types of the specialised semirings
VSIZE = {"BOOL": 1, "INT32": 4, "UINT32": 4, "FP32": 4, "INT64": 8, "UINT64": 8, "FP64": 8}


def kernel_mul(mul, vxm):
    """The multiply the run kernels see: x = the matrix entry, y = u's (FIRST and SECOND swap in vxm form)."""
    return {"FIRST": "SECOND", "SECOND": "FIRST"}.get(mul, mul) if vxm else mul


def hot_reads_u(mul, vxm):
    """The multiply reads u: only then is there a gather for the hot table to serve (else the plain run kernel)."""
    return kernel_mul(mul, vxm) not in ("FIRST", "PAIR")


def hot_reads_a(mul, vxm):
    """The multiply reads A's values: the warp stage holds them beside the ids (mul_reads_x)."""
    return kernel_mul(mul, vxm) not in ("SECOND", "PAIR")


def hot_henc(S, vxm=False):
    """henc of spmv_hot_plan: the referenced columns of the CSR the kernel pulls along (A for mxv, A' for vxm), at most HOT_EXT."""
    deg = np.diff(S.indptr) if vxm else np.bincount(S.indices, minlength=S.shape[1])
    return min(int(np.count_nonzero(deg)), HOT_EXT)


def hot_id_bits(S, vxm=False):
    """The id width spmv_hot_plan picks: 3 bytes when ncols + henc < 2^24 (ncols of the pulled CSR), else 4."""
    ncols = S.shape[0] if vxm else S.shape[1]
    return 24 if ncols + hot_henc(S, vxm) < (1 << 24) else 32


def hot_table_cap(typ, reads_a, id_bits, henc, limit_bytes, max_optin):
    """Restates hot2_table_entries: the table entries left after the warp stages and barriers, at most limit_bytes."""
    idb = id_bits // 8
    stage = 256 * idb + (256 * VSIZE[typ] if reads_a else 0)
    fixed = 32 * stage + 33 * 8 + 8
    avail = min(max(max_optin - fixed - 256, 0), limit_bytes)
    return min(henc, avail // VSIZE[typ]) & ~15


def hot_tiers(henc, cap, C, t0kb, vsize):
    """Restates hot2_tiers: (C, T0, T1, slice)."""
    if C == 1 or henc - cap < 16:
        return 1, cap, 0, 0
    t0 = min(((t0kb << 10) // vsize) & ~15, cap)
    need = henc - t0
    sl = min(cap - t0, (-(-need // C) + 15) & ~15)
    if sl == 0:
        return 1, cap, 0, 0
    return C, t0, min(need, sl * C), sl


def max_optin():
    """The device's opt-in shared memory per block (what hot2_table_entries asks the driver for)."""
    import torch
    return int(torch.cuda.get_device_properties(0).shared_memory_per_block_optin)


def expected_hot_launch(S, vxm, typ, mul, hot_kb, C, t0kb, smem_optin):
    """(C, T0, T1, henc) and the id width of a hot-table call on the CSR S (A; the kernel pulls along A' in vxm form)."""
    henc, bits = hot_henc(S, vxm), hot_id_bits(S, vxm)
    cap = hot_table_cap(typ, hot_reads_a(mul, vxm), bits, henc, hot_kb << 10, smem_optin)
    c, t0, t1, _ = hot_tiers(henc, cap, C, t0kb, VSIZE[typ])
    return (c, t0, t1, henc), bits


def hot_tokens():
    """(kernel entries, {key: value}) of the last call's seam reading."""
    ks = last_kernel().split(";")
    return entries(ks), dict(k.split("=", 1) for k in ks if "=" in k)


def hot_launch_of(tok):
    """(C, T0, T1, henc) and the id width the library reports for a hot-table call."""
    return (int(tok["hot-cluster"]),) + tuple(int(x) for x in tok["hot-tiers"].split(",")), int(tok["ids"])


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


def oracle_spmv(typ, sr, S, vals, uv, vxm):
    """The oracle's mxv (A = S) or vxm (u' S) with dense u, on the entries of u that S references only: the referenced
    indices are renumbered in order (the oracle's fold order is kept), so a u of 2^24 entries costs what S does."""
    if vxm:
        keep = np.flatnonzero(np.diff(S.indptr))
        T = sp.csr_matrix((np.ones(S.nnz, np.int8), S.indices, np.r_[0, np.cumsum(np.diff(S.indptr)[keep])]), shape=(len(keep), S.shape[1]))
        uo = orc.SpVec(typ, len(keep), np.arange(len(keep)), uv[keep])
        return orc.vxm(orc.SpVec(typ, S.shape[1]), None, None, sr, uo, o_csr(typ, T, vals), "")
    keep, inv = np.unique(S.indices, return_inverse=True)
    T = sp.csr_matrix((np.ones(S.nnz, np.int8), inv.astype(np.int64), S.indptr), shape=(S.shape[0], len(keep)))
    uo = orc.SpVec(typ, len(keep), np.arange(len(keep)), uv[keep])
    return orc.mxv(orc.SpVec(typ, S.shape[0]), None, None, sr, o_csr(typ, T, vals), uo, "")


def uniform_pattern(ncols, deg, cols=None):
    """Every referenced column (cols, default all ncols) referenced exactly deg times: the stable degree sort then ranks the
    j-th referenced column as j, so every hot rank (and so both sides of every tier boundary) is gathered.  Square when
    every column is referenced, else one row per referenced column."""
    cols = np.arange(ncols, dtype=np.int64) if cols is None else np.asarray(cols, np.int64)
    nrows = ncols if len(cols) == ncols else len(cols)
    j = np.repeat(cols, deg)
    t = np.tile(np.arange(deg, dtype=np.int64), len(cols))
    r = (np.repeat(np.arange(len(cols), dtype=np.int64), deg) * 7 + t * 4099) % nrows
    S = sp.csr_matrix((np.ones(len(j), np.int8), (r, j)), shape=(nrows, ncols))
    S.sort_indices()
    assert S.nnz == len(cols) * deg
    return S


def spread_columns(ncols, low, nspread):
    """The columns 0 .. low-1 and nspread columns spread evenly over the rest, the last column included."""
    return np.concatenate([np.arange(low), np.linspace(low, ncols - 1, nspread).astype(np.int64)])


# ------------------------------------------------------------------ coverage ledgers
def full_count(module, ledger):
    """The number of cases in the module but its ledger test: every test function times its parametrisations."""
    n = 0
    for name, f in vars(module).items():
        if name.startswith("test_") and callable(f) and name != ledger:
            k = 1
            for m in getattr(f, "pytestmark", []):
                if m.name == "parametrize":
                    k *= len(m.args[1])
            n += k
    return n
