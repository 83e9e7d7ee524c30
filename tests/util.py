"""Shared helpers for the tests: golden dict <-> oracle containers <-> product containers."""
import numpy as np
from oracle import oracle as orc


# ------------------------------------------------------------------ oracle side
def o_mat(d):
    return orc.SpMat(d["type"], d["nrows"], d["ncols"], d["I"], d["J"], d["X"])


def o_vec(d):
    return orc.SpVec(d["type"], d["size"], d["I"], d["X"])


def oracle_run(case):
    sr = tuple(case["semiring"])
    acc = tuple(case["accum"]) if case["accum"] else None
    if case["op"] == "mxm":
        return orc.mxm(o_mat(case["C"]), o_mat(case["mask"]) if case["mask"] else None, acc, sr, o_mat(case["A"]), o_mat(case["B"]), case["desc"])
    if case["op"] == "mxv":
        return orc.mxv(o_vec(case["w"]), o_vec(case["mask"]) if case["mask"] else None, acc, sr, o_mat(case["A"]), o_vec(case["u"]), case["desc"])
    return orc.vxm(o_vec(case["w"]), o_vec(case["mask"]) if case["mask"] else None, acc, sr, o_vec(case["u"]), o_mat(case["A"]), case["desc"])


def same_mat(a, d, rtol=0.0):
    """oracle/product result `a` (with .type, I, J, X arrays) equals golden dict d."""
    e = o_mat(d)
    if a.type != e.type or (a.nrows, a.ncols) != (e.nrows, e.ncols):
        return False
    if not (np.array_equal(a.I, e.I) and np.array_equal(a.J, e.J)):
        return False
    return np.array_equal(a.X, e.X) if rtol == 0 else np.allclose(a.X, e.X, rtol=rtol, atol=0)


def same_vec(a, d, rtol=0.0):
    e = o_vec(d)
    if a.type != e.type or a.size != e.size or not np.array_equal(a.I, e.I):
        return False
    return np.array_equal(a.X, e.X) if rtol == 0 else np.allclose(a.X, e.X, rtol=rtol, atol=0)


# ------------------------------------------------------------------ product side
def g_type(name):
    import pygraphblas_b200 as gb
    return gb.types.by_name(name)


def g_mat(d):
    import pygraphblas_b200 as gb
    return gb.Matrix.from_lists(d["I"], d["J"], d["X"], d["nrows"], d["ncols"], g_type(d["type"]))


def g_vec(d):
    import pygraphblas_b200 as gb
    return gb.Vector.from_lists(d["I"], d["X"], d["size"], g_type(d["type"]))


def g_semiring(sr):
    add, mul, t = sr
    return getattr(g_type(t), f"{add}_{mul}")


def g_accum(acc):
    return getattr(g_type(acc[1]), acc[0]) if acc else None


def g_desc(desc):
    import pygraphblas_b200 as gb
    return getattr(gb.descriptor, desc) if desc else None


def product_run(case):
    """Run a golden-style case through the product's public API; returns an oracle container."""
    sr = g_semiring(case["semiring"])
    acc = g_accum(case["accum"])
    desc = g_desc(case["desc"])
    if case["op"] == "mxm":
        A, B = g_mat(case["A"]), g_mat(case["B"])
        C = A if case["C"] is case["A"] else g_mat(case["C"])
        M = g_mat(case["mask"]) if case["mask"] else None
        out = A.mxm(B, semiring=sr, out=C, mask=M, accum=acc, desc=desc)
        I, J, X = out.to_arrays()
        return orc.SpMat(out.type.name, out.nrows, out.ncols, I, J, X)
    A, u = g_mat(case["A"]), g_vec(case["u"])
    w = u if case["w"] is case["u"] else g_vec(case["w"])
    m = g_vec(case["mask"]) if case["mask"] else None
    if case["op"] == "mxv":
        out = A.mxv(u, semiring=sr, out=w, mask=m, accum=acc, desc=desc)
    else:
        out = u.vxm(A, semiring=sr, out=w, mask=m, accum=acc, desc=desc)
    I, X = out.to_arrays()
    return orc.SpVec(out.type.name, out.size, I, X)


# ------------------------------------------------------------------ random cases
INT_T = ["INT8", "INT16", "INT32", "INT64", "UINT8", "UINT16", "UINT32", "UINT64"]
ALL_T = ["BOOL"] + INT_T + ["FP32", "FP64"]
DESCS_M = ["", "T0", "T1", "T0T1", "C", "R", "RC", "S", "SC", "RS", "RSC", "RCT0", "ST1", "RSCT0T1"]


def rand_values(rng, typ, n):
    dt = orc.DTYPES[typ]
    if typ == "BOOL":
        return rng.integers(0, 2, n).astype(dt)
    if typ in ("FP32", "FP64"):
        return (rng.integers(-8, 9, n) / 4.0).astype(dt)      # exactly representable: order-independent sums
    info = np.iinfo(dt)
    lo = max(info.min, -5)
    return rng.integers(lo, 6, n).astype(dt)


def rand_mat(rng, typ, nrows, ncols, density):
    nnz = int(round(nrows * ncols * density))
    flat = rng.choice(nrows * ncols, size=min(nnz, nrows * ncols), replace=False) if nnz else np.zeros(0, np.int64)
    I, J = np.divmod(flat, ncols)
    return {"type": typ, "nrows": nrows, "ncols": ncols, "I": I.tolist(), "J": J.tolist(), "X": rand_values(rng, typ, len(I)).tolist()}


def rand_vec(rng, typ, size, density):
    nnz = int(round(size * density))
    I = rng.choice(size, size=min(nnz, size), replace=False) if nnz else np.zeros(0, np.int64)
    return {"type": typ, "size": size, "I": I.tolist(), "X": rand_values(rng, typ, len(I)).tolist()}


def semirings_for(typ):
    """A representative slice of the builtin semirings on operand type typ."""
    if typ == "BOOL":
        return [("LOR", "LAND", "BOOL"), ("ANY", "PAIR", "BOOL"), ("LXOR", "LAND", "BOOL"), ("EQ", "LOR", "BOOL"),
                ("LAND", "LOR", "BOOL"), ("LOR", "FIRST", "BOOL"), ("LOR", "SECOND", "BOOL")]
    out = [("PLUS", "TIMES", typ), ("MIN", "PLUS", typ), ("PLUS", "SECOND", typ), ("PLUS", "FIRST", typ),
           ("PLUS", "PAIR", typ), ("MAX", "MIN", typ), ("MIN", "FIRST", typ), ("MIN", "SECOND", typ),
           ("MAX", "PLUS", typ), ("PLUS", "MINUS", typ), ("TIMES", "PLUS", typ), ("PLUS", "LAND", typ),
           ("LOR", "EQ", typ), ("LOR", "GT", typ), ("LXOR", "LT", typ), ("ANY", "PAIR", typ)]
    return out


# ------------------------------------------------------------------ edge values
FP_T = ["FP32", "FP64"]


def edge_values(typ):
    """A fixed pool of the values where kernels and CPU references part ways, for each type: the ends of the integer
    range (and UINT* values at and above 2^(w-1)), and for FP NaN, +-Inf, +-0, the smallest and largest subnormal, the
    smallest normal and the largest finite value (both signs), and a few ordinary values."""
    dt = orc.DTYPES[typ]
    if typ == "BOOL":
        return np.array([False, True])
    if typ in FP_T:
        fi = np.finfo(dt)
        sub_lo, sub_hi, norm_lo = fi.smallest_subnormal, fi.tiny - fi.smallest_subnormal, fi.tiny
        vals = [np.nan, np.inf, -np.inf, 0.0, -0.0, sub_lo, -sub_lo, sub_hi, -sub_hi, norm_lo, -norm_lo,
                fi.max, -fi.max, 1.0, -1.0, 0.5, 3.0]
        return np.array(vals, dtype=dt)
    info = np.iinfo(dt)
    if info.min < 0:
        vals = [info.min, info.min + 1, -2, -1, 0, 1, 2, info.max - 1, info.max]
    else:
        half = 1 << (info.bits - 1)
        vals = [0, 1, 2, half - 1, half, info.max - 1, info.max]
    return np.array(vals, dtype=dt)


def rand_edge_values(rng, typ, n, ratio=0.5, pool=None):
    """n values: each drawn from `pool` (default edge_values(typ)) with probability `ratio`, else from rand_values."""
    pool = edge_values(typ) if pool is None else np.asarray(pool, dtype=orc.DTYPES[typ])
    out = rand_values(rng, typ, n)
    pick = rng.random(n) < ratio
    out[pick] = pool[rng.integers(0, len(pool), int(pick.sum()))]
    return out


def rand_edge_mat(rng, typ, nrows, ncols, density, ratio=0.5, pool=None):
    d = rand_mat(rng, typ, nrows, ncols, density)
    d["X"] = rand_edge_values(rng, typ, len(d["I"]), ratio, pool).tolist()
    return d


def rand_edge_vec(rng, typ, size, density, ratio=0.5, pool=None):
    d = rand_vec(rng, typ, size, density)
    d["X"] = rand_edge_values(rng, typ, len(d["I"]), ratio, pool).tolist()
    return d
