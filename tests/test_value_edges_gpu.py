"""Every mxv / vxm / mxm kernel path against the CPU oracle, with operands drawn from the edges of each type.

The parity suite uses gentle values (small integers, multiples of 1/4) so that every fold order gives the same answer.
This module feeds the kernels what those values never reach: INT*_MIN / *_MAX, UINT* values >= 2^(w-1), NaN, +-Inf,
-0.0, subnormals and the largest finite floats, and float -> integer casts that saturate.  Each case forces one kernel
path with the B200GRB_* switches and the operand shape, asserts through B200_debug_last_kernel that the path was taken,
and compares with the oracle:

* BOOL and integer results: bit-exact.
* FP, with operands chosen so that every fold order gives the same result (MIN / MAX over the whole pool; PLUS and
  TIMES over dyadic values, +-0, +-Inf and NaN, without the largest finite values): identical bit patterns, except that
  any NaN matches any NaN and, for MIN / MAX monoids, +0 matches -0 (IEEE leaves the sign of fmin(+0, -0) open).
* ANY monoid: the value must be one of the products of that entry.
* Presence is always identical: a NaN result is still an entry.

test_fp_sums_within_error_bound checks PLUS_TIMES on general FP values (also scaled into the subnormal range) against
the dot-product error bound instead of the oracle's bits, on every path that can carry it.

Large operands are built once per module (the R-MAT graph of the hot-table SpMV kernel, the SpGEMM patterns) and
their values once per type and value pool; the semirings of a type run in a loop inside one test case."""
import functools

import numpy as np
import pytest
import scipy.sparse as sp

from pygraphblas_b200 import Matrix, Vector, descriptor
from pygraphblas_b200.generators import rmat_csr
from oracle import oracle as orc
import util
from kernel_check import (compare, entries, fp_pool_for as _fp_pool_for, last_kernel, o_csr, products_by_entry, record_kernels,
                          seed_of, semiring, spmv_specialised, tunables, values, vec_products as _vec_products)

pytestmark = pytest.mark.gpu

INT_T, FP_T, ALL_T = util.INT_T, util.FP_T, util.ALL_T
SIGNED = {"INT8", "INT16", "INT32", "INT64"}
INT_MULS = ["TIMES", "PLUS", "MINUS", "RMINUS", "DIV", "RDIV", "FIRST", "SECOND", "MIN", "MAX"]
FP_MULS = ["TIMES", "PLUS", "MINUS", "DIV", "FIRST", "SECOND"]
BOOL_MULS = ["LAND", "LOR", "LXOR", "FIRST", "SECOND"]
ANY_MULS = ["FIRST", "SECOND", "TIMES"]


def semirings(typ, only=None):
    """(pool, [(add, mul, typ), ...]) groups for operand type typ.  only: a predicate on (add, mul, typ)."""
    groups = {}
    if typ == "BOOL":
        for add in ("LOR", "LAND", "LXOR", "EQ"):
            groups.setdefault("edge", []).extend((add, m, typ) for m in BOOL_MULS)
        groups["edge"].extend(("ANY", m, typ) for m in ("FIRST", "SECOND", "LAND"))
    elif typ in FP_T:
        for add in ("PLUS", "TIMES", "MIN", "MAX", "ANY"):
            for m in (ANY_MULS if add == "ANY" else FP_MULS):
                groups.setdefault(_fp_pool_for(add, m), []).append((add, m, typ))
        groups["subnormal"] = [("PLUS", m, typ) for m in ("TIMES", "FIRST", "SECOND")]
    else:
        adds = ["PLUS", "TIMES", "MIN", "MAX"] + ([] if typ in SIGNED else ["BOR", "BAND", "BXOR", "BXNOR"])
        groups["edge"] = [(a, m, typ) for a in adds for m in INT_MULS] + [("ANY", m, typ) for m in ANY_MULS]
    out = []
    for pool, srs in groups.items():
        srs = [s for s in srs if only is None or only(*s)]
        if srs:
            out.append((pool, srs))
    return out


# ------------------------------------------------------------------ the kernel-path seam
REACHED = set()


def _kernels():
    return record_kernels(REACHED)


# ------------------------------------------------------------------ operands
def pattern(seed, nrows, ncols, per_row):
    rng = np.random.default_rng(seed)
    cols = [np.sort(rng.choice(ncols, per_row, replace=False)) for _ in range(nrows)]
    indptr = np.arange(nrows + 1, dtype=np.int64) * per_row
    return sp.csr_matrix((np.ones(nrows * per_row, bool), np.concatenate(cols), indptr), shape=(nrows, ncols))


@functools.lru_cache(maxsize=None)
def rmat17():
    n, indptr, indices = rmat_csr(17)
    S = sp.csr_matrix((np.ones(len(indices), bool), indices, indptr), shape=(n, n))
    S.sort_indices()
    return S


# SpMV paths: pattern, the switches, the expected kernel, the semirings it serves
SPMV = {
    "tile-4": dict(shape="small", env={"B200GRB_SPMV_ITEMS": 4}, kernel="tile (specialised, 4 items)", only=spmv_specialised),
    "tile-8": dict(shape="small", env={}, kernel="tile", only=None),
    "tile-16": dict(shape="small", env={"B200GRB_SPMV_ITEMS": 16}, kernel="tile (specialised, 16 items)", only=spmv_specialised),
    "run": dict(shape="run", env={}, kernel="run", only=None),
    "run-sparse-u": dict(shape="run", env={}, kernel="run (sparse u)", only=None, sparse_u=True),
    "hot": dict(shape="rmat", env={"B200GRB_SPMV_HOT": 128}, kernel="run+hot-table (TMA-staged)", only=spmv_specialised),
    "hot-pipe": dict(shape="rmat", env={"B200GRB_SPMV_HOT": 128, "B200GRB_SPMV_PIPE": 1}, kernel="run+hot-table (TMA-staged, pipelined)",
                     only=spmv_specialised),
    "pull": dict(shape="pull", env={}, kernel="pull", only=lambda a, m, t: a in ("LOR", "LAND", "ANY"), mask=True),
    "push": dict(shape="pull", env={"B200GRB_FORCE_PUSH": 1}, kernel="push", only=lambda a, m, t: a in ("LOR", "LAND", "ANY"),
                 mask=True, sparse_u=True),
}
HOT_T = ["BOOL", "INT32", "UINT64", "FP32", "FP64"]


@functools.lru_cache(maxsize=None)
def spmv_pattern(shape):
    if shape == "small":
        return pattern(11, 300, 400, 6)                       # 1800 entries: the tile kernel
    if shape == "run":
        return pattern(12, 3000, 2500, 6)                     # 18000 entries: the run kernel
    if shape == "rmat":
        return rmat17()                                        # 1.9M entries, >= 2^16 columns: the hot-table kernel
    # masked pull: mostly short rows, a few rows longer than the pull kernel's long-row cut (4096)
    S = pattern(13, 6000, 6000, 4).tolil()
    rng = np.random.default_rng(14)
    for r in (5, 77, 3001):
        S[r, np.sort(rng.choice(6000, 5000, replace=False))] = True
    S = S.tocsr(); S.sort_indices()
    return S


def _spmv_expect(path, cfg, typ, add, mul, vxm):
    k = cfg["kernel"]
    if path == "tile-8":
        return None                                            # specialised (8 items) or run-time operators: checked by prefix
    if path.startswith("hot") and mul == ("SECOND" if vxm else "FIRST"):
        return "run"                                           # the multiply ignores u: no gathers for the hot table to serve
    if path == "hot-pipe" and orc.DTYPES[typ]().itemsize > 4:
        return "run+hot-table (TMA-staged)"                   # the pipelined kernel serves types of up to 4 bytes
    return k


def run_spmv_path(path, typ):
    cfg = SPMV[path]
    S = spmv_pattern(cfg["shape"])
    nrows, ncols = S.shape
    errors, calls = [], 0
    with tunables(**cfg["env"]):
        for pool, srs in semirings(typ, cfg["only"]):
            seed = seed_of(path, typ, pool)
            av = values(seed, typ, S.nnz, pool, 0)
            A = Matrix.from_csr(S.indptr, S.indices, av, nrows, ncols, util.g_type(typ))
            Ao = o_csr(typ, S, av)
            for vxm in (False, True):
                n_in = nrows if vxm else ncols
                uv = values(seed + 1 + vxm, typ, n_in, pool, 1)
                upres = np.random.default_rng(seed + 3).random(n_in) < (0.02 if path == "push" else 0.6) if cfg.get("sparse_u") else np.ones(n_in, bool)
                u = Vector.from_numpy(uv, present=upres if cfg.get("sparse_u") else None, typ=util.g_type(typ))
                uo = orc.SpVec(typ, n_in, np.flatnonzero(upres), uv[upres])
                mask = mo = None
                n_out = ncols if vxm else nrows
                if cfg.get("mask"):
                    mp = np.random.default_rng(seed + 4).random(n_out) < 0.7
                    mask = Vector.from_numpy(np.ones(n_out, bool), present=mp)
                    mo = orc.SpVec("BOOL", n_out, np.flatnonzero(mp), np.ones(int(mp.sum()), bool))
                if path == "push" and not vxm:
                    Vector.from_numpy(np.ones(nrows, typ == "BOOL" and bool or orc.DTYPES[typ]), typ=util.g_type(typ)).vxm(A, semiring=semiring("ANY", "FIRST", typ))
                for sr in srs:
                    s = semiring(*sr)
                    desc = descriptor.S if mask is not None else None
                    w = (u.vxm(A, semiring=s, mask=mask, desc=desc) if vxm else A.mxv(u, semiring=s, mask=mask, desc=desc))
                    ks = _kernels()
                    calls += 1
                    want_k = _spmv_expect(path, cfg, typ, sr[0], sr[1], vxm)
                    form = "vxm" if vxm else "mxv"
                    if want_k is None:
                        assert len(ks) == 1 and ks[0].startswith("tile"), (path, sr, form, ks)
                    else:
                        assert entries(ks) == [want_k], (path, sr, form, ks)
                    gI, gX = w.to_arrays()
                    ref = (orc.vxm(orc.SpVec(w.type.name, n_out), mo, None, sr, uo, Ao, "S" if mo else "") if vxm else
                           orc.mxv(orc.SpVec(w.type.name, n_out), mo, None, sr, Ao, uo, "S" if mo else ""))
                    cands = _vec_products(uv, upres, S, av, sr[1], vxm) if sr[0] == "ANY" else None
                    e = compare(gI, gX, ref.I, ref.X, typ, sr[0], f"{form} {'_'.join(sr)}", cands)
                    if e:
                        errors.append(e)
    assert calls > 0
    assert not errors, f"{len(errors)} of {calls} calls differ on the {path} path:\n" + "\n".join(errors[:40])


@pytest.mark.parametrize("typ", ALL_T)
@pytest.mark.parametrize("path", ["tile-4", "tile-8", "tile-16", "run", "run-sparse-u", "pull", "push"])   # SPMV_CASES
def test_spmv_edges(path, typ):
    if not semirings(typ, SPMV[path]["only"]):
        pytest.skip(f"no specialised SpMV kernel on {typ}")
    run_spmv_path(path, typ)


@pytest.mark.parametrize("typ", HOT_T)
@pytest.mark.parametrize("path", ["hot", "hot-pipe"])
def test_spmv_hot_table_edges(path, typ):
    """R-MAT scale 17: edge values land at hot and cold columns of u and inside hub rows that span many runs, whose
    partials the fix-up kernel folds."""
    run_spmv_path(path, typ)


# ------------------------------------------------------------------ SpGEMM
# path: (A, B, mask patterns, descriptor, switches, expected kernels)
def _gemm_patterns(path):
    if path in ("esc-small", "hash-small"):
        return pattern(21, 200, 200, 6), pattern(22, 200, 200, 6), None, ""
    if path in ("esc-medium", "hash-medium"):
        return pattern(23, 150, 300, 30), pattern(24, 300, 300, 30), None, ""
    if path == "spa":
        return pattern(25, 64, 400, 60), pattern(26, 400, 3000, 60), None, ""
    if path == "masked-warp":
        return pattern(27, 300, 300, 10), pattern(28, 300, 300, 10), pattern(29, 300, 300, 60), "S"
    if path == "stream-S":
        return pattern(30, 100, 2000, 10), pattern(31, 2000, 2000, 15), pattern(32, 100, 2000, 300), "S"
    if path == "stream-M":
        return pattern(33, 60, 4000, 10), pattern(34, 4000, 4000, 15), pattern(35, 60, 4000, 1000), "S"
    if path == "stream-L":
        return pattern(36, 40, 5000, 20), pattern(37, 5000, 5000, 20), pattern(38, 40, 5000, 3000), "S"
    if path == "split":
        # 40 x 1000 = 40000 products per row (> 32768): every row is cut into two chunks whose partials are combined in HBM;
        # rows 0-3 have mask rows of 400 entries (class S), rows 4-7 of 2100 (class L)
        M = sp.vstack([pattern(41, 4, 2200, 400), pattern(42, 4, 2200, 2100)]).tocsr()
        M.sort_indices()
        return pattern(39, 8, 2000, 40), pattern(40, 2000, 2200, 1000), M, "S"
    if path == "dot":
        return pattern(43, 200, 300, 10), pattern(44, 200, 300, 10), pattern(45, 200, 200, 20), "ST1"
    if path == "st1-transpose":
        return pattern(46, 200, 3000, 5), pattern(47, 3000, 3000, 90), pattern(48, 200, 3000, 50), "ST1"
    raise KeyError(path)


GEMM = {
    "esc-small": ({}, ["esc-small"]), "hash-small": ({"B200GRB_SPGEMM_ESC": 0}, ["hash-small"]),
    "esc-medium": ({}, ["esc-medium"]), "hash-medium": ({"B200GRB_SPGEMM_ESC": 0}, ["hash-medium"]),
    "spa": ({}, ["spa"]), "masked-warp": ({}, ["masked-warp"]),
    "stream-S": ({}, ["stream-S"]), "stream-M": ({}, ["stream-M"]), "stream-L": ({}, ["stream-L"]),
    "split": ({}, ["stream-S", "stream-L"]), "dot": ({}, ["dot"]), "st1-transpose": ({}, ["masked-warp"]),
}


@functools.lru_cache(maxsize=None)
def gemm_patterns(path):
    A, B, M, desc = _gemm_patterns(path)
    assert B.nnz >= (1 << 18) if path == "st1-transpose" else True
    return A, B, M, desc


def run_gemm(path, typ, srs_filter=None, pools=None, extra=None):
    env, want = GEMM[path]
    SA, SB, SM, desc = gemm_patterns(path)
    Bt = SB.T.tocsr() if "T1" in desc else SB
    Bt.sort_indices()
    nrows, ncols = SA.shape[0], Bt.shape[1]
    errors, calls = [], 0
    with tunables(**env):
        M = Matrix.from_csr(SM.indptr, SM.indices, None, *SM.shape) if SM is not None else None
        Mo = o_csr("BOOL", SM, np.ones(SM.nnz, bool)) if SM is not None else None
        for pool, srs in semirings(typ, srs_filter):
            if pools is not None and pool not in pools:
                continue
            seed = seed_of(path, typ, pool)
            av, bv = values(seed, typ, SA.nnz, pool, 0), values(seed + 1, typ, SB.nnz, pool, 1)
            gt = util.g_type(typ)
            A = Matrix.from_csr(SA.indptr, SA.indices, av, *SA.shape, gt)
            B = Matrix.from_csr(SB.indptr, SB.indices, bv, *SB.shape, gt)
            Ao, Bo = o_csr(typ, SA, av), o_csr(typ, SB, bv)
            for sr in srs:
                s = semiring(*sr)
                C = Matrix.sparse(util.g_type(orc.semiring_ztype(sr)), nrows, ncols)
                A.mxm(B, semiring=s, out=C, mask=M, desc=getattr(descriptor, desc) if desc else None)
                ks = _kernels()
                calls += 1
                assert all(k in ks for k in want), (path, sr, ks)
                if path == "st1-transpose":
                    assert "dot" not in ks, (path, sr, ks)
                gI, gJ, gX = C.to_arrays()
                ref = orc.mxm(orc.SpMat(C.type.name, nrows, ncols), Mo, None, sr, Ao, Bo, desc)
                cands = None
                if sr[0] == "ANY":
                    if "T1" in desc:
                        bvt = sp.csr_matrix((bv, SB.indices, SB.indptr), shape=SB.shape).T.tocsr()
                        bvt.sort_indices()
                        Bp, Bc, Bvv = bvt.indptr, bvt.indices, bvt.data
                    else:
                        Bp, Bc, Bvv = SB.indptr, SB.indices, bv
                    Ar = np.repeat(np.arange(nrows), np.diff(SA.indptr))
                    cands = products_by_entry(Ar, SA.indices.astype(np.int64), av, Bp, Bc, Bvv, ncols, sr[1])
                gK = gI.astype(np.int64) * ncols + gJ.astype(np.int64)
                rK = ref.I.astype(np.int64) * ncols + ref.J.astype(np.int64)
                e = compare(gK, gX, rK, ref.X, typ, sr[0], "_".join(sr), cands)
                if e:
                    errors.append(e)
    assert calls > 0
    assert not errors, f"{len(errors)} of {calls} mxm calls differ on the {path} path:\n" + "\n".join(errors[:40])


@pytest.mark.parametrize("typ", ALL_T)
@pytest.mark.parametrize("path", list(GEMM))
def test_spgemm_edges(path, typ):
    run_gemm(path, typ)


# ------------------------------------------------------------------ operands and outputs of other types
# The multiply's operands are cast on the device (dev_cast_values) and the result is cast into C / w, through an
# accumulator: NaN -> 0, saturation, wrap-around, Inf into integer types.
MIXED = [
    # (operand type, semiring, output type, accumulator)
    ("FP64", ("PLUS", "TIMES", "INT8"), "FP32", ("PLUS", "FP32")),
    ("FP32", ("MAX", "PLUS", "FP64"), "INT16", None),
    ("UINT64", ("MIN", "FIRST", "INT32"), "UINT8", ("MAX", "INT64")),
    ("INT64", ("MIN", "SECOND", "FP32"), "UINT32", ("PLUS", "FP64")),
    ("FP64", ("TIMES", "FIRST", "UINT16"), "INT8", ("TIMES", "INT8")),
]


@pytest.mark.parametrize("case", range(len(MIXED)))
@pytest.mark.parametrize("path", ["tile-8", "run", "esc-small", "spa", "masked-warp", "stream-L", "dot"])   # MIXED_PATHS
def test_mixed_types(path, case):
    otyp, sr, ctyp, acc = MIXED[case]
    rng = np.random.default_rng(case)
    accum = util.g_accum(acc)
    if path in SPMV:
        S = spmv_pattern(SPMV[path]["shape"])
        nrows, ncols = S.shape
        av = util.rand_edge_values(rng, otyp, S.nnz, 0.5)
        uv = util.rand_edge_values(rng, otyp, ncols, 0.5)
        A = Matrix.from_csr(S.indptr, S.indices, av, nrows, ncols, util.g_type(otyp))
        u = Vector.from_numpy(uv, typ=util.g_type(otyp))
        wp = rng.random(nrows) < 0.5
        wv = util.rand_edge_values(rng, ctyp, nrows, 0.5)
        w = Vector.from_lists(np.flatnonzero(wp), wv[wp], nrows, util.g_type(ctyp))
        A.mxv(u, semiring=semiring(*sr), out=w, accum=accum)
        assert _kernels()[0].startswith("tile" if path == "tile-8" else "run"), last_kernel()
        gI, gX = w.to_arrays()
        ref = orc.mxv(orc.SpVec(ctyp, nrows, np.flatnonzero(wp), wv[wp]), None, acc, sr, o_csr(otyp, S, av),
                      orc.SpVec(otyp, ncols, np.arange(ncols), uv))
        e = compare(gI, gX, ref.I, ref.X, ctyp, sr[0], f"{path} {MIXED[case]}")
    else:
        SA, SB, SM, desc = gemm_patterns(path)
        av = util.rand_edge_values(rng, otyp, SA.nnz, 0.5)
        bv = util.rand_edge_values(rng, otyp, SB.nnz, 0.5)
        A = Matrix.from_csr(SA.indptr, SA.indices, av, *SA.shape, util.g_type(otyp))
        B = Matrix.from_csr(SB.indptr, SB.indices, bv, *SB.shape, util.g_type(otyp))
        M = Matrix.from_csr(SM.indptr, SM.indices, None, *SM.shape) if SM is not None else None
        ncols = SB.shape[0] if "T1" in desc else SB.shape[1]
        Sc = pattern(99, SA.shape[0], ncols, min(ncols, 7))
        cv = util.rand_edge_values(rng, ctyp, Sc.nnz, 0.5)
        C = Matrix.from_csr(Sc.indptr, Sc.indices, cv, SA.shape[0], ncols, util.g_type(ctyp))
        A.mxm(B, semiring=semiring(*sr), out=C, mask=M, accum=accum, desc=getattr(descriptor, desc) if desc else None)
        assert GEMM[path][1][0] in _kernels(), last_kernel()
        gI, gJ, gX = C.to_arrays()
        ref = orc.mxm(o_csr(ctyp, Sc, cv), o_csr("BOOL", SM, np.ones(SM.nnz, bool)) if SM is not None else None, acc, sr,
                      o_csr(otyp, SA, av), o_csr(otyp, SB, bv), desc)
        e = compare(gI.astype(np.int64) * ncols + gJ.astype(np.int64), gX, ref.I.astype(np.int64) * ncols + ref.J.astype(np.int64),
                    ref.X, ctyp, sr[0], f"{path} {MIXED[case]}")
    assert e is None, e


# ------------------------------------------------------------------ FP sums against the dot-product error bound
def _expand(Ar, Ac, Av, Bp, Bc, Bv, ncols):
    lens = (Bp[Ac + 1] - Bp[Ac]).astype(np.int64)
    rows = np.repeat(Ar, lens)
    starts = np.repeat(Bp[Ac].astype(np.int64) - np.concatenate(([0], np.cumsum(lens)[:-1])), lens)
    pos = np.arange(int(lens.sum())) + starts
    return rows.astype(np.int64) * ncols + Bc[pos].astype(np.int64), np.repeat(Av, lens), Bv[pos]


def check_bound(gK, gX, keys, a, b, typ, label):
    """|got - exact| <= gamma_n * sum |a b| + n * eta for every entry, n = its product count + 1."""
    dt = orc.DTYPES[typ]
    hp = np.float64 if typ == "FP32" else np.longdouble
    uk, inv = np.unique(keys, return_inverse=True)
    prod = a.astype(hp) * b.astype(hp)
    exact = np.zeros(len(uk), hp); np.add.at(exact, inv, prod)
    mag = np.zeros(len(uk), hp); np.add.at(mag, inv, np.abs(prod))
    n = np.bincount(inv, minlength=len(uk)).astype(np.float64) + 1
    u = float(np.finfo(dt).eps) / 2
    eta = hp(np.finfo(dt).smallest_subnormal) / 2          # in hp: half the FP64 subnormal is 0 in float64
    gamma = n * u / (1 - n * u)
    assert np.array_equal(np.asarray(gK, np.int64), uk), f"{label}: presence differs"
    err = np.abs(np.asarray(gX).astype(hp) - exact)
    bound = gamma.astype(hp) * mag + n.astype(hp) * eta
    bad = np.flatnonzero(~(err <= bound))
    assert len(bad) == 0, (f"{label}: {len(bad)} of {len(uk)} entries outside the error bound, e.g. got "
                           f"{np.asarray(gX)[bad[:3]].tolist()}, exact {exact[bad[:3]].astype(np.float64).tolist()}, bound {bound[bad[:3]].astype(np.float64).tolist()}")


def _general_values(rng, typ, n, scale):
    dt = orc.DTYPES[typ]
    x = rng.standard_normal(n) * np.exp2(rng.integers(-6, 7, n).astype(np.float64))
    if scale == "subnormal":        # products and sums spread over the subnormal range of the type
        x = x * (2.0 ** (-135 if typ == "FP32" else -1040))
    return x.astype(dt)


BOUND_SPMV = ["tile-8", "run", "run-sparse-u", "hot", "hot-pipe"]


@pytest.mark.parametrize("scale", ["normal", "subnormal"])
@pytest.mark.parametrize("typ", FP_T)
@pytest.mark.parametrize("path", BOUND_SPMV + [p for p in GEMM])
def test_fp_sums_within_error_bound(path, typ, scale):
    rng = np.random.default_rng(seed_of(path, typ, scale))
    s = semiring("PLUS", "TIMES", typ)
    if path in SPMV:
        cfg = SPMV[path]
        S = spmv_pattern(cfg["shape"])
        nrows, ncols = S.shape
        av = _general_values(rng, typ, S.nnz, "normal")
        uv = _general_values(rng, typ, ncols, scale)
        upres = rng.random(ncols) < 0.6 if cfg.get("sparse_u") else np.ones(ncols, bool)
        A = Matrix.from_csr(S.indptr, S.indices, av, nrows, ncols, util.g_type(typ))
        u = Vector.from_numpy(uv, present=upres if cfg.get("sparse_u") else None, typ=util.g_type(typ))
        with tunables(**cfg["env"]):
            w = A.mxv(u, semiring=s)
            ks = _kernels()
        assert entries(ks) == [_spmv_expect(path, cfg, typ, "PLUS", "TIMES", False)] if path != "tile-8" else ks[0].startswith("tile"), ks
        gI, gX = w.to_arrays()
        Ar = np.repeat(np.arange(nrows), np.diff(S.indptr))
        keep = upres[S.indices]
        check_bound(gI, gX, Ar[keep].astype(np.int64), av[keep], uv[S.indices][keep], typ, f"{path} {typ} {scale}")
    else:
        env, want = GEMM[path]
        SA, SB, SM, desc = gemm_patterns(path)
        av = _general_values(rng, typ, SA.nnz, "normal")
        bv = _general_values(rng, typ, SB.nnz, scale)
        A = Matrix.from_csr(SA.indptr, SA.indices, av, *SA.shape, util.g_type(typ))
        B = Matrix.from_csr(SB.indptr, SB.indices, bv, *SB.shape, util.g_type(typ))
        M = Matrix.from_csr(SM.indptr, SM.indices, None, *SM.shape) if SM is not None else None
        C = Matrix.sparse(util.g_type(typ), SA.shape[0], SB.shape[0] if "T1" in desc else SB.shape[1])
        with tunables(**env):
            A.mxm(B, semiring=s, out=C, mask=M, desc=getattr(descriptor, desc) if desc else None)
            ks = _kernels()
        assert all(k in ks for k in want), ks
        if "T1" in desc:
            Bt = sp.csr_matrix((bv, SB.indices, SB.indptr), shape=SB.shape).T.tocsr()
            Bt.sort_indices()
            Bp, Bc, Bvv, ncols = Bt.indptr, Bt.indices, Bt.data, SB.shape[0]
        else:
            Bp, Bc, Bvv, ncols = SB.indptr, SB.indices, bv, SB.shape[1]
        Ar = np.repeat(np.arange(SA.shape[0]), np.diff(SA.indptr))
        keys, a, b = _expand(Ar, SA.indices.astype(np.int64), av, Bp, Bc, Bvv, ncols)
        if SM is not None:
            mk = np.repeat(np.arange(SM.shape[0]), np.diff(SM.indptr)).astype(np.int64) * ncols + SM.indices
            keep = np.isin(keys, mk)
            keys, a, b = keys[keep], a[keep], b[keep]
        gI, gJ, gX = C.to_arrays()
        check_bound(gI.astype(np.int64) * ncols + gJ.astype(np.int64), gX, keys, a, b, typ, f"{path} {typ} {scale}")


# ------------------------------------------------------------------ every path of the table was reached
ALL_PATHS = {"tile (specialised, 4 items)", "tile (specialised, 8 items)", "tile (specialised, 16 items)", "tile (run-time operators)",
             "run", "run (sparse u)", "run+hot-table (TMA-staged)", "run+hot-table (TMA-staged, pipelined)", "pull", "push",
             "esc-small", "esc-medium", "hash-small", "hash-medium", "spa", "masked-warp", "stream-S", "stream-M", "stream-L", "dot"}


SPMV_CASES = ["tile-4", "tile-8", "tile-16", "run", "run-sparse-u", "pull", "push"]
MIXED_PATHS = ["tile-8", "run", "esc-small", "spa", "masked-warp", "stream-L", "dot"]
FULL_COUNT = (len(SPMV_CASES) * len(ALL_T) + 2 * len(HOT_T) + len(GEMM) * len(ALL_T) + len(MIXED_PATHS) * len(MIXED)
              + (len(BOUND_SPMV) + len(GEMM)) * len(FP_T) * 2)


def test_every_kernel_path_was_reached(request):
    mine = [it for it in request.session.items if it.module is request.module and it is not request.node]
    if len(mine) < FULL_COUNT:
        pytest.skip("only part of the module was selected")
    missing = ALL_PATHS - REACHED
    assert not missing, f"kernel paths no case reached: {sorted(missing)}"
