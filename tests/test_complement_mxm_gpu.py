"""GrB_mxm under a complemented mask, C<!M> = accum(C, A (+).(x) B): the unmasked bins (esc-small, esc-medium, spa) run with
the filter of the mask entries that block, so no blocked product is formed, and rows above SPLIT_FLOPS products run on
spa-split, spread over the GPU.  Checked against the oracle at the bin, SPLIT_FLOPS and split-group boundaries, over mask shapes, mask types, descriptors, aliasing and the other callers of the product, through the reported
nnz of the product, under allocation failures, and in multi-source BFS and the betweenness centrality of gap/bcmark.py."""
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.csgraph as csgraph

import pygraphblas_b200 as gb
from pygraphblas_b200 import Matrix, descriptor, ffi, lib
from pygraphblas_b200.generators import rmat_csr
from oracle import oracle as orc
import positional_model as pm
import util
from kernel_check import compare, entries, fp_pool_for, o_csr, record_kernels, seed_of, semiring, values
from test_alloc_failure_gpu import _sweep

pytestmark = pytest.mark.gpu

REACHED = set()
SMALL, MEDIUM = 128, 2048          # the product counts that bound the esc-small and esc-medium bins
SPLIT_FLOPS, SPLIT_BUDGET = 1 << 18, 1 << 28     # spa-split: rows above SPLIT_FLOPS, HBM buffers of one group of rows
SRS = [("PLUS", "TIMES", "FP32"), ("MIN", "PLUS", "INT32"), ("LOR", "LAND", "BOOL"), ("PLUS", "PAIR", "INT64"),
       ("MAX", "MINUS", "FP64"), ("ANY", "PAIR", "BOOL"), ("PLUS", "TIMES", "UINT8")]


# ------------------------------------------------------------------ operands
def csr(lens, ncols, seed):
    """A sorted CSR pattern with the given row lengths (capped at ncols), random distinct columns."""
    rng = np.random.default_rng(seed)
    lens = np.minimum(np.asarray(lens, np.int64), ncols)
    cols = [np.sort(rng.choice(ncols, size=int(k), replace=False)) for k in lens]
    S = sp.csr_matrix((np.ones(int(lens.sum())), np.concatenate(cols).astype(np.int64) if len(cols) else np.zeros(0, np.int64),
                       np.r_[0, np.cumsum(lens)]), shape=(len(lens), ncols))
    S.sort_indices()
    return S


def flops(SA, SB):
    return np.bincount(np.repeat(np.arange(SA.shape[0]), np.diff(SA.indptr)), weights=np.diff(SB.indptr)[SA.indices],
                       minlength=SA.shape[0]).astype(np.int64)


def route(SA, SB, blocks=True):
    """The bins of the product, chosen by the unfiltered product count of each row; when the mask blocks anything, the rows
    above SPLIT_FLOPS leave spa for spa-split."""
    f = flops(SA, SB)
    out = []
    if ((f > 0) & (f <= SMALL)).any():
        out.append("esc-small")
    if ((f > SMALL) & (f <= MEDIUM)).any():
        out.append("esc-medium")
    top = SPLIT_FLOPS if blocks else np.inf
    if ((f > MEDIUM) & (f <= top)).any():
        out.append("spa")
    if (f > top).any():
        out.append("spa-split")
    return out


def split_group_rows(ncols, zsize):
    """Rows per group of spa-split: the buffers of one row are an accumulator word per column and two bitmaps."""
    words = (ncols + 31) // 32
    return max(1, SPLIT_BUDGET // (ncols * (8 if zsize == 8 else 4) + 2 * words * 4))


def product_pattern(SA, SB):
    P = (sp.csr_matrix((np.ones(SA.nnz), SA.indices, SA.indptr), SA.shape) @
         sp.csr_matrix((np.ones(SB.nnz), SB.indices, SB.indptr), SB.shape)).tocsr()
    P.sort_indices()
    return P


def mask_shapes(SA, SB, seed):
    """A mask over the product: row 0 empty, row 1 full (ncols entries), row 2 the whole product row (blocks every product),
    the rest random entries, half of them at columns with no product."""
    P = product_pattern(SA, SB)
    nrows, ncols = P.shape
    rng = np.random.default_rng(seed)
    rows = []
    for i in range(nrows):
        pc = P.indices[P.indptr[i]:P.indptr[i + 1]]
        if i % 4 == 0:
            r = np.zeros(0, np.int64)
        elif i % 4 == 1:
            r = np.arange(ncols)
        elif i % 4 == 2:
            r = pc
        else:
            hit = rng.choice(pc, size=len(pc) // 2, replace=False) if len(pc) else np.zeros(0, np.int64)
            miss = np.setdiff1d(np.arange(ncols), pc)
            miss = rng.choice(miss, size=min(len(miss), 1 + len(pc) // 2), replace=False) if len(miss) else miss
            r = np.union1d(hit, miss)
        rows.append(np.sort(np.asarray(r, np.int64)))
    lens = [len(r) for r in rows]
    S = sp.csr_matrix((np.ones(sum(lens)), np.concatenate(rows) if rows else [], np.r_[0, np.cumsum(lens)]), shape=(nrows, ncols))
    S.sort_indices()
    return S


def mask_vals(typ, n, seed):
    """n mask values of typ: about a third false (0, and -0.0 for FP), FP NaN among the true ones."""
    rng = np.random.default_rng(seed)
    dt = orc.DTYPES[typ]
    if typ == "BOOL":
        return rng.random(n) < 0.6
    v = rng.integers(1, 100, n).astype(dt)
    z = rng.random(n) < 0.35
    v[z] = 0
    if typ in util.FP_T:
        v[z & (rng.random(n) < 0.5)] = -0.0
        v[(~z) & (rng.random(n) < 0.1)] = np.nan
    return v


def blocked_pattern(SM, mv, struct):
    """M' as a set of keys i * ncols + j: every mask entry (structural) or the entries whose value is != 0 (NaN is true)."""
    keys = np.repeat(np.arange(SM.shape[0], dtype=np.int64), np.diff(SM.indptr)) * SM.shape[1] + SM.indices
    return keys if struct else keys[np.asarray(mv) != 0]


def stats():
    fl, no = ffi.new("uint64_t*"), ffi.new("uint64_t*")
    lib.B200_last_mxm_stats(fl, no)
    return int(fl[0]), int(no[0])


def run(SA, SB, SM, label, srs=SRS, desc="C", mtype=None, accum=False, c_init=False, alias=None, want_route=True):
    """C<!M> = accum(C, A (+).(x) B) for each semiring against the oracle; asserts the bins and, for calls into an empty C
    without an accumulator, that nnz_out counts only the positions the mask does not block."""
    errors = []
    for sr in srs:
        typ, zt = sr[2], orc.semiring_ztype(sr)
        seed = seed_of("comp", label, sr)
        pool = fp_pool_for(sr[0], sr[1]) if typ in util.FP_T else "edge"
        av, bv = values(seed, typ, SA.nnz, pool, 0), values(seed + 1, typ, SB.nnz, pool, 1)
        if sr[0] == "ANY":                      # the one product value of PAIR: the fold is determined
            av, bv = np.ones(SA.nnz, bool), np.ones(SB.nnz, bool)
        A = Matrix.from_csr(SA.indptr, SA.indices, av, *SA.shape, util.g_type(typ))
        B = Matrix.from_csr(SB.indptr, SB.indices, bv, *SB.shape, util.g_type(typ))
        Ao, Bo = o_csr(typ, SA, av), o_csr(typ, SB, bv)
        nrows, ncols = SA.shape[0], SB.shape[1]
        M = Mo = None
        mv = None
        if SM is not None:
            mt = mtype or "BOOL"
            mv = np.ones(SM.nnz, bool) if mtype is None else mask_vals(mt, SM.nnz, seed + 2)
            M = Matrix.from_csr(SM.indptr, SM.indices, mv, *SM.shape, util.g_type(mt))
            Mo = o_csr(mt, SM, mv)
        if alias == "A":
            C, Co = A, Ao
        elif alias == "B":
            C, Co = B, Bo
        elif alias == "M":
            C, Co = M, Mo
        elif c_init:
            Sc = csr(np.random.default_rng(seed).integers(0, 6, nrows), ncols, seed + 3)
            cv = values(seed + 4, zt, Sc.nnz, "edge", 0)
            C, Co = Matrix.from_csr(Sc.indptr, Sc.indices, cv, nrows, ncols, util.g_type(zt)), o_csr(zt, Sc, cv)
        else:
            C, Co = Matrix.sparse(util.g_type(zt), nrows, ncols), orc.SpMat(zt, nrows, ncols)
        acc = (sr[0] if sr[0] != "ANY" else "FIRST", zt) if accum else None
        ref = orc.mxm(Co, Mo, acc, sr, Ao, Bo, desc)
        A.mxm(B, semiring=semiring(*sr), out=C, mask=M, accum=util.g_accum(acc), desc=getattr(descriptor, desc))
        ks = record_kernels(REACHED)
        if want_route:
            want = route(SA, SB, len(blocked_pattern(SM, mv, "S" in desc)) > 0)
            assert [k for k in ks if k] == want, (label, sr, ks, want)
        if SM is not None and alias is None and not c_init and not accum:
            P = product_pattern(SA, SB)
            pk = np.repeat(np.arange(nrows, dtype=np.int64), np.diff(P.indptr)) * ncols + P.indices
            free = int((~np.isin(pk, blocked_pattern(SM, mv, "S" in desc))).sum())
            assert stats()[1] == free, (label, sr, stats(), free)
        gI, gJ, gX = C.to_arrays()
        e = compare(gI.astype(np.int64) * ncols + gJ.astype(np.int64), gX, ref.I.astype(np.int64) * ncols + ref.J.astype(np.int64),
                    ref.X, zt, sr[0], f"{label} {'_'.join(sr)}")
        if e:
            errors.append(e)
    assert not errors, "\n".join(errors[:20])


# ------------------------------------------------------------------ every bin on both sides of its boundary
# row r of A has lens[r] entries into a B whose rows have one entry each: row r has exactly lens[r] products
BOUNDARY = {"128": [SMALL] * 6, "129": [SMALL + 1] * 6, "2048": [MEDIUM] * 4, "2049": [MEDIUM + 1] * 4,
            "mixed": [1, SMALL, SMALL + 1, MEDIUM, MEDIUM + 1, 5000, 0, 3]}


@pytest.mark.parametrize("ncols", [1, 31, 32, 33, 1000])
@pytest.mark.parametrize("case", list(BOUNDARY))
def test_bins_at_their_boundaries(case, ncols):
    lens = BOUNDARY[case]
    inner = max(lens) + 7
    SA = csr(lens, inner, seed_of("bnd-a", case, ncols))
    SB = csr([1] * inner, ncols, seed_of("bnd-b", case, ncols))
    assert (flops(SA, SB) == np.minimum(lens, inner)).all()
    run(SA, SB, mask_shapes(SA, SB, 3), f"bnd-{case}-{ncols}", desc="SC")
    run(SA, SB, mask_shapes(SA, SB, 4), f"bnd-{case}-{ncols}-v", srs=SRS[:3], desc="RC", mtype="FP32")


# ------------------------------------------------------------------ spa-split: SPLIT_FLOPS and the group boundary
def split_operands(nrows, ncols, extra, seed):
    """nrows rows of 256 A entries into B rows of 1024 entries: SPLIT_FLOPS products per row, plus `extra[i]` (one B row of
    1024 + extra[i] entries) for row i."""
    rng = np.random.default_rng(seed)
    inner = 256 * nrows + 1
    blen = np.full(inner, 1024)
    blen[-1] = 1024 + max(extra) if max(extra) else 1024
    SB = csr(blen, ncols, seed + 1)
    rows = [np.r_[np.arange(256 * i, 256 * i + 255), inner - 1 if extra[i] else 256 * i + 255] for i in range(nrows)]
    rows = [np.sort(r) for r in rows]
    SA = sp.csr_matrix((np.ones(256 * nrows), np.concatenate(rows), np.arange(nrows + 1) * 256), shape=(nrows, inner))
    SA.sort_indices()
    f = flops(SA, SB)
    assert (f == SPLIT_FLOPS + np.asarray(extra) * (blen[-1] - 1024 > 0)).all(), f
    return SA, SB


@pytest.mark.parametrize("extra", [0, 1])
def test_split_flops_boundary(extra):
    """Rows of exactly SPLIT_FLOPS products stay on spa, one more product takes them to spa-split."""
    SA, SB = split_operands(4, 1 << 16, [extra] * 4, seed_of("split-bnd", extra))
    SM = mask_shapes(SA, SB, 14)
    run(SA, SB, SM, f"split-bnd-{extra}", srs=SRS[:5], desc="RSC")
    run(SA, SB, SM, f"split-bnd-{extra}-v", srs=SRS[:2], desc="C", mtype="FP64", c_init=True, accum=True)
    assert ("spa-split" in REACHED) or not extra


def test_split_groups():
    """More split rows than one group holds: rows on both sides of the group boundary, and a row whose mask blocks all."""
    ncols = 1 << 22
    g = split_group_rows(ncols, 4)
    n = g + 1
    SA, SB = split_operands(n, ncols, [1] * n, seed_of("split-groups"))
    SM = mask_shapes(SA, SB, 15)
    run(SA, SB, SM, "split-groups", srs=[("PLUS", "TIMES", "FP32"), ("MIN", "PLUS", "INT32"), ("ANY", "PAIR", "BOOL")], desc="SC")
    assert "spa-split" in REACHED


def test_split_allocation_failures():
    """Allocation failures on spa-split with two groups."""
    ncols = 1 << 22
    n = split_group_rows(ncols, 4) + 1
    SA, SB = split_operands(n, ncols, [1] * n, seed_of("split-alloc"))
    SM = mask_shapes(SA, SB, 16)

    def make():
        A = Matrix.from_csr(SA.indptr, SA.indices, np.ones(SA.nnz, np.float32), *SA.shape, gb.FP32)
        B = Matrix.from_csr(SB.indptr, SB.indices, np.ones(SB.nnz, np.float32), *SB.shape, gb.FP32)
        M = Matrix.from_csr(SM.indptr, SM.indices, np.ones(SM.nnz, bool), *SM.shape, gb.BOOL)
        return A, B, M

    def call(A, B, M):
        C = A.mxm(B, semiring=gb.FP32.PLUS_TIMES, mask=M, desc=descriptor.RSC)
        assert "spa-split" in record_kernels(REACHED)
        return C

    def check(ref):
        I, J, X = ref
        P = product_pattern(SA, SB)
        pk = np.repeat(np.arange(P.shape[0], dtype=np.int64), np.diff(P.indptr)) * ncols + P.indices
        keep = ~np.isin(pk, blocked_pattern(SM, None, True))
        assert np.array_equal(np.asarray(I, np.int64) * ncols + J, pk[keep]) and np.array_equal(X, P.data[keep].astype(np.float32))

    assert _sweep(make, call, check) > 1


# ------------------------------------------------------------------ mask shapes
def _operands(seed, nrows=60, ncols=700, heavy=True):
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, 40, nrows)
    if heavy:
        lens[:3] = [300, 600, 2]                 # with B rows of ~12: spa, spa and esc rows
    SA = csr(lens, 800, seed)
    SB = csr(rng.integers(0, 24, 800), ncols, seed + 1)
    return SA, SB


@pytest.mark.parametrize("shape", ["empty", "all-false", "no-rows", "full-rows", "blocks-all", "off-product"])
def test_mask_shapes(shape):
    SA, SB = _operands(seed_of("shape", shape))
    nrows, ncols = SA.shape[0], SB.shape[1]
    P = product_pattern(SA, SB)
    mtype = None
    if shape == "empty":
        SM = sp.csr_matrix((nrows, ncols))
    elif shape == "all-false":
        SM = mask_shapes(SA, SB, 5)
        mtype = "ZERO"
    elif shape == "no-rows":
        SM = csr([0] * (nrows - 1) + [5], ncols, 1)
    elif shape == "full-rows":
        SM = csr([ncols] * nrows, ncols, 1)
    elif shape == "blocks-all":
        SM = P.copy()
    else:                                       # only columns where the row has no product
        SM = (sp.csr_matrix(np.ones((nrows, ncols))) - P.astype(bool).astype(float)).tocsr()
        SM.eliminate_zeros()
        SM.sort_indices()
    if mtype == "ZERO":                         # a valued mask whose every entry is false: nothing blocks
        for d in ("C", "RC"):
            _run_valued_zero(SA, SB, SM, d)
        return
    for d in ("C", "SC", "RSC"):
        run(SA, SB, SM, f"shape-{shape}-{d}", desc=d)


def _run_valued_zero(SA, SB, SM, desc):
    for typ in ("FP32", "INT8"):
        sr = ("PLUS", "TIMES", "INT64")
        A = Matrix.from_csr(SA.indptr, SA.indices, np.ones(SA.nnz, np.int64), *SA.shape, gb.INT64)
        B = Matrix.from_csr(SB.indptr, SB.indices, np.ones(SB.nnz, np.int64), *SB.shape, gb.INT64)
        mv = np.zeros(SM.nnz, orc.DTYPES[typ])
        if typ == "FP32":
            mv[::2] = -0.0
        M = Matrix.from_csr(SM.indptr, SM.indices, mv, *SM.shape, util.g_type(typ))
        C = A.mxm(B, semiring=semiring(*sr), mask=M, desc=getattr(descriptor, desc))
        assert entries(record_kernels(REACHED)) == route(SA, SB)
        P = product_pattern(SA, SB)
        I, J, X = C.to_arrays()
        assert np.array_equal(np.asarray(I, np.int64) * SB.shape[1] + J, np.repeat(np.arange(P.shape[0]), np.diff(P.indptr)) * SB.shape[1] + P.indices)
        assert np.array_equal(X, P.data.astype(np.int64))


# ------------------------------------------------------------------ mask types
MASK_T = ["BOOL", "INT8", "UINT16", "INT32", "FP32", "UINT64", "FP64"]


@pytest.mark.parametrize("struct", [False, True])
@pytest.mark.parametrize("mtype", MASK_T)
def test_mask_types(mtype, struct):
    SA, SB = _operands(seed_of("mtype", mtype))
    SM = mask_shapes(SA, SB, seed_of("mtype-m", mtype))
    run(SA, SB, SM, f"mtype-{mtype}-{struct}", srs=SRS[:4], desc="SC" if struct else "C", mtype=mtype)
    run(SA, SB, SM, f"mtype-{mtype}-{struct}-r", srs=SRS[4:], desc="RSC" if struct else "RC", mtype=mtype)


# ------------------------------------------------------------------ descriptors, accumulator, C, aliasing, casts
@pytest.mark.parametrize("c_init", [False, True])
@pytest.mark.parametrize("accum", [False, True])
@pytest.mark.parametrize("desc", ["C", "RC", "SC", "RSC"])
def test_descriptors(desc, accum, c_init):
    SA, SB = _operands(seed_of("desc", desc, accum, c_init))
    SM = mask_shapes(SA, SB, 9)
    run(SA, SB, SM, f"desc-{desc}-{accum}-{c_init}", desc=desc, accum=accum, c_init=c_init,
        mtype=None if "S" in desc else "INT16")


@pytest.mark.parametrize("desc", ["C", "RC", "SC", "RSC"])
@pytest.mark.parametrize("who", ["A", "B", "M"])
def test_output_aliases_an_input(who, desc):
    n = 500
    rng = np.random.default_rng(seed_of("alias", who, desc))
    lens = rng.integers(0, 20, n)
    lens[:2] = [400, 150]
    S = csr(lens, n, 7)
    SM = csr(rng.integers(0, 60, n), n, 8)
    srs = [("PLUS", "TIMES", "FP32"), ("MIN", "PLUS", "INT32"), ("LOR", "LAND", "BOOL")]
    if who == "M":
        # C is the mask itself: the mask keeps its type, the semiring's z type is the mask's type
        for sr in srs:
            run(S, S, SM, f"alias-M-{desc}-{sr}", srs=[sr], desc=desc, mtype=sr[2], alias="M")
    else:
        run(S, S, SM if who == "A" else S, f"alias-{who}-{desc}", srs=srs, desc=desc, alias=who)


@pytest.mark.parametrize("desc", ["CT0", "RSCT0"])
def test_transposed_a(desc):
    """T0: A's cached transpose feeds the bins; the mask rows are rows of A'."""
    SA, SB = _operands(seed_of("t0", desc))
    SAt = SA.T.tocsr()
    SAt.sort_indices()
    SM = mask_shapes(SA, SB, 10)
    for sr in SRS[:4]:
        typ, zt = sr[2], orc.semiring_ztype(sr)
        seed = seed_of("t0v", desc, sr)
        pool = fp_pool_for(sr[0], sr[1]) if typ in util.FP_T else "edge"
        av, bv = values(seed, typ, SAt.nnz, pool, 0), values(seed + 1, typ, SB.nnz, pool, 1)
        At = Matrix.from_csr(SAt.indptr, SAt.indices, av, *SAt.shape, util.g_type(typ))
        B = Matrix.from_csr(SB.indptr, SB.indices, bv, *SB.shape, util.g_type(typ))
        M = Matrix.from_csr(SM.indptr, SM.indices, np.ones(SM.nnz, bool), *SM.shape, gb.BOOL)
        C = Matrix.sparse(util.g_type(zt), SA.shape[0], SB.shape[1])
        for rep in range(2):                    # the second call reuses the cached transpose
            At.mxm(B, semiring=semiring(*sr), out=C, mask=M, desc=getattr(descriptor, desc))
            assert entries(record_kernels(REACHED)) == route(SA, SB)
        ref = orc.mxm(orc.SpMat(zt, SA.shape[0], SB.shape[1]), o_csr("BOOL", SM, np.ones(SM.nnz, bool)), None, sr,
                      o_csr(typ, SAt, av), o_csr(typ, SB, bv), desc)
        gI, gJ, gX = C.to_arrays()
        n = SB.shape[1]
        assert compare(gI.astype(np.int64) * n + gJ, gX, ref.I.astype(np.int64) * n + ref.J, ref.X, zt, sr[0], desc) is None


@pytest.mark.parametrize("desc", ["CT1", "RSCT1"])
def test_transposed_b(desc):
    """T1: B's cached transpose feeds the same bins."""
    SA, SB = _operands(seed_of("t1", desc))
    SBt = SB.T.tocsr()
    SBt.sort_indices()
    SM = mask_shapes(SA, SB, 11)
    for sr in SRS[:4]:
        typ, zt = sr[2], orc.semiring_ztype(sr)
        seed = seed_of("t1v", desc, sr)
        pool = fp_pool_for(sr[0], sr[1]) if typ in util.FP_T else "edge"
        av, bv = values(seed, typ, SA.nnz, pool, 0), values(seed + 1, typ, SBt.nnz, pool, 1)
        A = Matrix.from_csr(SA.indptr, SA.indices, av, *SA.shape, util.g_type(typ))
        Bt = Matrix.from_csr(SBt.indptr, SBt.indices, bv, *SBt.shape, util.g_type(typ))
        M = Matrix.from_csr(SM.indptr, SM.indices, np.ones(SM.nnz, bool), *SM.shape, gb.BOOL)
        C = Matrix.sparse(util.g_type(zt), SA.shape[0], SB.shape[1])
        for rep in range(2):                    # the second call reuses the cached transpose
            A.mxm(Bt, semiring=semiring(*sr), out=C, mask=M, desc=getattr(descriptor, desc))
            assert entries(record_kernels(REACHED)) == route(SA, SB)
        ref = orc.mxm(orc.SpMat(zt, SA.shape[0], SB.shape[1]), o_csr("BOOL", SM, np.ones(SM.nnz, bool)), None, sr,
                      o_csr(typ, SA, av), o_csr(typ, SBt, bv), desc)
        gI, gJ, gX = C.to_arrays()
        n = SB.shape[1]
        assert compare(gI.astype(np.int64) * n + gJ, gX, ref.I.astype(np.int64) * n + ref.J, ref.X, zt, sr[0], desc) is None


def test_casts():
    """INT8 operands into an FP64 semiring, a FP32 C: operand and output casts around the filtered product."""
    SA, SB = _operands(seed_of("casts"))
    SM = mask_shapes(SA, SB, 12)
    rng = np.random.default_rng(5)
    av, bv = rng.integers(-4, 5, SA.nnz).astype(np.int8), rng.integers(-4, 5, SB.nnz).astype(np.int8)
    A = Matrix.from_csr(SA.indptr, SA.indices, av, *SA.shape, gb.INT8)
    B = Matrix.from_csr(SB.indptr, SB.indices, bv, *SB.shape, gb.INT8)
    M = Matrix.from_csr(SM.indptr, SM.indices, np.ones(SM.nnz, bool), *SM.shape, gb.BOOL)
    for desc in ("SC", "RSC"):
        C = Matrix.sparse(gb.FP32, SA.shape[0], SB.shape[1])
        A.mxm(B, semiring=gb.FP64.PLUS_TIMES, out=C, mask=M, desc=getattr(descriptor, desc))
        ref = orc.mxm(orc.SpMat("FP32", *C.shape), o_csr("BOOL", SM, np.ones(SM.nnz, bool)), None, ("PLUS", "TIMES", "FP64"),
                      o_csr("INT8", SA, av), o_csr("INT8", SB, bv), desc)
        gI, gJ, gX = C.to_arrays()
        n = SB.shape[1]
        assert compare(gI.astype(np.int64) * n + gJ, gX, ref.I.astype(np.int64) * n + ref.J, ref.X, "FP32", "PLUS", desc) is None


# ------------------------------------------------------------------ the other callers of the product
POS_SR = [("MIN", "SECONDI", "INT64"), ("PLUS", "FIRSTJ1", "INT32"), ("MAX", "FIRSTI", "INT64"), ("PLUS", "SECONDJ1", "INT32")]


def _dict(M):
    I, J, X = M.to_lists()
    return {(int(i), int(j)): x for i, j, x in zip(I, J, X)}


def _mat(d, typ, nrows, ncols):
    I, J = zip(*sorted(d)) if d else ((), ())
    return Matrix.from_lists(list(I), list(J), [d[e] for e in sorted(d)], nrows, ncols, util.g_type(typ))


def _pdesc(form):
    return dict(replace="R" in form, mask_comp="C" in form, mask_struct="S" in form, tran0="T0" in form, tran1="T1" in form)


@pytest.mark.parametrize("hyper", [False, True])
@pytest.mark.parametrize("desc", ["SC", "RC"])
def test_positional_and_hypersparse(desc, hyper):
    """Positional semirings in the inner (FIRSTJ / SECONDI) and count (FIRSTI / SECONDJ) forms, and 2^60-sized operands whose
    product runs in the compact space, under a complemented mask."""
    rng = np.random.default_rng(seed_of("pos", desc, hyper))
    n = 150
    A = {(int(i), int(j)): float(v) for i, j, v in zip(rng.integers(0, n, 2500), rng.integers(0, n, 2500), rng.integers(1, 5, 2500))}
    for j in range(n):
        A[(0, j)] = 1.0                                 # row 0: n * ~17 products, the spa bin
    B = {(int(i), int(j)): 1 for i, j in zip(rng.integers(0, n, 3000), rng.integers(0, n, 3000))}
    Mv = {(int(i), int(j)): bool(rng.random() < 0.7) for i, j in zip(rng.integers(0, n, 6000), rng.integers(0, n, 6000))}
    dim = (1 << 60) if hyper else n
    sh = (lambda d: {(i * (1 << 40) + 5, j * (1 << 40) + 5): v for (i, j), v in d.items()}) if hyper else (lambda d: d)
    A, B, Mv = sh(A), sh(B), sh(Mv)
    Am, Bm, Mm = _mat(A, "FP32", dim, dim), _mat(B, "INT8", dim, dim), _mat(Mv, "BOOL", dim, dim)
    for sr in POS_SR:
        C = Matrix.sparse(util.g_type(sr[2]), dim, dim)
        Am.mxm(Bm, semiring=getattr(util.g_type(sr[2]), f"{sr[0]}_{sr[1]}"), out=C, mask=Mm, desc=getattr(descriptor, desc))
        ks = record_kernels(REACHED)
        form = "positional=inner" if sr[1].rstrip("1") in ("FIRSTJ", "SECONDI") else "positional=count"
        assert form in ks and "spa" in ks, (sr, ks)
        want, _ = pm.mxm({}, sr[2], Mv, None, sr, A, B, _pdesc(desc))
        got = {k: int(v) for k, v in _dict(C).items()}
        assert got == {k: int(v) for k, v in want.items()}, (desc, hyper, sr)
    # a value semiring (small integers: every sum is exact) against a dict model
    want = {}
    rows_b = {}
    for (k, j), v in B.items():
        rows_b.setdefault(k, []).append((j, v))
    for (i, k), a in A.items():
        for j, b in rows_b.get(k, ()):
            want[(i, j)] = want.get((i, j), 0.0) + a * b
    block = {k for k, v in Mv.items() if v or "S" in desc}
    want = {k: v for k, v in want.items() if k not in block}
    Bf = _mat({k: float(v) for k, v in B.items()}, "FP32", dim, dim)
    C = Am.mxm(Bf, semiring=gb.FP32.PLUS_TIMES, mask=Mm, desc=getattr(descriptor, desc))
    assert "spa" in record_kernels(REACHED)
    assert {k: float(v) for k, v in _dict(C).items()} == want, (desc, hyper)


# ------------------------------------------------------------------ allocation failures
@pytest.mark.parametrize("valued", [False, True])
def test_allocation_failures(valued):
    SA, SB = _operands(seed_of("alloc", valued))
    SM = mask_shapes(SA, SB, 13)
    mv = mask_vals("FP32", SM.nnz, 3) if valued else np.ones(SM.nnz, bool)

    def make():
        A = Matrix.from_csr(SA.indptr, SA.indices, np.ones(SA.nnz, np.float32), *SA.shape, gb.FP32)
        B = Matrix.from_csr(SB.indptr, SB.indices, np.ones(SB.nnz, np.float32), *SB.shape, gb.FP32)
        M = Matrix.from_csr(SM.indptr, SM.indices, mv, *SM.shape, gb.FP32 if valued else gb.BOOL)
        return A, B, M

    def call(A, B, M):
        return A.mxm(B, semiring=gb.FP32.PLUS_TIMES, mask=M, desc=descriptor.RC if valued else descriptor.RSC)

    def check(ref):
        I, J, X = ref
        P = product_pattern(SA, SB)
        n = SB.shape[1]
        pk = np.repeat(np.arange(P.shape[0], dtype=np.int64), np.diff(P.indptr)) * n + P.indices
        keep = ~np.isin(pk, blocked_pattern(SM, mv, not valued))
        assert np.array_equal(np.asarray(I, np.int64) * n + J, pk[keep]) and np.array_equal(X, P.data[keep].astype(np.float32))

    assert _sweep(make, call, check) > 1


# ------------------------------------------------------------------ algorithms
def _rmat(scale, seed=1, ef=8):
    n, indptr, indices = rmat_csr(scale, ef, seed=seed)
    S = sp.csr_matrix((np.ones(len(indices), np.float32), indices, indptr), shape=(n, n))
    S.sort_indices()
    return n, S


def ms_bfs(A, n, sources, semiring_):
    """Levels of a k-source BFS: F<!V, R> = F (+).(x) A, V += F.  Returns a k x n level array (-1 unreached) and the bins."""
    k = len(sources)
    F = Matrix.from_lists(list(range(k)), list(sources), [True] * k, k, n, gb.BOOL)
    V = F.dup()
    lev = np.full((k, n), -1, np.int64)
    lev[np.arange(k), sources] = 0
    seen = set()
    for d in range(1, n + 1):
        F.mxm(A, semiring=semiring_, out=F, mask=V, desc=descriptor.RSC)
        seen.update(entries(record_kernels(REACHED)))
        if F.nvals == 0:
            break
        I, J, _ = F.to_arrays()
        assert (lev[I, J] == -1).all()
        lev[I, J] = d
        V.eadd(F, gb.BOOL.LOR, out=V)
    return lev, seen


@pytest.mark.parametrize("scale,k", [(10, 4), (11, 64), (12, 4), (17, 4)])
def test_multi_source_bfs(scale, k):
    n, S = _rmat(scale, ef=16 if scale > 12 else 8)
    A = Matrix.from_csr(S.indptr, S.indices, np.ones(S.nnz, bool), n, n, gb.BOOL)
    deg = np.diff(S.indptr)
    sources = np.argsort(-deg, kind="stable")[:k]
    want = csgraph.shortest_path(S, unweighted=True, indices=sources)
    want = np.where(np.isinf(want), -1, want).astype(np.int64)
    for sr in (gb.BOOL.ANY_PAIR, gb.BOOL.LOR_LAND):
        lev, seen = ms_bfs(A, n, sources, sr)
        assert np.array_equal(lev, want)
        assert ("spa-split" if scale > 12 else "spa") in seen, seen


def brandes(S, sources):
    """Sum over the sources of the dependencies delta_s(v) (v != s), unweighted directed graph, in float64."""
    n = S.shape[0]
    out = np.zeros(n)
    for s in sources:
        dist = csgraph.shortest_path(S, unweighted=True, indices=[s])[0]
        sigma = np.zeros(n)
        sigma[s] = 1
        levels = []
        d = 0
        while True:
            lv = np.flatnonzero(dist == d)
            if not len(lv):
                break
            levels.append(lv)
            d += 1
        C = S.tocoo()
        for d in range(1, len(levels)):
            e = (dist[C.row] == d - 1) & (dist[C.col] == d)
            np.add.at(sigma, C.col[e], sigma[C.row[e]])
        delta = np.zeros(n)
        for d in range(len(levels) - 1, 0, -1):
            e = (dist[C.row] == d - 1) & (dist[C.col] == d)
            np.add.at(delta, C.row[e], sigma[C.row[e]] / sigma[C.col[e]] * (1 + delta[C.col[e]]))
        delta[s] = 0
        out += delta
    return out


def bc_round(sources, AT, A, n):
    """gap/bcmark.py's bc(), with RC for its `oocr` descriptor and GrB_Matrix_assign for `assign_matrix`."""
    ns = len(sources)
    paths = Matrix.from_lists(np.repeat(np.arange(ns), n), np.tile(np.arange(n), ns), np.zeros(ns * n, np.float32), ns, n, gb.FP32)
    frontier = Matrix.sparse(gb.FP32, ns, n)
    for i, s in enumerate(sources):
        paths[i, int(s)] = 1.0
        frontier[i, int(s)] = 1.0
    frontier.mxm(A, out=frontier, mask=paths, semiring=gb.FP32.PLUS_FIRST, desc=descriptor.RC)
    seen = set(entries(record_kernels(REACHED)))
    S = []
    depth = 0
    for depth in range(n):
        if frontier.nvals == 0:
            break
        s = Matrix.sparse(gb.BOOL, ns, n)
        frontier.apply(gb.BOOL.ONE, out=s)
        S.append(s)
        gb.base._check(lib.GrB_Matrix_assign(paths._matrix[0], ffi.NULL, gb.FP32.PLUS.get_op(), frontier._matrix[0],
                                             lib.GrB_ALL, ns, lib.GrB_ALL, n, ffi.NULL))
        frontier.mxm(A, out=frontier, mask=paths, semiring=gb.FP32.PLUS_FIRST, desc=descriptor.RC)
        seen.update(entries(record_kernels(REACHED)))
    bc = Matrix.from_lists(np.repeat(np.arange(ns), n), np.tile(np.arange(n), ns), np.ones(ns * n, np.float32), ns, n, gb.FP32)
    W = Matrix.sparse(gb.FP32, ns, n)
    for i in range(depth - 1, 0, -1):
        bc.emult(paths, gb.FP32.DIV, out=W, mask=S[i], desc=descriptor.R)
        W.mxm(AT, out=W, mask=S[i - 1], semiring=gb.FP32.PLUS_FIRST, desc=descriptor.R)
        W.emult(paths, gb.FP32.TIMES, out=bc, accum=gb.FP32.PLUS)
    _, J, X = bc.to_arrays()
    cent = np.full(n, -float(ns))
    np.add.at(cent, J, X.astype(np.float64))
    return cent, seen


@pytest.mark.parametrize("scale", [10, 11])
def test_betweenness_centrality(scale):
    n, S = _rmat(scale, seed=3)
    A = Matrix.from_csr(S.indptr, S.indices, np.ones(S.nnz, np.float32), n, n, gb.FP32)
    ST = S.T.tocsr()
    ST.sort_indices()
    AT = Matrix.from_csr(ST.indptr, ST.indices, np.ones(ST.nnz, np.float32), n, n, gb.FP32)
    deg = np.diff(S.indptr)
    order = np.argsort(-deg, kind="stable")
    seen = set()
    for r in range(2):
        sources = order[4 * r:4 * r + 4]
        cent, sn = bc_round(sources, AT, A, n)
        seen |= sn
        want = brandes(S, sources)
        assert np.allclose(cent, want, rtol=1e-4, atol=1e-5 * max(1.0, np.abs(want).max())), (scale, r)
    assert "spa" in seen, seen
