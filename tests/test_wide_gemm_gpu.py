"""The wide route of the unmasked and complemented-mask bins of mxm (C = A (+).(x) B and C<!M> = A (+).(x) B) on matrices with
2^32 or more entries.

The wide route runs the esc-small, esc-medium, spa and spa-split bins on row panels of A and of M' (the mask's blocking
entries), whose offsets are rebased to 32 bits, and reads B's 64-bit offsets when B is wide.  B200_debug_wide_gemm(chunk,
limit, budget) puts every such product on that route with panels of at most `chunk` entries, so the first part runs each case
narrow and then wide on fresh operands at chunks 7, 3000 and 2^30.  Each wide run must list the narrow entries with
`offsets=64` after the first, form the same pattern and the same value bits (the ESC bins fold in Gustavson order; the value
pools make the atomic folds of spa / spa-split exact in any order, and general FP values are checked against the exact sum
within the gamma_n bound), and agree with the oracle.  The size rule (results of 2^32 or more entries are refused) is reached
with a small limit.  The second part builds a real matrix of 2^32 + 2^26 entries on the device as kron(G, J) and checks the
coarsening products A P and P' A and a multi-source BFS against identities on the small factors; it skips, with the reason,
when the card lacks the free memory."""
import contextlib

import numpy as np
import pytest
import scipy.sparse as sp

import pygraphblas_b200 as gb
from pygraphblas_b200 import Matrix, Vector, descriptor, ffi, lib
from oracle import oracle as orc
import kernel_check as kc
import positional_model as pm
import util
from test_alloc_failure_gpu import _mat, _same_csr, _sweep
from test_complement_mxm_gpu import SPLIT_FLOPS, route as comp_route
from test_route_edges_gpu import partial_mask
from test_structure_edges_gpu import GEMM_SRS, csr, mask_values, pool_of, unmasked_operands
from test_value_edges_gpu import _expand, check_bound
from test_wide_mxm_gpu import trim_pool
from test_wide_offsets_gpu import GB_, Memory, factor

pytestmark = pytest.mark.gpu

ENTRIES = ("esc-small", "esc-medium", "spa", "spa-split")
CHUNKS = (7, 3000, 1 << 30)


@contextlib.contextmanager
def wide_gemm(chunk, limit=0, budget=0):
    lib.B200_debug_wide_gemm(chunk, limit, budget)
    try:
        yield
    finally:
        lib.B200_debug_wide_gemm(0, 0, 0)


def _keys(I, J, ncols):
    return np.asarray(I, np.int64) * ncols + np.asarray(J, np.int64)


def _tokens():
    return kc.last_kernel().split(";")


def _stats():
    f, o = ffi.new("uint64_t*"), ffi.new("uint64_t*")
    lib.B200_last_mxm_stats(f, o)
    return int(f[0]), int(o[0])


def widened(nt):
    """The tokens of the wide route: the narrow ones with offsets=64 after the first bin"""
    if not any(k in ENTRIES for k in nt):
        return nt
    at = next(i for i, k in enumerate(nt) if k in ENTRIES) + 1
    return nt[:at] + ["offsets=64"] + nt[at:]


def twice(run, add, zt, chunks=CHUNKS, bits=True):
    """run() builds fresh operands, makes one mxm and returns (C, tokens); it runs narrow, then wide at each chunk.  Each wide
    result must have the narrow tokens (plus offsets=64), pattern, stats and, when `bits` (and add is not ANY), values as
    kernel_check.compare has them.  Returns the narrow tuples and tokens and the wide tuples of each chunk."""
    C, nt = run()
    stats = _stats()
    nI, nJ, nX = C.to_arrays()
    ncols = C.ncols
    assert "offsets=64" not in nt, nt
    wides = []
    for chunk in chunks:
        with wide_gemm(chunk):
            C, gt = run()
            assert _stats() == stats, (chunk, _stats(), stats)
        gI, gJ, gX = C.to_arrays()
        assert gt == widened(nt), (chunk, nt, gt)
        assert np.array_equal(nI, gI) and np.array_equal(nJ, gJ), chunk
        if bits and add != "ANY":
            e = kc.compare(_keys(gI, gJ, ncols), gX, _keys(nI, nJ, ncols), nX, zt, add, f"wide {chunk} vs narrow")
            assert e is None, e
        wides.append((gI, gJ, gX))
    return (nI, nJ, nX), nt, wides


def gemm_twice(SA, SB, desc, label, sr, SM=None, mask_type=None, c_init=False, accum=False, alias=False, chunks=CHUNKS):
    """C<!M> = accum(C, op(A) (+).(x) op(B)) (SM None: no mask) narrow and wide, then the oracle.  SA is op(A) (stored
    transposed when desc holds T0), SB is B as stored; mask_type: None (structural BOOL) or a valued type with false entries
    and an all-false row; alias: C = A = B (SB ignored).  Returns the narrow tokens."""
    add, _, typ = sr
    zt, pool = orc.semiring_ztype(sr), pool_of(sr)
    seed = kc.seed_of("wide-gemm", label, sr)
    if alias:
        SB = SA
    t0 = "T0" in desc
    SAs = SA.T.tocsr() if t0 else SA
    SAs.sort_indices()
    av = kc.values(seed, typ, SAs.nnz, pool, 0)
    bv = av if alias else kc.values(seed + 1, typ, SB.nnz, pool, 1)
    nrows, ncols = SA.shape[0], (SB.shape[0] if "T1" in desc else SB.shape[1])
    mt, mv = "BOOL", None
    if SM is not None:
        mv = np.ones(SM.nnz, bool)
        if mask_type is not None:
            mt = mask_type
            mv = mask_values(mask_type, SM.nnz, np.random.default_rng(seed + 2))
            r = int(np.argmax(np.diff(SM.indptr) > 0))            # the first non-empty mask row: all false
            mv[SM.indptr[r]:SM.indptr[r + 1]] = 0
    Sc = cv = None
    if c_init:
        Sc = csr(np.minimum(np.random.default_rng(seed).integers(0, 6, nrows), ncols), ncols, seed + 3)
        cv = kc.values(seed + 4, zt, Sc.nnz, pool if zt == typ else "edge", 0)
    acc = (add if add != "ANY" else "FIRST", zt) if accum else None

    def run():
        A = Matrix.from_csr(SAs.indptr, SAs.indices, av, *SAs.shape, util.g_type(typ))
        B = A if alias else Matrix.from_csr(SB.indptr, SB.indices, bv, *SB.shape, util.g_type(typ))
        M = None if SM is None else Matrix.from_csr(SM.indptr, SM.indices, mv, *SM.shape, util.g_type(mt))
        if alias:
            C = A
        elif c_init:
            C = Matrix.from_csr(Sc.indptr, Sc.indices, cv, nrows, ncols, util.g_type(zt))
        else:
            C = Matrix.sparse(util.g_type(zt), nrows, ncols)
        A.mxm(B, semiring=kc.semiring(*sr), out=C, mask=M, accum=util.g_accum(acc), desc=getattr(descriptor, desc) if desc else None)
        return C, _tokens()

    (nI, nJ, nX), nt, wides = twice(run, add, zt, chunks)
    Bop = SB.T.tocsr() if "T1" in desc else SB
    blocks = SM is not None and (mv != 0).any()
    assert [k for k in nt if k] == comp_route(SA, Bop, blocks), (label, sr, nt)
    Ao, Bo = kc.o_csr(typ, SAs, av), kc.o_csr(typ, SB, bv)
    Mo = None if SM is None else kc.o_csr(mt, SM, mv)
    Co = Ao if alias else (kc.o_csr(zt, Sc, cv) if c_init else orc.SpMat(zt, nrows, ncols))
    ref = orc.mxm(Co, Mo, acc, sr, Ao, Bo, desc)
    cands = None
    if add == "ANY":
        if accum or c_init or alias or "T" in desc:
            return nt
        cands = kc.products_by_entry(np.repeat(np.arange(nrows), np.diff(SA.indptr)), SA.indices.astype(np.int64), av,
                                     Bop.indptr, Bop.indices, bv, ncols, sr[1])
    for gI, gJ, gX in [(nI, nJ, nX)] + wides:
        e = kc.compare(_keys(gI, gJ, ncols), gX, _keys(ref.I, ref.J, ncols), ref.X, zt, add, f"{label} {'_'.join(sr)}", cands)
        assert e is None, e
    return nt


# ------------------------------------------------------------------ operands
def _pad_rows(S, before, after):
    """S with empty rows before and after it: panels of empty rows only"""
    Z = lambda k: sp.csr_matrix((k, S.shape[1]), dtype=S.dtype)
    T = sp.vstack([Z(before), S, Z(after)], format="csr")
    T.sort_indices()
    return T


def bins_operands():
    """unmasked_operands (rows of 0, 1, 128, 129, 2048, 2049, 200, 2100 and 200 products) with empty rows around them"""
    SA, SB = unmasked_operands()
    return _pad_rows(SA, 3, 20), SB


def split_operands():
    """B: 130 rows of 2048 entries, then rows of 1 entry.  A: rows of exactly SPLIT_FLOPS products (spa) and one more B row
    (spa-split), an esc-medium row of 2048 products and esc-small rows; empty rows."""
    nc = 4096
    SB = csr([2048] * 130 + [1] * 200, nc, seed=31)
    arows = [[], list(range(128)), [5], list(range(129)), [], list(range(130, 140)), [7], list(range(130)) + [200], []]
    SA = csr([len(r) for r in arows], SB.shape[0], cols={i: r for i, r in enumerate(arows) if r})
    f = np.bincount(np.repeat(np.arange(SA.shape[0]), np.diff(SA.indptr)), weights=np.diff(SB.indptr)[SA.indices], minlength=SA.shape[0])
    assert f[1] == SPLIT_FLOPS and f[3] == SPLIT_FLOPS + 2048 and f[6] == 2048
    return SA, SB


# ------------------------------------------------------------------ every bin, every chunk of the panels
def test_bins_fast_and_generic():
    """esc-small / esc-medium on both sides of 128 and 2048 products, spa above; rows longer than the chunk; empty rows and
    panels of empty rows; every semiring of GEMM_SRS (fast and generic instantiations, BOOL, ANY, the edge values)."""
    SA, SB = bins_operands()
    for sr in GEMM_SRS:
        assert gemm_twice(SA, SB, "", "bins", sr) == ["esc-small", "esc-medium", "spa"]


@pytest.mark.parametrize("case", [("SC", None), ("RSC", None), ("C", "INT32"), ("RC", "FP64")], ids=lambda c: c[0] + (c[1] or ""))
def test_complemented_split(case):
    """A complemented structural or valued mask (with an all-false row) that blocks part of every row: the bins on both sides
    of SPLIT_FLOPS (spa / spa-split)."""
    desc, mt = case
    SA, SB = split_operands()
    SM = partial_mask(SA, SB, 41)
    srs = GEMM_SRS if desc == "SC" else GEMM_SRS[::3]
    for sr in srs:
        nt = gemm_twice(SA, SB, desc, f"split-{desc}", sr, SM=SM, mask_type=mt, c_init="R" in desc)
        assert nt == ["esc-small", "esc-medium", "spa", "spa-split"], nt


def test_complemented_bins():
    SA, SB = bins_operands()
    SM = partial_mask(SA, SB, 43)
    for sr in GEMM_SRS[:4]:
        gemm_twice(SA, SB, "SC", "bins-sc", sr, SM=SM)


# (name, desc, C holds entries, accum)
WRITE_BACK = [("accum", "", True, True), ("T0", "T0", False, False), ("T1", "T1", False, False),
              ("accum-comp", "SC", True, True)]


@pytest.mark.parametrize("case", WRITE_BACK, ids=[c[0] for c in WRITE_BACK])
def test_write_back(case):
    name, desc, c_init, accum = case
    SA, SB = bins_operands()
    SM = partial_mask(SA, SB, 47) if "C" in desc else None
    if "T1" in desc:
        SB = SB.T.tocsr()
        SB.sort_indices()
    for sr in GEMM_SRS[:5]:
        gemm_twice(SA, SB, desc, f"wb-{name}", sr, SM=SM, c_init=c_init, accum=accum)


def test_alias():
    """C = A = B: A = A (+).(x) A in place"""
    SA = csr(np.random.default_rng(11).integers(0, 30, 400), 400, seed=12)
    for sr in [("PLUS", "TIMES", "INT64"), ("MIN", "PLUS", "INT32"), ("PLUS", "TIMES", "FP64"), ("LOR", "LAND", "BOOL")]:
        gemm_twice(SA, None, "", "alias", sr, alias=True)


def test_one_side_shapes():
    """The shapes of the coarsening products: A P (P an n x k one-hot assignment: the wide operand is A) and P' A (the wide
    operand is B), with spa rows on P' A.  The seam makes every operand wide, so B's offsets are 64-bit in both here; the
    uint32_t instantiations on the wide route (A or the mask wide, B narrow) run in the real-size A P below, as on the masked
    route."""
    n, k = 3000, 8
    SA = csr(np.random.default_rng(13).integers(0, 40, n), n, seed=14)
    rng = np.random.default_rng(15)
    P = sp.csr_matrix((np.ones(n), (np.arange(n), rng.integers(0, k, n))), shape=(n, k))
    P.sort_indices()
    Pt = P.T.tocsr()
    Pt.sort_indices()
    for sr in [("PLUS", "TIMES", "INT64"), ("PLUS", "TIMES", "FP64"), ("MIN", "PLUS", "INT32")]:
        gemm_twice(SA, P, "", "a-p", sr)
        assert "spa" in gemm_twice(Pt, SA, "", "pt-a", sr)


def test_general_fp_sums():
    """General FP values (not exact in every order) on the spa and spa-split rows: narrow and wide each within the gamma_n bound
    of the exact sum; the ESC rows bit for bit"""
    SA, SB = split_operands()
    SM = partial_mask(SA, SB, 49)
    for typ in ("FP32", "FP64"):
        dt = orc.DTYPES[typ]
        rng = np.random.default_rng(51)
        av = rng.standard_normal(SA.nnz).astype(dt)
        bv = rng.standard_normal(SB.nnz).astype(dt)
        ncols = SB.shape[1]
        Ar = np.repeat(np.arange(SA.shape[0], dtype=np.int64), np.diff(SA.indptr))
        keys, a, b = _expand(Ar, SA.indices.astype(np.int64), av, SB.indptr, SB.indices, bv, ncols)
        for desc in ("", "SC"):
            def run():
                A = Matrix.from_csr(SA.indptr, SA.indices, av, *SA.shape, util.g_type(typ))
                B = Matrix.from_csr(SB.indptr, SB.indices, bv, *SB.shape, util.g_type(typ))
                M = Matrix.from_csr(SM.indptr, SM.indices, np.ones(SM.nnz, bool), *SM.shape, gb.BOOL) if desc else None
                C = Matrix.sparse(util.g_type(typ), *SA.shape[:1], ncols)
                A.mxm(B, semiring=getattr(util.g_type(typ), "PLUS_TIMES"), out=C, mask=M, desc=descriptor.SC if desc else None)
                return C, _tokens()
            (nI, nJ, nX), nt, wides = twice(run, "PLUS", typ, bits=False)
            assert "spa" in nt
            kk, aa, bb = keys, a, b
            if desc:
                blocked = np.isin(keys, _keys(np.repeat(np.arange(SM.shape[0]), np.diff(SM.indptr)), SM.indices, ncols))
                kk, aa, bb = keys[~blocked], a[~blocked], b[~blocked]
            f = np.bincount(Ar, weights=np.diff(SB.indptr)[SA.indices], minlength=SA.shape[0])
            for gI, gJ, gX in [(nI, nJ, nX)] + wides:
                check_bound(_keys(gI, gJ, ncols), gX, kk, aa, bb, typ, f"general {typ} {desc}")
                esc = f[gI] <= 2048
                assert np.array_equal(kc._bits(gX[esc]), kc._bits(nX[esc])), (typ, desc)


@pytest.mark.parametrize("sr", [("MIN", "SECONDI", "INT64"), ("PLUS", "FIRSTI", "INT64"), ("MAX", "FIRSTJ", "INT32")])
@pytest.mark.parametrize("comp", [False, True])
def test_positional(sr, comp):
    """Positional semirings on the bins: the inner form (SECONDI, FIRSTJ) and the count form (FIRSTI)"""
    add, mul, typ = sr
    rng = np.random.default_rng(kc.seed_of("wide-gemm-positional", sr))
    SA = csr(rng.integers(0, 12, 300), 200, seed=13)
    SB = csr(rng.integers(0, 9, 200), 250, seed=14)
    SM = csr(rng.integers(0, 40, 300), 250, seed=15)
    form = "count" if mul == "FIRSTI" else "inner"

    def run():
        A = Matrix.from_csr(SA.indptr, SA.indices, np.ones(SA.nnz, np.int32), *SA.shape, gb.INT32)
        B = Matrix.from_csr(SB.indptr, SB.indices, np.ones(SB.nnz, np.int32), *SB.shape, gb.INT32)
        M = Matrix.from_csr(SM.indptr, SM.indices, np.ones(SM.nnz, bool), *SM.shape, gb.BOOL) if comp else None
        C = Matrix.sparse(util.g_type(typ), 300, 250)
        A.mxm(B, semiring=getattr(util.g_type(typ), f"{add}_{mul}"), out=C, mask=M, desc=descriptor.SC if comp else None)
        return C, _tokens()

    (nI, nJ, nX), nt, wides = twice(run, add, typ)
    assert f"positional={form}" in nt, nt

    def d(S):
        C = S.tocoo()
        return {(int(i), int(j)): 1 for i, j in zip(C.row, C.col)}
    desc = dict(mask_struct=True, mask_comp=True) if comp else {}
    want, _ = pm.mxm({}, typ, d(SM) if comp else None, None, sr, d(SA), d(SB), desc)
    for gI, gJ, gX in wides:
        assert {(int(i), int(j)): int(x) for i, j, x in zip(gI, gJ, gX)} == {k: int(v) for k, v in want.items()}


def test_workspace_reuse_wide_narrow_wide():
    """The grow-only workspaces across routes: wide panels of one size, a narrow call on larger operands, wide again with
    larger panels, then narrow on the first operands."""
    small, large = bins_operands(), split_operands()
    for name, (SA, SB), chunk in [("wide", small, 300), ("narrow", large, None), ("wide-large", large, 1 << 30), ("narrow-small", small, None)]:
        A = Matrix.from_csr(SA.indptr, SA.indices, np.arange(SA.nnz) % 7, *SA.shape, gb.INT64)
        B = Matrix.from_csr(SB.indptr, SB.indices, np.arange(SB.nnz) % 5, *SB.shape, gb.INT64)
        if chunk:
            with wide_gemm(chunk):
                C = A.mxm(B, semiring=gb.INT64.PLUS_TIMES)
                assert "offsets=64" in _tokens(), name
        else:
            C = A.mxm(B, semiring=gb.INT64.PLUS_TIMES)
            assert "offsets=64" not in _tokens(), name
        want = (sp.csr_matrix((np.arange(SA.nnz) % 7, SA.indices, SA.indptr), shape=SA.shape) @
                sp.csr_matrix((np.arange(SB.nnz) % 5, SB.indices, SB.indptr), shape=SB.shape)).tocoo()
        I, J, X = C.to_arrays()
        got = sp.csr_matrix((X, (I, J)), shape=C.shape)
        assert (got != want.tocsr()).nnz == 0, name


@pytest.mark.parametrize("ctas", [1, 2])
def test_spa_budget(ctas):
    """The dense-accumulator byte budget of the wide route set so that it caps the CTAs at 1 and 2, unmasked and complemented.
    The CTA count is not reported, so this checks the results under the cap (every spa row through one or two persistent CTAs,
    each reusing its accumulator across rows), not the count itself."""
    SA, SB = split_operands()
    SM = partial_mask(SA, SB, 53)
    ncols = SB.shape[1]
    for desc, comp in (("", False), ("SC", True)):
        budget = ctas * (ncols * 8 + (ncols + 31) // 32 * 4 * (2 if comp else 1))
        A = Matrix.from_csr(SA.indptr, SA.indices, np.arange(SA.nnz) % 7, *SA.shape, gb.INT64)
        B = Matrix.from_csr(SB.indptr, SB.indices, np.arange(SB.nnz) % 5, *SB.shape, gb.INT64)
        M = Matrix.from_csr(SM.indptr, SM.indices, np.ones(SM.nnz, bool), *SM.shape, gb.BOOL) if comp else None
        C0 = A.mxm(B, semiring=gb.INT64.PLUS_TIMES, mask=M, desc=getattr(descriptor, desc) if desc else None)
        with wide_gemm(500, 0, budget):
            C = A.mxm(B, semiring=gb.INT64.PLUS_TIMES, mask=M, desc=getattr(descriptor, desc) if desc else None)
            assert "spa" in _tokens() and "offsets=64" in _tokens()
        for x, y in zip(C.to_arrays(), C0.to_arrays()):
            assert np.array_equal(x, y), (ctas, desc)


@pytest.mark.parametrize("comp", [False, True])
def test_alloc_failure(comp):
    """A failed allocation anywhere on the wide route returns GrB_OUT_OF_MEMORY, frees what the call allocated, and a retry
    gets the clean result."""
    from pygraphblas_b200.generators import rmat_csr
    n, indptr, indices = rmat_csr(10, 16, seed=5)
    S = sp.csr_matrix((np.ones(len(indices), np.int64), indices, indptr), shape=(n, n))
    want = (S @ S).tocsr()
    if comp:
        want = (want - want.multiply(S.astype(bool))).tocsr()
    want.eliminate_zeros()
    want.sort_indices()
    with wide_gemm(S.nnz // 3):
        k = _sweep(lambda: (_mat(S, gb.INT64),),
                   lambda A: A.mxm(A, mask=A if comp else None, semiring=gb.INT64.PLUS_TIMES, desc=descriptor.SC if comp else None),
                   _same_csr(want))
        assert "offsets=64" in _tokens()
    assert k > 10


@pytest.mark.parametrize("shape", [(5, 4, 0), (5, 0, 6), (0, 4, 6), (0, 0, 0)], ids=lambda s: "x".join(map(str, s)))
def test_empty_shapes(shape):
    """m x k times k x n with a zero dimension (A holds entries when it has positions: rows of A, no column of B), unmasked and
    under a complemented structural mask: an empty product on the wide route as on the narrow one, accumulated into a C with
    entries when it has any positions"""
    m, k, n = shape
    rng = np.random.default_rng(71)
    for desc in ("", "SC"):
        for c_init in (False, True):
            def run():
                A = Matrix.from_lists([0, m - 1], [k - 1, 0], [2, 5], m, k, gb.INT64) if m and k else Matrix.sparse(gb.INT64, m, k)
                B = Matrix.sparse(gb.INT64, k, n)
                if k and n:
                    B = Matrix.from_lists([0, k - 1], [n - 1, 0], [3, 4], k, n, gb.INT64)
                M = None
                if desc:
                    M = Matrix.from_lists([0], [0], [True], m, n, gb.BOOL) if m and n else Matrix.sparse(gb.BOOL, m, n)
                C = Matrix.sparse(gb.INT64, m, n)
                if c_init and m and n:
                    C = Matrix.from_lists([m - 1], [n - 1], [int(rng.integers(1, 9))], m, n, gb.INT64)
                before = C.to_arrays()
                A.mxm(B, semiring=gb.INT64.PLUS_TIMES, out=C, mask=M, accum=gb.INT64.PLUS if c_init else None,
                      desc=descriptor.SC if desc else None)
                return C, before
            C, want = run()
            assert C.shape == (m, n)
            for x, y in zip(C.to_arrays(), want):
                assert np.array_equal(x, y), (shape, desc, c_init)
            for chunk in CHUNKS:
                with wide_gemm(chunk):
                    C, want = run()
                assert C.shape == (m, n)
                for x, y in zip(C.to_arrays(), want):
                    assert np.array_equal(x, y), (shape, desc, c_init, chunk)


# ------------------------------------------------------------------ the size rule
def test_result_limit():
    """L (the longest B row named by each row of A, less what M' holds of that row, summed) >= limit: refused before any panel
    runs; L < limit <= nnz(T): refused after the panels' symbolic counts; nnz(T) = limit - 1: runs.  A refusal leaves C's
    tuples and the live allocations as they were."""
    SA, SB = bins_operands()
    Sc = csr(np.full(SA.shape[0], 2), SB.shape[1], seed=61)
    for comp in (False, True):
        SM = partial_mask(SA, SB, 63) if comp else None
        blen = np.diff(SB.indptr)
        longest = np.array([blen[SA.indices[SA.indptr[i]:SA.indptr[i + 1]]].max(initial=0) for i in range(SA.shape[0])])
        if comp:
            longest = longest - np.diff(SM.indptr)
        L = int(np.maximum(longest, 0).sum())
        P = (SA.astype(np.int64) @ SB.astype(np.int64)).tocsr()
        if comp:
            P = (P - P.multiply(SM.astype(bool))).tocsr()
            P.eliminate_zeros()
        nnz = P.nnz
        assert 0 < L < nnz, (L, nnz)

        A = Matrix.from_csr(SA.indptr, SA.indices, np.ones(SA.nnz, np.int64), *SA.shape, gb.INT64)
        B = Matrix.from_csr(SB.indptr, SB.indices, np.ones(SB.nnz, np.int64), *SB.shape, gb.INT64)
        M = Matrix.from_csr(SM.indptr, SM.indices, np.ones(SM.nnz, bool), *SM.shape, gb.BOOL) if comp else None

        def call(limit, chunk=3000):
            C = Matrix.from_csr(Sc.indptr, Sc.indices, np.arange(Sc.nnz, dtype=np.int64), SA.shape[0], SB.shape[1], gb.INT64)
            before = C.to_arrays()
            live = lib.B200_debug_live_allocs()
            try:
                with wide_gemm(chunk, limit, 0):
                    A.mxm(B, semiring=gb.INT64.PLUS_PAIR, out=C, mask=M, accum=gb.INT64.PLUS, desc=descriptor.SC if comp else None)
            except gb.base.InvalidValue as e:
                assert "2^32 entries are not supported" in str(e), e
                assert lib.B200_debug_live_allocs() == live, (comp, limit)
                for x, y in zip(C.to_arrays(), before):
                    assert np.array_equal(x, y), (comp, limit)
                return None
            return C

        C = call(nnz + 1)                   # runs: the operands' device forms and the panels' workspace are in place
        assert C is not None and _stats()[1] == nnz
        union = sp.csr_matrix((np.ones(Sc.nnz), Sc.indices, Sc.indptr), shape=P.shape).maximum(P.astype(bool).astype(np.float64))
        assert C.nvals == union.nnz
        # chunk 3000: several panels, the one that reaches the limit refused; 2^30: one panel, refused after its scan, before its
        # entries are allocated
        for chunk in (3000, 1 << 30):
            for limit, stage in ((L, "bound"), (L + 1, "counted"), (nnz, "counted")):
                assert call(limit, chunk) is None, (comp, limit, chunk)
                flops, _ = _stats()
                assert (flops == 0) == (stage == "bound"), (comp, limit, chunk, stage, flops)


# ------------------------------------------------------------------ a real wide matrix: A = kron(G, J), nnz(A) = 2^32 + 2^26
NG, NJ = 4096, 4096                            # n = 2^24 rows and columns
NNZ_G, NNZ_J = (1 << 16) + (1 << 10), 1 << 16
NNZ = NNZ_G * NNZ_J                            # 4 362 076 160
n = NG * NJ
K = 8                                          # P = PG (x) PJ assigns every vertex to one of K * K = 64 groups
SOURCES = 16
# A: col 4 B + value 1 B per entry, rowptr 8 B per row.  A P (~9·10^8 entries in UINT8): the panels' CSRs and T while they are
# joined, 5 B per entry and 12 B of row offsets per row each, and a result of the same size from the write-back.  A panel:
# ~40 B per row (2^26 rows at most).  P' A: the dense accumulators (2^32 B) and a result of ~8·10^8 entries.  The BFS: F, V and
# the next F, 16 x n BOOL each at most.  The checks: two dense vectors of n entries and the run plans of the results.
PLAN_A = NNZ * 5 + 8 * n
PLAN_AP = 3 * (9e8 * 5 + 12 * n)
PLAN_PANEL = (1 << 26) * 40
PLAN_CHECKS = 2 * n * 9 + 9e8 * 1
PLANNED = PLAN_A + PLAN_AP + PLAN_PANEL + PLAN_CHECKS + 1 * GB_


@pytest.fixture(scope="module")
def memory():
    m = Memory()
    if m.start < PLANNED + 2 * GB_:
        pytest.skip(f"needs {PLANNED / GB_:.1f} GB of free device memory for a matrix of {NNZ} entries, "
                    f"{m.start / GB_:.1f} GB free")
    yield m
    print(f"\nwide unmasked mxm: {NNZ} entries, planned peak {PLANNED / GB_:.1f} GB, observed peak {m.peak / GB_:.1f} GB "
          f"on {m.torch.cuda.get_device_name()}")
    trim_pool(m.torch)


@pytest.fixture(scope="module")
def real(memory):
    G, J = factor(1, NG, NNZ_G), factor(2, NJ, NNZ_J)
    A = kron(G, J, "UINT8")
    memory.note()
    assert A.nvals == NNZ and NNZ >= (1 << 32) + (1 << 26)
    yield G, J, A
    del A
    trim_pool(memory.torch)


def kron(X, Y, typ):
    """kron(X, Y) on the device in `typ` (X, Y scipy CSR of any shapes)"""
    tg = util.g_type(typ)
    Xm = Matrix.from_csr(X.indptr, X.indices, X.data.astype(tg.dtype), *X.shape, tg)
    Ym = Matrix.from_csr(Y.indptr, Y.indices, Y.data.astype(tg.dtype), *Y.shape, tg)
    C = Matrix.sparse(tg, X.shape[0] * Y.shape[0], X.shape[1] * Y.shape[1])
    gb.base._check(lib.GrB_Matrix_kronecker_BinaryOp(C._matrix[0], ffi.NULL, ffi.NULL, gb.UINT8.TIMES.get_op(), Xm._matrix[0],
                                                     Ym._matrix[0], ffi.NULL))
    return C


def one_hot(seed, nn):
    rng = np.random.default_rng(seed)
    S = sp.csr_matrix((rng.integers(1, 4, nn).astype(np.uint8), (np.arange(nn), rng.integers(0, K, nn))), shape=(nn, K))
    S.sort_indices()
    return S


def _check_kron(T, Zg, Zj, label, memory, rows=(), cols=()):
    """T = Zg (x) Zj in UINT8 (values mod 256, entries whose sum is 0 mod 256 kept): nvals, the PLUS row sums against the
    outer product of the factors' row sums, rows `rows` through vxm and columns `cols` through mxv."""
    nj = Zj.shape[1]
    assert T.nvals == Zg.nnz * Zj.nnz, (label, T.nvals, Zg.nnz * Zj.nnz)
    r = T.reduce_vector(gb.UINT8.PLUS_MONOID)
    memory.note()
    sg, sj = np.asarray(Zg.sum(axis=1)).ravel(), np.asarray(Zj.sum(axis=1)).ravel()
    I, X = r.to_arrays()
    nzr = np.flatnonzero(np.outer(np.diff(Zg.indptr) > 0, np.diff(Zj.indptr) > 0).ravel())
    assert np.array_equal(I, nzr), label
    assert np.array_equal(X.astype(np.int64), np.outer(sg, sj).ravel()[nzr] % 256), label
    for i in rows:
        ig, ij = divmod(int(i), Zj.shape[0])
        w = Vector.from_lists([int(i)], [1], T.nrows, gb.UINT8).vxm(T, semiring=gb.UINT8.PLUS_TIMES)
        memory.note()
        rg, rj = Zg[ig], Zj[ij]
        keys = (rg.indices[:, None].astype(np.int64) * nj + rj.indices[None, :]).ravel()
        vals = (rg.data[:, None].astype(np.int64) * rj.data[None, :]).ravel() % 256
        o = np.argsort(keys)
        I, X = w.to_arrays()
        assert np.array_equal(I, keys[o]) and np.array_equal(X.astype(np.int64), vals[o]), (label, "row", i)
    ZgT, ZjT = Zg.T.tocsr(), Zj.T.tocsr()
    for jg, jj in cols:
        w = T.mxv(Vector.from_lists([jg * nj + jj], [1], T.ncols, gb.UINT8), semiring=gb.UINT8.PLUS_TIMES)
        memory.note()
        cg, cj = ZgT[jg], ZjT[jj]
        keys = (cg.indices[:, None].astype(np.int64) * Zj.shape[0] + cj.indices[None, :]).ravel()
        vals = (cg.data[:, None].astype(np.int64) * cj.data[None, :]).ravel() % 256
        o = np.argsort(keys)
        I, X = w.to_arrays()
        assert np.array_equal(I, keys[o]) and np.array_equal(X.astype(np.int64), vals[o]), (label, "col", jg, jj)


def test_real_coarsening_a_p(real, memory):
    """A (+).(x) P in UINT8, A wide on the left in several panels, P narrow: (G PG) (x) (J PJ) mod 256"""
    G, J, A = real
    PG, PJ = one_hot(3, NG), one_hot(4, NJ)
    P = kron(PG, PJ, "UINT8")
    Zg, Zj = (G.astype(np.int64) @ PG.astype(np.int64)).tocsr(), (J.astype(np.int64) @ PJ.astype(np.int64)).tocsr()
    Zg.sort_indices(); Zj.sort_indices()
    C = A.mxm(P, semiring=gb.UINT8.PLUS_TIMES)
    memory.note()
    ks = _tokens()
    assert ks[0] in ENTRIES and ks[1] == "offsets=64", ks
    flops, nout = _stats()
    assert flops == NNZ and nout == Zg.nnz * Zj.nnz, (flops, nout)
    # rows whose A entries lie past offset 2^32: the last ones
    rpG = G.indptr.astype(np.int64)
    past = int(np.searchsorted(rpG * NNZ_J, 1 << 32)) * NJ
    rows = list(range(0, n, n // 7)) + [past + 5, n - 1]
    _check_kron(C, Zg, Zj, "a-p", memory, rows=rows, cols=[(0, 0), (3, 5), (7, 7)])
    del C, P
    trim_pool(memory.torch)


def test_real_wide_b(real, memory):
    """P' (+).(x) A in UINT8, A the wide right operand: (PG' G) (x) (PJ' J) mod 256; 64 rows on the spa bin over 2^24 columns"""
    G, J, A = real
    PG, PJ = one_hot(5, NG), one_hot(6, NJ)
    PGt, PJt = PG.T.tocsr(), PJ.T.tocsr()
    PGt.sort_indices(); PJt.sort_indices()
    Pt = kron(PGt, PJt, "UINT8")
    Zg, Zj = (PGt.astype(np.int64) @ G.astype(np.int64)).tocsr(), (PJt.astype(np.int64) @ J.astype(np.int64)).tocsr()
    Zg.sort_indices(); Zj.sort_indices()
    C = Pt.mxm(A, semiring=gb.UINT8.PLUS_TIMES)
    memory.note()
    assert _tokens()[:2] == ["spa", "offsets=64"], _tokens()
    _check_kron(C, Zg, Zj, "wide-b", memory, rows=[0, 9, 63], cols=[(0, 0), (NG - 1, 17), (2000, NJ - 1)])
    del C, Pt
    trim_pool(memory.torch)


def _walk_sets(S, src, steps):
    """the vertices reached from src by walks of exactly L steps, L = 0 .. steps"""
    Sb = S.astype(bool).astype(np.int64)
    w = np.zeros(S.shape[0], np.int64)
    w[src] = 1
    out = [w > 0]
    for _ in range(steps):
        w = ((Sb.T @ w) > 0).astype(np.int64)
        out.append(w > 0)
    return out


def test_real_msbfs_complemented(real, memory):
    """F<!V, R> = F any.pair A for 16 sources to the last level.  Vertex (g', j') is at level L from (g, j) for the least L with
    g' reached from g by a walk of exactly L steps in G and j' from j by one of exactly L steps in J."""
    G, J, A = real
    rng = np.random.default_rng(9)
    sg, sj = rng.integers(0, NG, SOURCES), rng.integers(0, NJ, SOURCES)
    src = sg.astype(np.int64) * NJ + sj
    F = Matrix.from_lists(list(range(SOURCES)), src.tolist(), [True] * SOURCES, SOURCES, n, gb.BOOL)
    V = Matrix.from_lists(list(range(SOURCES)), src.tolist(), [True] * SOURCES, SOURCES, n, gb.BOOL)
    ones = Vector.from_numpy(np.ones(n, np.int64), typ=gb.INT64)
    counts, small = [], {}
    while True:
        Fn = Matrix.sparse(gb.BOOL, SOURCES, n)
        F.mxm(A, semiring=gb.BOOL.ANY_PAIR, out=Fn, mask=V, desc=descriptor.RSC)
        memory.note()
        ks = _tokens()
        F = Fn
        if F.nvals == 0:
            break
        assert ks[0] in ENTRIES and ks[1] == "offsets=64", ks
        c = np.zeros(SOURCES, np.int64)
        I, X = F.mxv(ones, semiring=gb.INT64.PLUS_PAIR).to_arrays()
        c[I] = X
        counts.append(c)
        if F.nvals < 2e7:
            small[len(counts)] = F.to_arrays()[:2]
        V.eadd(F, gb.BOOL.LOR, out=V)
        memory.note()
        assert len(counts) < 40
    levels = len(counts)
    for s in range(SOURCES):
        WG, WJ = _walk_sets(G, sg[s], levels + 1), _walk_sets(J, sj[s], levels + 1)
        reached = np.zeros(n, bool)
        reached[src[s]] = True
        for L in range(1, levels + 2):
            new = np.outer(WG[L], WJ[L]).ravel() & ~reached
            reached |= new
            got = counts[L - 1][s] if L <= levels else 0
            assert got == int(new.sum()), (s, L, got, int(new.sum()))
            if L in small:
                I, Jc = small[L]
                assert np.array_equal(Jc[I == s], np.flatnonzero(new)), (s, L)
