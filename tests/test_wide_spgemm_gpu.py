"""The wide route of the masked CSR x CSR methods of mxm (C<M> = A (+).(x) B, the mask not complemented) on matrices with 2^32
or more entries.

The wide route runs the masked-warp, stream and dot kernels on row panels of A and M, whose offsets are rebased to 32 bits,
and reads B's 64-bit offsets when B is wide.  B200_debug_wide(chunk) puts every operand on that route with panels of at most
`chunk` entries of A and of M, so the first part runs each case twice at small sizes -- narrow, then wide on fresh operands --
and requires the same route (plus the `offsets=64` token after the route's entry), the same pattern and value bits, and one
agreement with the oracle.  The second part builds a real matrix of 2^32 + 2^26 entries on the device as kron(G, J) and checks
the triangle-shaped product C<A> = A (+.pair) A and its relatives against identities on the small factors; it skips, with the
reason, when the card lacks the free memory."""
import numpy as np
import pytest
import scipy.sparse as sp

import pygraphblas_b200 as gb
from pygraphblas_b200 import Matrix, Vector, descriptor
from oracle import oracle as orc
import kernel_check as kc
import positional_model as pm
import util
from test_alloc_failure_gpu import _mat, _same_csr, _sweep
from test_structure_edges_gpu import GEMM_SRS, csr, gemm_route, mask_values, masked, pool_of, uniform_masked
from test_wide_mxm_gpu import trim_pool
from test_wide_offsets_gpu import GB_, Memory, factor, kron, wide

pytestmark = pytest.mark.gpu

ENTRIES = ("dot", "masked-warp", "stream-S", "stream-M", "stream-L")


def _keys(I, J, ncols):
    return np.asarray(I, np.int64) * ncols + np.asarray(J, np.int64)


def twice(run, add, zt, chunk=7):
    """run() builds fresh operands, makes one mxm and returns (C, tokens); it runs narrow, then wide.  The wide result must
    have the narrow pattern and values (bit for bit; any NaN for a NaN and, under MIN / MAX, either zero for a zero, as in
    kernel_check.compare; under ANY the pattern only).  Returns the wide C's tuples and the narrow tokens."""
    C, nt = run()
    nI, nJ, nX = C.to_arrays()
    ncols = C.ncols
    with wide(chunk):
        C, gt = run()
        gI, gJ, gX = C.to_arrays()
    assert "offsets=64" not in nt, nt
    at = next(i for i, k in enumerate(nt) if k in ENTRIES) + 1
    assert gt == nt[:at] + ["offsets=64"] + nt[at:], (nt, gt)
    assert np.array_equal(nI, gI) and np.array_equal(nJ, gJ)
    if add != "ANY":
        e = kc.compare(_keys(gI, gJ, ncols), gX, _keys(nI, nJ, ncols), nX, zt, add, "wide vs narrow")
        assert e is None, e
    return (gI, gJ, gX), nt


def gemm_twice(SA, SB, SM, desc, label, sr, chunk=7, mask_type=None, c_init=False, accum=False, alias=False):
    """C<M> = accum(C, op(A) (+).(x) op(B)) narrow and wide: the route restated by gemm_route, then the oracle.  SA is op(A)
    (stored transposed when desc holds T0); mask_type as in run_gemm; alias: C = A, the mask and both operands (SB, SM
    ignored)."""
    add, _, typ = sr
    zt, pool = orc.semiring_ztype(sr), pool_of(sr)
    seed = kc.seed_of("wide-spgemm", label, sr)
    if alias:
        SB = SM = SA
    t0 = "T0" in desc
    SAs = SA.T.tocsr() if t0 else SA
    SAs.sort_indices()
    av = kc.values(seed, typ, SAs.nnz, pool, 0)
    bv = av if alias else kc.values(seed + 1, typ, SB.nnz, pool, 1)
    nrows, ncols = SA.shape[0], (SB.shape[0] if "T1" in desc else SB.shape[1])
    mt, mv = "BOOL", np.ones(SM.nnz, bool)
    if alias:
        mt, mv = typ, av
    elif mask_type is not None:
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
        M = A if alias else Matrix.from_csr(SM.indptr, SM.indices, mv, *SM.shape, util.g_type(mt))
        if alias:
            C = A
        elif c_init:
            C = Matrix.from_csr(Sc.indptr, Sc.indices, cv, nrows, ncols, util.g_type(zt))
        else:
            C = Matrix.sparse(util.g_type(zt), nrows, ncols)
        A.mxm(B, semiring=kc.semiring(*sr), out=C, mask=M, accum=util.g_accum(acc), desc=getattr(descriptor, desc) if desc else None)
        return C, kc.last_kernel().split(";")

    (gI, gJ, gX), nt = twice(run, add, zt, chunk)
    want = gemm_route(SA, SB, SM, desc.replace("T0", ""), {})
    assert [k for k in nt if k] == want, (label, sr, nt, want)
    Ao, Bo = kc.o_csr(typ, SAs, av), kc.o_csr(typ, SB, bv)
    Mo = Ao if alias else kc.o_csr(mt, SM, mv)
    Co = Ao if alias else (kc.o_csr(zt, Sc, cv) if c_init else orc.SpMat(zt, nrows, ncols))
    ref = orc.mxm(Co, Mo, acc, sr, Ao, Bo, desc)
    cands = None
    if add == "ANY":
        if accum or c_init or alias or "T" in desc:
            return nt
        cands = kc.products_by_entry(np.repeat(np.arange(nrows), np.diff(SA.indptr)), SA.indices.astype(np.int64), av,
                                     SB.indptr, SB.indices, bv, ncols, sr[1])
    e = kc.compare(_keys(gI, gJ, ncols), gX, _keys(ref.I, ref.J, ncols), ref.X, zt, add, f"{label} {'_'.join(sr)} wide", cands)
    assert e is None, e
    return nt


# ------------------------------------------------------------------ every masked entry, every chunk of the panels
# 7: every row a panel of its own, and rows longer than the chunk; 3000: panels of several rows; 2^30: one panel
@pytest.mark.parametrize("chunk", [7, 3000, 1 << 30])
def test_classes_chunks_long_rows(chunk):
    """The warp class and the three stream classes (exact filters), at every class and chunk boundary of chunk_count_kernel
    and with long B rows, over every semiring of GEMM_SRS (fast and generic instantiations, the edge values of each type)."""
    SA, SB, SM = masked(4096)
    srs = GEMM_SRS if chunk == 7 else GEMM_SRS[::3]
    for sr in srs:
        nt = gemm_twice(SA, SB, SM, "S", f"classes-{chunk}", sr, chunk)
        assert nt == ["masked-warp", "stream-S", "filter=exact", "stream-M", "filter=exact", "stream-L", "filter=exact"], nt


@pytest.mark.parametrize("cls", ["S", "M", "L"])
def test_bloom_filters(cls):
    """One column past the exact-bitmap limit of each stream class: the Bloom filter."""
    bits = {"S": 14, "M": 16, "L": 20}[cls]
    SA, SB, SM = uniform_masked(cls, (1 << bits) + 1)
    for sr in GEMM_SRS[::2]:
        nt = gemm_twice(SA, SB, SM, "S", f"bloom-{cls}", sr, 1000)
        assert nt == [f"stream-{cls}", "filter=bloom"], nt


def test_dot():
    """C<M> = A B' by row intersections (nnz(B) < 2^18): every semiring, valued mask with an all-false row."""
    SB = csr(np.full(1 << 10, 40), 4096, seed=5)
    SA = csr(np.random.default_rng(6).integers(0, 40, 200), 4096, seed=7)
    SM = csr(np.random.default_rng(8).integers(0, 60, 200), 1 << 10, seed=9)
    for sr in GEMM_SRS:
        assert gemm_twice(SA, SB, SM, "ST1", "dot", sr, 50) == ["dot"]
    assert gemm_twice(SA, SB, SM, "T1", "dot-valued", GEMM_SRS[0], 7, mask_type="FP32") == ["dot"]


# (name, desc, mask type, C holds entries, accum)
WRITE_BACK = [("valued-int", "", "INT32", False, False),
              ("valued-fp", "", "FP64", False, False),
              ("accum", "S", None, True, True),
              ("replace", "RS", None, True, False),
              ("replace-valued-accum", "R", "UINT8", True, True),
              ("T0", "ST0", None, False, False),
              ("T1", "ST1", None, False, False)]


@pytest.mark.parametrize("case", WRITE_BACK, ids=[c[0] for c in WRITE_BACK])
def test_write_back(case):
    name, desc, mt, c_init, accum = case
    SA, SB, SM = uniform_masked("S", 4096)
    if "T1" in desc:
        SB = SB.T.tocsr()                      # stored B', transposed back by the call (nnz(B) >= 2^18 would take the dot method
        SB.sort_indices()                      # below it; this B is small, so the call takes the dot method)
    for sr in GEMM_SRS[:5]:
        gemm_twice(SA, SB, SM, desc, f"wb-{name}", sr, 500, mask_type=mt, c_init=c_init, accum=accum)


def test_alias():
    """C = A, the mask and both operands: A<A> = A (+).(x) A in place."""
    SA = csr(np.random.default_rng(11).integers(0, 30, 400), 400, seed=12)
    for sr in [("PLUS", "TIMES", "INT64"), ("MIN", "PLUS", "INT32"), ("PLUS", "TIMES", "FP64"), ("LOR", "LAND", "BOOL")]:
        gemm_twice(SA, None, None, "S", "alias", sr, 40, alias=True)


@pytest.mark.parametrize("sr", [("MIN", "SECONDI", "INT64"), ("PLUS", "FIRSTI", "INT64"), ("MAX", "FIRSTJ", "INT32")])
def test_positional(sr):
    """Positional semirings, rewritten onto the masked methods: the inner form (SECONDI, FIRSTJ: the values of the sparser
    operand become their inner index) and the count form (FIRSTI: PLUS_PAIR counts, then the row index folded)."""
    add, mul, typ = sr
    rng = np.random.default_rng(kc.seed_of("wide-positional", sr))
    SA = csr(rng.integers(0, 12, 300), 200, seed=13)
    SB = csr(rng.integers(0, 9, 200), 250, seed=14)
    SM = csr(rng.integers(0, 40, 300), 250, seed=15)
    form = "count" if mul == "FIRSTI" else "inner"

    def run():
        A = Matrix.from_csr(SA.indptr, SA.indices, np.ones(SA.nnz, np.int32), *SA.shape, gb.INT32)
        B = Matrix.from_csr(SB.indptr, SB.indices, np.ones(SB.nnz, np.int32), *SB.shape, gb.INT32)
        M = Matrix.from_csr(SM.indptr, SM.indices, np.ones(SM.nnz, bool), *SM.shape, gb.BOOL)
        C = Matrix.sparse(util.g_type(typ), 300, 250)
        A.mxm(B, semiring=getattr(util.g_type(typ), f"{add}_{mul}"), out=C, mask=M, desc=descriptor.S)
        return C, kc.last_kernel().split(";")

    (gI, gJ, gX), nt = twice(run, add, typ, 11)
    assert f"positional={form}" in nt, nt

    def d(S):
        C = S.tocoo()
        return {(int(i), int(j)): 1 for i, j in zip(C.row, C.col)}
    want, _ = pm.mxm({}, typ, d(SM), None, sr, d(SA), d(SB), dict(mask_struct=True))
    got = {(int(i), int(j)): int(x) for i, j, x in zip(gI, gJ, gX)}
    assert got == {k: int(v) for k, v in want.items()}


def test_complemented_mask_stays_narrow():
    """A complemented mask under the switch runs the unmasked bins on their 32-bit kernels: no `offsets=64`."""
    SA, SB, SM = uniform_masked("S", 4096)
    sr = ("PLUS", "TIMES", "INT64")
    for desc in ("SC", "RSC"):
        A = Matrix.from_csr(SA.indptr, SA.indices, np.ones(SA.nnz, np.int64), *SA.shape, gb.INT64)
        B = Matrix.from_csr(SB.indptr, SB.indices, np.ones(SB.nnz, np.int64), *SB.shape, gb.INT64)
        M = Matrix.from_csr(SM.indptr, SM.indices, np.ones(SM.nnz, bool), *SM.shape, gb.BOOL)
        with wide(7):
            C = A.mxm(B, semiring=gb.INT64.PLUS_TIMES, mask=M, desc=getattr(descriptor, desc))
            t = kc.last_kernel().split(";")
        assert "offsets=64" not in t and not any(k in ENTRIES for k in t), t
        want = orc.mxm(orc.SpMat("INT64", *C.shape), kc.o_csr("BOOL", SM, np.ones(SM.nnz, bool)), None, sr,
                       kc.o_csr("INT64", SA, np.ones(SA.nnz, np.int64)), kc.o_csr("INT64", SB, np.ones(SB.nnz, np.int64)), desc)
        gI, gJ, gX = C.to_arrays()
        e = kc.compare(_keys(gI, gJ, C.ncols), gX, _keys(want.I, want.J, C.ncols), want.X, "INT64", "PLUS", desc)
        assert e is None, e


def test_workspace_reuse_wide_narrow_wide():
    """The grow-only workspaces across routes: wide panels of one size, a narrow call on larger operands, wide again with
    larger panels, then narrow on the first operands."""
    small, large = uniform_masked("S", 4096), uniform_masked("L", (1 << 20) + 1)
    for name, ops, chunk in [("wide", small, 300), ("narrow", large, None), ("wide-large", large, 1 << 30), ("narrow-small", small, None)]:
        SA, SB, SM = ops
        sr = ("PLUS", "TIMES", "INT64")
        A = Matrix.from_csr(SA.indptr, SA.indices, np.arange(SA.nnz) % 7, *SA.shape, gb.INT64)
        B = Matrix.from_csr(SB.indptr, SB.indices, np.arange(SB.nnz) % 5, *SB.shape, gb.INT64)
        M = Matrix.from_csr(SM.indptr, SM.indices, np.ones(SM.nnz, bool), *SM.shape, gb.BOOL)
        if chunk:
            with wide(chunk):
                C = A.mxm(B, semiring=gb.INT64.PLUS_TIMES, mask=M, desc=descriptor.S)
                assert "offsets=64" in kc.last_kernel().split(";"), name
        else:
            C = A.mxm(B, semiring=gb.INT64.PLUS_TIMES, mask=M, desc=descriptor.S)
        want = (sp.csr_matrix((np.arange(SA.nnz) % 7, SA.indices, SA.indptr), shape=SA.shape) @
                sp.csr_matrix((np.arange(SB.nnz) % 5, SB.indices, SB.indptr), shape=SB.shape))
        want = want.multiply(SM.astype(bool)).tocsr()
        want.eliminate_zeros()
        I, J, X = C.to_arrays()
        W = want.tocoo()
        order = np.lexsort((W.col, W.row))
        pat = (_keys(W.row, W.col, SM.shape[1])[order])
        # entries whose products sum to 0 are still present in C: compare on the pattern of nonzero sums
        nz = X != 0
        assert np.array_equal(_keys(I, J, SM.shape[1])[nz], pat) and np.array_equal(X[nz], W.data[order]), name


@pytest.mark.parametrize("dot", [False, True])
def test_alloc_failure(dot):
    """A failed allocation anywhere on the wide route returns GrB_OUT_OF_MEMORY, frees what the call allocated, and a
    retry gets the clean result."""
    from pygraphblas_b200.generators import rmat_csr
    n, indptr, indices = rmat_csr(11, 16, seed=3)
    S = sp.csr_matrix((np.ones(len(indices), np.int64), indices, indptr), shape=(n, n))
    want = ((S @ (S.T if dot else S)).multiply(S)).tocsr()
    want.eliminate_zeros()
    with wide(S.nnz // 3):
        k = _sweep(lambda: (_mat(S, gb.INT64),),
                   lambda A: A.mxm(A, mask=A, semiring=gb.INT64.PLUS_PAIR, desc=descriptor.ST1 if dot else descriptor.S),
                   _same_csr(want))
        assert "offsets=64" in kc.last_kernel().split(";")
    assert k > 10


# ------------------------------------------------------------------ a real wide matrix: A = kron(G, J), nnz(A) >= 2^32 + 2^26
# Sparser, larger factors than the other wide modules: n = 2^28 rows, ~16 entries per row of A, so that A (+).pair A is
# ~10^11 products.  Cliques planted in both factors give a sizeable share of the mask entries products.
NG = NJ = 1 << 14
NNZ_G, NNZ_J = (1 << 16) + (1 << 10), 1 << 16
NNZ = NNZ_G * NNZ_J                            # 4 362 076 160
n = NG * NJ
# (first row, size): small cliques every 160 rows, and one of 24 in the last rows, whose rows of A lie past 2^32
CLIQUES = [(r, 8) for r in range(0, NG - 64, 160)] + [(NG - 40, 24)]
# A: col 4 B + value 1 B per entry, rowptr 8 B per row.  A panel (at most 2^30 entries of M and 2^26 rows): accumulator words 4 B
# + found flag 1 B per mask entry (+ 1 B narrowed for UINT8), 5 int64 and two 32-bit offsets per row.  T (~1.8·10^8 entries in
# UINT32): the panels' CSRs and T itself, each with 12 B of row offsets per row.  The checks: three dense vectors of n entries.
PLAN_A = NNZ * 5 + 8 * n
PLAN_PANEL = (1 << 30) * (4 + 1 + 1) + (1 << 26) * (5 * 8 + 2 * 4)
PLAN_T = 2 * (1.8e8 * (4 + 4) + 12 * n)
PLAN_CHECKS = 3 * n * (4 + 1)
PLANNED = PLAN_A + PLAN_PANEL + PLAN_T + PLAN_CHECKS + 1 * GB_


def factor_cliques(seed, nn, nnz):
    """factor(), with CLIQUES planted: dense blocks on the diagonal, the entries they add taken back from elsewhere so that
    the factor keeps exactly nnz entries."""
    S = factor(seed, nn, nnz).tolil()
    rng = np.random.default_rng(seed + 100)
    add = 0
    for r0, k in CLIQUES:
        for i in range(r0, r0 + k):
            for j in range(r0, r0 + k):
                if S[i, j] == 0:
                    S[i, j] = 1
                    add += 1
    S = S.tocsr()
    S.sort_indices()
    # drop `add` entries outside the cliques, from rows that keep at least one entry
    inside = np.zeros(nn, bool)
    for r0, k in CLIQUES:
        inside[r0:r0 + k] = True
    rows = np.repeat(np.arange(nn), np.diff(S.indptr))
    deg = np.diff(S.indptr)
    cand = np.flatnonzero(~inside[rows] & (deg[rows] > 1) & (S.indices != S.indices[S.indptr[rows]]))
    drop = np.zeros(S.nnz, bool)
    picked = 0
    for e in rng.permutation(cand):
        r = rows[e]
        if deg[r] > 1:
            drop[e] = True
            deg[r] -= 1
            picked += 1
            if picked == add:
                break
    assert picked == add
    S = sp.csr_matrix((S.data[~drop], S.indices[~drop], np.concatenate([[0], np.cumsum(np.bincount(rows[~drop], minlength=nn))])),
                      shape=(nn, nn))
    S.sort_indices()
    assert S.nnz == nnz and (np.diff(S.indptr) > 0).all()
    return S


@pytest.fixture(scope="module")
def memory():
    m = Memory()
    if m.start < PLANNED + 2 * GB_:
        pytest.skip(f"needs {PLANNED / GB_:.1f} GB of free device memory for a matrix of {NNZ} entries, "
                    f"{m.start / GB_:.1f} GB free")
    yield m
    print(f"\nwide masked mxm: {NNZ} entries, planned peak {PLANNED / GB_:.1f} GB, observed peak {m.peak / GB_:.1f} GB "
          f"on {m.torch.cuda.get_device_name()}")
    trim_pool(m.torch)


def _tokens():
    return kc.last_kernel().split(";")


def _masked_counts(X, Y, P):
    """(X @ Y) restricted to the pattern of P, as int64 counts / sums (scipy)"""
    Z = (X.astype(np.int64) @ Y.astype(np.int64)).multiply(P.astype(bool)).tocsr()
    Z.sort_indices()
    return Z


def _check_kron(T, Zg, Zj, mod, label, memory, cols=()):
    """T = Zg (x) Zj (values mod `mod`, entries with a zero product sum kept): nvals, the PLUS row reduction against the
    outer product of the factors' row sums, and the columns `cols` through mxv."""
    typ = T.type
    assert T.nvals == Zg.nnz * Zj.nnz, (label, T.nvals, Zg.nnz * Zj.nnz)
    r = T.reduce_vector(getattr(typ, "PLUS_MONOID"))
    memory.note()
    sg, sj = np.asarray(Zg.sum(axis=1)).ravel(), np.asarray(Zj.sum(axis=1)).ravel()
    I, X = r.to_arrays()
    nzr = np.flatnonzero(np.outer(np.diff(Zg.indptr) > 0, np.diff(Zj.indptr) > 0).ravel())
    assert np.array_equal(I, nzr), label
    assert np.array_equal(X.astype(np.int64) % mod, (np.outer(sg, sj).ravel()[nzr]) % mod), label
    ZgT, ZjT = Zg.T.tocsr(), Zj.T.tocsr()
    for jg, jj in cols:
        j = jg * NJ + jj
        w = T.mxv(Vector.from_lists([j], [1], n, typ), semiring=getattr(typ, "PLUS_TIMES"))
        memory.note()
        cg, cj = ZgT[jg], ZjT[jj]
        rows = (cg.indices[:, None].astype(np.int64) * NJ + cj.indices[None, :]).ravel()
        vals = (cg.data[:, None].astype(np.int64) * cj.data[None, :]).ravel() % mod
        order = np.argsort(rows)
        I, X = w.to_arrays()
        assert np.array_equal(I, rows[order]) and np.array_equal(X.astype(np.int64) % mod, vals[order]), (label, jg, jj)


def test_real_wide_masked(memory):
    G, J = factor_cliques(1, NG, NNZ_G), factor_cliques(2, NJ, NNZ_J)
    Gb, Jb = G.astype(bool).astype(np.int64), J.astype(bool).astype(np.int64)
    A = kron(G, J, "UINT8")
    memory.note()
    assert A.nvals == NNZ and NNZ >= (1 << 32) + (1 << 26)
    assert max(np.diff(G.indptr)) * max(np.diff(J.indptr)) <= 2048     # no hub mask row: stream-L's maps would be ncols per CTA
    rpG, rpJ, dG = G.indptr.astype(np.int64), J.indptr.astype(np.int64), np.diff(G.indptr).astype(np.int64)
    # columns of the last clique of G: their entries in the last rows of A lie past 2^32
    lastG = CLIQUES[-1][0]
    cols = [(lastG + 3, CLIQUES[0][0] + 5), (lastG + 20, CLIQUES[1][0] + 2), (CLIQUES[5][0] + 1, CLIQUES[-1][0] + 7)]
    first_last = rpG[lastG] * NNZ_J + dG[lastG] * rpJ[CLIQUES[0][0]]
    assert first_last >= 1 << 32

    # C<A> = A (+.pair) A in UINT32 (the triangle form): A, B and M wide, the fast PLUS_PAIR kernel
    Zg, Zj = _masked_counts(Gb, Gb, G), _masked_counts(Jb, Jb, J)
    assert Zg.nnz > 0.1 * G.nnz and Zj.nnz > 0.1 * J.nnz
    C = Matrix.sparse(gb.UINT32, n, n)
    A.mxm(A, mask=A, semiring=gb.UINT32.PLUS_PAIR, out=C, desc=descriptor.S)
    memory.note()
    ks = _tokens()
    assert ks[1] == "offsets=64" and ks[0] in ENTRIES, ks
    _check_kron(C, Zg, Zj, 1 << 32, "pair", memory, cols)
    del C
    trim_pool(memory.torch)
    memory.note()

    # the same in UINT8 PLUS_TIMES, mod 256, on the generic kernel
    Zg8, Zj8 = _masked_counts(G, G, G), _masked_counts(J, J, J)
    C = Matrix.sparse(gb.UINT8, n, n)
    A.mxm(A, mask=A, semiring=gb.UINT8.PLUS_TIMES, out=C, desc=descriptor.S)
    memory.note()
    assert _tokens()[1] == "offsets=64", _tokens()
    _check_kron(C, Zg8, Zj8, 256, "uint8", memory, cols)
    del C
    trim_pool(memory.torch)
    memory.note()

    # P = Pg (x) Pj, narrow (nnz(P) < 2^18): dense blocks on G's last clique and J's first, so that the products reach A's rows
    # past 2^32 and hit the mask
    def block(nn, r0, k):
        I, J = np.meshgrid(np.arange(r0, r0 + k), np.arange(r0, r0 + k), indexing="ij")
        X = sp.csr_matrix((np.ones(k * k, np.uint8), (I.ravel(), J.ravel())), shape=(nn, nn))
        X.sort_indices()
        return X
    rng = np.random.default_rng(7)
    Pg, Pj = block(NG, lastG, 20), block(NJ, CLIQUES[0][0], 20)
    P = kron(Pg, Pj, "UINT8")
    assert P.nvals == Pg.nnz * Pj.nnz < 1 << 18
    Pgb, Pjb = Pg.astype(np.int64), Pj.astype(np.int64)

    # the dot method: C<A> = A (+.pair) P', A and M wide, B narrow
    C = Matrix.sparse(gb.UINT32, n, n)
    A.mxm(P, mask=A, semiring=gb.UINT32.PLUS_PAIR, out=C, desc=descriptor.ST1)
    memory.note()
    assert _tokens()[:2] == ["dot", "offsets=64"], _tokens()
    _check_kron(C, _masked_counts(Gb, Pgb.T, G), _masked_counts(Jb, Pjb.T, J), 1 << 32, "dot", memory, cols)
    del C
    trim_pool(memory.torch)

    # the stream kernel with a narrow B: C<A> = A (+.pair) P
    C = Matrix.sparse(gb.UINT32, n, n)
    A.mxm(P, mask=A, semiring=gb.UINT32.PLUS_PAIR, out=C, desc=descriptor.S)
    memory.note()
    ks = _tokens()
    assert ks[1] == "offsets=64" and ks[0] in ENTRIES, ks
    _check_kron(C, _masked_counts(Gb, Pgb, G), _masked_counts(Jb, Pjb, J), 1 << 32, "narrow-b", memory, cols)
    del C
    trim_pool(memory.torch)

    # B wide only: C<Mg (x) Mj> = P (+.pair) A under a narrow mask, with 4 x 4 blocks: a mask row stays within 2048 entries
    # (a longer one would take the hub class, whose column maps are ncols entries per CTA)
    del P
    Pg, Pj = block(NG, lastG, 4), block(NJ, CLIQUES[0][0], 4)
    P = kron(Pg, Pj, "UINT8")
    Pgb, Pjb = Pg.astype(np.int64), Pj.astype(np.int64)

    def near(nn, Px, X):
        """the pattern of Px X, and 200 entries anywhere"""
        Y = ((Px.astype(np.int64) @ X.astype(bool).astype(np.int64)) + sp.random(nn, nn, density=200 / nn / nn, format="csr",
                                                                                 random_state=rng)).tocsr()
        Y.eliminate_zeros()
        Y = sp.csr_matrix((np.ones(Y.nnz, np.uint8), Y.indices, Y.indptr), shape=Y.shape)
        Y.sort_indices()
        return Y
    Mg, Mj = near(NG, Pg, G), near(NJ, Pj, J)
    assert np.diff(Mg.indptr).max() * np.diff(Mj.indptr).max() <= 2048
    M = kron(Mg, Mj, "UINT8")
    C = Matrix.sparse(gb.UINT32, n, n)
    P.mxm(A, mask=M, semiring=gb.UINT32.PLUS_PAIR, out=C, desc=descriptor.S)
    memory.note()
    ks = _tokens()
    assert ks[1] == "offsets=64" and ks[0] in ENTRIES, ks
    _check_kron(C, _masked_counts(Pgb, Gb, Mg), _masked_counts(Pjb, Jb, Mj), 1 << 32, "wide-b", memory,
                [(lastG + 3, CLIQUES[0][0] + 5)])
    del C, M, P
    trim_pool(memory.torch)

    # an unmasked product of a wide operand is still refused
    with pytest.raises(gb.base.InvalidValue, match="2\\^32 entries are not supported"):
        A.mxm(A, semiring=gb.UINT8.PLUS_TIMES)
    del A
    memory.note()
