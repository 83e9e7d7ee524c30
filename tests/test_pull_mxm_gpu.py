"""GrB_mxm under a complemented mask with a saturating monoid (LOR, LAND, ANY) on the pull route (DESIGN.md section 3.2):
the rows GxB_AxB_DOT or the B200GRB_MXM_PULL rule picks walk the columns M' leaves open.  Checked against the oracle, with ANY
held to the product at the smallest inner index p, over types, value edges, mask kinds, descriptors, casts, positional
multiplies, 2^60-sized operands, the lane / warp and group boundaries, the route tokens of the rule, allocation failures, and
in multi-source BFS against scipy and against the push route at every level."""
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.csgraph as csgraph

import pygraphblas_b200 as gb
from pygraphblas_b200 import Matrix, descriptor, ffi, lib
from pygraphblas_b200.generators import rmat_csr
from oracle import oracle as orc
import util
from kernel_check import compare, entries, o_csr, record_kernels, seed_of, semiring, tunables, values
from test_alloc_failure_gpu import _sweep
from test_complement_mxm_gpu import csr, flops, mask_vals
from test_pull_mxm import MXM_PULL_LONG, axb, pull_rows

pytestmark = pytest.mark.gpu

REACHED = set()
SMALL, MEDIUM, SPLIT_FLOPS = 128, 2048, 1 << 18
PULL_T = ["BOOL", "INT8", "UINT16", "INT32", "INT64", "FP32", "FP64"]
# LOR and LAND are BOOL monoids: on the other types they fold the comparison multiplies (x of the type, z BOOL)
BOOL_SR = [("LOR", "LAND"), ("LOR", "PAIR"), ("LAND", "LOR"), ("ANY", "PAIR"), ("ANY", "FIRST"), ("ANY", "SECOND"), ("LOR", "EQ")]
NUM_SR = [("LOR", "GT"), ("LAND", "NE"), ("LOR", "EQ"), ("ANY", "PAIR"), ("ANY", "FIRST"), ("ANY", "SECOND")]


def srs_for(typ, n=None):
    return (BOOL_SR if typ == "BOOL" else NUM_SR)[:n]


def _mul(mul, a, b, dt):
    with np.errstate(all="ignore"):
        if mul == "FIRST":
            return a
        if mul == "SECOND":
            return b
        if mul == "PAIR":
            return np.ones(len(a), dt)
        raise ValueError(mul)


def smallest_p(SA, av, SB, bv, mul, dt):
    """key i * ncols + j -> the product at the smallest p of T(i,j) = fold_p A(i,p) (x) B(p,j)."""
    ncols = SB.shape[1]
    A = SA.tocoo()                                      # CSR order: the value of entry e is av[e]
    lens = np.diff(SB.indptr)[A.col].astype(np.int64)
    rows, ps = np.repeat(A.row.astype(np.int64), lens), np.repeat(A.col.astype(np.int64), lens)
    pos = np.concatenate([np.arange(SB.indptr[c], SB.indptr[c + 1]) for c in A.col]) if A.nnz else np.zeros(0, np.int64)
    pos = pos.astype(np.int64)
    keys = rows * ncols + SB.indices[pos].astype(np.int64)
    prod = _mul(mul, np.repeat(np.asarray(av), lens), np.asarray(bv)[pos], dt)
    o = np.lexsort((ps, keys))
    keys, prod = keys[o], prod[o]
    first = np.r_[True, keys[1:] != keys[:-1]] if len(keys) else np.zeros(0, bool)
    return dict(zip(keys[first].tolist(), prod[first]))


def _bits(x):
    x = np.asarray(x)
    return x.view(f"u{x.dtype.itemsize}").tolist() if x.dtype != np.bool_ else x.tolist()


def run(SA, SB, SM, label, nsr=None, types=("BOOL",), method="DOT", desc="C", mtype=None, accum=False, c_init=False, alias=False,
        want=None):
    """C<!M> = accum(C, A (+).(x) B) with GxB_AxB_<method> against the oracle; ANY values are the smallest-p product.  want:
    the expected entry tokens (default: just "pull" when a row has products)."""
    errors = []
    d = getattr(descriptor, desc) & axb(method)
    for typ in types:
        for add, mul in srs_for(typ, nsr):
            sr = (add, mul, typ)
            zt = orc.semiring_ztype(sr)
            dt = orc.DTYPES[zt]
            seed = seed_of("pull", label, sr)
            av, bv = values(seed, typ, SA.nnz, "edge", 0), values(seed + 1, typ, SB.nnz, "edge", 1)
            A = Matrix.from_csr(SA.indptr, SA.indices, av, *SA.shape, util.g_type(typ))
            B = Matrix.from_csr(SB.indptr, SB.indices, bv, *SB.shape, util.g_type(typ))
            Ao, Bo = o_csr(typ, SA, av), o_csr(typ, SB, bv)
            nrows, ncols = SA.shape[0], SB.shape[1]
            mt = mtype or "BOOL"
            mv = np.ones(SM.nnz, bool) if mtype is None else mask_vals(mt, SM.nnz, seed + 2)
            M = Matrix.from_csr(SM.indptr, SM.indices, mv, *SM.shape, util.g_type(mt))
            Mo = o_csr(mt, SM, mv)
            if alias:                                   # out = A: the BFS form F<!V> = F (+).(x) A
                C, Co = A, Ao
            elif c_init:
                Sc = csr(np.random.default_rng(seed).integers(0, 6, nrows), ncols, seed + 3)
                cv = values(seed + 4, zt, Sc.nnz, "edge", 0)
                C, Co = Matrix.from_csr(Sc.indptr, Sc.indices, cv, nrows, ncols, util.g_type(zt)), o_csr(zt, Sc, cv)
            else:
                C, Co = Matrix.sparse(util.g_type(zt), nrows, ncols), orc.SpMat(zt, nrows, ncols)
            acc = (("LOR" if add == "LOR" else "FIRST"), zt) if accum else None
            ref = orc.mxm(Co, Mo, acc, sr, Ao, Bo, desc)
            A.mxm(B, semiring=semiring(add, mul, typ), out=C, mask=M, accum=util.g_accum(acc), desc=d)
            ks = record_kernels(REACHED)
            w = want if want is not None else (["pull"] if flops(SA, SB).any() else [])
            if method == "DOT" and w != entries([k for k in ks if k]):
                errors.append(f"{label} {sr}: tokens {ks}, want {w}")
            gI, gJ, gX = C.to_arrays()
            gk = gI.astype(np.int64) * ncols + gJ.astype(np.int64)
            rk = ref.I.astype(np.int64) * ncols + ref.J.astype(np.int64)
            if add == "ANY" and not alias and not accum and not c_init:
                sm = smallest_p(SA, av, SB, bv, mul, dt)
                if not np.array_equal(gk, rk):
                    errors.append(f"{label} {sr}: presence differs from the oracle")
                elif _bits(gX) != _bits(np.asarray([sm[k] for k in gk.tolist()], dt)):
                    errors.append(f"{label} {sr}: ANY is not the smallest-p product")
                continue
            if add == "ANY":                            # the write-back's own rules: only presence is pinned here
                e = None if np.array_equal(gk, rk) else f"{label} {sr}: presence differs"
            else:
                e = compare(gk, gX, rk, ref.X, zt, add, f"{label} {sr}")
            if e:
                errors.append(e)
    assert not errors, "\n".join(errors[:20])


def mask_for(SA, SB, seed, share=0.4):
    """A mask over the product's pattern and beyond: about `share` of each product row blocked, row 1 blocks every column."""
    rng = np.random.default_rng(seed)
    nrows, ncols = SA.shape[0], SB.shape[1]
    lens = rng.binomial(ncols, share, nrows)
    if nrows > 1:
        lens[1] = ncols
    return csr(lens, ncols, seed + 1)


def _operands(seed, nrows=40, inner=300, ncols=500, alen=30, blen=20):
    rng = np.random.default_rng(seed)
    SA = csr(rng.integers(0, alen, nrows), inner, seed)
    SB = csr(rng.integers(0, blen, inner), ncols, seed + 1)
    return SA, SB


# ------------------------------------------------------------------ semirings, types, value edges
@pytest.mark.parametrize("typ", PULL_T)
def test_semirings_and_types(typ):
    SA, SB = _operands(seed_of("sr", typ))
    SM = mask_for(SA, SB, 3)
    run(SA, SB, SM, f"sr-{typ}", None, types=[typ], desc="SC")
    run(SA, SB, SM, f"sr-{typ}-r", 4, types=[typ], desc="RSC")


@pytest.mark.parametrize("struct", [False, True])
@pytest.mark.parametrize("mtype", ["BOOL", "INT8", "UINT16", "INT32", "FP32", "FP64"])
def test_mask_kinds(mtype, struct):
    SA, SB = _operands(seed_of("mk", mtype, struct))
    SM = mask_for(SA, SB, 4)
    run(SA, SB, SM, f"mk-{mtype}-{struct}", 4, types=["BOOL", "FP32"], desc="SC" if struct else "C", mtype=mtype)


@pytest.mark.parametrize("c_init,accum", [(False, True), (True, False), (True, True)])
@pytest.mark.parametrize("desc", ["C", "RC", "SC", "RSC"])
def test_descriptors_accum_and_c(desc, accum, c_init):
    SA, SB = _operands(seed_of("dc", desc, accum, c_init))
    SM = mask_for(SA, SB, 5)
    run(SA, SB, SM, f"dc-{desc}", 4, types=["BOOL", "INT32"], desc=desc, accum=accum, c_init=c_init,
        mtype=None if "S" in desc else "INT16")


def test_output_aliases_the_frontier():
    n = 400
    rng = np.random.default_rng(9)
    S = csr(rng.integers(0, 12, n), n, 7)
    SM = csr(rng.integers(0, 150, n), n, 8)
    run(S, S, SM, "alias", 4, types=["BOOL", "FP64"], desc="RSC", alias=True)


# ------------------------------------------------------------------ transposes, casts, positional, hypersparse
@pytest.mark.parametrize("desc", ["SCT0", "SCT1", "RSCT0T1"])
def test_transposed_operands(desc):
    SA, SB = _operands(seed_of("tr", desc), nrows=30, inner=200, ncols=250)
    SM = mask_for(SA, SB, 6)
    t0, t1 = "T0" in desc, "T1" in desc
    SAs = SA.T.tocsr() if t0 else SA
    SBs = SB.T.tocsr() if t1 else SB
    for S in (SAs, SBs):
        S.sort_indices()
    for typ in ("BOOL", "INT64", "FP32"):
        for add, mul in srs_for(typ):
            sr = (add, mul, typ)
            zt = orc.semiring_ztype(sr)
            seed = seed_of("trv", desc, sr)
            av, bv = values(seed, typ, SAs.nnz, "edge", 0), values(seed + 1, typ, SBs.nnz, "edge", 1)
            A = Matrix.from_csr(SAs.indptr, SAs.indices, av, *SAs.shape, util.g_type(typ))
            B = Matrix.from_csr(SBs.indptr, SBs.indices, bv, *SBs.shape, util.g_type(typ))
            M = Matrix.from_csr(SM.indptr, SM.indices, np.ones(SM.nnz, bool), *SM.shape, gb.BOOL)
            C = Matrix.sparse(util.g_type(zt), SA.shape[0], SB.shape[1])
            for _ in range(2):                              # the second call reuses the cached transpose
                A.mxm(B, semiring=semiring(add, mul, typ), out=C, mask=M, desc=getattr(descriptor, desc) & axb("DOT"))
                assert entries(record_kernels(REACHED)) == ["pull"]
            ref = orc.mxm(orc.SpMat(zt, SA.shape[0], SB.shape[1]), o_csr("BOOL", SM, np.ones(SM.nnz, bool)), None, sr,
                          o_csr(typ, SAs, av), o_csr(typ, SBs, bv), desc)
            gI, gJ, gX = C.to_arrays()
            n = SB.shape[1]
            gk, rk = gI.astype(np.int64) * n + gJ, ref.I.astype(np.int64) * n + ref.J
            if add == "ANY":
                # op(A), op(B) in CSR with their values
                oa = sp.csr_matrix((np.arange(SAs.nnz), SAs.indices, SAs.indptr), SAs.shape)
                ob = sp.csr_matrix((np.arange(SBs.nnz), SBs.indices, SBs.indptr), SBs.shape)
                oa, ob = (oa.T.tocsr() if t0 else oa), (ob.T.tocsr() if t1 else ob)
                oa.sort_indices(); ob.sort_indices()
                sm = smallest_p(oa, np.asarray(av)[oa.data.astype(np.int64)], ob, np.asarray(bv)[ob.data.astype(np.int64)], mul,
                                orc.DTYPES[typ])
                assert np.array_equal(gk, rk), (desc, sr)
                assert _bits(gX) == _bits(np.asarray([sm[k] for k in gk.tolist()], orc.DTYPES[typ])), (desc, sr)
            else:
                assert compare(gk, gX, rk, ref.X, zt, add, f"{desc} {sr}") is None


def test_casts():
    """INT8 and FP64 operands into FP32 LOR_GT / ANY_SECOND / ANY_FIRST: the casts of op(A) and of op(B)' around the pull."""
    SA, SB = _operands(seed_of("casts"))
    SM = mask_for(SA, SB, 12)
    rng = np.random.default_rng(5)
    av, bv = rng.integers(-2, 3, SA.nnz).astype(np.int8), (rng.integers(-2, 3, SB.nnz) / 2).astype(np.float64)
    A = Matrix.from_csr(SA.indptr, SA.indices, av, *SA.shape, gb.INT8)
    B = Matrix.from_csr(SB.indptr, SB.indices, bv, *SB.shape, gb.FP64)
    M = Matrix.from_csr(SM.indptr, SM.indices, np.ones(SM.nnz, bool), *SM.shape, gb.BOOL)
    Af, Bf = av.astype(np.float32), bv.astype(np.float32)
    for add, mul in (("LOR", "GT"), ("ANY", "SECOND"), ("ANY", "FIRST")):
        zt = orc.semiring_ztype((add, mul, "FP32"))
        C = Matrix.sparse(util.g_type(zt), SA.shape[0], SB.shape[1])
        A.mxm(B, semiring=semiring(add, mul, "FP32"), out=C, mask=M, desc=descriptor.RSC & axb("DOT"))
        assert entries(record_kernels(REACHED)) == ["pull"]
        ref = orc.mxm(orc.SpMat(zt, *C.shape), o_csr("BOOL", SM, np.ones(SM.nnz, bool)), None, (add, mul, "FP32"),
                      o_csr("FP32", SA, Af), o_csr("FP32", SB, Bf), "RSC")
        gI, gJ, gX = C.to_arrays()
        n = SB.shape[1]
        gk, rk = gI.astype(np.int64) * n + gJ, ref.I.astype(np.int64) * n + ref.J
        if add == "ANY":
            sm = smallest_p(SA, Af, SB, Bf, mul, np.float32)
            assert np.array_equal(gk, rk) and _bits(gX) == _bits(np.asarray([sm[k] for k in gk.tolist()], np.float32)), mul
        else:
            assert compare(gk, gX, rk, ref.X, zt, add, mul) is None


def _dict(M):
    I, J, X = M.to_lists()
    return {(int(i), int(j)): x for i, j, x in zip(I, J, X)}


def _mat(d, typ, nrows, ncols):
    I, J = zip(*sorted(d)) if d else ((), ())
    return Matrix.from_lists(list(I), list(J), [d[e] for e in sorted(d)], nrows, ncols, util.g_type(typ))


@pytest.mark.parametrize("hyper", [False, True])
@pytest.mark.parametrize("side", ["A", "B"])
def test_positional_smallest_p(side, hyper):
    """ANY_SECONDI and ANY_FIRSTJ give p: the smallest p of every entry, whichever operand the inner form rewrites
    (the one with fewer entries), also for 2^60-sized operands."""
    rng = np.random.default_rng(seed_of("pos", side, hyper))
    n = 120
    na, nb = (600, 2400) if side == "A" else (2400, 600)
    A = {(int(i), int(j)): 1.0 for i, j in zip(rng.integers(0, n, na), rng.integers(0, n, na))}
    B = {(int(i), int(j)): 1 for i, j in zip(rng.integers(0, n, nb), rng.integers(0, n, nb))}
    Mv = {(int(i), int(j)): True for i, j in zip(rng.integers(0, n, 3000), rng.integers(0, n, 3000))}
    want = {}
    for (i, p), _ in sorted(A.items(), key=lambda e: e[0][1]):
        for (q, j), _ in B.items():
            if q == p and (i, j) not in Mv and (i, j) not in want:
                want[(i, j)] = p
    dim = (1 << 60) if hyper else n
    sh = (lambda d: {(i * (1 << 40) + 5, j * (1 << 40) + 5): v for (i, j), v in d.items()}) if hyper else (lambda d: d)
    off = (1 << 40) if hyper else 1
    Am, Bm, Mm = _mat(sh(A), "FP32", dim, dim), _mat(sh(B), "INT8", dim, dim), _mat(sh(Mv), "BOOL", dim, dim)
    for mul in ("SECONDI", "FIRSTJ"):
        C = Matrix.sparse(gb.INT64, dim, dim)
        Am.mxm(Bm, semiring=getattr(gb.INT64, f"ANY_{mul}"), out=C, mask=Mm, desc=descriptor.SC & axb("DOT"))
        ks = record_kernels(REACHED)
        assert "pull" in ks and "positional=inner" in ks, ks
        got = _dict(C)
        if hyper:                                       # the compact index space: p is the rank of the inner index
            inner = sorted({p for (_, p) in A} | {q for (q, _) in B})
            rank = {v * off + 5: r for r, v in enumerate(inner)}
            assert set(got) == {(i * off + 5, j * off + 5) for (i, j) in want}, (side, mul)
            assert all(int(got[(i * off + 5, j * off + 5)]) in (p * off + 5, rank.get(p * off + 5, -1)) for (i, j), p in want.items())
        else:
            assert got == want, (side, mul)


# ------------------------------------------------------------------ structure edges
@pytest.mark.parametrize("ncols", [1, 31, 32, 33])
@pytest.mark.parametrize("inner", [1, 31, 32, 33])
def test_small_dimensions(ncols, inner):
    rng = np.random.default_rng(seed_of("dim", ncols, inner))
    SA = csr(rng.integers(0, inner + 1, 20), inner, 1)
    SB = csr(rng.integers(0, ncols + 1, inner), ncols, 2)
    SM = csr(rng.integers(0, ncols + 1, 20), ncols, 3)
    run(SA, SB, SM, f"dim-{ncols}-{inner}", 5, types=["BOOL", "INT32"], desc="RSC")


@pytest.mark.parametrize("clen", [MXM_PULL_LONG - 1, MXM_PULL_LONG, MXM_PULL_LONG + 1, 4 * MXM_PULL_LONG + 5])
def test_column_lengths_at_the_lane_warp_threshold(clen):
    """Columns of op(B) of clen entries next to short ones, and A rows meeting each column at its first, last or no entry."""
    inner, ncols, nrows = 4 * MXM_PULL_LONG + 40, 70, 50
    rng = np.random.default_rng(seed_of("clen", clen))
    Bt = [np.sort(rng.choice(inner, clen if j % 3 == 0 else int(rng.integers(0, 8)), replace=False)) for j in range(ncols)]
    SBt = sp.csr_matrix((np.ones(sum(map(len, Bt))), np.concatenate(Bt), np.r_[0, np.cumsum([len(b) for b in Bt])]), (ncols, inner))
    SB = SBt.T.tocsr()
    SB.sort_indices()
    lens = rng.integers(0, 4, nrows)
    SA = csr(lens, inner, 5).tolil()
    for i in range(0, nrows, 5):                        # the last entry of a long column only: a full walk to find it
        SA[i, int(Bt[0][-1])] = 1
    SA = SA.tocsr()
    SA.sort_indices()
    SM = csr(rng.integers(0, ncols // 2, nrows), ncols, 6)
    run(SA, SB, SM, f"clen-{clen}", None, types=["BOOL", "FP64"], desc="RSC")


def test_blocked_rows_and_empty_rows():
    SA, SB = _operands(seed_of("blk"))
    SA = SA.tolil()
    SA[3, :] = 0
    SA[4, :] = 0
    SA = SA.tocsr()
    SA.eliminate_zeros()
    SM = mask_for(SA, SB, 7).tolil()
    SM[0, :] = 1                                        # row 0 blocks every column; rows 3, 4 have no products
    SM = SM.tocsr()
    SM.sort_indices()
    run(SA, SB, SM, "blk", 5, types=["BOOL", "INT64"], desc="SC")
    empty = csr([0] * SA.shape[0], SB.shape[1], 1)      # a mask with no entries: every column open
    run(SA, SB, empty, "open", 5, types=["BOOL"], desc="SC")


def group_rows(inner, ncols, budget):
    words, iwords = (ncols + 31) // 32, (inner + 31) // 32
    return max(1, budget // ((iwords + 2 * words) * 4 + words * 8))


def test_many_groups():
    SA, SB = _operands(seed_of("grp"), nrows=90)
    SM = mask_for(SA, SB, 8)
    budget = 3000
    assert group_rows(SA.shape[1], SB.shape[1], budget) < 20
    with tunables(B200GRB_MXM_PULL_BUDGET=budget):
        run(SA, SB, SM, "grp", None, types=["BOOL", "FP32"], desc="RSC")
    with tunables(B200GRB_MXM_PULL_BUDGET=1):           # one row per group
        run(SA, SB, SM, "grp1", 4, types=["INT8"], desc="SC")


# ------------------------------------------------------------------ which rows pull: the route tokens
def bins(f):
    out = []
    for name, lo, hi in (("esc-small", 0, SMALL), ("esc-medium", SMALL, MEDIUM), ("spa", MEDIUM, SPLIT_FLOPS), ("spa-split", SPLIT_FLOPS, np.inf)):
        if ((f > lo) & (f <= hi)).any():
            out.append(name)
    return out


def rule_operands():
    """Rows from 1 to ~3000 products and masks from none to most of the row: rows on both sides of the rule at alpha 4."""
    rng = np.random.default_rng(11)
    inner, ncols = 2000, 3000
    SB = csr(rng.integers(0, 10, inner), ncols, 2)
    SA = csr(np.r_[[1, 2, 5, 20, 60, 200, 600], rng.integers(0, 40, 25)], inner, 3)
    SM = csr(np.r_[[0, 2900, 10, 2990, 1000, 0, 2500], rng.integers(0, ncols, 25)], ncols, 4)
    return SA, SB, SM


@pytest.mark.parametrize("method,alpha", [("DOT", 0), ("SAXPY", 4), ("HASH", 4), ("GUSTAVSON", 4), ("DEFAULT", 0), ("DEFAULT", 1),
                                          ("DEFAULT", 4), ("DEFAULT", 32)])
def test_route_tokens_follow_the_rule(method, alpha):
    SA, SB, SM = rule_operands()
    f = flops(SA, SB)
    pr = pull_rows(f, np.diff(SM.indptr), SB.shape[1], SB.nnz, method, alpha)
    if method == "DEFAULT" and alpha == 4:
        assert pr.any() and (~pr & (f > 0)).any()       # both sides of the inequality
    want = bins(np.where(pr, 0, f)) + (["pull"] if pr.any() else [])
    with tunables(B200GRB_MXM_PULL=alpha):
        for add, mul in (("LOR", "LAND"), ("ANY", "PAIR")):
            A = Matrix.from_csr(SA.indptr, SA.indices, np.ones(SA.nnz, bool), *SA.shape, gb.BOOL)
            B = Matrix.from_csr(SB.indptr, SB.indices, np.ones(SB.nnz, bool), *SB.shape, gb.BOOL)
            M = Matrix.from_csr(SM.indptr, SM.indices, np.ones(SM.nnz, bool), *SM.shape, gb.BOOL)
            C = A.mxm(B, semiring=semiring(add, mul, "BOOL"), mask=M, desc=descriptor.SC & axb(method))
            ks = record_kernels(REACHED)
            assert entries(ks) == want, (method, alpha, ks, want)
            if pr.any():
                assert ks[-1] == ("pull=dot" if method == "DOT" else "pull=auto"), ks
            ref = orc.mxm(orc.SpMat("BOOL", *C.shape), o_csr("BOOL", SM, np.ones(SM.nnz, bool)), None, (add, mul, "BOOL"),
                          o_csr("BOOL", SA, np.ones(SA.nnz, bool)), o_csr("BOOL", SB, np.ones(SB.nnz, bool)), "SC")
            gI, gJ, gX = C.to_arrays()
            n = SB.shape[1]
            assert compare(gI.astype(np.int64) * n + gJ, gX, ref.I.astype(np.int64) * n + ref.J, ref.X, "BOOL", add, method) is None


def test_dot_on_ineligible_calls_changes_nothing():
    SA, SB, SM = rule_operands()
    A = Matrix.from_csr(SA.indptr, SA.indices, np.ones(SA.nnz, np.float32), *SA.shape, gb.FP32)
    B = Matrix.from_csr(SB.indptr, SB.indices, np.ones(SB.nnz, np.float32), *SB.shape, gb.FP32)
    M = Matrix.from_csr(SM.indptr, SM.indices, np.ones(SM.nnz, bool), *SM.shape, gb.BOOL)
    Ab = Matrix.from_csr(SA.indptr, SA.indices, np.ones(SA.nnz, bool), *SA.shape, gb.BOOL)
    Bb = Matrix.from_csr(SB.indptr, SB.indices, np.ones(SB.nnz, bool), *SB.shape, gb.BOOL)
    cases = [(A, B, gb.FP32.PLUS_TIMES, M, "SC"), (A, B, gb.FP32.MIN_PLUS, M, "C"),        # other monoids
             (Ab, Bb, gb.BOOL.LOR_LAND, M, "S"), (Ab, Bb, gb.BOOL.ANY_PAIR, None, "")]       # a mask that is not complemented, none
    for X, Y, s, m, d in cases:
        base = getattr(descriptor, d) if d else descriptor.Default
        X.mxm(Y, semiring=s, mask=m, desc=base)
        plain = record_kernels(REACHED)
        C = X.mxm(Y, semiring=s, mask=m, desc=(base & axb("DOT")) if d else axb("DOT"))
        assert record_kernels(REACHED) == plain and "pull" not in plain, (s, d, plain)
    with tunables(B200GRB_MXM_PULL=1000):
        A.mxm(B, semiring=gb.FP32.PLUS_TIMES, mask=M, desc=descriptor.SC)
        assert "pull" not in record_kernels(REACHED)
    del C


def stats():
    fl, no = ffi.new("uint64_t*"), ffi.new("uint64_t*")
    lib.B200_last_mxm_stats(fl, no)
    return int(fl[0]), int(no[0])


def test_determinism_and_stats():
    SA, SB, SM = rule_operands()
    for add, mul, typ in (("LOR", "GT", "FP32"), ("ANY", "SECOND", "INT64"), ("LAND", "LOR", "BOOL")):
        av, bv = values(1, typ, SA.nnz, "edge", 0), values(2, typ, SB.nnz, "edge", 1)
        A = Matrix.from_csr(SA.indptr, SA.indices, av, *SA.shape, util.g_type(typ))
        B = Matrix.from_csr(SB.indptr, SB.indices, bv, *SB.shape, util.g_type(typ))
        M = Matrix.from_csr(SM.indptr, SM.indices, np.ones(SM.nnz, bool), *SM.shape, gb.BOOL)
        s = semiring(add, mul, typ)
        A.mxm(B, semiring=s, mask=M, desc=descriptor.SC)
        push = stats()
        outs = []
        for _ in range(2):
            C = A.mxm(B, semiring=s, mask=M, desc=descriptor.SC & axb("DOT"))
            assert entries(record_kernels(REACHED)) == ["pull"]
            assert stats() == push, (typ, stats(), push)
            I, J, X = C.to_arrays()
            outs.append((I.tolist(), J.tolist(), _bits(X)))
        assert outs[0] == outs[1]


def test_allocation_failures():
    SA, SB, SM = rule_operands()

    def make():
        A = Matrix.from_csr(SA.indptr, SA.indices, np.ones(SA.nnz, np.int8), *SA.shape, gb.INT8)
        B = Matrix.from_csr(SB.indptr, SB.indices, np.ones(SB.nnz, np.int8), *SB.shape, gb.INT8)
        M = Matrix.from_csr(SM.indptr, SM.indices, np.ones(SM.nnz, bool), *SM.shape, gb.BOOL)
        return A, B, M

    def call(A, B, M):                                   # INT8 operands of an INT32 multiply: op(B)' is built and cast
        C = Matrix.sparse(gb.BOOL, *M.shape)
        A.mxm(B, semiring=semiring("LOR", "EQ", "INT32"), out=C, mask=M, desc=descriptor.RSC & axb("DOT"))
        assert "pull" in record_kernels(REACHED)
        return C

    def check(ref):
        I, J, X = ref
        P = (sp.csr_matrix((np.ones(SA.nnz), SA.indices, SA.indptr), SA.shape) @ sp.csr_matrix((np.ones(SB.nnz), SB.indices, SB.indptr), SB.shape)).tocsr()
        P.sort_indices()
        n = SB.shape[1]
        pk = np.repeat(np.arange(P.shape[0], dtype=np.int64), np.diff(P.indptr)) * n + P.indices
        mk = np.repeat(np.arange(SM.shape[0], dtype=np.int64), np.diff(SM.indptr)) * n + SM.indices
        keep = ~np.isin(pk, mk)
        assert np.array_equal(np.asarray(I, np.int64) * n + J, pk[keep])
        assert np.array_equal(X, np.ones(int(keep.sum()), bool))

    assert _sweep(make, call, check) > 1


# ------------------------------------------------------------------ multi-source BFS
def _rmat(scale, seed=1, ef=8):
    n, indptr, indices = rmat_csr(scale, ef, seed=seed)
    S = sp.csr_matrix((np.ones(len(indices), np.float32), indices, indptr), shape=(n, n))
    S.sort_indices()
    return n, S


@pytest.mark.parametrize("scale,k", [(10, 4), (11, 64), (13, 16), (17, 4)])
def test_multi_source_bfs_dot_and_auto(scale, k):
    """Levels equal to scipy's, and F equal to the push route's at every level, with DOT on every level and with auto."""
    n, S = _rmat(scale, ef=16 if scale > 12 else 8)
    A = Matrix.from_csr(S.indptr, S.indices, np.ones(S.nnz, bool), n, n, gb.BOOL)
    sources = np.argsort(-np.diff(S.indptr), kind="stable")[:k]
    want = csgraph.shortest_path(S, unweighted=True, indices=sources)
    want = np.where(np.isinf(want), -1, want).astype(np.int64)
    for sr in (gb.BOOL.ANY_PAIR, gb.BOOL.LOR_LAND):
        for arm, alpha in (("DOT", 0), ("DEFAULT", 14)):
            with tunables(B200GRB_MXM_PULL=alpha):
                F = Matrix.from_lists(list(range(k)), list(sources), [True] * k, k, n, gb.BOOL)
                Fp, V = F.dup(), F.dup()
                lev = np.full((k, n), -1, np.int64)
                lev[np.arange(k), sources] = 0
                seen = set()
                for d in range(1, n + 1):
                    Fp.mxm(A, semiring=sr, out=Fp, mask=V, desc=descriptor.RSC & axb("SAXPY"))
                    assert "pull" not in record_kernels(REACHED)
                    F.mxm(A, semiring=sr, out=F, mask=V, desc=descriptor.RSC & axb(arm))
                    seen.update(entries(record_kernels(REACHED)))
                    assert F.nvals == Fp.nvals
                    if F.nvals == 0:
                        break
                    I, J, X = F.to_arrays()
                    Ip, Jp, Xp = Fp.to_arrays()
                    assert np.array_equal(I, Ip) and np.array_equal(J, Jp) and np.array_equal(X, Xp), (arm, d)
                    assert (lev[I, J] == -1).all()
                    lev[I, J] = d
                    V.eadd(F, gb.BOOL.LOR, out=V)
                assert np.array_equal(lev, want), (arm, str(sr))
                assert "pull" in seen, (arm, seen)


@pytest.mark.parametrize("scale", [10, 14])
def test_parent_bfs(scale):
    """P<!V> = F ANY_SECONDI A with DOT: every parent is a frontier in-neighbour, and the smallest one."""
    n, S = _rmat(scale, seed=2)
    k = 8
    A = Matrix.from_csr(S.indptr, S.indices, np.ones(S.nnz, bool), n, n, gb.BOOL)
    ST = S.T.tocsr()
    ST.sort_indices()
    sources = np.argsort(-np.diff(S.indptr), kind="stable")[:k]
    F = Matrix.from_lists(list(range(k)), list(sources), [True] * k, k, n, gb.BOOL)
    V = F.dup()
    fr = [np.array([s]) for s in sources]
    for d in range(1, n + 1):
        P = Matrix.sparse(gb.INT64, k, n)
        F.mxm(A, semiring=gb.INT64.ANY_SECONDI, out=P, mask=V, desc=descriptor.RSC & axb("DOT"))
        assert "pull" in record_kernels(REACHED)
        if P.nvals == 0:
            break
        I, J, X = P.to_arrays()
        for s in range(k):
            sel = I == s
            for j, par in zip(J[sel].tolist(), X[sel].tolist()):
                ins = ST.indices[ST.indptr[j]:ST.indptr[j + 1]]
                cand = np.intersect1d(ins, fr[s])
                assert len(cand) and par == cand.min(), (d, s, j, par)
        fr = [J[I == s] for s in range(k)]
        F = Matrix.from_lists(I.tolist(), J.tolist(), [True] * len(I), k, n, gb.BOOL)
        V.eadd(F, gb.BOOL.LOR, out=V)
