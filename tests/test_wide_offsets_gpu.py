"""The wide route of mxv / vxm and the chunked transpose: the code that serves matrices with 2^32 or more entries.

A matrix without 32-bit row offsets (nnz >= 2^32) runs mxv / vxm on 64-bit-offset plan, pull and push kernels and is
transposed in chunks.  B200_debug_wide(chunk) puts every matrix on that route, so the first part runs each case twice at
small sizes -- narrow, then wide on fresh copies of the operands -- and requires the same route (plus the `offsets=64`
token) and the same bits, with one comparison against the oracle per case.  The second part builds a real matrix of
2^32 + 2^26 entries on the device as kron(G, J) and checks mxv, vxm (a BFS), the row reduce and the refusal of mxm
against identities computed on the small factors; it skips, with the reason, when the card lacks the free memory."""
import contextlib

import numpy as np
import pytest
import scipy.sparse as sp

import pygraphblas_b200 as gb
from pygraphblas_b200 import Matrix, Vector, descriptor, ffi, lib
from oracle import oracle as orc
import util
from kernel_check import compare, fp_pool_for, last_kernel, o_csr, seed_of, semiring, tunables, values, vec_products
from test_structure_edges_gpu import csr
from test_value_edges_gpu import spmv_pattern

pytestmark = pytest.mark.gpu


@contextlib.contextmanager
def wide(chunk):
    lib.B200_debug_wide(chunk)
    try:
        yield
    finally:
        lib.B200_debug_wide(0)


def _bits(x):
    x = np.ascontiguousarray(x)
    return x.view(f"u{x.dtype.itemsize}") if x.dtype != np.bool_ else x


# ------------------------------------------------------------------ shapes
def run_ends():
    """Rows ending on, before and after run ends (256 entries), rows straddling several runs, empty rows between."""
    lens = [0, 256, 255, 1, 0, 0, 257, 511, 3, 0, 1024, 7, 0, 300, 2, 0] * 3
    return csr(lens, 1500, seed=3)


SHAPES = {"run-ends": run_ends, "run": lambda: spmv_pattern("run"), "rmat": lambda: spmv_pattern("rmat"),
          "pull": lambda: spmv_pattern("pull")}

# (name, shape, semiring, form, options): form is "mxv" or "vxm"; options: sparse_u (density), mask ("value", "struct"),
# comp (complemented mask), accum, replace, desc ("T0" / "T1"), env, kernel (the route's entry), pos (positional semiring)
CASES = [
    ("run-specialised", "run-ends", ("PLUS", "TIMES", "FP64"), "mxv", dict(kernel="run")),
    ("run-specialised-vxm", "run-ends", ("MIN", "PLUS", "INT32"), "vxm", dict(kernel="run")),
    ("run-specialised-T0", "run", ("PLUS", "TIMES", "FP32"), "mxv", dict(kernel="run", desc="T0")),
    ("run-specialised-vxm-T1", "run", ("PLUS", "SECOND", "UINT64"), "vxm", dict(kernel="run", desc="T1")),
    ("run-generic", "run-ends", ("MAX", "MINUS", "INT16"), "mxv", dict(kernel="run")),
    ("run-generic-vxm", "run", ("BXOR", "TIMES", "UINT8"), "vxm", dict(kernel="run")),
    ("run-generic-fp", "run", ("PLUS", "MINUS", "FP32"), "mxv", dict(kernel="run")),
    ("run-bool", "run-ends", ("LOR", "LAND", "BOOL"), "mxv", dict(kernel="run")),
    ("sparse-u", "run-ends", ("PLUS", "TIMES", "INT64"), "mxv", dict(kernel="run (sparse u)", sparse_u=0.6)),
    ("sparse-u-vxm", "run", ("MAX", "DIV", "FP64"), "vxm", dict(kernel="run (sparse u)", sparse_u=0.5)),
    ("accum-mask", "run", ("PLUS", "TIMES", "INT32"), "mxv", dict(kernel="run", mask="value", accum=True)),
    ("replace-struct", "run", ("MIN", "PLUS", "FP64"), "vxm", dict(kernel="run", mask="struct", replace=True, accum=True)),
    ("hot-c1", "rmat", ("PLUS", "TIMES", "FP32"), "mxv", dict(kernel="run+hot-table (TMA-staged)",
                                                                env={"B200GRB_SPMV_HOT": 128, "B200GRB_SPMV_CLUSTER": 1})),
    ("hot-c2", "rmat", ("LOR", "LAND", "BOOL"), "mxv", dict(kernel="run+hot-table (TMA-staged)",
                                                            env={"B200GRB_SPMV_HOT": 128, "B200GRB_SPMV_CLUSTER": 2})),
    ("hot-c2-int", "rmat", ("MIN", "PLUS", "UINT64"), "vxm", dict(kernel="run+hot-table (TMA-staged)",
                                                                  env={"B200GRB_SPMV_HOT": 128, "B200GRB_SPMV_CLUSTER": 2})),
    ("pull", "pull", ("LOR", "LAND", "BOOL"), "mxv", dict(kernel="pull", mask="value", comp=True, replace=True)),
    ("pull-vxm", "pull", ("LAND", "LOR", "BOOL"), "vxm", dict(kernel="pull", mask="struct")),
    ("pull-any", "pull", ("ANY", "SECOND", "INT64"), "mxv", dict(kernel="pull", mask="value")),
    ("push", "pull", ("LOR", "LAND", "BOOL"), "mxv", dict(kernel="push", mask="struct", comp=True, sparse_u=0.003)),
    ("push-vxm", "pull", ("LOR", "LAND", "BOOL"), "vxm", dict(kernel="push", mask="value", sparse_u=0.003)),
    ("push-forced", "pull", ("ANY", "TIMES", "FP32"), "mxv", dict(kernel="push", mask="struct", sparse_u=0.2,
                                                                  env={"B200GRB_FORCE_PUSH": 1})),
    ("positional-run", "run", ("MIN", "SECONDI", "INT64"), "mxv", dict(kernel="run", pos=True)),
    ("positional-count", "run-ends", ("PLUS", "FIRSTI", "INT64"), "vxm", dict(kernel="run", pos=True)),
    ("positional-pull", "pull", ("ANY", "SECONDI", "INT64"), "mxv", dict(kernel="pull", pos=True, mask="struct")),
]


def _desc(o):
    name = ("R" if o.get("replace") else "") + ("S" if o.get("mask") == "struct" else "") + ("C" if o.get("comp") else "")
    name += o.get("desc", "")
    return name


def _call(S, av, sr, form, o, uv, upres, mask, w0, typ):
    """One mxv / vxm on fresh operands; returns (I, X, tokens)."""
    nrows, ncols = S.shape
    add, mul, _ = sr
    A = Matrix.from_csr(S.indptr, S.indices, av, nrows, ncols, util.g_type(typ))
    vxm = form == "vxm"
    if o.get("kernel") == "push" and not vxm:      # A' in HBM: the other orientation the push kernel walks, as a BFS has it
        Vector.sparse(util.g_type(typ), nrows).vxm(A, semiring=semiring("LOR" if typ == "BOOL" else "ANY", "FIRST", typ))
    u = Vector.from_numpy(uv, present=None if upres.all() else upres, typ=util.g_type(typ))
    zt = orc.semiring_ztype(sr) if not o.get("pos") else sr[2]
    M = None
    if mask is not None:
        M = Vector.from_lists(mask[1], mask[2], mask[3], util.g_type(mask[0]))
    wI, wX, wn = w0
    w = Vector.from_lists(wI, wX, wn, util.g_type(zt)) if len(wI) else Vector.sparse(util.g_type(zt), wn)
    s = getattr(util.g_type(typ), f"{add}_{mul}") if o.get("pos") else semiring(*sr)
    acc = util.g_accum((add if add != "ANY" else "FIRST", zt)) if o.get("accum") else None
    d = _desc(o)
    d = getattr(descriptor, d) if d else None
    if vxm:
        u.vxm(A, semiring=s, out=w, mask=M, accum=acc, desc=d)
    else:
        A.mxv(u, semiring=s, out=w, mask=M, accum=acc, desc=d)
    ks = last_kernel().split(";")
    I, X = w.to_arrays()
    return I, X, ks


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_wide_equals_narrow(case):
    name, shape, sr, form, o = case
    add, mul, typ = sr
    S = SHAPES[shape]()
    nrows, ncols = S.shape
    vxm = form == "vxm"
    tran = (o.get("desc") == "T1") if vxm else (o.get("desc") == "T0")
    pulled_T = vxm != tran                         # the call pulls along A' (vxm without T1, mxv with T0)
    n_in, n_out = (nrows, ncols) if pulled_T else (ncols, nrows)
    rng = np.random.default_rng(seed_of("wide", name, bits=32))
    pool = fp_pool_for(add, mul) if typ in util.FP_T else "edge"
    av = values(seed_of("wide-a", name), typ, S.nnz, pool, 0)
    if o.get("pos"):
        av = np.ones(S.nnz, orc.DTYPES[typ])
    uv = values(seed_of("wide-u", name), typ, n_in, pool, 1)
    upres = rng.random(n_in) < o["sparse_u"] if "sparse_u" in o else np.ones(n_in, bool)
    zt = orc.semiring_ztype(sr) if not o.get("pos") else typ
    mask = None
    if o.get("mask"):
        idx = np.flatnonzero(rng.random(n_out) < 0.7)
        if o["mask"] == "struct":
            mask = ("BOOL", idx, np.ones(len(idx), bool), n_out)
        else:
            mask = ("INT32", idx, rng.integers(0, 3, len(idx)).astype(np.int32), n_out)
    wI = np.flatnonzero(rng.random(n_out) < 0.5) if o.get("accum") else np.zeros(0, np.int64)
    wX = values(seed_of("wide-w", name), zt, len(wI), pool if zt == typ else "edge", 1)
    w0 = (wI, wX, n_out)
    with tunables(**o.get("env", {})):
        nI, nX, nks = _call(S, av, sr, form, o, uv, upres, mask, w0, typ)
        with wide(7 if S.nnz < 20000 else S.nnz // 5 + 1):      # transposes in thousands of chunks, or in 5 for the large shapes
            gI, gX, gks = _call(S, av, sr, form, o, uv, upres, mask, w0, typ)
    assert o["kernel"] in nks, (name, nks)
    assert "offsets=64" not in nks, (name, nks)
    assert gks == nks[:1] + ["offsets=64"] + nks[1:], (name, nks, gks)
    assert np.array_equal(nI, gI), name
    if add != "ANY":
        assert np.array_equal(_bits(nX), _bits(gX)), (name, nX[:5], gX[:5])
    if o.get("pos"):
        return                                     # positional calls are checked against their model in test_positional_gpu.py
    # the oracle, once per case
    Ao = o_csr(typ, S, av)
    uo = orc.SpVec(typ, n_in, np.flatnonzero(upres), uv[upres])
    Mo = orc.SpVec(mask[0], n_out, mask[1], mask[2]) if mask is not None else None
    wo = orc.SpVec(zt, n_out, wI, wX)
    acc = (add if add != "ANY" else "FIRST", zt) if o.get("accum") else None
    d = _desc(o) or None
    ref = orc.vxm(wo, Mo, acc, sr, uo, Ao, d) if vxm else orc.mxv(wo, Mo, acc, sr, Ao, uo, d)
    cands = vec_products(uv, upres, S, av, mul, vxm) if add == "ANY" else None
    e = compare(gI, gX, ref.I, ref.X, zt, add, f"{name} wide", cands)
    assert e is None, e


# ------------------------------------------------------------------ the chunked transpose
@pytest.mark.parametrize("chunk", [1, 7, 256, 1 << 30])
@pytest.mark.parametrize("typ", ["BOOL", "UINT16", "FP32", "FP64"])
def test_chunked_transpose(chunk, typ):
    S = run_ends() if chunk == 1 else spmv_pattern("pull")
    nrows, ncols = S.shape
    av = values(seed_of("wide-t", typ), typ, S.nnz, "edge", 0)
    A0 = Matrix.from_csr(S.indptr, S.indices, av, nrows, ncols, util.g_type(typ))
    P0, J0, X0 = A0.transpose().to_csr()
    with wide(chunk):
        A1 = Matrix.from_csr(S.indptr, S.indices, av, nrows, ncols, util.g_type(typ))
        P1, J1, X1 = A1.transpose().to_csr()
    assert np.array_equal(P0, P1) and np.array_equal(J0, J1) and np.array_equal(_bits(X0), _bits(X1))
    T = sp.csr_matrix((np.arange(S.nnz), S.indices, S.indptr), shape=S.shape).T.tocsr()
    T.sort_indices()
    assert np.array_equal(P1, T.indptr) and np.array_equal(J1, T.indices)
    assert np.array_equal(_bits(X1), _bits(av[T.data]))


# ------------------------------------------------------------------ a real wide matrix: A = kron(G, J), nnz(A) = 2^32 + 2^26
NG, NJ = 4096, 4096                            # n = 2^24 rows and columns
NNZ_G, NNZ_J = (1 << 16) + (1 << 10), 1 << 16
NNZ = NNZ_G * NNZ_J                            # 4 362 076 160
GB_ = 1e9
# per entry: col 4 B + value 1 B; the run plan ~0.5 B; the hot plan's encoded columns 4 B; A' 5 B.  The transpose's chunk
# scratch ~3.2 GB, and 16 B per column while it runs.
PLAN_MXV = NNZ * (5 + 0.5 + 4) + 1 * GB_       # A, its run and hot plans
PLAN_BFS = NNZ * (5 + 5) + 3.5 * GB_           # A and A', plus the transpose's scratch while it runs
PLANNED = max(PLAN_MXV, PLAN_BFS)


def factor(seed, n, nnz):
    """A random n x n pattern with exactly nnz entries, every row non-empty, and its values 1..3."""
    rng = np.random.default_rng(seed)
    first = np.arange(n, dtype=np.int64) * n + rng.integers(0, n, n)           # one entry in every row
    rest = np.setdiff1d(rng.choice(n * n, nnz * 2, replace=False), first)
    keys = np.sort(np.concatenate([first, rng.choice(rest, nnz - n, replace=False)]))
    S = sp.csr_matrix((rng.integers(1, 4, nnz).astype(np.uint8), (keys // n, keys % n)), shape=(n, n))
    S.sort_indices()
    assert S.nnz == nnz and (np.diff(S.indptr) > 0).all()
    return S


class Memory:
    """Free device memory as torch sees it, and the lowest reading since start."""

    def __init__(self):
        import torch
        self.torch = torch
        self.start = torch.cuda.mem_get_info()[0]
        self.low = self.start

    def note(self):
        self.low = min(self.low, self.torch.cuda.mem_get_info()[0])

    @property
    def peak(self):
        return self.start - self.low


@pytest.fixture(scope="module")
def memory():
    m = Memory()
    if m.start < PLANNED + 2 * GB_:
        pytest.skip(f"needs {PLANNED / GB_:.1f} GB of free device memory for a matrix of {NNZ} entries, "
                    f"{m.start / GB_:.1f} GB free")
    yield m
    print(f"\nwide matrix: {NNZ} entries, planned peak {PLANNED / GB_:.1f} GB, observed peak {m.peak / GB_:.1f} GB "
          f"on {m.torch.cuda.get_device_name()}")


def kron(G, J, typ):
    n = G.shape[0] * J.shape[0]
    tg = util.g_type(typ)
    Gm = Matrix.from_csr(G.indptr, G.indices, G.data.astype(tg.dtype) if typ != "BOOL" else np.ones(G.nnz, bool), *G.shape, tg)
    Jm = Matrix.from_csr(J.indptr, J.indices, J.data.astype(tg.dtype) if typ != "BOOL" else np.ones(J.nnz, bool), *J.shape, tg)
    A = Matrix.sparse(tg, n, n)
    op = (gb.BOOL.LAND if typ == "BOOL" else gb.UINT8.TIMES).get_op()
    gb.base._check(lib.GrB_Matrix_kronecker_BinaryOp(A._matrix[0], ffi.NULL, ffi.NULL, op, Gm._matrix[0], Jm._matrix[0], ffi.NULL))
    return A


def _tokens():
    return last_kernel().split(";")


def test_real_wide_mxv(memory):
    G, J = factor(1, NG, NNZ_G), factor(2, NJ, NNZ_J)
    n = NG * NJ
    A = kron(G, J, "UINT8")
    memory.note()
    assert A.nvals == NNZ and NNZ >= (1 << 32) + (1 << 26)
    dG, dJ = np.diff(G.indptr), np.diff(J.indptr)
    # degrees: PLUS_PAIR against a dense u
    w = A.mxv(Vector.from_numpy(np.ones(n, np.int64), typ=gb.INT64), semiring=gb.INT64.PLUS_PAIR)
    memory.note()
    ks = _tokens()
    assert ks[:2] == ["run", "offsets=64"], ks
    I, X = w.to_arrays()
    assert np.array_equal(I, np.arange(n)) and np.array_equal(X, np.outer(dG, dJ).ravel())
    # separable PLUS_TIMES in UINT8 (mod 256): (A_G u_G) (x) (A_J u_J)
    rng = np.random.default_rng(3)
    uG, uJ = rng.integers(0, 256, NG).astype(np.uint8), rng.integers(0, 256, NJ).astype(np.uint8)
    w = A.mxv(Vector.from_numpy(np.outer(uG, uJ).ravel().astype(np.uint8), typ=gb.UINT8), semiring=gb.UINT8.PLUS_TIMES)
    memory.note()
    ks = _tokens()
    assert ks[:2] == ["run", "offsets=64"], ks
    yG = (G.astype(np.int64) @ uG.astype(np.int64)) % 256
    yJ = (J.astype(np.int64) @ uJ.astype(np.int64)) % 256
    I, X = w.to_arrays()
    assert np.array_equal(I, np.arange(n)) and np.array_equal(X.astype(np.int64), np.outer(yG, yJ).ravel() % 256)
    # row sums through the row reduce (UINT8 PLUS, mod 256)
    r = A.reduce_vector(gb.UINT8.PLUS_MONOID)
    memory.note()
    sG = np.asarray(G.astype(np.int64).sum(axis=1)).ravel()
    sJ = np.asarray(J.astype(np.int64).sum(axis=1)).ravel()
    I, X = r.to_arrays()
    assert np.array_equal(I, np.arange(n)) and np.array_equal(X.astype(np.int64), np.outer(sG, sJ).ravel() % 256)
    # LOR_SECOND with a dense BOOL u on the hot-table kernel
    bG, bJ = rng.random(NG) < 0.01, rng.random(NJ) < 0.01
    with tunables(B200GRB_SPMV_HOT=128):
        w = A.mxv(Vector.from_numpy(np.outer(bG, bJ).ravel(), typ=gb.BOOL), semiring=gb.BOOL.LOR_SECOND)
    memory.note()
    ks = _tokens()
    assert ks[:2] == ["run+hot-table (TMA-staged)", "offsets=64"] and any(k.startswith("hot-cluster=") for k in ks), ks
    hG = (G.astype(bool).astype(np.int64) @ bG.astype(np.int64)) > 0
    hJ = (J.astype(bool).astype(np.int64) @ bJ.astype(np.int64)) > 0
    I, X = w.to_arrays()
    assert np.array_equal(I, np.arange(n)) and np.array_equal(X, np.outer(hG, hJ).ravel())
    # mxm keeps refusing a wide operand
    with pytest.raises(gb.base.InvalidValue, match="2\\^32 entries are not supported"):
        A.mxm(A, semiring=gb.UINT8.PLUS_TIMES)
    del A, w, r
    memory.note()


def test_real_wide_bfs(memory):
    """BFS by level with vxm under a complemented structural mask: push at the first levels (small frontier), then pull,
    both along 64-bit offsets; pulling along A' needs the chunked transpose."""
    G, J = factor(1, NG, NNZ_G), factor(2, NJ, NNZ_J)
    n = NG * NJ
    A = kron(G, J, "BOOL")
    memory.note()
    assert A.nvals == NNZ
    deg = A.reduce_vector(gb.INT64.PLUS_MONOID, out=Vector.sparse(gb.INT64, n))
    I, X = deg.to_arrays()
    assert np.array_equal(X, np.outer(np.diff(G.indptr), np.diff(J.indptr)).ravel())
    del deg
    # expected levels: the smallest l with i in W_G(l) and j in W_J(l), W(l) = ends of walks of exactly l steps
    sG, sJ = 5, 9
    GT, JT = G.T.tocsr().astype(bool), J.T.tocsr().astype(bool)
    wG, wJ = np.zeros(NG, bool), np.zeros(NJ, bool)
    wG[sG] = wJ[sJ] = True
    want = np.full(n, -1, np.int64)
    seen = set()
    for l in range(4 * (NG + NJ)):
        new = np.outer(wG, wJ).ravel() & (want < 0)
        want[new] = l
        key = (wG.tobytes(), wJ.tobytes())
        if key in seen:
            break
        seen.add(key)
        wG, wJ = (GT @ wG) > 0, (JT @ wJ) > 0
    got = np.full(n, -1, np.int64)
    q = Vector.from_lists([sG * NJ + sJ], [True], n, gb.BOOL)
    visited = np.zeros(n, bool)
    routes = set()
    level = 0
    while q.nvals:
        qi = q.to_arrays()[0].astype(np.int64)
        got[qi] = level
        visited[qi] = True
        mask = Vector.from_numpy(np.ones(n, bool), present=visited)
        q = q.vxm(A, mask=mask, semiring=gb.BOOL.LOR_LAND, desc=descriptor.RSC)
        memory.note()
        ks = _tokens()
        assert ks[1] == "offsets=64", ks
        routes.add(ks[0])
        level += 1
    assert {"push", "pull"} <= routes, routes
    assert np.array_equal(got, want)
    del A, q, mask
    memory.note()
