"""The SpMV fix-up kernel (spmv_run.cuh) at the boundary between its two paths: a row still open at the end of its run that
reaches at most FIX_LONG = 8 runs further is folded by one thread, a longer one by a whole warp in trips of 32 x 8 runs.  The
matrix holds rows whose open span sits just below, at and above that boundary, rows that need one, two and three trips of
the warp, rows that end exactly at a run's end, and a long last row that ends inside a partial last run.  Every route that
runs the fix-up (hot-table kernel at every cluster size, plain run kernel, sparse u) must give the oracle's values (the value
pools make every fold exact in any order) and identical bytes on every call.  The matrix is built twice: on 2^18 columns the
hot-table kernel streams 3-byte ids, on 2^24 + 4096 columns 4-byte ids, whose bulk copy of the partial last run is rounded
up to 16 bytes rather than taking a whole padded run."""
import numpy as np
import pytest
import scipy.sparse as sp

from pygraphblas_b200 import Matrix, Vector
from oracle import oracle as orc
import util
from kernel_check import compare, entries, hot_id_bits, last_kernel, o_csr, semiring, seed_of, tunables, values, fp_pool_for

RUN = 256
FIX_LONG = 8
NCOLS = {"ids24": 1 << 18, "ids32": (1 << 24) + 4096}
# open spans (runs past the run the row starts in) of the rows placed at an offset of 100 inside a run; "end" rows end on
# the last entry of a run
SPANS = [1, 7, 8, 9, 31, 32, 33, 255, 256, 257, 600]
END_SPANS = [5, 20]
LAST_SPAN = 12


def build_pattern(ncols):
    """(S, spans): a CSR pattern of >= 2^20 entries (the hot-table kernel's minimum) and the open span of every long row."""
    rng = np.random.default_rng(11)
    lens, spans = [], []
    pos = 0

    def pad_to(offset):
        nonlocal pos
        while pos % RUN != offset:
            k = min(int(rng.integers(1, 40)), (offset - pos) % RUN)
            lens.append(k)
            pos += k

    def long_row(span, length):
        nonlocal pos
        lens.append(length)
        spans.append(span)
        assert (pos + length - 1) // RUN - pos // RUN == span
        pos += length

    for s in SPANS:
        pad_to(100)
        long_row(s, RUN * s + 10)
    for s in END_SPANS:
        pad_to(100)
        long_row(s, RUN * s + RUN - 100)
        assert pos % RUN == 0
    while pos < (1 << 20):                       # short rows up to the size the hot-table kernel needs
        k = int(rng.integers(1, 40))
        lens.append(k)
        pos += k
    pad_to(100)
    long_row(LAST_SPAN, RUN * LAST_SPAN + 77 - 100)    # the last run holds 77 entries
    assert pos % RUN == 77
    lens = np.asarray(lens, np.int64)
    # an empty row between every two rows: absent output rows sit between the long ones
    nrows = 2 * len(lens)
    row_len = np.zeros(nrows, np.int64)
    row_len[1::2] = lens
    indptr = np.concatenate(([0], np.cumsum(row_len)))
    indices = np.empty(int(indptr[-1]), np.int64)
    for r in np.flatnonzero(row_len):
        L = int(row_len[r])
        indices[indptr[r]:indptr[r + 1]] = np.sort(rng.choice(ncols, L, replace=False))
    S = sp.csr_matrix((np.ones(len(indices), np.int8), indices, indptr), shape=(nrows, ncols))
    return S, spans


def open_spans(S):
    """Restates the run plan: for every run whose last row start opens a row, how many runs past it that row reaches."""
    starts = S.indptr[:-1][np.diff(S.indptr) > 0]
    ends = S.indptr[1:][np.diff(S.indptr) > 0]
    run_of = starts // RUN
    last = np.r_[run_of[1:] != run_of[:-1], True]             # the last row start inside each run
    return (ends[last] - 1) // RUN - run_of[last]


@pytest.fixture(scope="module", params=list(NCOLS))
def pattern(request):
    S, spans = build_pattern(NCOLS[request.param])
    assert hot_id_bits(S) == int(request.param[3:])          # the width the plan picks (ncols + henc against 2^24)
    got = open_spans(S)
    # every designed span is an open span of the plan, on both sides of the boundary, and one needs three warp trips
    assert set(spans) <= set(got.tolist())
    assert (got == FIX_LONG).any() and (got == FIX_LONG + 1).any() and got.max() > 2 * 32 * 8
    assert S.nnz % RUN == 77
    return S


SRS = [("PLUS", "TIMES", "FP32"), ("PLUS", "TIMES", "FP64"), ("MIN", "PLUS", "FP32"), ("PLUS", "TIMES", "INT64")]


def call(A, u, sr):
    w = A.mxv(u, semiring=semiring(*sr))
    ks = last_kernel().split(";")
    ent = entries(ks)
    if ent[0].startswith("run+hot"):
        ent = [f"{ent[0]} {k}" for k in ks if k.startswith("ids=")]
    x, p = w.to_numpy()
    return ent[0], (np.ascontiguousarray(x).tobytes(), np.ascontiguousarray(p).tobytes()), w.to_arrays()


@pytest.mark.gpu
@pytest.mark.parametrize("sr", SRS, ids=["_".join(s) for s in SRS])
def test_long_open_rows(pattern, sr):
    S = pattern
    nrows, ncols = S.shape
    typ = sr[2]
    pool = fp_pool_for(sr[0], sr[1]) if typ in util.FP_T else "edge"
    av = values(seed_of("fixup", typ), typ, S.nnz, pool, 0)
    uv = values(seed_of("fixup", sr, "u"), typ, ncols, pool, 1)
    A = Matrix.from_csr(S.indptr, S.indices, av, nrows, ncols, util.g_type(typ))
    Ao = o_csr(typ, S, av)
    errors = []

    # dense u: the hot-table kernel (forced on: the columns are spread evenly) at every cluster size, and the plain run kernel
    u = Vector.from_numpy(uv, typ=util.g_type(typ))
    ref = orc.mxv(orc.SpVec(typ, nrows), None, None, sr, Ao, orc.SpVec(typ, ncols, np.arange(ncols), uv), "")
    base = None
    hot = f"run+hot-table (TMA-staged) ids={hot_id_bits(S)}"
    settings = [(hot, {"B200GRB_SPMV_HOT": 128, "B200GRB_SPMV_CLUSTER": C, "B200GRB_SPMV_HOT_REPL": t0})
                for C, t0 in ((1, 0), (2, 32), (4, 0), (8, 96), (16, 32))]
    settings += [("run", {"B200GRB_SPMV_HOT": 0})]
    for route, env in settings:
        with tunables(**env):
            for rep in range(2):
                got_route, got, (gI, gX) = call(A, u, sr)
                assert got_route == route, (sr, env, got_route)
                if base is None:
                    base = got
                elif got != base:
                    errors.append(f"{sr} {env} call {rep}: bytes differ from the first call")
        e = compare(gI, gX, ref.I, ref.X, typ, sr[0], f"{sr} {env}")
        if e:
            errors.append(e)

    # sparse u: the run kernel and fix-up that carry presence
    rng = np.random.default_rng(seed_of("fixup", sr, "holes"))
    upres = rng.random(ncols) < 0.7
    us = Vector.from_numpy(uv, present=upres, typ=util.g_type(typ))
    idx = np.flatnonzero(upres)
    ref = orc.mxv(orc.SpVec(typ, nrows), None, None, sr, Ao, orc.SpVec(typ, ncols, idx, uv[idx]), "")
    first = None
    for rep in range(2):
        got_route, got, (gI, gX) = call(A, us, sr)
        assert got_route == "run (sparse u)", (sr, got_route)
        if first is None:
            first = got
        elif got != first:
            errors.append(f"{sr} sparse u: bytes differ between calls")
    e = compare(gI, gX, ref.I, ref.X, typ, sr[0], f"{sr} sparse u")
    if e:
        errors.append(e)
    assert not errors, "\n".join(errors[:20])
