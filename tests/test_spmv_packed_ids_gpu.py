"""The hot-table SpMV kernel on 3-byte column ids (spmv_run.cuh, spmv_hot_plan): the plan stores the encoded ids in 3 bytes,
packed run by run, when every id fits (ncols + henc < 2^24), and in 4 bytes otherwise.  The library reports the width it
launched (`ids=24` / `ids=32` beside `hot-tiers=`); every result must match the oracle and be bit-identical to the plain run
kernel (B200GRB_SPMV_HOT=0), which shares the runs, the fold and the fix-up and reads every value of u from u itself.

The matrices are skewed (most entries on a few thousand columns, so the default route takes the hot-table kernel), reference
at least 2^17 columns (henc = 2^17) including the last one (the largest id, ncols - 1 + henc), have a number of entries that
is not a multiple of 256 (the last run is padded) and a hub row that spans hundreds of runs (the fix-up's long-row path)."""
import numpy as np
import pytest
import scipy.sparse as sp

from pygraphblas_b200 import Matrix, Vector
from oracle import oracle as orc
import util
from kernel_check import compare, entries, last_kernel, o_csr, semiring, seed_of, tunables, values, fp_pool_for

HOT_EXT = 1 << 17
RUN = 256
HOT_ROUTE = "run+hot-table (TMA-staged)"
SRS = [("PLUS", "TIMES", "FP32"), ("PLUS", "TIMES", "FP64"), ("PLUS", "TIMES", "INT64"), ("LOR", "LAND", "BOOL")]
HUB = 60_000

# ncols of each case: the 3-byte ids of a graph of ~1 M columns, and ncols + henc one below and at 2^24
CASES = {
    "skewed": (1 << 20) + 4099,
    "below-2^24": (1 << 24) - HOT_EXT - 1,
    "at-2^24": (1 << 24) - HOT_EXT,
}


def skewed_pattern(ncols, seed):
    rng = np.random.default_rng(seed)
    nrows = 24576
    cold = rng.integers(0, ncols, 400_000)
    hot = (HOT_EXT * rng.random(700_000) ** 3).astype(np.int64)          # concentrated on the lowest columns
    cols = np.concatenate([cold, hot, np.arange(HOT_EXT), [ncols - 2, ncols - 1]])
    rows = rng.integers(0, nrows, len(cols))
    rows[:HUB] = 777                                                      # the hub row: cold columns, mostly distinct
    S = sp.csr_matrix((np.ones(len(cols), np.int32), (rows, cols)), shape=(nrows, ncols))
    S.sort_indices()
    if S.nnz % RUN == 0:                                                  # drop the last entry: the last run is partial
        S = sp.csr_matrix((S.data[:-1], S.indices[:-1], np.minimum(S.indptr, S.nnz - 1)), shape=S.shape)
    deg = np.bincount(S.indices, minlength=ncols)
    assert S.nnz % RUN and S.nnz >= (1 << 20) and deg[ncols - 1] > 0
    assert np.count_nonzero(deg) >= HOT_EXT                               # henc = 2^17
    assert np.diff(S.indptr).max() > 100 * RUN                            # the hub row spans more than 100 runs
    return S


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_packed_ids_match_oracle_and_plain_run_kernel(case):
    ncols = CASES[case]
    S = skewed_pattern(ncols, seed_of("packed-ids", case, bits=32))
    nrows = S.shape[0]
    want_ids = "24" if ncols + HOT_EXT < (1 << 24) else "32"
    errors = []
    for sr in SRS:
        typ = sr[2]
        pool = fp_pool_for(sr[0], sr[1]) if typ in util.FP_T else "edge"
        av = values(seed_of(case, typ, "a"), typ, S.nnz, pool, 0)
        uv = values(seed_of(case, typ, "u"), typ, ncols, pool, 1)
        A = Matrix.from_csr(S.indptr, S.indices, av, nrows, ncols, util.g_type(typ))
        u = Vector.from_numpy(uv, typ=util.g_type(typ))
        label = f"{case} {'_'.join(sr)}"

        w = A.mxv(u, semiring=semiring(*sr))
        ks = last_kernel().split(";")
        tok = dict(k.split("=", 1) for k in ks if "=" in k)
        assert entries(ks)[0] == HOT_ROUTE, (label, ks)
        assert tok.get("ids") == want_ids, (label, ks)
        assert int(tok["hot-tiers"].split(",")[2]) == HOT_EXT, (label, ks)
        x, p = w.to_numpy()
        hot_bytes = (np.ascontiguousarray(x).tobytes(), np.ascontiguousarray(p).tobytes())
        ref = orc.mxv(orc.SpVec(typ, nrows), None, None, sr, o_csr(typ, S, av), orc.SpVec(typ, ncols, np.arange(ncols), uv), "")
        e = compare(*w.to_arrays(), ref.I, ref.X, typ, sr[0], label)
        if e:
            errors.append(e)

        with tunables(B200GRB_SPMV_HOT=0):
            w0 = A.mxv(u, semiring=semiring(*sr))
            ks0 = last_kernel().split(";")
        assert entries(ks0)[0] == "run" and not any(k.startswith("ids=") for k in ks0), (label, ks0)
        x0, p0 = w0.to_numpy()
        if (np.ascontiguousarray(x0).tobytes(), np.ascontiguousarray(p0).tobytes()) != hot_bytes:
            errors.append(f"{label}: the hot-table kernel's bytes differ from the plain run kernel's")
    assert not errors, "\n".join(errors)
