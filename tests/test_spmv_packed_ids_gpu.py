"""The hot-table SpMV kernel on 3-byte and 4-byte column ids (spmv_run.cuh, spmv_hot_plan): the plan stores the encoded ids in
3 bytes, packed run by run, when every id fits (ncols + henc < 2^24), and in 4 bytes otherwise.  The library reports the width
it launched (`ids=24` / `ids=32` beside `hot-tiers=`); every result must match the oracle and be bit-identical to the plain
run kernel (B200GRB_SPMV_HOT=0), which shares the runs, the fold and the fix-up and reads every value of u from u itself.

Every specialised semiring runs on every type it is specialised for, in both forms: mxv pulls along A, vxm along A'
(here A is the transposed pattern, so A' is the same skewed pattern).  The width is restated from the CSR the kernel pulls
along; a multiply that ignores u gathers nothing and takes the plain run kernel.

The matrices are skewed (most entries on a few thousand columns, so the default route takes the hot-table kernel), reference
at least 2^17 columns (henc = 2^17) including the last one (the largest id, ncols - 1 + henc), have a number of entries that
is not a multiple of 256 (the last run is padded) and a hub row that spans hundreds of runs (the fix-up's long-row path)."""
import functools

import numpy as np
import pytest
import scipy.sparse as sp

from pygraphblas_b200 import Matrix, Vector
import util
from kernel_check import (HOT_EXT, HOT_T, compare, expected_hot_launch, fp_pool_for, hot_launch_of, hot_reads_u, hot_tokens,
                          max_optin, oracle_spmv, seed_of, semiring, spmv_specialised, tunables, values)

RUN = 256
HOT_ROUTE = "run+hot-table (TMA-staged)"
HUB = 60_000
DEFAULT_C, DEFAULT_T0_KB, DEFAULT_HOT_KB = 2, 32, 128          # the library's defaults (common.cuh, spmv.cu)
PAIRS = [("PLUS", m) for m in ("TIMES", "SECOND", "FIRST", "PAIR")] + [("MIN", m) for m in ("PLUS", "FIRST", "SECOND")] + \
        [("LOR", m) for m in ("LAND", "PAIR", "SECOND", "FIRST")] + [("ANY", "PAIR")]
SRS = [(a, m, t) for t in HOT_T for a, m in PAIRS if spmv_specialised(a, m, t)]
FORMS = ("mxv", "vxm")

# ncols of each case: the 3-byte ids of a graph of ~1 M columns, ncols + henc one below and at 2^24, and 4-byte ids well past it
CASES = {
    "skewed": (1 << 20) + 4099,
    "below-2^24": (1 << 24) - HOT_EXT - 1,
    "at-2^24": (1 << 24) - HOT_EXT,
    "well-above": (1 << 24) + (1 << 20) + 4099,
}
# (case, add, mul, typ, form, "ids=24" / "ids=32" / "run") of every call made
REACHED = set()


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


@functools.lru_cache(maxsize=1)
def operands(case):
    """The pattern of mxv (A = S) and of vxm (A = S', so that the kernel pulls along A' = S): {form: CSR of A}."""
    S = skewed_pattern(CASES[case], seed_of("packed-ids", case, bits=32))
    St = S.T.tocsr()
    St.sort_indices()
    return {"mxv": S, "vxm": St}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_packed_ids_match_oracle_and_plain_run_kernel(case):
    pats = operands(case)
    smem = max_optin()
    errors = []
    for form in FORMS:
        vxm = form == "vxm"
        S = pats[form]
        nrows, ncols = S.shape
        n_in = nrows if vxm else ncols
        mats, vecs = {}, {}
        for sr in SRS:
            add, mul, typ = sr
            pool = fp_pool_for(add, mul) if typ in util.FP_T else "edge"
            if (typ, pool) not in mats:
                av = values(seed_of(case, typ, pool, form, "a"), typ, S.nnz, pool, 0)
                uv = values(seed_of(case, typ, pool, form, "u"), typ, n_in, pool, 1)
                mats = {(typ, pool): (Matrix.from_csr(S.indptr, S.indices, av, nrows, ncols, util.g_type(typ)), av)}
                vecs = {(typ, pool): (Vector.from_numpy(uv, typ=util.g_type(typ)), uv)}
            (A, av), (u, uv) = mats[(typ, pool)], vecs[(typ, pool)]
            s = semiring(*sr)
            label = f"{case} {form} {'_'.join(sr)}"

            w = u.vxm(A, semiring=s) if vxm else A.mxv(u, semiring=s)
            ent, tok = hot_tokens()
            if hot_reads_u(mul, vxm):
                want_launch, want_bits = expected_hot_launch(S, vxm, typ, mul, DEFAULT_HOT_KB, DEFAULT_C, DEFAULT_T0_KB, smem)
                assert ent[0] == HOT_ROUTE, (label, ent)
                got_launch, got_bits = hot_launch_of(tok)
                assert got_bits == want_bits, (label, tok, want_bits)
                assert got_launch == want_launch and want_launch[3] == HOT_EXT, (label, got_launch, want_launch)
                REACHED.add((case, add, mul, typ, form, f"ids={got_bits}"))
            else:                                  # the multiply ignores u: nothing to gather, the plain run kernel
                assert ent[0] == "run" and "ids" not in tok, (label, ent, tok)
                REACHED.add((case, add, mul, typ, form, "run"))
            x, p = w.to_numpy()
            hot_bytes = (np.ascontiguousarray(x).tobytes(), np.ascontiguousarray(p).tobytes())
            ref = oracle_spmv(typ, sr, S, av, uv, vxm)
            e = compare(*w.to_arrays(), ref.I, ref.X, typ, add, label)
            if e:
                errors.append(e)

            with tunables(B200GRB_SPMV_HOT=0):
                w0 = u.vxm(A, semiring=s) if vxm else A.mxv(u, semiring=s)
                ent0, tok0 = hot_tokens()
            assert ent0[0] == "run" and "ids" not in tok0, (label, ent0, tok0)
            x0, p0 = w0.to_numpy()
            if (np.ascontiguousarray(x0).tobytes(), np.ascontiguousarray(p0).tobytes()) != hot_bytes:
                errors.append(f"{label}: the hot-table kernel's bytes differ from the plain run kernel's")
    assert not errors, "\n".join(errors[:40])


def expected_reach():
    """Every (case, semiring, type, form) with the width its CSR gives, or "run" where the multiply ignores u."""
    out = set()
    for case, ncols in CASES.items():
        bits = 24 if ncols + HOT_EXT < (1 << 24) else 32       # every case references >= 2^17 columns: henc = 2^17
        for add, mul, typ in SRS:
            for form in FORMS:
                out.add((case, add, mul, typ, form, f"ids={bits}" if hot_reads_u(mul, form == "vxm") else "run"))
    return out


def test_every_semiring_type_form_and_width_was_reached(request):
    mine = [it for it in request.session.items if it.module is request.module and it is not request.node and "gpu" in it.keywords]
    if len(mine) < len(CASES) or not REACHED:
        pytest.skip("the GPU cases of the module did not all run")
    want = expected_reach()
    assert REACHED == want, (sorted(want - REACHED)[:20], sorted(REACHED - want)[:20])
    # both widths, each at every type and in both forms
    for bits in ("ids=24", "ids=32"):
        assert {(t, f) for _, _, _, t, f, b in REACHED if b == bits} == {(t, f) for t in HOT_T for f in FORMS}, bits
