"""The hot-table SpMV kernel (spmv_run.cuh) where its two id widths meet what the other modules cannot take as one more input:

* a table capped by the device's shared memory rather than by B200GRB_SPMV_HOT: hot2_table_entries leaves the table
  max_optin - fixed - 256 bytes, and `fixed` (the warp stages and barriers) depends on the id width and on whether the
  multiply reads A's values;
* the width rule of spmv_hot_plan (3-byte ids while ncols + henc < 2^24) at henc < 2^17, where every referenced column is
  hot: every id is a rank below henc and no gather reads u in place;
* calls that alternate between a 3-byte and a 4-byte matrix on one kernel instantiation, whose launch caches (the
  dynamic shared-memory limit and the co-scheduled clusters) are kept per instantiation and see two `fixed` sizes.

Every call asserts the route, the id width and the tiers the library reports against the restatement in kernel_check
(never against device output), and compares the result with the oracle and, where stated, with other calls' bytes."""
import functools

import numpy as np
import pytest
import scipy.sparse as sp

from pygraphblas_b200 import Matrix, Vector
import util
from kernel_check import (HOT_EXT, VSIZE, compare, expected_hot_launch, fp_pool_for, hot_launch_of, hot_tokens, max_optin,
                          oracle_spmv, seed_of, semiring, spread_columns, tunables, uniform_pattern, values)

HOT_ROUTE = "run+hot-table (TMA-staged)"
WIDE = (1 << 24) + 4096
REACHED = set()          # (test, case, width) of every checked launch


@functools.lru_cache(maxsize=None)
def even_pattern(bits):
    """2^17 + 4096 referenced columns, each 8 times (henc = 2^17, 4096 cold columns read from u): on 2^17 + 4096 columns
    (3-byte ids), or with the cold ones spread up to the last of 2^24 + 4096 (4-byte ids)."""
    if bits == 24:
        return uniform_pattern((1 << 17) + 4096, 8)
    return uniform_pattern(WIDE, 8, spread_columns(WIDE, HOT_EXT, 4096))


def mxv_bytes(A, u, sr):
    w = A.mxv(u, semiring=semiring(*sr))
    ent, tok = hot_tokens()
    x, p = w.to_numpy()
    return ent, tok, (np.ascontiguousarray(x).tobytes(), np.ascontiguousarray(p).tobytes()), w


def operands(S, sr, label):
    typ = sr[2]
    pool = fp_pool_for(sr[0], sr[1]) if typ in util.FP_T else "edge"
    nrows, ncols = S.shape
    av = values(seed_of(label, typ, pool, "a"), typ, S.nnz, pool, 0)
    uv = values(seed_of(label, typ, pool, "u"), typ, ncols, pool, 1)
    A = Matrix.from_csr(S.indptr, S.indices, av, nrows, ncols, util.g_type(typ))
    u = Vector.from_numpy(uv, typ=util.g_type(typ))
    ref = oracle_spmv(typ, sr, S, av, uv, False)
    return A, u, ref


# ------------------------------------------------------------------ a table capped by shared memory
CAP_SRS = [("PLUS", "TIMES", "FP32"), ("PLUS", "SECOND", "FP32"), ("PLUS", "TIMES", "FP64"), ("PLUS", "SECOND", "FP64")]
CAP_KB = 1024            # more than any SM holds: the shared memory left after the stages binds


@pytest.mark.gpu
@pytest.mark.parametrize("bits", [24, 32])
def test_table_capped_by_shared_memory(bits):
    """B200GRB_SPMV_HOT=1024 at C = 1 and C = 8: the table the library reports is the restated shared-memory cap (different
    per id width, value type and stage layout), and the results match the oracle and the C = 1 bytes."""
    S = even_pattern(bits)
    smem = max_optin()
    errors = []
    for sr in CAP_SRS:
        typ, label = sr[2], f"cap ids={bits} {'_'.join(sr)}"
        A, u, ref = operands(S, sr, label)
        base = None
        for C in (1, 8):
            with tunables(B200GRB_SPMV_HOT=CAP_KB, B200GRB_SPMV_CLUSTER=C, B200GRB_SPMV_HOT_REPL=32):
                ent, tok, got, w = mxv_bytes(A, u, sr)
            assert ent[0] == HOT_ROUTE, (label, C, ent)
            got_t, got_bits = hot_launch_of(tok)
            want_t, want_bits = expected_hot_launch(S, False, typ, sr[1], CAP_KB, C, 32, smem)
            assert (got_t, got_bits) == (want_t, want_bits), (label, C, tok, want_t, want_bits)
            if C == 1:                                   # the cap binds: the table is smaller than both henc and the KB limit
                assert want_t[1] < want_t[3] and want_t[1] * VSIZE[typ] < (CAP_KB << 10), (label, want_t)
                base = got
            else:
                assert want_t[0] == C, (label, want_t)
                if got != base:
                    errors.append(f"{label} C={C}: bytes differ from C=1")
            e = compare(*w.to_arrays(), ref.I, ref.X, typ, sr[0], f"{label} C={C}")
            if e:
                errors.append(e)
            REACHED.add(("cap", f"{'_'.join(sr)} C={C}", got_bits))
    assert not errors, "\n".join(errors)


# ------------------------------------------------------------------ the width rule at henc < 2^17
RULE_NCOLS = (1 << 24) - 4096
RULE_SRS = [("PLUS", "TIMES", "FP32"), ("MIN", "PLUS", "FP64"), ("PLUS", "SECOND", "INT32"), ("LOR", "LAND", "BOOL")]


def few_columns_pattern(nhot):
    """>= 2^20 entries on exactly nhot distinct columns, spread over all RULE_NCOLS columns (the last one included), on 8192
    rows; the number of entries is not a multiple of 256."""
    rng = np.random.default_rng(nhot)
    cols = np.linspace(0, RULE_NCOLS - 1, nhot).astype(np.int64)
    k = np.concatenate([np.arange(nhot), rng.integers(0, nhot, 1_200_000)])
    rows = rng.integers(0, 8192, len(k))
    S = sp.csr_matrix((np.ones(len(k), np.int32), (rows, cols[k])), shape=(8192, RULE_NCOLS))
    S.sort_indices()
    if S.nnz % 256 == 0:                                                  # drop the last entry: the last run is partial
        S = sp.csr_matrix((S.data[:-1], S.indices[:-1], np.minimum(S.indptr, S.nnz - 1)), shape=S.shape)
    assert S.nnz >= (1 << 20) and S.nnz % 256
    assert np.count_nonzero(np.bincount(S.indices, minlength=RULE_NCOLS)) == nhot
    return S


@pytest.mark.gpu
@pytest.mark.parametrize("nhot", [4095, 4096])
def test_width_rule_below_hot_ext(nhot):
    """ncols + henc = 2^24 - 1 gives 3-byte ids, 2^24 gives 4-byte ids; every referenced column is hot (ids < henc).  With
    the defaults (C = 2, T0 = 32 KB, a 128 KB table) one table holds every rank but the last henc mod 16: plain CTAs."""
    S = few_columns_pattern(nhot)
    smem = max_optin()
    want_bits = 24 if RULE_NCOLS + nhot < (1 << 24) else 32
    errors = []
    for sr in RULE_SRS:
        typ, label = sr[2], f"rule nhot={nhot} {'_'.join(sr)}"
        A, u, ref = operands(S, sr, label)
        ent, tok, got, w = mxv_bytes(A, u, sr)
        assert ent[0] == HOT_ROUTE, (label, ent)
        want_t, bits = expected_hot_launch(S, False, typ, sr[1], 128, 2, 32, smem)
        assert bits == want_bits and want_t[3] == nhot
        assert hot_launch_of(tok) == (want_t, want_bits), (label, tok, want_t, want_bits)
        e = compare(*w.to_arrays(), ref.I, ref.X, typ, sr[0], label)
        if e:
            errors.append(e)
        with tunables(B200GRB_SPMV_HOT=0):
            ent0, tok0, got0, _ = mxv_bytes(A, u, sr)
        assert ent0[0] == "run" and "ids" not in tok0, (label, ent0)
        if got0 != got:
            errors.append(f"{label}: the hot-table kernel's bytes differ from the plain run kernel's")
        REACHED.add(("rule", f"{'_'.join(sr)} nhot={nhot}", want_bits))
    assert not errors, "\n".join(errors)


# ------------------------------------------------------------------ alternating widths on one instantiation
# (semiring, table KB): at 128 KB a BOOL table holds every hot rank (plain CTAs whatever C); at 64 KB it is spread
ALT = [(("PLUS", "TIMES", "FP32"), 128), (("LOR", "LAND", "BOOL"), 64)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(ALT)), ids=["FP32-PLUS_TIMES", "BOOL-LOR_LAND"])
def test_alternating_widths_on_one_instantiation(case):
    """Calls of one semiring on a 3-byte and a 4-byte matrix at C = 1, 2 and 16, twice in a row each and then alternating:
    every call launches the restated tiers, and gives the bytes of the first call of its width (the oracle's result)."""
    sr, hot_kb = ALT[case]
    typ = sr[2]
    smem = max_optin()
    ops = {bits: operands(even_pattern(bits), sr, f"alt {'_'.join(sr)} ids={bits}") for bits in (24, 32)}
    errors = []
    for C in (1, 2, 16):
        with tunables(B200GRB_SPMV_HOT=hot_kb, B200GRB_SPMV_CLUSTER=C, B200GRB_SPMV_HOT_REPL=32):
            alone = {}
            want = {bits: expected_hot_launch(even_pattern(bits), False, typ, sr[1], hot_kb, C, 32, smem) for bits in (24, 32)}
            for bits in (24, 24, 32, 32, 24, 32, 24, 32):
                A, u, ref = ops[bits]
                label = f"alt {'_'.join(sr)} C={C} ids={bits}"
                ent, tok, got, w = mxv_bytes(A, u, sr)
                assert ent[0] == HOT_ROUTE, (label, ent)
                assert hot_launch_of(tok) == want[bits], (label, tok, want[bits])
                assert C == 1 or want[bits][0][0] == C, (label, want[bits])
                if bits not in alone:
                    alone[bits] = got
                    e = compare(*w.to_arrays(), ref.I, ref.X, typ, sr[0], label)
                    if e:
                        errors.append(e)
                elif got != alone[bits]:
                    errors.append(f"{label}: bytes differ from the same call made on its own")
                REACHED.add(("alt", f"{'_'.join(sr)} C={C}", bits))
    assert not errors, "\n".join(errors)


def test_every_case_reached_its_width(request):
    mine = [it for it in request.session.items if it.module is request.module and it is not request.node and "gpu" in it.keywords]
    if len(mine) < 2 + 2 + len(ALT) or not REACHED:
        pytest.skip("the GPU cases of the module did not all run")
    want = {("cap", f"{'_'.join(sr)} C={C}", bits) for sr in CAP_SRS for C in (1, 8) for bits in (24, 32)}
    want |= {("rule", f"{'_'.join(sr)} nhot={n}", 24 if n == 4095 else 32) for sr in RULE_SRS for n in (4095, 4096)}
    want |= {("alt", f"{'_'.join(sr)} C={C}", bits) for sr, _ in ALT for C in (1, 2, 16) for bits in (24, 32)}
    assert REACHED == want, (sorted(want - REACHED), sorted(REACHED - want))
