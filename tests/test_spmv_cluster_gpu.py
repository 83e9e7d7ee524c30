"""The hot-table SpMV kernel as thread-block clusters (spmv_run.cuh): every cluster size and replicated tier gives the same
bytes as plain CTAs, and the oracle's result, with gathers on every side of every tier boundary.

The tiers are restated from hot2_tiers: a CTA's table holds `cap` entries; with C > 1 the replicated tier T0 is the
B200GRB_SPMV_HOT_REPL request (entries, multiple of 16, at most cap), the rest of the table is this CTA's slice of the
distributed tier T1, and the hot ranks past T0 + T1 up to henc are read from u_hot in L2.  Plain CTAs are launched when
one table holds every hot rank or T0 takes the whole table.  Every call asserts the cluster size and the tiers the
library reports (`hot-cluster=`, `hot-tiers=T0,T1,henc`) against this restatement; an H100 co-schedules every C <= 16.
Each call also asserts the id width (`ids=24` / `ids=32`, spmv_hot_plan: 4-byte ids once ncols + henc reaches 2^24), and
every cluster size is reached at both widths.  The SASS checks need no GPU."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import scipy.sparse as sp

from pygraphblas_b200 import Matrix, Vector
from pygraphblas_b200.generators import rmat_csr
import util
from kernel_check import (HOT_EXT, compare, expected_hot_launch, hot_launch_of, hot_tokens, max_optin, oracle_spmv, semiring, seed_of,
                          spread_columns, tunables, uniform_pattern, values, fp_pool_for)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pygraphblas_b200", "libb200grb.so")
CLUSTERS = (1, 2, 4, 8, 16)
HOT_SRS = [("PLUS", "TIMES"), ("MIN", "PLUS"), ("PLUS", "SECOND")]
SRS = [sr + (t,) for t in ("FP32", "FP64", "INT32", "UINT64") for sr in HOT_SRS] + [("LOR", "LAND", "BOOL")]
ROUTES = {"run+hot-table (TMA-staged)"}
REACHED_C, SIDES = set(), set()         # REACHED_C: (C, id width) of every launch


def rmat_pattern(scale):
    n, indptr, indices = rmat_csr(scale, 16, seed=3)
    return sp.csr_matrix((np.ones(len(indices), np.int8), indices, indptr), shape=(n, n))


def run_all(S, label, settings, srs=SRS, forms=("mxv", "vxm"), hot_kb=128):
    """For each semiring and form: the C = 1 result, then each (C, T0 KB) of settings must give the same bytes; every
    result is compared with the oracle, and the launch the library reports (tiers and id width) with the restatement
    (kernel_check.expected_hot_launch: the table is capped by hot_kb and by the shared memory left after the stages).
    Returns the set of (C, T0, T1, henc) launched."""
    nrows, ncols = S.shape
    smem = max_optin()
    errors, launched = [], set()
    for sr0 in srs:
        typ = sr0[2]
        pool = fp_pool_for(sr0[0], sr0[1]) if typ in util.FP_T else "edge"
        av = values(seed_of(label, typ), typ, S.nnz, pool, 0)
        A = Matrix.from_csr(S.indptr, S.indices, av, nrows, ncols, util.g_type(typ))
        for form in forms:
            vxm = form == "vxm"
            # SECOND reads u in mxv form; in vxm form FIRST does (the other one gathers nothing and takes the plain run kernel)
            sr = (sr0[0], "FIRST", typ) if vxm and sr0[1] == "SECOND" else sr0
            n_in = nrows if vxm else ncols
            uv = values(seed_of(label, sr, form), typ, n_in, pool, 1)
            u = Vector.from_numpy(uv, typ=util.g_type(typ))
            ref = oracle_spmv(typ, sr, S, av, uv, vxm)
            base = None
            for C, t0kb in [(1, 0)] + list(settings):
                with tunables(B200GRB_SPMV_CLUSTER=C, B200GRB_SPMV_HOT_REPL=t0kb):
                    w = u.vxm(A, semiring=semiring(*sr)) if vxm else A.mxv(u, semiring=semiring(*sr))
                    ent, tok = hot_tokens()
                assert ent[0] in ROUTES, (label, sr, form, C, ent)
                got_t, got_bits = hot_launch_of(tok)
                want_t, want_bits = expected_hot_launch(S, vxm, typ, sr[1], hot_kb, C, t0kb, smem)
                assert got_t == want_t, (label, sr, form, C, t0kb, got_t, want_t)
                assert got_bits == want_bits, (label, sr, form, C, t0kb, tok, want_bits)
                launched.add(got_t)
                REACHED_C.add((got_t[0], got_bits))
                x, p = w.to_numpy()
                got = (np.ascontiguousarray(x).tobytes(), np.ascontiguousarray(p).tobytes())
                if base is None:
                    base = got
                elif got != base:
                    errors.append(f"{label} {form} {'_'.join(sr)} C={C} T0={t0kb}KB: bytes differ from C=1")
                gI, gX = w.to_arrays()
                e = compare(gI, gX, ref.I, ref.X, typ, sr[0], f"{label} {form} {'_'.join(sr)} C={C} T0={t0kb}KB")
                if e:
                    errors.append(e)
    assert not errors, "\n".join(errors[:20])
    return launched


@pytest.mark.gpu
@pytest.mark.parametrize("pattern", ["rmat18", "even", "even-ids32"])
def test_cluster_sizes_are_bit_identical(pattern):
    # even-ids32: the columns of "even" with the cold ones spread up to the last of 2^24 + 4096, so mxv pulls along a CSR
    # whose ids take 4 bytes (vxm along A', of 2^17 + 4096 columns: 3 bytes)
    S = {"rmat18": lambda: rmat_pattern(18), "even": lambda: uniform_pattern((1 << 17) + 4096, 8),
         "even-ids32": lambda: uniform_pattern(WIDE, 8, spread_columns(WIDE, HOT_EXT, 4096))}[pattern]()
    settings = [(C, t0) for C in CLUSTERS[1:] for t0 in (0, 32, 96)]
    with tunables(B200GRB_SPMV_HOT=128):
        launched = run_all(S, pattern, settings, srs=SRS[:-1])
    assert {c for c, *_ in launched} == set(CLUSTERS), launched
    # a BOOL table of 128 KB holds all 2^17 hot ranks (plain CTAs); capped at 64 KB, the 1-byte values are spread too
    with tunables(B200GRB_SPMV_HOT=64):
        launched = run_all(S, pattern, settings, srs=SRS[-1:], hot_kb=64)
    assert {c for c, *_ in launched} == set(CLUSTERS), launched


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["fp32-table-64", "fp64-table-96", "bool-fits"])
def test_plain_ctas_when_nothing_is_spread(case):
    """A request for C = 8 and T0 = 96 KB launches plain CTAs when T0 takes the whole table (a table cap of 96 KB or
    less) and when one table already holds every hot rank (BOOL: 128 K entries >= henc)."""
    S = rmat_pattern(18)
    typ, hot_kb = {"fp32-table-64": ("FP32", 64), "fp64-table-96": ("FP64", 96), "bool-fits": ("BOOL", 128)}[case]
    sr = ("LOR", "LAND", "BOOL") if typ == "BOOL" else ("PLUS", "TIMES", typ)
    with tunables(B200GRB_SPMV_HOT=hot_kb):
        launched = run_all(S, case, [(8, 96)], srs=[sr], forms=("mxv",), hot_kb=hot_kb)
    assert {c for c, *_ in launched} == {1}, launched
    SIDES.add(f"plain-{case}")


# (ncols, per-column degree, C, T0 KB, referenced columns or None for all): FP32 tables of 128 KB (cap = 32768 entries).
# The -ids32 cases reference the same number of columns, spread up to the last of 2^24 + 4096 (4-byte ids)
WIDE = (1 << 24) + 4096
TIER_CASES = {
    "c8-rest-and-u": ((1 << 17) + 4096, 8, 8, 96, None),        # T0 + T1 < henc = 2^17 < ncols: every tier and u
    "c4-no-repl": ((1 << 17) + 4096, 8, 4, 0, None),            # T0 = 0: the table is all slices
    "c16-short": ((1 << 16) + 40, 16, 16, 0, None),             # fewer hot columns than C * cap: partly filled slices
    "c2-short-repl": ((1 << 16) + 40, 16, 2, 64, None),
    "c8-rest-and-u-ids32": (WIDE, 8, 8, 96, (HOT_EXT, 4096)),   # ranks 0 .. 2^17 - 1 on the lowest columns, 4096 cold ones
    "c16-short-ids32": (WIDE, 16, 16, 0, (0, (1 << 16) + 40)),  # every referenced column hot, spread over all of u
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(TIER_CASES))
def test_tier_boundaries(case):
    ncols, deg, C, t0kb, spread = TIER_CASES[case]
    S = uniform_pattern(ncols, deg, None if spread is None else spread_columns(ncols, *spread))
    srs = [("PLUS", "TIMES", "FP32"), ("MIN", "PLUS", "FP32")]
    with tunables(B200GRB_SPMV_HOT=128):
        launched = run_all(S, case, [(C, t0kb)], srs=srs, forms=("mxv",))
    # the tiers the library reported for the cluster launch (rank j = the j-th referenced column: every rank is gathered, so
    # each boundary inside the hot ranks has a gathered rank on both of its sides)
    (c, t0, t1, henc), = [t for t in launched if t[0] > 1]
    assert c == C
    for b in (t0, t0 + t1, henc):
        if 0 < b < S.nnz // deg:
            SIDES.add(f"{case}-{b - 1}|{b}")
    if t0 + t1 < henc:
        SIDES.add(f"{case}-rest")
    if t1 % (16 * C):                                     # slices are multiples of 16 entries: full ones sum to a multiple of 16 C
        SIDES.add(f"{case}-partial-slices")


def test_every_cluster_size_and_tier_was_reached(request):
    mine = [it for it in request.session.items if it.module is request.module and it is not request.node and "gpu" in it.keywords]
    gpu_count = 3 + 3 + len(TIER_CASES)
    if len(mine) < gpu_count or not REACHED_C:
        pytest.skip("the GPU cases of the module did not all run")
    assert REACHED_C >= {(c, bits) for c in CLUSTERS for bits in (24, 32)}, sorted(REACHED_C)
    assert {s for s in SIDES if s.endswith("-rest")} and {s for s in SIDES if s.endswith("-partial-slices")}, SIDES
    assert all(any(s.startswith(c + "-") for s in SIDES) for c in TIER_CASES), SIDES
    assert len({s for s in SIDES if s.startswith("plain-")}) == 3, SIDES


# ------------------------------------------------------------------ SASS (no GPU)
@pytest.fixture(scope="module")
def hot2_sass():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe) or not os.path.exists(LIB):
        pytest.skip("cuobjdump or the built library is not available")
    out = subprocess.run([exe, "-sass", LIB], capture_output=True, text=True, timeout=600).stdout
    funcs, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            continue
        if name and "spmv_run_hot2_kernel" in name:
            m = re.search(r"/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_.]*)", line)
            if m:
                funcs.setdefault(name, []).append(m.group(1))
    if not funcs:
        pytest.skip("no SASS found in the library")
    return funcs


def test_every_hot2_instantiation_has_both_cluster_barriers_and_remote_loads(hot2_sass):
    assert len(hot2_sass) >= 20
    for name, ops in hot2_sass.items():
        arv = [i for i, o in enumerate(ops) if o == "UCGABAR_ARV"]
        wait = [i for i, o in enumerate(ops) if o == "UCGABAR_WAIT"]
        assert len(arv) >= 2 and len(wait) >= 2, name               # after the table is in, and before the CTA exits
        assert arv[0] < wait[0] and arv[-1] < wait[-1], name
        # ld.shared::cluster compiles to a generic LD (not LDS / LDG) of the address mapa gives; the instantiations whose
        # multiply ignores u (FIRST = 0, PAIR = 2) gather nothing
        mul = int(re.search(r"Li(\d+)ELi(\d+)E", name).group(2))
        assert (mul in (0, 2)) or any(re.fullmatch(r"LD(\.[A-Z0-9]+)*", o) for o in ops), name
        assert "MEMBAR.ALL.GPU" in ops, name                         # barrier.cluster.arrive.release
