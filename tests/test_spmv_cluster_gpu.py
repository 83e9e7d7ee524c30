"""The hot-table SpMV kernel as thread-block clusters (spmv_run.cuh): every cluster size and replicated tier gives the same
bytes as plain CTAs, and the oracle's result, with gathers on every side of every tier boundary.

The tiers are restated from hot2_tiers: a CTA's table holds `cap` entries; with C > 1 the replicated tier T0 is the
B200GRB_SPMV_HOT_REPL request (entries, multiple of 16, at most cap), the rest of the table is this CTA's slice of the
distributed tier T1, and the hot ranks past T0 + T1 up to henc are read from u_hot in L2.  Plain CTAs are launched when
one table holds every hot rank or T0 takes the whole table.  Every call asserts the cluster size and the tiers the
library reports (`hot-cluster=`, `hot-tiers=T0,T1,henc`) against this restatement; an H100 co-schedules every C <= 16.
The SASS checks need no GPU."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import scipy.sparse as sp

from pygraphblas_b200 import Matrix, Vector
from pygraphblas_b200.generators import rmat_csr
from oracle import oracle as orc
import util
from kernel_check import compare, entries, last_kernel, o_csr, semiring, seed_of, tunables, values, fp_pool_for

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pygraphblas_b200", "libb200grb.so")
HOT_EXT = 1 << 17
CLUSTERS = (1, 2, 4, 8, 16)
HOT_SRS = [("PLUS", "TIMES"), ("MIN", "PLUS"), ("PLUS", "SECOND")]
SRS = [sr + (t,) for t in ("FP32", "FP64", "INT32", "UINT64") for sr in HOT_SRS] + [("LOR", "LAND", "BOOL")]
VSIZE = {"FP32": 4, "FP64": 8, "INT32": 4, "UINT64": 8, "BOOL": 1}
ROUTES = {"run+hot-table (TMA-staged)"}
REACHED_C, SIDES = set(), set()


def tokens():
    ks = last_kernel().split(";")
    return entries(ks), dict(k.split("=", 1) for k in ks if "=" in k)


def uniform_pattern(ncols, deg):
    """Every column referenced exactly deg times: the stable degree sort then ranks column j as j, so every hot rank
    (and so both sides of every tier boundary) is gathered."""
    nrows = ncols
    j = np.repeat(np.arange(ncols, dtype=np.int64), deg)
    t = np.tile(np.arange(deg, dtype=np.int64), ncols)
    r = (j * 7 + t * 4099) % nrows
    S = sp.csr_matrix((np.ones(len(j), np.int8), (r, j)), shape=(nrows, ncols))
    S.sort_indices()
    assert S.nnz == ncols * deg
    return S


def rmat_pattern(scale):
    n, indptr, indices = rmat_csr(scale, 16, seed=3)
    return sp.csr_matrix((np.ones(len(indices), np.int8), indices, indptr), shape=(n, n))


def tiers(henc, cap, C, t0kb, vsize):
    """Restates hot2_tiers: (C, T0, T1, slice)."""
    if C == 1 or henc - cap < 16:
        return 1, cap, 0, 0
    t0 = min(((t0kb << 10) // vsize) & ~15, cap)
    need = henc - t0
    sl = min(cap - t0, (-(-need // C) + 15) & ~15)
    if sl == 0:
        return 1, cap, 0, 0
    return C, t0, min(need, sl * C), sl


def expected_tiers(S, vxm, typ, hot_kb, C, t0kb):
    """(C, T0, T1, henc) of a call: henc from the column degrees of the CSR the kernel pulls along (A' for vxm), cap from
    the table limit (128 KB or B200GRB_SPMV_HOT; the shared memory left after the stages exceeds 128 KB for these types)."""
    deg = np.diff(S.indptr) if vxm else np.bincount(S.indices, minlength=S.shape[1])
    henc = min(int(np.count_nonzero(deg)), HOT_EXT)
    cap = min(henc, (hot_kb << 10) // VSIZE[typ]) & ~15
    c, t0, t1, _ = tiers(henc, cap, C, t0kb, VSIZE[typ])
    return c, t0, t1, henc


def run_all(S, label, settings, srs=SRS, forms=("mxv", "vxm"), hot_kb=128):
    """For each semiring and form: the C = 1 result, then each (C, T0 KB) of settings must give the same bytes; every
    result is compared with the oracle, and the launch the library reports with the restated tiers.  Returns the set
    of (C, T0, T1, henc) launched."""
    nrows, ncols = S.shape
    errors, launched = [], set()
    for sr0 in srs:
        typ = sr0[2]
        pool = fp_pool_for(sr0[0], sr0[1]) if typ in util.FP_T else "edge"
        av = values(seed_of(label, typ), typ, S.nnz, pool, 0)
        A, Ao = Matrix.from_csr(S.indptr, S.indices, av, nrows, ncols, util.g_type(typ)), o_csr(typ, S, av)
        for form in forms:
            vxm = form == "vxm"
            # SECOND reads u in mxv form; in vxm form FIRST does (the other one gathers nothing and takes the plain run kernel)
            sr = (sr0[0], "FIRST", typ) if vxm and sr0[1] == "SECOND" else sr0
            n_in = nrows if vxm else ncols
            uv = values(seed_of(label, sr, form), typ, n_in, pool, 1)
            u = Vector.from_numpy(uv, typ=util.g_type(typ))
            uo = orc.SpVec(typ, n_in, np.arange(n_in), uv)
            ref = orc.vxm(orc.SpVec(typ, nrows if not vxm else ncols), None, None, sr, uo, Ao, "") if vxm else \
                orc.mxv(orc.SpVec(typ, nrows), None, None, sr, Ao, uo, "")
            base = None
            for C, t0kb in [(1, 0)] + list(settings):
                with tunables(B200GRB_SPMV_CLUSTER=C, B200GRB_SPMV_HOT_REPL=t0kb):
                    w = u.vxm(A, semiring=semiring(*sr)) if vxm else A.mxv(u, semiring=semiring(*sr))
                    ent, tok = tokens()
                assert ent[0] in ROUTES, (label, sr, form, C, ent)
                got_t = (int(tok["hot-cluster"]),) + tuple(int(x) for x in tok["hot-tiers"].split(","))
                want_t = expected_tiers(S, vxm, typ, hot_kb, C, t0kb)
                assert got_t == want_t, (label, sr, form, C, t0kb, got_t, want_t)
                launched.add(got_t)
                REACHED_C.add(got_t[0])
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
@pytest.mark.parametrize("pattern", ["rmat18", "even"])
def test_cluster_sizes_are_bit_identical(pattern):
    S = rmat_pattern(18) if pattern == "rmat18" else uniform_pattern((1 << 17) + 4096, 8)
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


# (ncols, per-column degree, C, T0 KB): FP32 tables of 128 KB (cap = 32768 entries)
TIER_CASES = {
    "c8-rest-and-u": ((1 << 17) + 4096, 8, 8, 96),        # T0 + T1 < henc = 2^17 < ncols: every tier and u
    "c4-no-repl": ((1 << 17) + 4096, 8, 4, 0),            # T0 = 0: the table is all slices
    "c16-short": ((1 << 16) + 40, 16, 16, 0),             # fewer hot columns than C * cap: partly filled slices
    "c2-short-repl": ((1 << 16) + 40, 16, 2, 64),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(TIER_CASES))
def test_tier_boundaries(case):
    ncols, deg, C, t0kb = TIER_CASES[case]
    S = uniform_pattern(ncols, deg)
    srs = [("PLUS", "TIMES", "FP32"), ("MIN", "PLUS", "FP32")]
    with tunables(B200GRB_SPMV_HOT=128):
        launched = run_all(S, case, [(C, t0kb)], srs=srs, forms=("mxv",))
    # the tiers the library reported for the cluster launch (rank j = column j: every rank is gathered, so each boundary
    # inside the hot ranks has a gathered rank on both of its sides)
    (c, t0, t1, henc), = [t for t in launched if t[0] > 1]
    assert c == C
    for b in (t0, t0 + t1, henc):
        if 0 < b < ncols:
            SIDES.add(f"{case}-{b - 1}|{b}")
    if t0 + t1 < henc:
        SIDES.add(f"{case}-rest")
    if t1 % (16 * C):                                     # slices are multiples of 16 entries: full ones sum to a multiple of 16 C
        SIDES.add(f"{case}-partial-slices")


def test_every_cluster_size_and_tier_was_reached(request):
    mine = [it for it in request.session.items if it.module is request.module and it is not request.node and "gpu" in it.keywords]
    gpu_count = 2 + 3 + len(TIER_CASES)
    if len(mine) < gpu_count or not REACHED_C:
        pytest.skip("the GPU cases of the module did not all run")
    assert REACHED_C >= set(CLUSTERS), sorted(REACHED_C)
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
