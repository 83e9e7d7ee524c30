"""Every mxv / vxm / mxm kernel path against the CPU oracle, with operands built to sit on both sides of the boundaries
where work is split and put back together.

test_value_edges_gpu.py varies the values and keeps the structure gentle; this module does the reverse.  Each operand
is built from explicit row lengths (csr()) and checks the structure it claims (a row of exactly 4097 entries, a B row
of 1025 entries starting at a position = 1 (mod 4), ...).  The routing rules of the library are restated in Python
(spmv_route, gemm_route); every call asserts through B200_debug_last_kernel that the library took the route the
restatement predicts, and every case asserts that the restatement puts it on the side of the boundary it claims to test
(side()).  Decisions the device makes (long-B-row pieces, the stream kernel's batch loop, the chunk count of a row, the
pull kernel's long rows) are asserted from the operand.

Values are drawn from the edge pools of util.rand_edge_values; FP PLUS / TIMES folds use the dyadic and unit pools so
that every fold order gives the same bits.  Results are compared with the rules of test_value_edges_gpu.py: bit-exact,
NaN matches NaN, +-0 match under MIN / MAX, and an ANY result must be one of its entry's products.

The last sections run call sequences that reuse cached state (the tile / run / hot plans and the cached transpose of a
matrix, the grow-only workspaces, mxv formed in place in w's buffers) and check every step against the oracle."""
import functools

import numpy as np
import pytest
import scipy.sparse as sp

from pygraphblas_b200 import Matrix, Vector, descriptor, lib, ffi
from oracle import oracle as orc
import util
from kernel_check import (compare, entries, fp_pool_for, o_csr, products_by_entry, record_kernels, seed_of, semiring,
                          spmv_specialised, tunables, values, vec_products)

pytestmark = pytest.mark.gpu

REACHED = set()      # kernel entries and variant tokens the seam reported
SIDES = set()        # boundary sides a case claimed and verified


def _kernels():
    return record_kernels(REACHED)


def side(name):
    assert name in ALL_SIDES, name
    SIDES.add(name)


# ------------------------------------------------------------------ the operand builder
def csr(row_lengths, ncols, seed=0, cols=None):
    """A sorted CSR pattern whose row r has exactly row_lengths[r] entries: at the columns cols[r] when given, else at
    distinct columns spread over [0, ncols) (vectorised: base + k * step mod ncols with step coprime to ncols)."""
    lens = np.asarray(row_lengths, np.int64)
    assert (lens <= ncols).all()
    nrows, nnz = len(lens), int(lens.sum())
    indptr = np.concatenate(([0], np.cumsum(lens)))
    rows = np.repeat(np.arange(nrows), lens)
    k = np.arange(nnz) - indptr[rows]
    rng = np.random.default_rng(seed)
    steps = np.array([s for s in (40503, 7919, 104729, 15485863, 1299709) if np.gcd(s, ncols) == 1] or [1])
    base = rng.integers(0, ncols, nrows)
    step = steps[rng.integers(0, len(steps), nrows)]
    c = (base[rows] + k * step[rows]) % ncols
    if cols:
        for r, cc in cols.items():
            cc = np.asarray(cc, np.int64)
            assert len(cc) == lens[r] and len(np.unique(cc)) == len(cc), r
            c[indptr[r]:indptr[r + 1]] = cc
    order = np.lexsort((c, rows))
    S = sp.csr_matrix((np.ones(nnz, bool), c[order].astype(np.int32), indptr), shape=(nrows, ncols))
    assert S.has_sorted_indices and S.nnz == nnz
    assert np.array_equal(np.diff(S.indptr), lens)
    return S


def row_span(S, r):
    """(first position, length) of row r."""
    return int(S.indptr[r]), int(S.indptr[r + 1] - S.indptr[r])


def assert_row(S, r, length, start_mod=None):
    """Row r has exactly `length` entries and (start_mod = (m, q)) starts at a position = q (mod m)."""
    s, n = row_span(S, r)
    assert n == length, (r, n, length)
    if start_mod is not None:
        assert s % start_mod[0] == start_mod[1], (r, s, start_mod)


def stack(*parts):
    S = sp.vstack(parts).tocsr()
    S.sort_indices()
    return S


# ------------------------------------------------------------------ the routing rules, restated
HOT_ENC, RUN, PULL_LONG, PUSH_CHUNK, STREAM_LONG_ROW = 40960, 256, 4096, 1024, 1024
CHUNK_FLOPS, WARP_FLOPS = 32768, 2048
COMMUTATIVE = {"TIMES", "PLUS", "MIN", "MAX", "PAIR", "LAND", "LOR", "LXOR", "EQ", "NE", "ISEQ", "ISNE"}


def _uses_x(op):
    return op not in ("SECOND", "PAIR")


def _uses_y(op):
    return op not in ("FIRST", "PAIR", "ANY")


@functools.lru_cache(maxsize=None)
def _hot_stats(key):
    """(number of hot columns, their share of the entries): hot_invert_kernel over the HOT_ENC most referenced columns."""
    S = _PULLED[key][1]
    deg =np.sort(np.bincount(S.indices, minlength=S.shape[1]))[::-1][:HOT_ENC]
    deg = deg[deg > 0]
    return len(deg), (float(deg.sum()) / S.nnz if S.nnz else 0.0)


_PULLED = {}        # (id(S), vxm) -> (S, pulled CSR); S is kept so that its id is never reused


def pulled(S, vxm):
    """The CSR the SpMV kernels pull along: A for mxv, A' for vxm (cached by identity)."""
    key = (id(S), vxm)
    if key not in _PULLED:
        if vxm:
            T = S.T.tocsr(); T.sort_indices()
            _PULLED[key] = (S, T)
        else:
            _PULLED[key] = (S, S)
    return key, _PULLED[key][1]


def forget(S):
    """Drop the cached pulled patterns (and hot statistics) of S."""
    for vxm in (False, True):
        _PULLED.pop((id(S), vxm), None)
    _hot_stats.cache_clear()


@pytest.fixture(autouse=True)
def _drop_pulled_patterns():
    yield
    _PULLED.clear()
    _hot_stats.cache_clear()


def spmv_route(S, sr, vxm, env, sparse_u=False, upres=None, masked=False):
    """Restates mxv_core's choice of kernel for w = A u (vxm: w' = u' A) on pattern S."""
    add, mul, typ = sr
    key, c = pulled(S, vxm)
    kmul, kflip = mul, vxm
    if vxm and mul in ("FIRST", "SECOND"):
        kmul, kflip = ("SECOND" if mul == "FIRST" else "FIRST"), False
    if vxm and mul in COMMUTATIVE:
        kflip = False
    need_u = _uses_x(kmul) if kflip else _uses_y(kmul)
    fast_sr = not kflip and spmv_specialised(add, kmul, typ)
    fast = fast_sr and not sparse_u
    if masked and add in ("LOR", "LAND", "ANY") and c.nnz > 0 and "B200GRB_NO_PULL" not in env:
        if sparse_u and "B200GRB_NO_PUSH" not in env and not (add in ("LOR", "LAND") and typ != "BOOL"):
            _, o = pulled(S, not vxm)
            count = int(upres.sum())
            edges = int(np.diff(o.indptr)[upres].sum())
            if not (edges * 16 > c.nnz or count * 32 > o.shape[0]) or "B200GRB_FORCE_PUSH" in env:
                return "push"
        return "pull"
    use_run = c.nnz >= 4096
    if "B200GRB_SPMV_RUN" in env:
        use_run = c.nnz > 0 and int(env["B200GRB_SPMV_RUN"]) != 0
    if use_run:
        hot_kb = int(env.get("B200GRB_SPMV_HOT", -1))
        hot = False
        if fast and need_u and (hot_kb if hot_kb >= 0 else 128) > 0 and c.nnz >= (1 << 20) and c.shape[1] >= (1 << 16):
            henc, cover = _hot_stats(key)
            hot = henc >= 16 and (hot_kb >= 0 or cover >= 0.25)
        if hot:
            pipe = orc.DTYPES[typ]().itemsize <= 4 and int(env.get("B200GRB_SPMV_PIPE", 0)) != 0
            return "run+hot-table (TMA-staged, pipelined)" if pipe else "run+hot-table (TMA-staged)"
        return "run (sparse u)" if sparse_u else "run"
    if c.nnz == 0:
        return "empty"
    if not fast:
        return "tile (run-time operators)"
    items = int(env.get("B200GRB_SPMV_ITEMS", 8))
    return f"tile (specialised, {items if items in (4, 16) else 8} items)"


def flops_per_row(SA, SB):
    return np.bincount(np.repeat(np.arange(SA.shape[0]), np.diff(SA.indptr)), weights=np.diff(SB.indptr)[SA.indices],
                       minlength=SA.shape[0]).astype(np.int64)


def masked_classes(SA, SB, SM):
    """chunk_count_kernel restated: per row the class ('' none, 'warp', 'S', 'M', 'L') and the number of chunks."""
    f = flops_per_row(SA, SB)
    ml = np.diff(SM.indptr).astype(np.int64)
    cls = np.full(len(f), "", dtype=object)
    live = (f > 0) & (ml > 0)
    cls[live & (ml <= 512)] = "S"
    cls[live & (ml > 512) & (ml <= 2048)] = "M"
    cls[live & (ml > 2048)] = "L"
    cls[live & (f <= WARP_FLOPS) & (ml <= 128)] = "warp"
    chunks = np.where(live & (cls != "warp"), (f + CHUNK_FLOPS - 1) // CHUNK_FLOPS, 0)
    return cls, chunks, f, ml


def gemm_route(SA, SB, SM, desc, env):
    """Restates GrB_mxm's choice of kernels: the entries (and filter tokens) B200_debug_last_kernel reports.
    SB is B as stored; desc may hold T1, C, S, R."""
    Bt = SB.T.tocsr() if "T1" in desc else SB
    if "T1" in desc:
        Bt.sort_indices()
    if SM is not None and "C" not in desc:
        if "T1" in desc and SB.nnz < (1 << 18):
            return ["dot"] if SM.nnz > 0 else []
        if SM.nnz == 0:
            return []
        cls, _, _, _ = masked_classes(SA, Bt, SM)
        out = ["masked-warp"] if (cls == "warp").any() else []
        ncols = Bt.shape[1]
        for k, bm in (("S", 14), ("M", 16), ("L", 20)):
            if (cls == k).any():
                out += [f"stream-{k}", "filter=exact" if ncols <= (1 << bm) else "filter=bloom"]
        return out
    if SM is None and "C" in desc:
        return []
    f = flops_per_row(SA, Bt)
    esc = int(env.get("B200GRB_SPGEMM_ESC", 1)) != 0
    out = []
    if ((f > 0) & (f <= 128)).any():
        out.append("esc-small" if esc else "hash-small")
    if ((f > 128) & (f <= 2048)).any():
        out.append("esc-medium" if esc else "hash-medium")
    if (f > 2048).any():
        out.append("spa")
    return out


# ------------------------------------------------------------------ semirings and values
# (add, mul, type): specialised and run-time-operator kernels, integer, FP and BOOL, and one ANY
SPMV_SRS = [("PLUS", "TIMES", "INT32"), ("MIN", "PLUS", "UINT64"), ("MAX", "MINUS", "INT16"), ("BXOR", "TIMES", "UINT8"),
            ("PLUS", "TIMES", "FP64"), ("MIN", "PLUS", "FP32"), ("PLUS", "SECOND", "FP32"), ("MAX", "DIV", "FP64"),
            ("PLUS", "MINUS", "FP32"), ("LOR", "LAND", "BOOL"), ("LXOR", "LAND", "BOOL"), ("ANY", "SECOND", "INT32")]
PULL_SRS = [("LOR", "LAND", "BOOL"), ("LAND", "LOR", "BOOL"), ("ANY", "SECOND", "INT64"), ("ANY", "TIMES", "FP32")]
GEMM_SRS = [("PLUS", "TIMES", "INT64"), ("MIN", "PLUS", "INT32"), ("PLUS", "TIMES", "FP64"), ("PLUS", "SECOND", "FP32"),
            ("MAX", "MINUS", "FP32"), ("LOR", "LAND", "BOOL"), ("LXOR", "LAND", "BOOL"), ("ANY", "TIMES", "UINT16")]


def pool_of(sr):
    return fp_pool_for(sr[0], sr[1]) if sr[2] in util.FP_T else "edge"


def ztype(sr):
    return orc.semiring_ztype(sr)


# ------------------------------------------------------------------ SpMV runner
def _mask_for(spec, n, seed):
    """spec: None, 'empty', 'struct' (BOOL, 70 % present) or a valued type: present entries of which about a third are
    false (0, -0.0 or integer zero); FP NaN entries count as true."""
    if spec is None:
        return None
    rng = np.random.default_rng(seed)
    if spec == "empty":
        return "BOOL", np.zeros(0, np.int64), np.zeros(0, bool)
    idx = np.flatnonzero(rng.random(n) < 0.7)
    typ = "BOOL" if spec == "struct" else spec
    if typ == "BOOL":
        return typ, idx, np.ones(len(idx), bool)
    return typ, idx, mask_values(typ, len(idx), rng)


def mask_values(typ, n, rng):
    """n mask values of typ, about a third false (0 and -0.0, or integer zero); the rest true, FP NaN among them."""
    dt = orc.DTYPES[typ]
    v = util.rand_edge_values(rng, typ, n, 0.5)
    v[v == 0] = 1
    if typ in util.FP_T:
        v[rng.random(n) < 0.1] = np.nan
    z = rng.random(n) < 0.35
    v[z] = np.where(rng.random(int(z.sum())) < 0.5, dt(0), dt(-0.0) if typ in util.FP_T else dt(0))
    return v


def run_spmv(S, label, env=None, srs=SPMV_SRS, forms=("mxv", "vxm"), sparse_u=None, mask=None, desc="", accum=False,
             w_init=False, seed=0):
    """Run each semiring of srs in each form on pattern S under the switches env; assert the route of every call and
    compare with the oracle.  Returns the set of routes taken.  sparse_u: None (dense) or the density of u.
    mask: see _mask_for.  accum: the semiring's monoid as accumulator.  w_init: w starts with entries."""
    env = env or {}
    nrows, ncols = S.shape
    routes, errors, calls = set(), [], 0
    mats = {}
    with tunables(**env):
        for sr in srs:
            typ = sr[2]
            pool = pool_of(sr)
            if (typ, pool) not in mats:
                av = values(seed_of(label, typ, pool), typ, S.nnz, pool, 0)
                mats[typ, pool] = (Matrix.from_csr(S.indptr, S.indices, av, nrows, ncols, util.g_type(typ)), o_csr(typ, S, av), av)
            A, Ao, av = mats[typ, pool]
            zt = ztype(sr)
            for form in forms:
                vxm = form == "vxm"
                n_in, n_out = (nrows, ncols) if vxm else (ncols, nrows)
                rng = np.random.default_rng(seed_of(label, sr, form, seed, bits=32))
                uv = values(int(rng.integers(1 << 30)), typ, n_in, pool, 1)
                upres = rng.random(n_in) < sparse_u if sparse_u is not None else np.ones(n_in, bool)
                u = Vector.from_numpy(uv, present=upres if sparse_u is not None else None, typ=util.g_type(typ))
                uo = orc.SpVec(typ, n_in, np.flatnonzero(upres), uv[upres])
                m = _mask_for(mask, n_out, int(rng.integers(1 << 30)))
                M = Mo = None
                if m is not None:
                    M = Vector.from_lists(m[1], m[2], n_out, util.g_type(m[0]))
                    Mo = orc.SpVec(m[0], n_out, m[1], m[2])
                wI = np.flatnonzero(rng.random(n_out) < 0.5) if w_init else np.zeros(0, np.int64)
                wX = values(int(rng.integers(1 << 30)), zt, len(wI), pool if zt == typ else "edge", 1)
                w = Vector.from_lists(wI, wX, n_out, util.g_type(zt)) if len(wI) else Vector.sparse(util.g_type(zt), n_out)
                wo = orc.SpVec(zt, n_out, wI, wX)
                acc = (sr[0] if sr[0] not in ("ANY",) else "FIRST", zt) if accum else None
                d = getattr(descriptor, desc) if desc else None
                if M is not None and sparse_u is not None and not vxm:      # A' in HBM: the other orientation the push kernel walks
                    Vector.sparse(util.g_type(typ), nrows).vxm(A, semiring=semiring("LOR" if typ == "BOOL" else "ANY", "FIRST", typ))
                if vxm:
                    u.vxm(A, semiring=semiring(*sr), out=w, mask=M, accum=util.g_accum(acc), desc=d)
                else:
                    A.mxv(u, semiring=semiring(*sr), out=w, mask=M, accum=util.g_accum(acc), desc=d)
                ks = _kernels()
                calls += 1
                want = spmv_route(S, sr, vxm, env, sparse_u is not None, upres, M is not None)
                assert entries(ks) == [want], (label, sr, form, ks, want)
                routes.add(want)
                gI, gX = w.to_arrays()
                ref = (orc.vxm(wo, Mo, acc, sr, uo, Ao, desc) if vxm else orc.mxv(wo, Mo, acc, sr, Ao, uo, desc))
                cands = vec_products(uv, upres, S, av, sr[1], vxm) if sr[0] == "ANY" and not accum and not w_init else None
                if sr[0] == "ANY" and cands is None:
                    continue
                e = compare(gI, gX, ref.I, ref.X, zt, sr[0], f"{label} {form} {'_'.join(sr)}", cands)
                if e:
                    errors.append(e)
    assert calls > 0
    assert not errors, f"{len(errors)} of {calls} calls differ ({label}):\n" + "\n".join(errors[:30])
    return routes


# ------------------------------------------------------------------ SpGEMM runner
def run_gemm(SA, SB, SM, desc, label, env=None, srs=GEMM_SRS, c_init=False, accum=False, mask_type=None, alias=False):
    """C<M> = accum(C, A (+).(x) B) for each semiring: assert the route, compare with the oracle.  Returns the routes.
    mask_type: None (structural BOOL mask of SM) or a valued type whose mask has false entries (see _mask_for), with a
    row whose every mask entry is false.  alias: C = A (+).(x) A computed into A itself (SB ignored)."""
    env = env or {}
    routes, errors, calls = [], [], 0
    with tunables(**env):
        for sr in srs:
            typ, zt, pool = sr[2], ztype(sr), pool_of(sr)
            seed = seed_of(label, sr)
            av = values(seed, typ, SA.nnz, pool, 0)
            bv = av if alias else values(seed + 1, typ, SB.nnz, pool, 1)
            SBx = SA if alias else SB
            A = Matrix.from_csr(SA.indptr, SA.indices, av, *SA.shape, util.g_type(typ))
            B = A if alias else Matrix.from_csr(SBx.indptr, SBx.indices, bv, *SBx.shape, util.g_type(typ))
            Ao, Bo = o_csr(typ, SA, av), o_csr(typ, SBx, bv)
            nrows, ncols = SA.shape[0], (SBx.shape[0] if "T1" in desc else SBx.shape[1])
            M = Mo = None
            if SM is not None:
                if mask_type is None:
                    mv = np.ones(SM.nnz, bool); mt = "BOOL"
                else:
                    mt = mask_type
                    mv = mask_values(mask_type, SM.nnz, np.random.default_rng(seed + 2))
                    r = int(np.argmax(np.diff(SM.indptr) > 0))            # the first non-empty mask row: all false
                    mv[SM.indptr[r]:SM.indptr[r + 1]] = 0
                M = Matrix.from_csr(SM.indptr, SM.indices, mv, *SM.shape, util.g_type(mt))
                Mo = o_csr(mt, SM, mv)
            if alias:
                C, Co = A, Ao
                assert zt == typ
            elif c_init:
                Sc = csr(np.minimum(np.random.default_rng(seed).integers(0, 6, nrows), ncols), ncols, seed + 3)
                cv = values(seed + 4, zt, Sc.nnz, pool if zt == typ else "edge", 0)
                C, Co = Matrix.from_csr(Sc.indptr, Sc.indices, cv, nrows, ncols, util.g_type(zt)), o_csr(zt, Sc, cv)
            else:
                C, Co = Matrix.sparse(util.g_type(zt), nrows, ncols), orc.SpMat(zt, nrows, ncols)
            acc = (sr[0] if sr[0] != "ANY" else "FIRST", zt) if accum else None
            A.mxm(B, semiring=semiring(*sr), out=C, mask=M, accum=util.g_accum(acc), desc=getattr(descriptor, desc) if desc else None)
            ks = _kernels()
            calls += 1
            want = gemm_route(SA, SBx, SM, desc, env)
            assert [k for k in ks if k] == want, (label, sr, ks, want)
            routes.append(want)
            ref = orc.mxm(Co, Mo, acc, sr, Ao, Bo, desc)
            gI, gJ, gX = C.to_arrays()
            cands = None
            if sr[0] == "ANY":
                if accum or c_init or alias or "T1" in desc:
                    continue
                cands = products_by_entry(np.repeat(np.arange(nrows), np.diff(SA.indptr)), SA.indices.astype(np.int64), av,
                                          SBx.indptr, SBx.indices, bv, ncols, sr[1])
            e = compare(gI.astype(np.int64) * ncols + gJ.astype(np.int64), gX, ref.I.astype(np.int64) * ncols + ref.J.astype(np.int64),
                        ref.X, zt, sr[0], f"{label} {'_'.join(sr)}", cands)
            if e:
                errors.append(e)
    assert calls > 0
    assert not errors, f"{len(errors)} of {calls} mxm calls differ ({label}):\n" + "\n".join(errors[:30])
    return routes


# ================================================================== SpMV: tile
def tile_pattern(items, tail):
    """Rows laid out against tiles of T = 256 * items entries: three leading empty rows; a row covering two whole tiles
    and more; a row ending at the last entry of tile 2; empty rows on that boundary; a row of one entry (ending at the
    first entry of tile 3); a row ending at the end of tile 3; 3000 empty rows; a row of 7; then rows up to
    nnz = 6 T + tail (tail in -1, 0, 1); five trailing empty rows."""
    T = 256 * items
    lens = [0, 0, 0, 2 * T + 3]
    lens += [3 * T - sum(lens)] + [0] * 4 + [1] + [4 * T - (3 * T + 1)] + [0] * 3000 + [7]
    while sum(lens) + T < 6 * T + tail:
        lens.append(T // 2)
    lens.append(6 * T + tail - sum(lens))
    lens += [0] * 5
    S = csr(lens, 2 * T + 64, seed=items * 10 + tail)
    assert S.nnz == 6 * T + tail and S.indptr[4] == 2 * T + 3
    for b in (3 * T, 3 * T + 1, 4 * T):
        assert b in set(S.indptr.tolist()), b              # rows end at the end of a tile and at the entry after it
    assert (np.diff(S.indptr)[4:4 + 1 + 4 + 1] == [3 * T - 2 * T - 3, 0, 0, 0, 0, 1]).all()
    return S


@pytest.mark.parametrize("tail", [-1, 0, 1])
@pytest.mark.parametrize("items", [4, 8, 16])
def test_tile_boundaries(items, tail):
    S = tile_pattern(items, tail)
    env = {"B200GRB_SPMV_RUN": 0, "B200GRB_SPMV_ITEMS": items}
    routes = run_spmv(S, f"tile-{items}-{tail}", env)
    assert f"tile (specialised, {items} items)" in routes and "tile (run-time operators)" in routes, routes
    side(f"tile-{items}-nnz{tail:+d}")


@pytest.mark.parametrize("shape", ["nrows=1", "ncols=1", "last-entry"])
def test_tile_degenerate_shapes(shape):
    if shape == "nrows=1":
        S = csr([300], 500, seed=1)
    elif shape == "ncols=1":
        S = csr(np.random.default_rng(2).integers(0, 2, 3000), 1)
    else:
        S = csr([0] * 2499 + [1], 777, cols={2499: [776]})
        assert S.indices[-1] == 776 and row_span(S, 2499) == (0, 1)
    routes = run_spmv(S, f"tile-{shape}")
    assert all(r.startswith("tile") for r in routes), routes
    side(f"tile-{shape}")


# ================================================================== SpMV: run
def run_pattern(tail, natural=False):
    """Rows laid out against runs of 256 entries and lane groups of 8: two leading empty rows; a row over three runs
    ending at a position = 7 (mod 8); rows starting at = 7, 0 and 1 (mod 8); a row ending at the end of run 3; 2000
    empty rows; a row covering exactly two whole runs; filler rows up to nnz = k * 256 + tail; trailing empty rows.
    natural: nnz = 4096 + tail, the size at which the run kernel is chosen without the switch."""
    lens = [0, 0, 3 * RUN + 7, 1, 1, 4 * RUN - (3 * RUN + 9)] + [0] * 2000 + [2 * RUN]
    total = (4096 if natural else 8 * RUN) + tail
    while sum(lens) + 100 < total:
        lens.append(97)
    lens.append(total - sum(lens))
    lens += [0] * 9
    S = csr(lens, 1500, seed=40 + tail + 7 * natural)
    assert row_span(S, 3)[0] % 8 == 7 and row_span(S, 4)[0] % 8 == 0 and row_span(S, 5)[0] % 8 == 1
    assert S.indptr[6] == 4 * RUN and row_span(S, 2006) == (4 * RUN, 2 * RUN)
    assert S.nnz == total
    return S


@pytest.mark.parametrize("u", ["dense", "sparse"])
@pytest.mark.parametrize("tail", [-1, 0, 1])
def test_run_boundaries(tail, u):
    S = run_pattern(tail)
    routes = run_spmv(S, f"run-{tail}-{u}", {"B200GRB_SPMV_RUN": 1}, sparse_u=0.6 if u == "sparse" else None)
    assert routes == ({"run"} if u == "dense" else {"run (sparse u)"}), routes
    side(f"run-nnz{tail:+d}")


@pytest.mark.parametrize("tail", [-1, 0])
def test_run_threshold(tail):
    """nnz = 4095: the tile kernel; nnz = 4096: the run kernel, without any switch."""
    S = run_pattern(tail, natural=True)
    routes = run_spmv(S, f"run-threshold{tail}", forms=("mxv",))
    assert all(r.startswith("tile") for r in routes) if tail < 0 else routes == {"run"}, routes
    side("run-threshold-below" if tail < 0 else "run-threshold-at")


# ================================================================== SpMV: hot table
@functools.lru_cache(maxsize=None)
def hot_pattern(ncols, nnz, hubs=True):
    """nnz entries over ncols columns, spread evenly (so the 40960 hottest columns carry 40960 / ncols of them), with
    hub rows of 3000 entries that cover many runs."""
    rng = np.random.default_rng(ncols + nnz)
    nrows = 1 << 16
    lens = rng.integers(0, 2 * nnz // nrows, nrows)
    if hubs:
        lens[[7, 4000, 65000]] = 3000
    d = nnz - int(lens.sum())
    i = 10000                                    # the adjustment stays clear of the hub rows
    while d:
        step = int(np.clip(d, -lens[i], 30 - lens[i]))
        lens[i] += step; d -= step; i += 1
    S = csr(lens, ncols, seed=ncols)
    assert S.nnz == nnz
    return S


HOT_CASES = {
    # name: (ncols, nnz, switches, expected family for PLUS_TIMES mxv)
    "at-threshold": ((1 << 16), (1 << 20), {}, "hot"),
    "nnz-below": ((1 << 16), (1 << 20) - 1, {}, "run"),
    "ncols-below": ((1 << 16) - 1, (1 << 20) + 1, {}, "run"),
    "table-64": ((1 << 16), (1 << 20) + 1, {"B200GRB_SPMV_HOT": 64}, "hot"),
    "pipe": ((1 << 16), (1 << 20) + 1, {"B200GRB_SPMV_PIPE": 1}, "hot"),
    "pipe-table-64": ((1 << 16), (1 << 20) + 1, {"B200GRB_SPMV_PIPE": 1, "B200GRB_SPMV_HOT": 64}, "hot"),
    "cover-below": ((1 << 20), (1 << 20) + 1, {}, "run"),
    "cover-below-forced": ((1 << 20), (1 << 20) + 1, {"B200GRB_SPMV_HOT": 128}, "hot"),
}
HOT_SRS = [("PLUS", "TIMES", "INT32"), ("MIN", "PLUS", "UINT64"), ("PLUS", "TIMES", "FP64"), ("MIN", "PLUS", "FP32"),
           ("PLUS", "FIRST", "FP32"), ("MAX", "MINUS", "INT16"), ("LOR", "LAND", "BOOL")]


@pytest.mark.parametrize("case", list(HOT_CASES))
def test_hot_table_boundaries(case):
    ncols, nnz, env, fam = HOT_CASES[case]
    S = hot_pattern(ncols, nnz)
    key, _ = pulled(S, False)
    henc, cover = _hot_stats(key)
    assert henc == min(HOT_ENC, ncols)                                # cold columns lie beyond the table
    assert (cover >= 0.25) == (ncols <= (1 << 16)), cover
    routes = run_spmv(S, f"hot-{case}", env, srs=HOT_SRS, forms=("mxv",))
    hot = {r for r in routes if r.startswith("run+hot")}
    assert bool(hot) == (fam == "hot"), routes
    run_spmv(S, f"hot-{case}", env, srs=HOT_SRS, forms=("vxm",))      # A' has 2^16 rows of up to 31 entries: its own side
    side(f"hot-{case}")


# ================================================================== SpMV: pull / push
@functools.lru_cache(maxsize=None)
def pull_pattern():
    """6000 x 6000.  Rows 5 and 77 have 4096 and 4097 entries (the pull kernel's CTA-per-row cut); column 5000 has 1024
    entries and column 5001 1025 (push chunks); columns 5002-5099 one entry each; columns 5100-5999 none; the rest of
    the entries (6700) spread over columns 0-4999."""
    rng = np.random.default_rng(77)
    n = 6000
    lens = np.zeros(n, np.int64)
    lens[:] = 1
    extra = 6700 - n
    lens[rng.choice(n, extra, replace=False)] += 1
    lens[5], lens[77] = 4096, 4097
    cols = {5: np.sort(rng.choice(5000, 4096, replace=False)), 77: np.sort(rng.choice(5000, 4097, replace=False))}
    base = csr(lens, 5000, seed=78, cols=cols)
    rows = [np.repeat(np.arange(n), np.diff(base.indptr)), np.arange(1000, 2024), np.arange(2100, 3125), np.arange(3200, 3298)]
    colv = [base.indices, np.full(1024, 5000), np.full(1025, 5001), np.arange(5002, 5100)]
    S = sp.csr_matrix((np.ones(sum(len(r) for r in rows), bool), (np.concatenate(rows), np.concatenate(colv))), shape=(n, n))
    S.sum_duplicates(); S.sort_indices()
    cl = np.bincount(S.indices, minlength=n)
    assert cl[5000] == 1024 and cl[5001] == 1025 and (cl[5002:5100] == 1).all() and (cl[5100:] == 0).all()
    assert np.diff(S.indptr)[5] == 4096 and np.diff(S.indptr)[77] == 4097
    return S


def frontier(S, kind):
    """A u pattern (mxv: a set of columns) on a chosen side of the push test edges * 16 > nnz or count * 32 > nin."""
    n, E = S.shape[1], S.nnz // 16
    p = np.zeros(n, bool)
    if kind in ("edges-at", "edges-over"):
        p[5000] = True                                      # 1024 edges in one push chunk ...
        p[5002:5002 + E - 1024 + (kind == "edges-over")] = True    # ... plus one-edge columns up to nnz / 16 (+1)
    elif kind in ("count-at", "count-over"):
        p[5001] = True                                      # 1025 edges: two push chunks ...
        p[5100:5100 + n // 32 - 1 + (kind == "count-over")] = True     # ... plus edge-less columns up to nin / 32 (+1)
    return p


@pytest.mark.parametrize("kind", ["edges-at", "edges-over", "count-at", "count-over"])
def test_push_heuristic_sides(kind):
    S = pull_pattern()
    up = frontier(S, kind)
    edges = int(np.diff(S.tocsc().indptr)[up].sum())
    push = not (edges * 16 > S.nnz or int(up.sum()) * 32 > S.shape[1])
    assert push == kind.endswith("-at"), (kind, edges, int(up.sum()))
    routes = set()
    for sr in PULL_SRS:
        routes |= _run_frontier(S, up, sr, kind)
    assert routes == {"push" if push else "pull"}, routes
    side(f"push-{kind}")


def _run_frontier(S, up, sr, label, desc="S"):
    typ = sr[2]
    n = S.shape[0]
    av = values(3, typ, S.nnz, pool_of(sr), 0)
    A = Matrix.from_csr(S.indptr, S.indices, av, n, n, util.g_type(typ))
    uv = values(4, typ, n, pool_of(sr), 1)
    u = Vector.from_numpy(uv, present=up, typ=util.g_type(typ))
    u.vxm(A, semiring=semiring("LOR", "FIRST", typ) if typ == "BOOL" else semiring("ANY", "FIRST", typ))      # A' in HBM
    mp = np.random.default_rng(5).random(n) < 0.7
    M = Vector.from_numpy(np.ones(n, bool), present=mp)
    w = A.mxv(u, semiring=semiring(*sr), mask=M, desc=getattr(descriptor, desc))
    ks = _kernels()
    want = spmv_route(S, sr, False, {}, True, up, True)
    assert entries(ks) == [want], (label, sr, ks, want)
    ref = orc.mxv(orc.SpVec(ztype(sr), n), orc.SpVec("BOOL", n, np.flatnonzero(mp), np.ones(int(mp.sum()), bool)), None, sr,
                  o_csr(typ, S, av), orc.SpVec(typ, n, np.flatnonzero(up), uv[up]), desc)
    gI, gX = w.to_arrays()
    cands = vec_products(uv, up, S, av, sr[1], False) if sr[0] == "ANY" else None
    e = compare(gI, gX, ref.I, ref.X, ztype(sr), sr[0], f"{label} {'_'.join(sr)}", cands)
    assert e is None, e
    return {want}


PULL_MASKS = {
    # name: (mask spec, descriptor, w starts with entries)
    "struct": ("struct", "S", False), "empty": ("empty", "", True), "valued-FP32": ("FP32", "", False),
    "valued-FP64": ("FP64", "", False), "valued-INT8": ("INT8", "", False), "valued-UINT16": ("UINT16", "", False),
    "valued-INT32": ("INT32", "", False), "valued-UINT64": ("UINT64", "", False),
    "complement": ("struct", "SC", True), "complement-replace": ("FP32", "RC", True),
}


@pytest.mark.parametrize("u", ["dense", "push"])
@pytest.mark.parametrize("mask", list(PULL_MASKS))
def test_pull_push_masks(mask, u):
    """Rows of 4096 / 4097 entries (the CTA-per-row cut) under every kind of mask; u dense (pull) or a 0.2 % frontier."""
    spec, desc, w_init = PULL_MASKS[mask]
    S = pull_pattern()
    routes = run_spmv(S, f"pull-{mask}-{u}", srs=PULL_SRS, mask=spec, desc=desc, w_init=w_init,
                      sparse_u=0.002 if u == "push" else None)
    assert ("push" in routes and routes <= {"pull", "push"}) if u == "push" else routes == {"pull"}, routes
    side(f"pull-{mask}")


# ================================================================== SpGEMM, unmasked
@functools.lru_cache(maxsize=None)
def unmasked_operands():
    """B: rows 0-4 of 1, 128, 129, 2048 and 2049 entries; rows 10-2200 single entries all at column 7; rows
    3000-3299 single entries at distinct columns.  A: rows with 0, 1, 128, 129, 2048, 2049 products; rows whose
    200 or 2100 products all hit column 7; a row whose 200 products all hit different columns."""
    nc = 4096
    blens = [1, 128, 129, 2048, 2049] + [0] * 5 + [1] * 2191 + [0] * 799 + [1] * 300
    bcols = {k: [7] for k in range(10, 2201)}
    bcols.update({3000 + k: [3000 + k] for k in range(300)})
    SB = csr(blens, nc, seed=90, cols=bcols)
    arows = [[], [0], [1], [2], [3], [4], list(range(10, 210)), list(range(10, 2110)), list(range(3000, 3200))]
    SA = csr([len(r) for r in arows], SB.shape[0], cols={i: r for i, r in enumerate(arows) if r})
    f = flops_per_row(SA, SB)
    assert f.tolist() == [0, 1, 128, 129, 2048, 2049, 200, 2100, 200]
    return SA, SB


@pytest.mark.parametrize("esc", [1, 0])
def test_unmasked_flops_bins(esc):
    SA, SB = unmasked_operands()
    routes = run_gemm(SA, SB, None, "", f"unmasked-esc{esc}", {"B200GRB_SPGEMM_ESC": esc})
    want = ["esc-small" if esc else "hash-small", "esc-medium" if esc else "hash-medium", "spa"]
    assert all(r == want for r in routes), routes
    side(f"unmasked-bins-esc{esc}")


@pytest.mark.parametrize("ncols", [1, 31, 32, 33, 4097])
def test_spa_widths(ncols):
    """The dense accumulator keeps ceil(ncols / 32) bit words: widths that are not a multiple of 32.  Row 0 has 2048
    products (hash / ESC), row 1 2049 (spa)."""
    per = min(ncols, 64)
    k0, r0 = divmod(2048, per)
    blens = [per] * k0 + ([r0] if r0 else []) + [1]
    SB = csr(blens, ncols, seed=ncols)
    arows = [list(range(len(blens) - 1)), list(range(len(blens)))]
    SA = csr([len(r) for r in arows], SB.shape[0], cols=dict(enumerate(arows)))
    assert flops_per_row(SA, SB).tolist() == [2048, 2049]
    routes = run_gemm(SA, SB, None, "", f"spa-{ncols}")
    assert all("spa" in r for r in routes), routes
    side(f"spa-ncols-{ncols}")


# ================================================================== SpGEMM, masked
def masked_operands(ncols, seed=0):
    """A, B, M with rows at every class and chunk boundary of chunk_count_kernel, and long B rows.

    B: rows 0-1999 of 1 entry, 2000-2099 of 16, 2100-2227 of 1024, then long rows of 1025 and 1151 entries starting
    at positions = 0, 1, 2, 3 (mod 4) (filler rows of one entry between them).
    A / M rows (flops, mask-row length -> class, chunks):"""
    rng = np.random.default_rng(seed + ncols)
    blens = [1] * 2000 + [16] * 100 + [1024] * 128
    long_rows = []
    for L in (1025, 1151):
        for q in range(4):
            while sum(blens) % 4 != q:
                blens.append(1)
            long_rows.append(len(blens)); blens.append(L)
    blens.append(1)
    SB = csr(blens, ncols, seed=seed + 1)
    for i, r in enumerate(long_rows):
        assert_row(SB, r, (1025, 1151)[i // 4], (4, i % 4))
    # the last long row ends one entry before the end of B and nnz(B) is not a multiple of 4: the 128-bit loads of its last
    # trip reach past the end of B's column ids
    assert SB.nnz % 4 != 0 and SB.indptr[long_rows[-1] + 1] == SB.nnz - 1
    ones, sixteen, k1024 = list(range(2000)), list(range(2000, 2100)), list(range(2100, 2228))

    def take(f):
        """distinct B rows whose lengths sum to exactly f"""
        n1024, rest = divmod(f, 1024)
        n16, n1 = divmod(rest, 16)
        assert n1024 <= 128
        return k1024[:n1024] + sixteen[:n16] + ones[:n1]

    spec = [  # (A row's B rows, mask-row length)
        (take(2048), 128),        # warp: flops and mask row at the limits
        (take(2049), 128),        # S: one flop too many for the warp class
        (take(100), 129),         # S: mask row one too long for the warp class
        (take(3000), 512),        # S
        (take(3000), 513),        # M
        (take(5000), 2048),       # M
        (take(5000), 2049),       # L
        (take(32768), 300),       # S, one chunk
        (take(32769), 300),       # S, two chunks
        (take(3 * 32768 + 5), 300),   # S, four chunks
        (take(100000), 3000),     # L, four chunks
        (take(70000), 600),       # M, three chunks
        (ones[:1100], 600),       # M: 1100 A entries in one chunk (batches of 256)
        (ones[:1100], 2500),      # L: 1100 A entries in one chunk (batches of 1024)
        (long_rows + ones[:50], 1000),   # every long B row in one batch
        (long_rows[1:2], 100),    # warp class with a long B row
        ([], 50),                 # a mask row whose A row is empty
        (take(500), 0),           # an A row with no mask row
    ]
    SA = csr([len(a) for a, _ in spec], SB.shape[0], cols={i: a for i, (a, _) in enumerate(spec) if a})
    # mask rows: half at columns the row's products reach, half anywhere; the last column in every long mask row
    mrows = {}
    for i, (a, ml) in enumerate(spec):
        reach = np.unique(SB.indices[np.concatenate([np.arange(SB.indptr[k], SB.indptr[k + 1]) for k in a])]) if a else np.zeros(0, np.int64)
        c = dict.fromkeys(([ncols - 1] if ml > 1000 else []) + rng.permutation(reach)[:ml // 2].tolist())
        for j in rng.permutation(ncols)[:2 * ml + 2].tolist():
            if len(c) >= ml:
                break
            c[j] = None
        mrows[i] = sorted(c)
    SM = csr([len(mrows[i]) for i in range(len(spec))], ncols, cols={i: c for i, c in mrows.items() if c})
    cls, chunks, f, ml = masked_classes(SA, SB, SM)
    assert cls.tolist() == ["warp", "S", "S", "S", "M", "M", "L", "S", "S", "S", "L", "M", "M", "L", "M", "warp", "", ""], cls
    assert chunks.tolist()[7:12] == [1, 2, 4, 4, 3], chunks
    assert np.diff(SA.indptr)[12] > 256 and np.diff(SA.indptr)[13] > 1024 and chunks[12] == chunks[13] == 1
    return SA, SB, SM


_MASKED = {}


def masked(ncols):
    if ncols not in _MASKED:
        _MASKED[ncols] = masked_operands(ncols)
    return _MASKED[ncols]


def mask_with_hits(SA, SB, lens, ncols, seed):
    """Mask rows of the given lengths: half at columns the row's products reach, the rest anywhere."""
    rng = np.random.default_rng(seed)
    rows = {}
    for i, ml in enumerate(lens):
        a = SA.indices[SA.indptr[i]:SA.indptr[i + 1]]
        reach = np.unique(np.concatenate([SB.indices[SB.indptr[k]:SB.indptr[k + 1]] for k in a])) if len(a) else np.zeros(0, np.int64)
        c = dict.fromkeys(rng.permutation(reach)[:ml // 2].tolist())
        for j in rng.permutation(ncols)[:2 * ml + 2].tolist():
            if len(c) >= ml:
                break
            c[j] = None
        rows[i] = sorted(c)
    return csr([len(rows[i]) for i in range(len(lens))], ncols, cols={i: c for i, c in rows.items() if c})


@functools.lru_cache(maxsize=None)
def uniform_masked(cls, ncols):
    """Operands of one stream class with uniform rows (the shapes of test_value_edges_gpu.py's stream paths), B and M
    over ncols columns: S = mask rows of 300, M = 1000, L = 3000 entries."""
    nrows, k, a_len, b_len, ml = {"S": (100, 2000, 10, 15, 300), "M": (60, 4000, 10, 15, 1000), "L": (40, 5000, 20, 20, 3000)}[cls]
    SA = csr([a_len] * nrows, k, seed=ncols + 1)
    SB = csr([b_len] * k, ncols, seed=ncols + 2)
    SM = mask_with_hits(SA, SB, [ml] * nrows, ncols, ncols + 3)
    assert set(masked_classes(SA, SB, SM)[0].tolist()) == {cls}
    return SA, SB, SM


@pytest.mark.parametrize("blk", [7, 12])
def test_masked_classes_chunks_long_rows(blk):
    SA, SB, SM = masked(4096)
    routes = run_gemm(SA, SB, SM, "S", f"masked-blk{blk}", {"B200GRB_STREAM_BLK": blk})
    assert all(r == ["masked-warp", "stream-S", "filter=exact", "stream-M", "filter=exact", "stream-L", "filter=exact"] for r in routes), routes
    for s in ("warp-limit", "mask-128-129", "mask-512-513", "mask-2048-2049", "chunks-1-2", "chunks-3-4", "a-batch-256",
              "a-batch-1024", "long-b-rows", "b-past-end"):
        side(f"masked-{s}")
    side(f"masked-blk{blk}")


@pytest.mark.parametrize("plus", [0, 1])
@pytest.mark.parametrize("cls", ["S", "M", "L"])
def test_masked_filter_limits(cls, plus):
    """ncols at the exact-bitmap limit of each class (2^14, 2^16, 2^20 columns) and one past it (the Bloom filter)."""
    bits = {"S": 14, "M": 16, "L": 20}[cls]
    ncols = (1 << bits) + plus
    SA, SB, SM = uniform_masked(cls, ncols)
    routes = run_gemm(SA, SB, SM, "S", f"filter-{cls}-{ncols}", srs=GEMM_SRS[::2])
    for r in routes:
        i = r.index(f"stream-{cls}")
        assert r[i + 1] == ("filter=bloom" if plus else "filter=exact"), r
    side(f"filter-{cls}{'+1' if plus else ''}")


@pytest.mark.parametrize("delta", [-1, 0])
def test_dot_threshold(delta):
    """C<M> = A B' by row intersections when nnz(B) < 2^18, through the cached transpose at 2^18."""
    nb = 1 << 12
    lens = np.full(nb, 64)
    lens[-1] += delta
    SB = csr(lens, 4096, seed=5)
    assert SB.nnz == (1 << 18) + delta
    SA = csr(np.random.default_rng(6).integers(0, 40, 200), 4096, seed=7)
    SM = csr(np.random.default_rng(8).integers(0, 60, 200), nb, seed=9)
    routes = run_gemm(SA, SB, SM, "ST1", f"dot{delta}", srs=GEMM_SRS[:6])
    assert all((r == ["dot"]) == (delta < 0) for r in routes), routes
    side("dot-below" if delta < 0 else "dot-at")


@pytest.mark.parametrize("case", ["mask-empty", "a-empty", "b-empty"])
def test_masked_empty_operands(case):
    SA, SB, SM = uniform_masked("S", 4096)
    if case == "mask-empty":
        SM = csr([0] * SA.shape[0], SM.shape[1])
    elif case == "a-empty":
        SA = csr([0] * SA.shape[0], SA.shape[1])
    else:
        SB = csr([0] * SB.shape[0], SB.shape[1])
    routes = run_gemm(SA, SB, SM, "S", f"masked-{case}", srs=GEMM_SRS[:4], c_init=True)
    assert all(r == [] for r in routes), routes
    side(f"masked-{case}")


# ================================================================== write-back on the large paths
WB_VARIANTS = {
    # name: (descriptor, accumulator, C starts with entries, mask: None / 'struct' / a valued type)
    "accum": ("", True, True, None),
    "masked-accum": ("S", True, True, "struct"),
    "replace": ("RS", False, True, "struct"),
    "complement": ("SC", False, True, "struct"),
    "complement-replace": ("RSC", True, True, "struct"),
    "valued-FP32": ("", False, True, "FP32"),
    "valued-UINT64": ("R", True, True, "UINT64"),
}
WB_GEMM_SRS = [("PLUS", "TIMES", "INT64"), ("MIN", "PLUS", "INT32"), ("PLUS", "TIMES", "FP64"), ("MAX", "MINUS", "FP32"),
               ("LOR", "LAND", "BOOL")]


def _wb_gemm_operands(path):
    if path == "spa":
        SA, SB = unmasked_operands()
        SM = csr(np.random.default_rng(1).integers(0, 300, SA.shape[0]), SB.shape[1], seed=2)
        return SA, SB, SM, ""
    if path == "dot":
        SB = csr(np.full(300, 10), 500, seed=3)
        return (csr(np.random.default_rng(4).integers(0, 20, 100), 500, seed=5), SB,
                csr(np.random.default_rng(6).integers(0, 50, 100), 300, seed=7), "T1")
    # 40 x 1000 = 40000 products per row: every row is cut into two chunks; mask rows of 400 (class S), 1000 (M) and 2100 (L)
    SA, SB = csr([40] * 12, 2000, seed=39), csr([1000] * 2000, 2200, seed=40)
    SM = mask_with_hits(SA, SB, [400] * 4 + [1000] * 4 + [2100] * 4, 2200, 41)
    cls, chunks, _, _ = masked_classes(SA, SB, SM)
    assert cls.tolist() == ["S"] * 4 + ["M"] * 4 + ["L"] * 4 and (chunks == 2).all()
    return SA, SB, SM, ""


# without a mask the stream and dot paths are not taken: the unmasked write-back with an accumulator runs on the spa path only
WB_CASES = [(p, v) for p in ("spa", "stream", "dot") for v in WB_VARIANTS if v != "accum" or p == "spa"]


@pytest.mark.parametrize("path,variant", WB_CASES)
def test_gemm_writeback(path, variant):
    """C<M> = accum(C, T) on the dense-accumulator, stream (S, M and L, split rows) and dot paths.  A complemented mask is
    computed unmasked and filtered in the write-back: on the spa path every masked variant takes the complement."""
    desc, accum, c_init, mspec = WB_VARIANTS[variant]
    SA, SB, SM, d0 = _wb_gemm_operands(path)
    use_mask = mspec is not None
    if path == "spa" and use_mask and "C" not in desc:
        desc += "C"                                     # a mask that is not complemented would select the stream kernels
    dd ="".join(sorted(set(desc + d0), key="RSCT1".index))
    routes = run_gemm(SA, SB, SM if use_mask else None, dd, f"wb-{path}-{variant}", srs=WB_GEMM_SRS, c_init=c_init,
                      accum=accum, mask_type=None if mspec in (None, "struct") else mspec)
    want = {"spa": ["spa"], "stream": ["stream-S", "stream-M", "stream-L"], "dot": ["dot"]}[path]
    if "C" in desc and path != "spa":           # computed unmasked, then filtered
        assert all(not any(k.startswith("stream") or k == "dot" for k in r) for r in routes), routes
    else:
        assert all(all(k in r for k in want) for r in routes), routes
    side(f"wb-{path}-{variant}")


@pytest.mark.parametrize("path", ["spa", "stream", "dot"])
def test_gemm_into_operand(path):
    """C = A (+).(x) A into A itself (square operands), unmasked and masked with A's own pattern."""
    if path == "spa":
        S = csr(np.r_[[2100], np.random.default_rng(1).integers(0, 30, 2999)], 3000, seed=11)
        routes = run_gemm(S, None, None, "", "alias-spa", srs=WB_GEMM_SRS, alias=True)
        assert all("spa" in r for r in routes), routes
    else:
        S = csr([200] * 50 + [20] * 2950, 3000, seed=12)             # rows 0-49: mask rows of 200, ~4600 products (class S)
        desc = "ST1" if path == "dot" else "S"
        routes = run_gemm(S, None, S, desc, f"alias-{path}", srs=WB_GEMM_SRS, alias=True)
        assert all(("dot" in r) if path == "dot" else ("stream-S" in r) for r in routes), routes
    side(f"alias-{path}")


SPMV_WB_PATHS = {"run": (lambda: run_pattern(0, natural=True), {}), "hot": (lambda: hot_pattern(1 << 16, (1 << 20) + 1), {}),
                 "tile": (lambda: tile_pattern(8, 1), {"B200GRB_SPMV_RUN": 0})}
WB_SPMV_SRS = [("PLUS", "TIMES", "INT32"), ("MIN", "PLUS", "FP32"), ("PLUS", "TIMES", "FP64"), ("MAX", "MINUS", "INT64"),
               ("LOR", "LAND", "BOOL")]


@pytest.mark.parametrize("variant", list(WB_VARIANTS))
@pytest.mark.parametrize("path", list(SPMV_WB_PATHS))
def test_spmv_writeback(path, variant):
    desc, accum, w_init, mspec = WB_VARIANTS[variant]
    build, env = SPMV_WB_PATHS[path]
    routes = run_spmv(build(), f"wb-{path}-{variant}", env, srs=WB_SPMV_SRS, mask=mspec, desc=desc, accum=accum, w_init=w_init)
    fam = {"run": "run", "hot": "run+hot", "tile": "tile"}[path]
    assert any(r.startswith(fam) for r in routes), routes
    side(f"wb-spmv-{path}-{variant}")


# ================================================================== call sequences over cached state
class Model:
    """A matrix as sorted (I, J, X) arrays: what the library's matrix must hold after each change."""

    def __init__(self, shape, I, J, X):
        self.shape = shape
        o = np.lexsort((J, I))
        self.I, self.J, self.X = np.asarray(I, np.int64)[o], np.asarray(J, np.int64)[o], np.asarray(X)[o]

    def set(self, i, j, x):
        hit = (self.I == i) & (self.J == j)
        X = self.X.copy()
        if hit.any():
            X[hit] = x
            return Model(self.shape, self.I, self.J, X)
        return Model(self.shape, np.r_[self.I, i], np.r_[self.J, j], np.r_[X, np.asarray([x], X.dtype)])

    def keep(self, sel):
        return Model(self.shape, self.I[sel], self.J[sel], self.X[sel])

    def csr(self):
        return sp.csr_matrix((self.X, self.J, np.r_[0, np.cumsum(np.bincount(self.I, minlength=self.shape[0]))]), shape=self.shape)


def _check_mxv(A, model, sr, env, label, forms=("mxv", "vxm", "T0")):
    """A must hold exactly `model`; then mxv / vxm / mxv with T0 against the oracle.  Returns the routes taken."""
    typ = sr[2]
    I, J, X = A.to_arrays()
    assert np.array_equal(I, model.I) and np.array_equal(J, model.J), f"{label}: pattern"
    assert np.array_equal(np.asarray(X).view(np.uint8), model.X.view(np.uint8)), f"{label}: values"
    S = model.csr()
    Ao = o_csr(typ, S, model.X)
    Sp = sp.csr_matrix((np.ones(S.nnz, bool), S.indices, S.indptr), shape=S.shape)
    kinds = []
    with tunables(**env):
        for form in forms:
            n_in = S.shape[0] if form != "mxv" else S.shape[1]
            n_out = S.shape[1] if form != "mxv" else S.shape[0]
            uv = values(seed_of(label, form), typ, n_in, pool_of(sr), 1)
            u = Vector.from_numpy(uv, typ=util.g_type(typ))
            uo = orc.SpVec(typ, n_in, np.arange(n_in), uv)
            if form == "mxv":
                w = A.mxv(u, semiring=semiring(*sr))
                ref = orc.mxv(orc.SpVec(ztype(sr), n_out), None, None, sr, Ao, uo, "")
            elif form == "vxm":
                w = u.vxm(A, semiring=semiring(*sr))
                ref = orc.vxm(orc.SpVec(ztype(sr), n_out), None, None, sr, uo, Ao, "")
            else:
                w = A.mxv(u, semiring=semiring(*sr), desc=descriptor.T0)
                ref = orc.mxv(orc.SpVec(ztype(sr), n_out), None, None, sr, Ao, uo, "T0")
            ks = _kernels()
            want = spmv_route(Sp, sr, form != "mxv", env)       # T0 pulls along A' as vxm does; SEQ_SRS multiply commutatively
            assert entries(ks) == [want], (label, form, ks, want)
            kinds.append(want)
            gI, gX = w.to_arrays()
            e = compare(gI, gX, ref.I, ref.X, ztype(sr), sr[0], f"{label} {form}")
            assert e is None, e
    forget(Sp)
    return kinds


SEQ_PATHS = {"tile": (lambda: tile_pattern(8, 0), {"B200GRB_SPMV_RUN": 0}),
             "run": (lambda: run_pattern(1, natural=True), {}),
             "hot": (lambda: hot_pattern(1 << 16, (1 << 20) + 1), {})}
SEQ_SRS = [("PLUS", "TIMES", "INT64"), ("MAX", "TIMES", "INT32"), ("PLUS", "TIMES", "FP32"), ("LOR", "LAND", "BOOL")]


@pytest.mark.parametrize("path", list(SEQ_PATHS))
def test_plans_dropped_when_matrix_changes(path):
    """Build the plans (and A' for vxm / T0) with a first round of calls, then change A and run them again:
    setElement (a new entry in an empty row, and an existing entry), GrB_Matrix_assign of a block, A as the output of
    select, GrB_transpose and mxm, and GrB_Matrix_clear followed by a rebuild through GrB_Matrix_assign."""
    build, env = SEQ_PATHS[path]
    S0 = build().copy()
    n = max(S0.shape)
    S0.resize((n, n))                                   # square: A can be its own transpose's output
    rows0 = np.repeat(np.arange(n), np.diff(S0.indptr))
    empty_row = int(np.flatnonzero(np.diff(S0.indptr) == 0)[0])
    for sr in SEQ_SRS:
        typ = sr[2]
        dt = orc.DTYPES[typ]
        gt = util.g_type(typ)
        vals = values(seed_of(path, sr), typ, S0.nnz, pool_of(sr), 0)
        model = Model((n, n), rows0, S0.indices, vals)
        A = Matrix.from_csr(S0.indptr, S0.indices, vals, n, n, gt)
        label = f"seq-{path}-{'_'.join(sr)}"
        first = _check_mxv(A, model, sr, env, label + " built")
        x = dt(3) if typ != "BOOL" else True
        A[empty_row, n - 1] = x
        model = model.set(empty_row, n - 1, x)
        A[int(model.I[0]), int(model.J[0])] = x
        model = model.set(int(model.I[0]), int(model.J[0]), x)
        _check_mxv(A, model, sr, env, label + " setElement")
        # C(1:2, 1:2) = [[., x], [x, .]]: the block's entries replace the region's
        blk = Matrix.from_lists([0, 1], [1, 0], [x, x], 2, 2, gt)
        idx = ffi.new("GrB_Index[]", [1, 2])
        assert lib.GrB_Matrix_assign(A._matrix[0], ffi.NULL, ffi.NULL, blk._matrix[0], idx, 2, idx, 2, ffi.NULL) == lib.GrB_SUCCESS
        model = model.keep(~(np.isin(model.I, [1, 2]) & np.isin(model.J, [1, 2]))).set(1, 2, x).set(2, 1, x)
        _check_mxv(A, model, sr, env, label + " assign")
        A.select(lib.GxB_TRIL, out=A)
        model = model.keep(model.J <= model.I)
        _check_mxv(A, model, sr, env, label + " select")
        A.transpose(out=A)
        model = Model((n, n), model.J, model.I, model.X)
        _check_mxv(A, model, sr, env, label + " transpose")
        # A = A (+).(first) I: the same content, written by a product
        Iden = Matrix.from_lists(np.arange(n), np.arange(n), np.ones(n, dt), n, n, gt)
        A.mxm(Iden, semiring=semiring("LOR" if typ == "BOOL" else "ANY", "FIRST", typ), out=A)
        _check_mxv(A, model, sr, env, label + " mxm")
        A.clear()
        _check_mxv(A, Model((n, n), [], [], np.zeros(0, dt)), sr, env, label + " cleared", forms=("mxv",))
        B = Matrix.from_csr(S0.indptr, S0.indices, vals, n, n, gt)
        assert lib.GrB_Matrix_assign(A._matrix[0], ffi.NULL, ffi.NULL, B._matrix[0], lib.GrB_ALL, n, lib.GrB_ALL, n, ffi.NULL) == lib.GrB_SUCCESS
        again = _check_mxv(A, Model((n, n), rows0, S0.indices, vals), sr, env, label + " rebuilt")
        assert again == first, (again, first)
    side(f"seq-{path}")


def test_alternating_semirings_rebuild_tile_plan():
    """Specialised (4 items) and run-time-operator (8 items) semirings alternate on one matrix: the tile plan is rebuilt
    for every call."""
    S = tile_pattern(4, 1)
    env = {"B200GRB_SPMV_RUN": 0, "B200GRB_SPMV_ITEMS": 4}
    srs = [("PLUS", "TIMES", "INT32"), ("MAX", "TIMES", "INT32")] * 3 + [("PLUS", "TIMES", "FP64"), ("MAX", "MINUS", "FP64")] * 2
    routes = run_spmv(S, "alternate", env, srs=srs, forms=("mxv",))
    assert routes == {"tile (specialised, 4 items)", "tile (run-time operators)"}, routes
    side("seq-alternate")


def test_workspace_reuse_wide_narrow_wide():
    """Stream class L on a wide matrix (the column -> position maps of WS_SPA_SLOT at ncols per CTA), then a narrow
    one, then the wide one again: the maps are reused without being set to -1 again.  Then a call that grows every
    workspace between two that do not."""
    wide, narrow = uniform_masked("L", (1 << 20) + 1), uniform_masked("L", 5000)
    seq = [("wide", wide), ("narrow", narrow), ("wide-again", wide)]
    SA, SB, SM = narrow
    big = (stack(*[SA] * 8), SB, stack(*[SM] * 8))                  # eight times the chunks: more CTAs, larger workspaces
    seq += [("grown", big), ("narrow-again", narrow)]
    for name, (SA, SB, SM) in seq:
        routes = run_gemm(SA, SB, SM, "S", f"ws-{name}", srs=GEMM_SRS[:5])
        assert all("stream-L" in r for r in routes), routes
    side("seq-workspace")


@pytest.mark.parametrize("inplace", [0, 1, 2])
def test_mxv_in_place_sequences(inplace):
    """A.mxv(u, out=w) repeated; then w as u, as the mask of the next call, and with an accumulator."""
    S = run_pattern(0, natural=True)
    n = S.shape[0]
    Ssq = csr(np.diff(S.indptr), n, seed=99)              # square: w can be the next u
    for sr in [("PLUS", "TIMES", "INT64"), ("MIN", "PLUS", "FP32"), ("LOR", "LAND", "BOOL")]:
        typ = sr[2]
        av = values(1, typ, Ssq.nnz, pool_of(sr), 0)
        A = Matrix.from_csr(Ssq.indptr, Ssq.indices, av, n, n, util.g_type(typ))
        Ao = o_csr(typ, Ssq, av)
        uv = values(2, typ, n, pool_of(sr), 1)
        u = Vector.from_numpy(uv, typ=util.g_type(typ))
        uo = orc.SpVec(typ, n, np.arange(n), uv)
        w = Vector.sparse(util.g_type(typ), n)
        took = []
        with tunables(B200GRB_MXV_INPLACE=inplace):
            for step in range(3):
                A.mxv(u, semiring=semiring(*sr), out=w)
                took.append("mxv=in-place" in _kernels())
                ref = orc.mxv(orc.SpVec(typ, n), None, None, sr, Ao, uo, "")
                e = compare(*w.to_arrays(), ref.I, ref.X, typ, sr[0], f"inplace{inplace} step{step}")
                assert e is None, e
            wo = ref
            # w as u of the next call, then as its mask, then with an accumulator
            w2 = Vector.sparse(util.g_type(typ), n)
            A.mxv(w, semiring=semiring(*sr), out=w2)
            ref2 = orc.mxv(orc.SpVec(typ, n), None, None, sr, Ao, wo, "")
            assert compare(*w2.to_arrays(), ref2.I, ref2.X, typ, sr[0], "w as u") is None
            A.mxv(u, semiring=semiring(*sr), out=w2, mask=w)
            ref3 = orc.mxv(ref2, wo, None, sr, Ao, uo, "")
            assert compare(*w2.to_arrays(), ref3.I, ref3.X, typ, sr[0], "w as mask") is None
            acc = ("PLUS" if typ != "BOOL" else "LOR", typ) if sr[0] != "MIN" else ("MIN", typ)
            A.mxv(u, semiring=semiring(*sr), out=w, accum=util.g_accum(acc))
            ref4 = orc.mxv(wo, None, acc, sr, Ao, uo, "")
            assert compare(*w.to_arrays(), ref4.I, ref4.X, typ, sr[0], "w with accum") is None
            A.mxv(u, semiring=semiring(*sr), out=w)
            took.append("mxv=in-place" in _kernels())
            assert compare(*w.to_arrays(), ref.I, ref.X, typ, sr[0], "after accum") is None
        # the first call forms T in fresh buffers (w has none yet); the repeated ones reuse w's when the switch allows
        assert not took[0] and took[1] == took[2] == (inplace > 0), (inplace, took)
    side(f"seq-inplace-{inplace}")


# ------------------------------------------------------------------ every entry, variant and boundary side was reached
ALL_ENTRIES = {"tile (specialised, 4 items)", "tile (specialised, 8 items)", "tile (specialised, 16 items)", "tile (run-time operators)",
               "run", "run (sparse u)", "run+hot-table (TMA-staged)", "run+hot-table (TMA-staged, pipelined)", "pull", "push",
               "esc-small", "esc-medium", "hash-small", "hash-medium", "spa", "masked-warp", "stream-S", "stream-M", "stream-L", "dot",
               "filter=exact", "filter=bloom", "mxv=in-place"}
ALL_SIDES = (
    {f"tile-{i}-nnz{t:+d}" for i in (4, 8, 16) for t in (-1, 0, 1)} | {"tile-nrows=1", "tile-ncols=1", "tile-last-entry"}
    | {f"run-nnz{t:+d}" for t in (-1, 0, 1)} | {"run-threshold-below", "run-threshold-at"}
    | {f"hot-{c}" for c in HOT_CASES} | {f"push-{k}" for k in ("edges-at", "edges-over", "count-at", "count-over")}
    | {f"pull-{m}" for m in PULL_MASKS}
    | {"unmasked-bins-esc1", "unmasked-bins-esc0"} | {f"spa-ncols-{n}" for n in (1, 31, 32, 33, 4097)}
    | {f"masked-{s}" for s in ("warp-limit", "mask-128-129", "mask-512-513", "mask-2048-2049", "chunks-1-2", "chunks-3-4",
                               "a-batch-256", "a-batch-1024", "long-b-rows", "b-past-end", "blk7", "blk12", "mask-empty", "a-empty",
                               "b-empty")}
    | {f"filter-{c}{p}" for c in "SML" for p in ("", "+1")} | {"dot-below", "dot-at"}
    | {f"wb-{p}-{v}" for p, v in WB_CASES} | {f"alias-{p}" for p in ("spa", "stream", "dot")}
    | {f"wb-spmv-{p}-{v}" for p in SPMV_WB_PATHS for v in WB_VARIANTS}
    | {f"seq-{p}" for p in SEQ_PATHS} | {"seq-alternate", "seq-workspace"} | {f"seq-inplace-{i}" for i in (0, 1, 2)}
)


def _full_count(module):
    """The number of cases in the module: every test function times its parametrisations."""
    n = 0
    for name, f in vars(module).items():
        if name.startswith("test_") and callable(f) and name != "test_every_entry_and_side_was_reached":
            k = 1
            for m in getattr(f, "pytestmark", []):
                if m.name == "parametrize":
                    k *= len(m.args[1])
            n += k
    return n


def test_every_entry_and_side_was_reached(request):
    mine = [it for it in request.session.items if it.module is request.module and it is not request.node]
    if len(mine) < _full_count(request.module):
        pytest.skip("only part of the module was selected")
    missing = ALL_ENTRIES - REACHED
    assert not missing, f"kernel entries or variants no case reached: {sorted(missing)}"
    unclaimed = ALL_SIDES - SIDES
    assert not unclaimed, f"boundary sides no case verified: {sorted(unclaimed)}"
