"""The wide route of mxm with a dense-form operand: SpMM (A (+).(x) X), the dense left operand (X (+).(x) A) and SDDMM under a
sparse mask (X (+).(x) Y' under M), on matrices with 2^32 or more entries.

Such a matrix has no 32-bit row offsets; the SpMM kernels then read the 64-bit ones, and SDDMM takes its mask in chunks of
entries.  B200_debug_wide(chunk) puts every matrix on that route, so the first part runs each case twice at small sizes --
narrow, then wide on fresh operands -- and requires the same route (plus the `offsets=64` token after the kernel entry), the
same bits and presence, and one agreement with the oracle.  The second part builds a real matrix of 2^32 + 2^26 entries on the
device as kron(G, J) and checks the three routes against identities on the small factors, in UINT8 arithmetic (mod 256); it
skips, with the reason, when the card lacks the free memory."""
import numpy as np
import pytest

import pygraphblas_b200 as gb
from pygraphblas_b200 import Matrix, Vector, descriptor
from oracle import oracle as orc
import kernel_check as kc
import util
from test_dense_gpu import SEG, check, dense_x, g_csr, g_dense, o_dense, rand_csr
from test_wide_offsets_gpu import GB_, NG, NJ, NNZ, NNZ_G, NNZ_J, Memory, factor, kron, wide

pytestmark = pytest.mark.gpu

ENTRIES = ("spmm-fast", "spmm-generic", "sddmm-fast", "sddmm-generic")


def _call(run):
    C, t = run()
    I, J, X = C.to_arrays()
    return I, J, X, t


def twice(run, chunk=7):
    """run() builds fresh operands, makes one mxm and returns (C, tokens); it runs narrow, then wide.  Returns the wide C's
    tuples and the narrow tokens."""
    nI, nJ, nX, nt = _call(run)
    with wide(chunk):
        gI, gJ, gX, gt = _call(run)
    assert "offsets=64" not in nt, nt
    at = next(i for i, k in enumerate(nt) if k in ENTRIES) + 1
    assert gt == nt[:at] + ["offsets=64"] + nt[at:], (nt, gt)
    assert np.array_equal(nI, gI) and np.array_equal(nJ, gJ)
    assert np.array_equal(kc._bits(nX), kc._bits(gX))
    return (gI, gJ, gX), nt


def agree(tuples, want, add, label):
    I, J, X = tuples
    wI = np.asarray(want.I, np.int64) * want.ncols + np.asarray(want.J, np.int64)
    msg = kc.compare(np.asarray(I, np.int64) * want.ncols + np.asarray(J, np.int64), X, wI, np.asarray(want.X), want.type, add, label)
    assert msg is None, msg


# ------------------------------------------------------------------ SpMM: A (+).(x) X
LENS = [0, 1, 0, SEG - 1, SEG, SEG + 1, 2 * SEG, 2 * SEG + 1, 0, 0, 3 * SEG - 1, 17, 700]   # both sides of SPMM_SEG, empty rows

# (name, semiring, A's type, X's type, fast)
SPMM = [("fast", ("PLUS", "TIMES", "INT64"), None, None, True),
        ("fast-fp", ("PLUS", "TIMES", "FP32"), None, None, True),
        ("fast-minplus", ("MIN", "PLUS", "UINT32"), None, None, True),
        ("bool", ("LOR", "LAND", "BOOL"), None, None, True),
        ("generic", ("MAX", "MINUS", "INT16"), None, None, False),
        ("cast", ("PLUS", "TIMES", "FP64"), "INT8", "FP32", True)]


@pytest.mark.parametrize("k", [1, 8, 33])
@pytest.mark.parametrize("case", SPMM, ids=[c[0] for c in SPMM])
def test_spmm(case, k):
    name, sr, atyp, xtyp, fast = case
    add, mul, typ = sr
    atyp, xtyp = atyp or typ, xtyp or typ
    n = 800
    rng = np.random.default_rng(kc.seed_of("wide-spmm", name, k))
    S = rand_csr(rng, atyp, len(LENS), n, None, lens=LENS)
    x, pres = dense_x(rng, xtyp, n, k, 0.8)
    if atyp in util.FP_T:
        S.data = kc.values(kc.seed_of("wide-spmm-a", name), atyp, S.nnz, kc.fp_pool_for(add, mul), 0)
    if xtyp in util.FP_T:
        x = kc.values(kc.seed_of("wide-spmm-x", name, k), xtyp, n * k, kc.fp_pool_for(add, mul), 1).reshape(n, k)

    def run():
        C = Matrix.sparse(util.g_type(sr[2]), len(LENS), k)
        g_csr(atyp, S).mxm(g_dense(xtyp, x, pres), semiring=kc.semiring(*sr), out=C)
        return C, kc.last_kernel().split(";")

    got, t = twice(run)
    assert ("spmm-fast" if fast else "spmm-generic") in t and "spmm-split" in t and "write=dense" in t, t
    want = orc.mxm(orc.SpMat(sr[2], len(LENS), k), None, None, sr, kc.o_csr(atyp, S, S.data), o_dense(xtyp, x, pres))
    agree(got, want, add, f"{name} k={k}")


def test_spmm_t0():
    rng = np.random.default_rng(21)
    S = rand_csr(rng, "FP64", len(LENS), 800, None, lens=LENS).T.tocsr()      # A, whose cached transpose has the rows of LENS
    S.sort_indices()
    x, pres = dense_x(rng, "FP64", S.shape[0], 8, 0.7)
    sr = ("PLUS", "TIMES", "FP64")

    def run():
        C = Matrix.sparse(gb.FP64, S.shape[1], 8)
        g_csr("FP64", S).mxm(g_dense("FP64", x, pres), semiring=gb.FP64.PLUS_TIMES, out=C, desc=descriptor.T0)
        return C, kc.last_kernel().split(";")

    got, t = twice(run)
    assert "spmm-fast" in t and "write=dense" in t, t
    want = orc.mxm(orc.SpMat("FP64", S.shape[1], 8), None, None, sr, kc.o_csr("FP64", S, S.data), o_dense("FP64", x, pres), "T0")
    agree(got, want, "PLUS", "T0")


@pytest.mark.parametrize("mask_kind", ["none", "csr"])
def test_spmm_accum_into_nonempty_c(mask_kind):
    rng = np.random.default_rng(kc.seed_of("wide-spmm-accum", mask_kind))
    m, n, k = len(LENS), 800, 6
    S = rand_csr(rng, "INT32", m, n, None, lens=LENS)
    x, pres = dense_x(rng, "INT32", n, k, 0.8)
    cx, cp = dense_x(rng, "INT64", m, k, 0.5)
    mp = (rng.random((m, k)) < 0.6).astype(np.uint8)
    mx = (rng.random((m, k)) < 0.5).astype(np.float32)
    sr, accum = ("PLUS", "TIMES", "INT32"), ("PLUS", "INT64")

    def run():
        I, J = np.nonzero(cp)
        C = Matrix.from_lists(I, J, cx[I, J], m, k, gb.INT64)
        M = None
        if mask_kind == "csr":
            I, J = np.nonzero(mp)
            M = Matrix.from_lists(I, J, mx[I, J], m, k, gb.FP32)
        g_csr("INT32", S).mxm(g_dense("INT32", x, pres), semiring=gb.INT32.PLUS_TIMES, out=C, mask=M, accum=util.g_accum(accum))
        return C, kc.last_kernel().split(";")

    got, t = twice(run)
    assert f"write={'csr' if mask_kind == 'csr' else 'dense'}" in t, t
    o_mask = o_dense("FP32", mx, mp) if mask_kind == "csr" else None
    want = orc.mxm(o_dense("INT64", cx, cp), o_mask, accum, sr, kc.o_csr("INT32", S, S.data), o_dense("INT32", x, pres))
    agree(got, want, "PLUS", mask_kind)


# ------------------------------------------------------------------ the dense left operand: X (+).(x) op(B)
# (name, desc, k, semiring, x-transpose, t-transpose)
LEFT = [("plain", None, 8, ("PLUS", "TIMES", "INT64"), True, True),
        ("k1", None, 1, ("MIN", "PLUS", "FP64"), False, True),
        ("k33", None, 33, ("MAX", "MINUS", "INT16"), True, True),
        ("T0", "T0", 8, ("PLUS", "SECOND", "FP32"), False, True),
        ("T1", "T1", 8, ("LOR", "LAND", "BOOL"), True, True),
        ("T0T1", "T0T1", 5, ("PLUS", "FIRST", "UINT32"), False, True)]


@pytest.mark.parametrize("case", LEFT, ids=[c[0] for c in LEFT])
def test_left(case):
    name, desc, k, sr, xtr, ttr = case
    add, mul, typ = sr
    rng = np.random.default_rng(kc.seed_of("wide-left", name))
    n, cols = 800, len(LENS)
    Bt = rand_csr(rng, typ, cols, n, None, lens=LENS)           # op(B)', the operand of the kernel: the rows of LENS
    if typ in util.FP_T:
        Bt.data = kc.values(kc.seed_of("wide-left-b", name), typ, Bt.nnz, kc.fp_pool_for(add, mul), 1)
    B = Bt if "T1" in (desc or "") else Bt.T.tocsr()              # op(B) = Bt' is n x cols
    B.sort_indices()
    x, pres = dense_x(rng, typ, n, k, 0.75) if "T0" in (desc or "") else dense_x(rng, typ, k, n, 0.75)
    if typ in util.FP_T:
        x = kc.values(kc.seed_of("wide-left-x", name), typ, x.size, kc.fp_pool_for(add, mul), 0).reshape(x.shape)

    def run():
        C = Matrix.sparse(util.g_type(typ), k, cols)
        g_dense(typ, x, pres).mxm(g_csr(typ, B), semiring=kc.semiring(*sr), out=C, desc=getattr(descriptor, desc) if desc else None)
        return C, kc.last_kernel().split(";")

    got, t = twice(run)
    assert "spmm-left" in t and ("x-transpose" in t) == xtr and ("t-transpose" in t) == ttr, t
    want = orc.mxm(orc.SpMat(typ, k, cols), None, None, sr, o_dense(typ, x, pres), kc.o_csr(typ, B, B.data), desc or "")
    agree(got, want, add, name)


# ------------------------------------------------------------------ SDDMM: X (+).(x) Y' under a sparse mask, in chunks of the mask
# chunk edges of 7 fall mid-row, on row starts and next to empty rows; 256 and one chunk larger than nnz(M) too
MLENS = [0, 7, 0, 0, 3, 4, 10, 0, 1, 13, 0, 0, 5, 2, 30, 0, 1, 6, 0, 9]

# (name, semiring, mask type, X presence, Y presence, accumulate, pattern)
SDDMM = [("mask", ("PLUS", "TIMES", "INT64"), "BOOL", None, None, False, "mask"),
         ("mask-generic", ("MAX", "MINUS", "INT16"), "BOOL", None, None, False, "mask"),
         ("mask-bool", ("LOR", "LAND", "BOOL"), "BOOL", None, None, False, "mask"),
         ("valued-mask", ("PLUS", "TIMES", "INT32"), "FP32", None, None, False, "compact"),
         ("x-pres", ("MIN", "PLUS", "UINT32"), "BOOL", 0.7, None, False, "compact"),
         ("y-pres", ("PLUS", "TIMES", "UINT8"), "BOOL", None, 0.6, False, "compact"),
         ("accum", ("PLUS", "TIMES", "INT32"), "BOOL", None, None, True, "mask")]


@pytest.mark.parametrize("chunk", [1, 7, 256, 1 << 30])
@pytest.mark.parametrize("d", [1, 33, 130])
@pytest.mark.parametrize("case", SDDMM, ids=[c[0] for c in SDDMM])
def test_sddmm(case, d, chunk):
    name, sr, mtyp, xdens, ydens, acc, pattern = case
    add, mul, typ = sr
    rng = np.random.default_rng(kc.seed_of("wide-sddmm", name, d))
    m, n = len(MLENS), 40
    S = rand_csr(rng, mtyp, m, n, None, lens=MLENS)
    if mtyp != "BOOL":
        S.data[rng.random(S.nnz) < 0.4] = 0                   # entries a valued mask switches off
    x, xp = dense_x(rng, typ, m, d, xdens)
    y, yp = dense_x(rng, typ, n, d, ydens)
    desc = "T1" if mtyp != "BOOL" else "ST1"
    cx, cp = dense_x(rng, typ, m, n, 0.5)
    accum = (add, typ) if acc else None

    def run():
        if acc:
            I, J = np.nonzero(cp)
            C = Matrix.from_lists(I, J, cx[I, J], m, n, util.g_type(typ))
        else:
            C = Matrix.sparse(util.g_type(typ), m, n)
        g_dense(typ, x, xp).mxm(g_dense(typ, y, yp), semiring=kc.semiring(*sr), mask=g_csr(mtyp, S), out=C,
                                accum=util.g_accum(accum), desc=getattr(descriptor, desc))
        return C, kc.last_kernel().split(";")

    got, t = twice(run, chunk)
    assert "sddmm" in t and f"pattern={pattern}" in t and "x-transpose" not in t and "y-transpose" not in t, t
    oc = o_dense(typ, cx, cp) if acc else orc.SpMat(typ, m, n)
    want = orc.mxm(oc, kc.o_csr(mtyp, S, S.data), accum, sr, o_dense(typ, x, xp), o_dense(typ, y, yp), desc)
    agree(got, want, add, f"{name} d={d} chunk={chunk}")


def test_csr_products_stay_narrow():
    """Under the switch, a CSR x CSR product still runs its 32-bit kernels: no `offsets=64` token."""
    rng = np.random.default_rng(5)
    S = rand_csr(rng, "INT64", 30, 30, 0.2)
    with wide(7):
        A = g_csr("INT64", S)
        C = A.mxm(A, semiring=gb.INT64.PLUS_TIMES)
        t = kc.last_kernel().split(";")
    assert "offsets=64" not in t and not any(k.startswith(("spmm", "sddmm")) for k in t), t
    want = orc.mxm(orc.SpMat("INT64", 30, 30), None, None, ("PLUS", "TIMES", "INT64"), kc.o_csr("INT64", S, S.data),
                   kc.o_csr("INT64", S, S.data))
    check(C, want, "PLUS", "csr x csr")


# ------------------------------------------------------------------ a real wide matrix: A = kron(G, J), nnz(A) = 2^32 + 2^26
n = NG * NJ
K_RIGHT, K_LEFT, D = 8, 8, 72                  # D > 64: two chunks of SPMM_SEG, folded by the chunk-partial tree
# A: col 4 B + value 1 B per entry.  SDDMM: T as much as A, X and Y n x D bytes, a chunk's row ids 0.5 GB; the run plan of T
# for the column checks ~0.5 B per entry.  The left route: A' as much as A, plus the transpose's scratch (~3.2 GB).
PLAN_SDDMM = NNZ * (5 + 5 + 0.5) + 2 * n * D + 1 * GB_
PLAN_LEFT = NNZ * (5 + 5) + 3.5 * GB_
PLANNED = max(PLAN_SDDMM, PLAN_LEFT)


def trim_pool(torch):
    """Hand the unused blocks of the device's stream-ordered pool back to the driver.  The library keeps freed blocks there for
    reuse, so without this the tens of GB this module freed would still read as used to the next module's free-memory check."""
    import ctypes
    gb.lib.B200_device_synchronize()
    cu = ctypes.CDLL("libcuda.so.1")
    dev, pool = ctypes.c_int(), ctypes.c_void_p()
    assert cu.cuDeviceGet(ctypes.byref(dev), torch.cuda.current_device()) == 0
    assert cu.cuDeviceGetDefaultMemPool(ctypes.byref(pool), dev) == 0
    assert cu.cuMemPoolTrimTo(pool, ctypes.c_size_t(0)) == 0


@pytest.fixture(scope="module")
def memory():
    m = Memory()
    if m.start < PLANNED + 2 * GB_:
        pytest.skip(f"needs {PLANNED / GB_:.1f} GB of free device memory for a matrix of {NNZ} entries, "
                    f"{m.start / GB_:.1f} GB free")
    yield m
    print(f"\nwide mxm: {NNZ} entries, planned peak {PLANNED / GB_:.1f} GB, observed peak {m.peak / GB_:.1f} GB "
          f"on {m.torch.cuda.get_device_name()}")
    trim_pool(m.torch)
    print(f"free after the module: {m.torch.cuda.mem_get_info()[0] / GB_:.1f} GB")


def _tokens():
    return kc.last_kernel().split(";")


def _u8(a):
    return (np.asarray(a, np.int64) % 256).astype(np.int64)


def test_real_wide_mxm(memory):
    G, J = factor(1, NG, NNZ_G), factor(2, NJ, NNZ_J)
    Gi, Ji = G.astype(np.int64), J.astype(np.int64)
    A = kron(G, J, "UINT8")
    memory.note()
    assert A.nvals == NNZ and NNZ >= (1 << 32) + (1 << 26)
    rng = np.random.default_rng(4)

    # A (+).(x) X, X's column c = u_c (x) v_c: column c of the result is (G u_c) (x) (J v_c)
    # the dense blocks are formed in uint8, whose products wrap mod 256 as the device's UINT8 arithmetic does
    U, V = rng.integers(0, 256, (NG, K_RIGHT), dtype=np.uint8), rng.integers(0, 256, (NJ, K_RIGHT), dtype=np.uint8)
    X = (U[:, None, :] * V[None, :, :]).reshape(n, K_RIGHT)
    T = A.mxm(Matrix.from_numpy(X, typ=gb.UINT8), semiring=gb.UINT8.PLUS_TIMES)
    memory.note()
    ks = _tokens()
    assert ks[:3] == ["spmm", "spmm-generic", "offsets=64"] and "write=dense" in ks, ks
    tx, tp = T.to_numpy()
    want = (_u8(Gi @ U.astype(np.int64))[:, None, :] * _u8(Ji @ V.astype(np.int64))[None, :, :]).reshape(n, K_RIGHT) % 256
    assert tp.all() and np.array_equal(tx.astype(np.int64), want)
    del T, tx, tp, X

    # X (+).(x) Y' under A (SDDMM), X(i, k) = xG[iG, k] xJ[iJ, k], Y likewise: the row sums of T, and its exact values in a few
    # columns, whose entries in the last rows of A lie past 2^32
    xG, xJ, yG, yJ = (rng.integers(0, 256, (s, D), dtype=np.uint8) for s in (NG, NJ, NG, NJ))
    Xd = Matrix.from_numpy((xG[:, None, :] * xJ[None, :, :]).reshape(n, D), typ=gb.UINT8)
    Yd = Matrix.from_numpy((yG[:, None, :] * yJ[None, :, :]).reshape(n, D), typ=gb.UINT8)
    T = Matrix.sparse(gb.UINT8, n, n)
    Xd.mxm(Yd, semiring=gb.UINT8.PLUS_TIMES, mask=A, out=T, desc=descriptor.ST1)
    memory.note()
    ks = _tokens()
    assert ks[:2] == ["sddmm", "sddmm-generic"] and ks[2] == "offsets=64" and "pattern=mask" in ks, ks
    assert T.nvals == NNZ
    del Xd, Yd
    r = T.reduce_vector(gb.UINT8.PLUS_MONOID)
    memory.note()
    sG = _u8(G.astype(bool).astype(np.int64) @ yG.astype(np.int64))       # per row of G, per k: sum of yG over the row's columns
    sJ = _u8(J.astype(bool).astype(np.int64) @ yJ.astype(np.int64))
    lhs, rhs = _u8(xG * sG).astype(np.float64), _u8(xJ * sJ).astype(np.float64)
    want = _u8(np.rint(lhs @ rhs.T)).ravel()                   # exact: every sum < 2^53
    I, Xr = r.to_arrays()
    assert np.array_equal(I, np.arange(n)) and np.array_equal(Xr.astype(np.int64), want)
    del r
    rpG, rpJ, dG = G.indptr.astype(np.int64), J.indptr.astype(np.int64), np.diff(G.indptr).astype(np.int64)
    # two columns of G's last rows (their entries in A's last rows lie past 2^32), and one from the middle
    for jG, jJ in ((G[NG - 1].indices[0], NJ - 1), (G[NG - 2].indices[-1], 17), (NG // 2, NJ - 3)):
        j = jG * NJ + jJ
        w = T.mxv(Vector.from_lists([j], [1], n, gb.UINT8), semiring=gb.UINT8.PLUS_TIMES)
        memory.note()
        assert _tokens()[1] == "offsets=64", _tokens()
        iG, iJ = G.T.tocsr()[jG].indices, J.T.tocsr()[jJ].indices
        rows = (iG[:, None] * NJ + iJ[None, :]).ravel()
        first = (rpG[iG][:, None] * NNZ_J + dG[iG][:, None] * rpJ[iJ][None, :]).ravel()     # A's offset of row i's first entry
        vals = _u8((xG[iG][:, None, :] * xJ[iJ][None, :, :] * yG[jG] * yJ[jJ]).sum(axis=2, dtype=np.int64)).ravel()
        order = np.argsort(rows)
        I, Xw = w.to_arrays()
        assert np.array_equal(I, rows[order]) and np.array_equal(Xw.astype(np.int64), vals[order]), (jG, jJ)
        if jG != NG // 2:
            assert (first >= 1 << 32).any()
    del T, w
    memory.note()

    # X (+).(x) A, X's row c = u_c (x) v_c: row c of the result is (u_c' G) (x) (v_c' J); runs on the chunked transpose of A
    U, V = rng.integers(0, 256, (K_LEFT, NG), dtype=np.uint8), rng.integers(0, 256, (K_LEFT, NJ), dtype=np.uint8)
    X = (U[:, :, None] * V[:, None, :]).reshape(K_LEFT, n)
    T = Matrix.from_numpy(X, typ=gb.UINT8).mxm(A, semiring=gb.UINT8.PLUS_TIMES)
    memory.note()
    ks = _tokens()
    assert ks[:4] == ["spmm", "spmm-left", "x-transpose", "spmm-generic"] and ks[4] == "offsets=64" and "t-transpose" in ks, ks
    tx, tp = T.to_numpy()
    want = (_u8((Gi.T @ U.T.astype(np.int64)).T)[:, :, None] * _u8((Ji.T @ V.T.astype(np.int64)).T)[:, None, :]).reshape(K_LEFT, n) % 256
    assert tp.all() and np.array_equal(tx.astype(np.int64), want)
    # CSR x CSR products keep refusing a wide operand
    with pytest.raises(gb.base.InvalidValue, match="2\\^32 entries are not supported"):
        A.mxm(A, semiring=gb.UINT8.PLUS_TIMES)
    del A, T, X
    memory.note()
