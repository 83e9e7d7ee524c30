"""Vectors and matrices checked against the dict model and the oracle through every change of form, and with overlapped host
copies in flight (DESIGN.md section 7).

(a) Ordering of the overlapped copies (B200_Vector_set_dense / export_dense with where = 2).  A read of a vector must wait for
    an import still running on the import stream, and an import must wait for every kernel that reads or writes the vector
    after the last recorded use.  The cases set the overlap up: a long import queued ahead on the import stream holds the
    import under test back, or a bounded sleep kernel on the library's stream holds the reader or writer back.  Nothing
    that synchronises the host runs between the import and the call it races.  DESIGN.md section 7 lists which cases show
    the race when the waits are missing.
(b) Every vector form (host tuples, pending tuples, device values with and without presence, an import or an export still
    running, a communicator view) through every entry point, each followed by a probe product against the oracle.
(c) A seeded random walk over a pool of matrices: every form (host tuples, pending tuples, device CSR, CSR with plans and a
    cached transpose, dense form, dense form with its CSR) through every operation, each step checked against the model and
    four products against the oracle.  The last test checks that the walk reached every (form, operation) pair of its table.
"""
import functools

import numpy as np
import pytest

import pygraphblas_b200 as gb
from pygraphblas_b200 import Matrix, Vector, descriptor, ffi, lib, types
from pygraphblas_b200.distributed import Comm
from oracle import oracle as orc
from oracle import vecmodel as vm
import kernel_check as kc
import util

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not gb.have_device(), reason="no CUDA device")]

NULL = ffi.NULL


# ------------------------------------------------------------------ helpers
def _torch():
    import torch
    torch.cuda.init()
    return torch


def _pinned(n, dtype):
    return _torch().empty(n, dtype=dtype).pin_memory().numpy()


def _ptr(a, ctype="void*"):
    return ffi.cast(ctype, a.ctypes.data) if a is not None else NULL


def delay(ms=4):
    """A sleep kernel of about `ms` milliseconds on the library's stream (at most a few ms: the clock is at most 2 GHz)."""
    torch = _torch()
    p = ffi.new("void**")
    assert lib.B200_get_stream(p) == 0
    s = torch.cuda.ExternalStream(int(ffi.cast("uintptr_t", p[0])))
    with torch.cuda.stream(s):
        torch.cuda._sleep(int(ms * 1_000_000))


def set_dense(v, x, p, where):
    assert lib.B200_Vector_set_dense(v._vector[0], _ptr(x), _ptr(p, "uint8_t*"), where) == 0


def export_dense(v, x, p, where):
    assert lib.B200_Vector_export_dense(v._vector[0], _ptr(x), _ptr(p, "uint8_t*"), where) == 0


def vwait(v):
    assert lib.GrB_Vector_wait(v._vector) == 0


def dense_arrays(x, p):
    """(I, X) of a dense image: the present positions and their values."""
    I = np.arange(len(x)) if p is None else np.flatnonzero(p)
    return I, x[I]


def assert_arrays(v, I, X, label):
    gI, gX = v.to_arrays()
    assert v.nvals == len(I), f"{label}: nvals {v.nvals}, want {len(I)}"
    assert np.array_equal(gI, I), f"{label}: presence differs"
    bad = np.flatnonzero(kc._bits(gX) != kc._bits(np.asarray(X, gX.dtype)))
    assert len(bad) == 0, f"{label}: {len(bad)} values differ, e.g. at {gI[bad[:4]].tolist()}: {gX[bad[:4]].tolist()} want {np.asarray(X)[bad[:4]].tolist()}"


# ------------------------------------------------------------------ (a) ordering of overlapped copies
NA = 1 << 24            # the vector whose import is held back behind the blocker
NB = 1 << 26            # the blocker: a 256 MB import queued ahead of it on the import stream (several ms on PCIe)
NW = 1 << 23            # the vector imported while a sleep holds its reader / writer back (a copy well under 4 ms)


@functools.lru_cache(maxsize=None)
def _vals(n):
    """old (positive), new (negative or -0.0: every value and every mask truth value can differ) and complementary presence."""
    rng = np.random.default_rng(n)
    old = (rng.integers(1, 8, n) / 4).astype(np.float32)
    new = -(rng.integers(0, 8, n) / 4).astype(np.float32)
    old_p = (rng.random(n) < 0.5).astype(np.uint8)
    new_pin, newp_pin = _pinned(n, _torch().float32), _pinned(n, _torch().uint8)
    new_pin[:] = new
    newp_pin[:] = 1 - old_p
    return old, old_p, new_pin, newp_pin


@functools.lru_cache(maxsize=None)
def _blocker():
    x = _pinned(NB, _torch().float32)
    x[:] = 1.0
    return Vector.from_numpy(np.zeros(NB, np.float32)), x


@functools.lru_cache(maxsize=None)
def _wide(n, rows=64, nnz=4096):
    """rows x n: mxv with it reads u (a few gathers)."""
    rng = np.random.default_rng(1)
    I, J = rng.integers(0, rows, nnz), rng.integers(0, n, nnz)
    return Matrix.from_lists(I, J, np.ones(nnz, np.float32), rows, n, types.FP32)


@functools.lru_cache(maxsize=None)
def _square(n, nnz=1 << 14):
    rng = np.random.default_rng(2)
    return Matrix.from_lists(rng.integers(0, n, nnz), rng.integers(0, n, nnz), np.ones(nnz, np.float32), n, n, types.FP32)


@functools.lru_cache(maxsize=None)
def _scratch(n):
    return _pinned(n, _torch().float32), _pinned(n, _torch().uint8)


def with_events(u):
    """An overlapped export of u, waited for: u gets the events of the overlapped copies, so that mxv records its use of u
    (the state of the vectors of an import -> mxv -> export loop)."""
    x, p = _scratch(u.size)
    export_dense(u, x, p, 2)
    vwait(u)
    return u


READS = ["nvals", "extractTuples", "extractElement", "dup", "setElement", "removeElement", "resize", "build"]


@pytest.mark.parametrize("pres", [True, False])
@pytest.mark.parametrize("read", READS)
def test_read_waits_for_an_import_in_flight(read, pres):
    """set_dense(v, where = 2) queued behind a long import, then at once a call that reads v on the compute stream: it must
    see exactly the imported data, never the old contents or a mix.  Everything the check needs is computed beforehand."""
    if read == "build" and not pres:
        pytest.skip("build needs an empty import: presence bytes all zero")
    old, old_p, new, new_p = _vals(NA)
    blocker, bx = _blocker()
    if read == "build":
        new_p = _pinned(NA, _torch().uint8)
        new_p[:] = 0
    I, X = dense_arrays(new, new_p if pres else None)
    i_in = int(I[len(I) // 2]) if len(I) else None            # present after the import (absent before it, with presence)
    i_out = int(np.flatnonzero(new_p == 0)[0]) if pres else None
    want_p = (new_p != 0) if pres else np.ones(NA, bool)
    if read == "setElement":
        j = i_out if pres else 3
        I = np.sort(np.append(I, j)) if pres else I
        X = new[I].copy()
        X[np.searchsorted(I, j)] = 5.0
    elif read == "removeElement":
        I = I[I != i_in]
        X = new[I]
    elif read == "resize":
        m = NA - 1000
        I = I[I < m]
        X = new[I]
    bi = np.array([7, 2, 7], np.uint64)
    bv = np.array([1.0, 2.0, 3.0], np.float32)
    v = Vector.from_numpy(old, old_p if pres else None)
    lib.B200_device_synchronize()
    set_dense(blocker, bx, None, 2)
    set_dense(v, new, new_p if pres else None, 2)
    label = f"{read} after an import in flight"
    if read == "nvals":
        got = v.nvals
        assert got == len(I), f"{label}: {got}, want {len(I)}"
    elif read == "extractTuples":
        assert_arrays(v, I, X, label)
    elif read == "extractElement":
        got = v.get(i_in)
        assert got is not None and np.float32(got) == new[i_in] and np.signbit(np.float32(got)) == np.signbit(new[i_in]), label
        if pres:
            assert v.get(i_out) is None, label
    elif read == "dup":
        d = v.dup()
        x, p = d.to_numpy()
        assert np.array_equal(p != 0, want_p), label
        assert np.array_equal(kc._bits(x[I]), kc._bits(X)), label
    elif read == "setElement":
        v[j] = 5.0
        assert_arrays(v, I, X, label)
    elif read == "removeElement":
        del v[i_in]
        assert_arrays(v, I, X, label)
    elif read == "resize":
        assert lib.GrB_Vector_resize(v._vector[0], m) == 0
        assert_arrays(v, I, X, label)
    elif read == "build":
        r = lib.GrB_Vector_build_FP32(v._vector[0], _ptr(bi, "GrB_Index*"), _ptr(bv, "float*"), 3, NULL)
        assert r == 0, f"{label}: build into a vector the import emptied returned {r}"
        assert_arrays(v, np.array([2, 7]), np.array([2.0, 3.0], np.float32), label)
    lib.B200_device_synchronize()


def _reader_expect(reader, old, p):
    I, X = dense_arrays(old, p)
    if reader == "eWiseAdd":
        return I, X
    if reader == "apply":
        return I, -X
    return I[X != 0], np.ones(int((X != 0).sum()), np.float32)       # mask


@pytest.mark.parametrize("export", [False, True])
@pytest.mark.parametrize("pres", [True, False])
@pytest.mark.parametrize("reader", ["eWiseAdd", "apply", "mask"])
def test_import_waits_for_a_reader_after_mxv(reader, pres, export):
    """mxv reads u (its use is recorded), a sleep holds the stream, another call reads u, then an import into u: the reader
    must see the old u, and u the import once it is waited for.  No call between the sleep and the import synchronises the
    host: the other operands are already in HBM and the export buffers already pinned.  (A reduce into a host scalar is no
    case here: it returns only once the reduction is done.)"""
    old, old_p, new, new_p = _vals(NW)
    p = old_p if pres else None
    u = with_events(Vector.from_numpy(old, p))
    A = _wide(NW)
    empty = Vector.from_numpy(np.zeros(NW, np.float32), np.zeros(NW, np.uint8))
    ones = Vector.from_numpy(np.ones(NW, np.float32))
    want = _reader_expect(reader, old, p)
    ex, ep = _pinned(NW, _torch().float32), _pinned(NW, _torch().uint8)
    w = A.mxv(u, semiring=types.FP32.PLUS_TIMES)
    lib.B200_device_synchronize()
    w = A.mxv(u, semiring=types.FP32.PLUS_TIMES, out=w)
    delay()
    if reader == "eWiseAdd":
        r = u.eadd(empty, types.FP32.PLUS)
    elif reader == "apply":
        r = u.apply(types.FP32.AINV)
    else:
        r = ones.apply(types.FP32.IDENTITY, mask=u)
    if export:
        export_dense(u, ex, ep, 2)
    set_dense(u, new, new_p if pres else None, 2)
    assert_arrays(r, *want, f"{reader} of u before the import")
    vwait(u)
    if export:
        assert np.array_equal(ep, p if pres else np.ones(NW, np.uint8))
        I, X = dense_arrays(old, p)
        assert np.array_equal(kc._bits(ex[I]), kc._bits(X)), "export in flight before the import"
    assert_arrays(u, *dense_arrays(new, new_p if pres else None), "u after the import")
    lib.B200_device_synchronize()


@pytest.mark.parametrize("export", [False, True])
@pytest.mark.parametrize("pres", [True, False])
@pytest.mark.parametrize("writer", ["eWiseAdd", "apply", "mxv_in_place"])
def test_import_waits_for_a_writer_after_mxv(writer, pres, export):
    """mxv reads u, a sleep holds the stream, a call rewrites u (new buffers from the pool, or in place), then an import into
    u: once waited for, u must hold exactly the import -- the rewrite may not land on top of it."""
    old, old_p, new, new_p = _vals(NW)
    p = old_p if pres else None
    u = with_events(Vector.from_numpy(old, p))
    src = Vector.from_numpy(old * 3, p)
    empty = Vector.from_numpy(np.zeros(NW, np.float32), np.zeros(NW, np.uint8))
    ex, ep = _pinned(NW, _torch().float32), _pinned(NW, _torch().uint8)
    sr = types.FP32.PLUS_TIMES
    if writer == "mxv_in_place":
        A = _square(NW)
        w = Vector.from_numpy(old, p)
        A.mxv(u, semiring=sr, out=w)
        if pres:
            A.mxv(w, semiring=sr, out=u)         # u owns buffers with presence bytes the product can be formed in
        lib.B200_device_synchronize()
        A.mxv(u, semiring=sr, out=w)             # ping ...
        delay()
        A.mxv(w, semiring=sr, out=u)             # ... pong
        assert ("mxv=in-place" in kc.last_kernel().split(";")) == pres, kc.last_kernel()
    else:
        A = _wide(NW)
        w = A.mxv(u, semiring=sr)
        lib.B200_device_synchronize()
        A.mxv(u, semiring=sr, out=w)
        delay()
        if writer == "eWiseAdd":
            src.eadd(empty, types.FP32.PLUS, out=u)
        else:
            src.apply(types.FP32.AINV, out=u)
    if export:
        export_dense(u, ex, ep, 2)
    set_dense(u, new, new_p if pres else None, 2)
    vwait(u)
    if export and writer != "mxv_in_place":
        I, X = dense_arrays(old * 3, p)
        assert np.array_equal(ep != 0, np.ones(NW, bool) if p is None else p != 0), "export in flight before the import"
        assert np.array_equal(kc._bits(ex[I]), kc._bits(X if writer == "eWiseAdd" else -X)), "export in flight before the import"
    assert_arrays(u, *dense_arrays(new, new_p if pres else None), f"u after {writer} and the import")
    lib.B200_device_synchronize()


# ------------------------------------------------------------------ (b) vector forms x entry points
VN = 208                 # a multiple of 16: the communicator moves slices as 16-byte words
VTYPES = ["BOOL", "INT8", "INT16", "FP32", "FP64"]
VFORMS = ["host", "pending", "device", "full", "import2", "export2", "view"]
VOPS = ["set", "remove", "extractElement", "build", "build_cleared", "dup", "clear", "resize", "nvals",
        "set_dense0", "set_dense1", "set_dense2", "export0", "export1", "export2", "device_ptrs",
        "mxv_u", "mxv_w", "mxv_mask", "eWiseAdd", "apply", "assign", "extract", "reduce"]
TORCH_DT = {"BOOL": "bool", "INT8": "int8", "INT16": "int16", "FP32": "float32", "FP64": "float64"}


def sr_of(typ):
    return ("LOR", "LAND", "BOOL") if typ == "BOOL" else ("PLUS", "TIMES", typ)


def o_vec(typ, n, d):
    k = sorted(d)
    return orc.SpVec(typ, n, np.array(k, np.uint64), np.array([d[i] for i in k], orc.DTYPES[typ]))


def o_mat(typ, nrows, ncols, d):
    k = sorted(d)
    return orc.SpMat(typ, nrows, ncols, np.array([a for a, _ in k], np.uint64), np.array([b for _, b in k], np.uint64),
                     np.array([d[x] for x in k], orc.DTYPES[typ]))


def check_vec(v, d, typ, label):
    k = sorted(d)
    assert v.nvals == len(d), f"{label}: nvals {v.nvals}, model {len(d)}"
    I, X = v.to_arrays()
    msg = kc.compare(I, X, np.array(k, np.int64), np.array([d[i] for i in k], orc.DTYPES[typ]), typ, None, label)
    assert msg is None, msg


def check_vec_result(v, want, typ, label):
    I, X = v.to_arrays()
    msg = kc.compare(I, X, want.I, want.X, typ, None, label)
    assert msg is None, msg


@functools.lru_cache(maxsize=None)
def _vmat(typ, n):
    rng = np.random.default_rng(kc.seed_of("vmat", typ, n))
    m = util.rand_mat(rng, typ, n, n, 0.05)
    d = {(i, j): x for i, j, x in zip(m["I"], m["J"], np.asarray(m["X"], orc.DTYPES[typ]))}
    return util.g_mat(m), o_mat(typ, n, n, d)


def probe(v, d, typ, n, label):
    """w = A v against the oracle: the product reads whatever form v is in."""
    A, Ao = _vmat(typ, n)
    sr = sr_of(typ)
    w = A.mxv(v, semiring=util.g_semiring(sr))
    want = orc.mxv(orc.SpVec(typ, n), None, None, sr, Ao, o_vec(typ, n, d))
    check_vec_result(w, want, typ, f"{label}: probe mxv")


def rand_dict(rng, typ, n, density):
    r = util.rand_vec(rng, typ, n, density)
    return dict(zip(r["I"], np.asarray(r["X"], orc.DTYPES[typ])))


def dense_of(typ, n, d, full=False):
    x = np.zeros(n, orc.DTYPES[typ])
    p = np.zeros(n, np.uint8)
    for i, val in d.items():
        x[i], p[i] = val, 1
    return x, (None if full else p)


def make_form(form, typ, n, rng, keep):
    """A vector in the named form and its model."""
    dt = orc.DTYPES[typ]
    full = form == "full"
    d = rand_dict(rng, typ, n, 1.0 if full else 0.4)
    x, p = dense_of(typ, n, d, full)
    if form == "host":
        return Vector.from_lists(sorted(d), [d[i] for i in sorted(d)], n, util.g_type(typ)), d
    if form == "pending":
        k = sorted(d)
        base = k[: len(k) // 2]
        v = Vector.from_lists(base, [d[i] for i in base], n, util.g_type(typ))
        for i in k[len(k) // 2:] + base[:2]:                     # pending tuples, two of them over host entries
            v[i] = d[i].item()
        return v, d
    if form in ("device", "full"):
        return Vector.from_numpy(x, p, util.g_type(typ)), d
    if form == "import2":
        v = Vector.from_numpy(np.zeros(n, dt), np.ones(n, np.uint8), util.g_type(typ))
        px, pp = _pinned(n, getattr(_torch(), TORCH_DT[typ])), _pinned(n, _torch().uint8)
        px[:], pp[:] = x, p
        keep += [px, pp]
        set_dense(v, px, pp, 2)
        return v, d
    if form == "export2":
        v = Vector.from_numpy(x, p, util.g_type(typ))
        px, pp = _pinned(n, getattr(_torch(), TORCH_DT[typ])), _pinned(n, _torch().uint8)
        keep += [px, pp]
        export_dense(v, px, pp, 2)
        return v, d
    assert form == "view"
    comm = Comm(n, util.g_type(typ), rank=0, world=1)
    keep.append(comm)
    view = comm.allgather(Vector.from_numpy(x, p, util.g_type(typ)), 0)
    return view, d


def _export_check(x, p, d, typ, label):
    want_x, want_p = dense_of(typ, len(x), d)
    assert np.array_equal(p != 0, want_p != 0), f"{label}: exported presence differs"
    I = np.flatnonzero(want_p)
    assert np.array_equal(kc._bits(x[I]), kc._bits(want_x[I])), f"{label}: exported values differ"


def apply_vop(op, v, d, typ, n, rng, keep):
    """Apply one entry point to v and to its model; returns (v, d, n)."""
    torch = _torch() if op in ("set_dense1", "export1", "set_dense2", "export2") else None
    g = util.g_type(typ)
    dt = orc.DTYPES[typ]
    label = op
    if op == "set":
        for i in rng.choice(n, 3, replace=False).tolist():
            x = util.rand_values(rng, typ, 1)[0]
            v[i] = x.item()
            d[i] = x
    elif op == "remove":
        for i in (sorted(d)[:1] + [int(rng.integers(n))]):
            del v[i]
            d.pop(i, None)
    elif op == "extractElement":
        for i in (sorted(d)[-1:] + rng.choice(n, 4, replace=False).tolist()):
            got = v.get(i)
            assert (got is None) == (i not in d), f"{label} at {i}"
            if got is not None:
                assert dt(got) == d[i] or (np.isnan(dt(got)) and np.isnan(d[i])), f"{label} at {i}: {got} vs {d[i]}"
    elif op in ("build", "build_cleared"):
        if op == "build_cleared":
            v.clear()
            d = {}
        bi = rng.integers(0, n, 12).astype(np.uint64)
        bx = util.rand_values(rng, typ, 12)
        r = g._Vector_build(v._vector[0], ffi.cast("GrB_Index*", bi.ctypes.data), ffi.cast(g.ptr, bx.ctypes.data), 12, NULL)
        if d:
            assert r == lib.GrB_OUTPUT_NOT_EMPTY, f"{label}: build into a non-empty vector returned {r}"
        else:
            assert r == 0, f"{label}: {r}"
            for i, x in zip(bi.tolist(), bx):         # no dup operator: the later tuple wins
                d[i] = x
    elif op == "dup":
        c = v.dup()
        check_vec(c, d, typ, "dup: the copy")
        c.clear()
    elif op == "clear":
        v.clear()
        d = {}
    elif op == "resize":
        n = n - 16
        assert lib.GrB_Vector_resize(v._vector[0], n) == 0
        d = {i: x for i, x in d.items() if i < n}
    elif op == "nvals":
        assert v.nvals == len(d)
    elif op.startswith("set_dense"):
        where = int(op[-1])
        d = rand_dict(rng, typ, n, 0.5 if rng.random() < 0.5 else 1.0)
        x, p = dense_of(typ, n, d, full=len(d) == n)
        if where == 0:
            set_dense(v, x, p, 0)
        elif where == 1:
            tx = torch.from_numpy(x).cuda()
            tp = torch.from_numpy(p).cuda() if p is not None else None
            torch.cuda.synchronize()
            assert lib.B200_Vector_set_dense(v._vector[0], ffi.cast("void*", tx.data_ptr()),
                                             ffi.cast("uint8_t*", tp.data_ptr()) if tp is not None else NULL, 1) == 0
            keep += [tx, tp]
        else:
            px = _pinned(n, getattr(torch, TORCH_DT[typ]))
            px[:] = x
            pp = None
            if p is not None:
                pp = _pinned(n, torch.uint8)
                pp[:] = p
            keep += [px, pp]
            set_dense(v, px, pp, 2)
    elif op.startswith("export"):
        where = int(op[-1])
        if where == 0:
            x, p = v.to_numpy()
        elif where == 1:
            tx = _torch().empty(n, dtype=getattr(_torch(), TORCH_DT[typ]), device="cuda")
            tp = _torch().empty(n, dtype=_torch().uint8, device="cuda")
            assert lib.B200_Vector_export_dense(v._vector[0], ffi.cast("void*", tx.data_ptr()), ffi.cast("uint8_t*", tp.data_ptr()), 1) == 0
            lib.B200_device_synchronize()
            x, p = tx.cpu().numpy(), tp.cpu().numpy()
        else:
            x, p = _pinned(n, getattr(torch, TORCH_DT[typ])), _pinned(n, torch.uint8)
            export_dense(v, x, p, 2)
            vwait(v)
        _export_check(x, p, d, typ, label)
    elif op == "device_ptrs":
        vals, pres = v.device_ptrs()
        nd = rand_dict(rng, typ, n, 0.5 if pres else 1.0)
        x, p = dense_of(typ, n, nd, full=not pres)
        src = Vector.from_numpy(x, p, g)
        assert lib.B200_Vector_export_dense(src._vector[0], ffi.cast("void*", vals), ffi.cast("uint8_t*", pres) if pres else NULL, 1) == 0
        d = nd
    elif op == "mxv_u":
        pass                                          # the probe below is this case
    elif op in ("mxv_w", "mxv_mask"):
        A, Ao = _vmat(typ, n)
        sr = sr_of(typ)
        zd = rand_dict(rng, typ, n, 0.5)
        z = Vector.from_lists(sorted(zd), [zd[i] for i in sorted(zd)], n, g)
        if op == "mxv_w":
            A.mxv(z, semiring=util.g_semiring(sr), out=v)
            want = orc.mxv(orc.SpVec(typ, n), None, None, sr, Ao, o_vec(typ, n, zd))
            d = dict(zip(want.I.tolist(), want.X))
        else:
            r = A.mxv(z, semiring=util.g_semiring(sr), mask=v)
            want = orc.mxv(orc.SpVec(typ, n), o_vec(typ, n, d), None, sr, Ao, o_vec(typ, n, zd))
            check_vec_result(r, want, typ, "mxv with v as the mask")
    elif op == "eWiseAdd":
        zd = rand_dict(rng, typ, n, 0.5)
        z = Vector.from_numpy(*dense_of(typ, n, zd), typ=g)
        v.eadd(z, g.FIRST, out=v)
        d = {**zd, **d}
    elif op == "apply":
        v.apply(g.AINV, out=v)
        d = {i: vm.unop("AINV", typ, x) for i, x in d.items()}
    elif op == "assign":
        idx = rng.choice(n, 20, replace=False)
        zd = rand_dict(rng, typ, 20, 0.5)
        z = Vector.from_lists(sorted(zd), [zd[i] for i in sorted(zd)], 20, g)
        v.assign(z, idx.tolist())
        for k, i in enumerate(idx.tolist()):
            if k in zd:
                d[i] = zd[k]
            else:
                d.pop(i, None)
    elif op == "extract":
        idx = rng.choice(n, 20, replace=False).tolist()
        r = v.extract(idx)
        check_vec(r, {k: d[i] for k, i in enumerate(idx) if i in d}, typ, "extract")
    elif op == "reduce":
        mon = g.LOR_MONOID if typ == "BOOL" else g.MAX_MONOID
        x = ffi.new(g.ptr)
        assert g._Vector_reduce(x, NULL, mon.get_op(), v._vector[0], NULL) == 0
        ident = False if typ == "BOOL" else (-np.inf if typ in util.FP_T else np.iinfo(dt).min)
        want = vm.reduce("LOR" if typ == "BOOL" else "MAX", typ, d, ident)
        assert dt(x[0]) == want, f"reduce: {x[0]} vs {want}"
    else:
        raise AssertionError(op)
    return v, d, n


@pytest.mark.parametrize("typ", VTYPES)
@pytest.mark.parametrize("form", VFORMS)
def test_vector_form_through_every_entry_point(form, typ):
    """Each entry point on a fresh vector in the form, then the vector against the model and a probe product."""
    bad = []
    for op in VOPS:
        rng = np.random.default_rng(kc.seed_of("vform", form, typ, op))
        keep = []
        v, d = make_form(form, typ, VN, rng, keep)
        try:
            v, d, n = apply_vop(op, v, d, typ, VN, rng, keep)
            check_vec(v, d, typ, f"{form} / {op}")
            probe(v, d, typ, n, f"{form} / {op}")
        except AssertionError as e:
            bad.append(f"{form} / {op}: {e}")
        lib.B200_device_synchronize()
        del v, keep
    assert not bad, "\n".join(bad)


# ------------------------------------------------------------------ (c) matrix forms x operations: a seeded random walk
MFORMS = ["host", "pending", "csr", "csr+plans+T", "dense", "dense+csr", "as_left"]
MOPS = ["setElement", "removeElement", "build_cleared", "resize", "dup", "Matrix_assign", "Row_assign", "Col_assign",
        "extract_self", "apply_self", "select_self", "transpose_self", "eWise_into_operand", "mxm_csr", "mxm_spmm",
        "dense_round_trip", "csr_round_trip"]
MTYPES = ["FP32", "FP32", "INT32", "BOOL"]        # two of one type: binary operations between pool matrices
WALK_SEEDS = range(8)
WALK_STEPS = 60
REACHED = set()


def m_sr(typ):
    return ("LOR", "LAND", "BOOL") if typ == "BOOL" else ("MIN", "PLUS", typ)      # folds exact in any order


def m_add(typ):
    return m_sr(typ)[0]


def mat_dict(M):
    I, J, X = M.to_arrays()
    return dict(zip(zip(I.tolist(), J.tolist()), X))


def check_mat(M, d, typ, label):
    assert M.nvals == len(d), f"{label}: nvals {M.nvals}, model {len(d)}"
    I, J, X = M.to_arrays()
    k = sorted(d)
    n = M.ncols
    msg = kc.compare(I.astype(np.int64) * n + J.astype(np.int64), X, np.array([a * n + b for a, b in k], np.int64),
                     np.array([d[x] for x in k], orc.DTYPES[typ]), typ, None, label)
    assert msg is None, msg


def check_mat_result(C, want, typ, label):
    I, J, X = C.to_arrays()
    n = C.ncols
    msg = kc.compare(I.astype(np.int64) * n + J.astype(np.int64), X, want.I.astype(np.int64) * n + want.J.astype(np.int64),
                     want.X, typ, m_add(typ), label)
    assert msg is None, msg


def status(M):
    p = ffi.new("int*")
    assert lib.GxB_Matrix_Option_get(M._matrix[0], lib.GxB_SPARSITY_STATUS, p) == lib.GrB_SUCCESS
    return p[0]


def lists_of(d):
    k = sorted(d)
    return [a for a, _ in k], [b for _, b in k], [d[x] for x in k]


def dense_mat(typ, n, m, d):
    x = np.zeros((n, m), orc.DTYPES[typ])
    p = np.zeros((n, m), np.uint8)
    for (a, b), val in d.items():
        x[a, b], p[a, b] = val, 1
    return x, p


def form_matrix(form, typ, n, d, rng):
    """A matrix holding d in the named form (built through the public calls that leave it so)."""
    g = util.g_type(typ)
    sr = util.g_semiring(m_sr(typ))
    I, J, X = lists_of(d)
    if form in ("host", "pending"):
        if form == "host" or not d:
            return Matrix.from_lists(I, J, np.asarray(X, orc.DTYPES[typ]), n, n, g)
        h = len(I) // 2
        M = Matrix.from_lists(I[:h], J[:h], np.asarray(X[:h], orc.DTYPES[typ]), n, n, g)
        for a, b, x in list(zip(I, J, X))[h:] + list(zip(I, J, X))[:1]:
            M[a, b] = x.item()
        return M
    if form in ("csr", "csr+plans+T"):
        x, p = dense_mat(typ, n, n, d)
        indptr = np.concatenate(([0], np.cumsum(p.sum(1)))).astype(np.int64)
        M = Matrix.from_csr(indptr, np.asarray(J, np.uint32), np.asarray(X, orc.DTYPES[typ]), n, n, g)
        if form == "csr+plans+T":
            u = Vector.from_numpy(util.rand_values(rng, typ, n), typ=g)
            M.mxv(u, semiring=sr)
            u.vxm(M, semiring=sr)
        return M
    x, p = dense_mat(typ, n, n, d)
    M = Matrix.from_numpy(x, None if p.all() else p, g)
    if form == "dense+csr":
        M.mxv(Vector.from_numpy(util.rand_values(rng, typ, n), typ=g), semiring=sr)
    return M


def check_products(M, d, typ, n, rng, label):
    """mxv, vxm, mxv with T0 and mxm with a dense X against the oracle."""
    g = util.g_type(typ)
    srn = m_sr(typ)
    sr = util.g_semiring(srn)
    Mo = o_mat(typ, n, n, d)
    uv = util.rand_values(rng, typ, n)
    up = (rng.random(n) < 0.7).astype(np.uint8)
    u = Vector.from_numpy(uv, up, g)
    uo = o_vec(typ, n, {i: uv[i] for i in np.flatnonzero(up).tolist()})
    check_vec_result(M.mxv(u, semiring=sr), orc.mxv(orc.SpVec(typ, n), None, None, srn, Mo, uo), typ, f"{label}: mxv")
    check_vec_result(u.vxm(M, semiring=sr), orc.vxm(orc.SpVec(typ, n), None, None, srn, uo, Mo), typ, f"{label}: vxm")
    check_vec_result(M.mxv(u, semiring=sr, desc=descriptor.T0), orc.mxv(orc.SpVec(typ, n), None, None, srn, Mo, uo, "T0"),
                     typ, f"{label}: mxv T0")
    xv = util.rand_values(rng, typ, n * 3).reshape(n, 3)
    X = Matrix.from_numpy(xv, typ=g)
    Xo = orc.SpMat(typ, n, 3, np.repeat(np.arange(n), 3), np.tile(np.arange(3), n), xv.ravel())
    C = Matrix.sparse(g, n, 3)
    M.mxm(X, semiring=sr, out=C)
    check_mat_result(C, orc.mxm(orc.SpMat(typ, n, 3), None, None, srn, Mo, Xo, ""), typ, f"{label}: mxm dense X")


def apply_mop(op, M, d, O, dO, typ, n, rng):
    """One operation on M (O: another pool matrix of M's type, or M itself); returns (M, d)."""
    g = util.g_type(typ)
    dt = orc.DTYPES[typ]
    srn = m_sr(typ)
    sr = util.g_semiring(srn)
    if op == "setElement":
        for _ in range(3):
            a, b = int(rng.integers(n)), int(rng.integers(n))
            x = util.rand_values(rng, typ, 1)[0]
            M[a, b] = x.item()
            d[(a, b)] = x
    elif op == "removeElement":
        for a, b in sorted(d)[:2] + [(int(rng.integers(n)), int(rng.integers(n)))]:
            del M[a, b]
            d.pop((a, b), None)
    elif op == "build_cleared":
        M.clear()
        k = 40
        bi, bj = rng.integers(0, n, k).astype(np.uint64), rng.integers(0, 8, k).astype(np.uint64)
        bx = util.rand_values(rng, typ, k)
        assert g._Matrix_build(M._matrix[0], ffi.cast("GrB_Index*", bi.ctypes.data), ffi.cast("GrB_Index*", bj.ctypes.data),
                               ffi.cast(g.ptr, bx.ctypes.data), k, NULL) == 0
        d = {}
        for a, b, x in zip(bi.tolist(), bj.tolist(), bx):
            d[(a, b)] = x
    elif op == "resize":
        assert lib.GrB_Matrix_resize(M._matrix[0], n - 5, n + 3) == 0
        assert lib.GrB_Matrix_resize(M._matrix[0], n, n) == 0
        d = {k: x for k, x in d.items() if k[0] < n - 5}
    elif op == "dup":
        M = M.dup()
    elif op == "Matrix_assign":
        ni, nj = 6, 9
        I, J = rng.choice(n, ni, replace=False), rng.choice(n, nj, replace=False)
        keys = [(a, b) for a in range(ni) for b in range(nj)]
        sd = {key: x for key, x, keep in zip(keys, util.rand_values(rng, typ, ni * nj), rng.random(ni * nj) < 0.5) if keep}
        Si, Sj, Sx = lists_of(sd)
        S = Matrix.from_lists(Si, Sj, np.asarray(Sx, dt), ni, nj, g)
        Ia, Ja = np.asarray(I, np.uint64), np.asarray(J, np.uint64)
        assert lib.GrB_Matrix_assign(M._matrix[0], NULL, NULL, S._matrix[0], ffi.cast("GrB_Index*", Ia.ctypes.data), ni,
                                     ffi.cast("GrB_Index*", Ja.ctypes.data), nj, NULL) == 0
        for a in range(ni):
            for b in range(nj):
                if (a, b) in sd:
                    d[(int(I[a]), int(J[b]))] = sd[(a, b)]
                else:
                    d.pop((int(I[a]), int(J[b])), None)
    elif op in ("Row_assign", "Col_assign"):
        k = 12
        idx = np.asarray(rng.choice(n, k, replace=False), np.uint64)
        line = int(rng.integers(n))
        ud = rand_dict(rng, typ, k, 0.5)
        u = Vector.from_lists(sorted(ud), [ud[i] for i in sorted(ud)], k, g)
        ip = ffi.cast("GrB_Index*", idx.ctypes.data)
        if op == "Row_assign":
            assert lib.GrB_Row_assign(M._matrix[0], NULL, NULL, u._vector[0], line, ip, k, NULL) == 0
        else:
            assert lib.GrB_Col_assign(M._matrix[0], NULL, NULL, u._vector[0], ip, k, line, NULL) == 0
        for q, i in enumerate(idx.tolist()):
            key = (line, i) if op == "Row_assign" else (i, line)
            if q in ud:
                d[key] = ud[q]
            else:
                d.pop(key, None)
    elif op == "extract_self":
        I, J = rng.permutation(n).astype(np.uint64), rng.permutation(n).astype(np.uint64)
        assert lib.GrB_Matrix_extract(M._matrix[0], NULL, NULL, M._matrix[0], ffi.cast("GrB_Index*", I.ctypes.data), n,
                                      ffi.cast("GrB_Index*", J.ctypes.data), n, NULL) == 0
        ri = {int(x): a for a, x in enumerate(I)}
        rj = {int(x): b for b, x in enumerate(J)}
        d = {(ri[a], rj[b]): x for (a, b), x in d.items()}
    elif op == "apply_self":
        M.apply(g.AINV, out=M)
        d = {k: vm.unop("AINV", typ, x) for k, x in d.items()}
    elif op == "select_self":
        off = int(rng.integers(-n // 4, n // 2))
        M.select(lib.GxB_TRIL, off, out=M)
        d = {(a, b): x for (a, b), x in d.items() if b <= a + off}
    elif op == "transpose_self":
        M.transpose(out=M)
        d = {(b, a): x for (a, b), x in d.items()}
    elif op == "eWise_into_operand":
        M.eadd(O, g.FIRST, out=M)
        d = {**dO, **d}
    elif op == "mxm_csr":
        # a CSR right operand (a dense-form one would take the SpMM); a dense-form M on the left takes the batched vxm
        dense = (lib.GxB_FULL, lib.GxB_BITMAP)
        R = O if status(O) not in dense else form_matrix("csr", typ, n, dO, rng)
        left_dense = status(M) in dense
        want = orc.mxm(orc.SpMat(typ, n, n), None, None, srn, o_mat(typ, n, n, d), o_mat(typ, n, n, dO), "")
        M.mxm(R, semiring=sr, out=M)
        assert left_dense or "spmm" not in kc.last_kernel().split(";"), kc.last_kernel()
        d = dict(zip(zip(want.I.tolist(), want.J.tolist()), want.X))
    elif op == "mxm_spmm":
        xv = util.rand_values(rng, typ, n * n).reshape(n, n)
        xp = (rng.random((n, n)) < 0.02).astype(np.uint8)         # a sparse bitmap keeps the product (and the walk) small
        D = Matrix.from_numpy(xv, xp, g)
        Di, Dj = np.nonzero(xp)
        Do = orc.SpMat(typ, n, n, Di, Dj, xv[Di, Dj])
        want = orc.mxm(orc.SpMat(typ, n, n), None, None, srn, o_mat(typ, n, n, d), Do, "")
        M.mxm(D, semiring=sr, out=M)
        toks = kc.last_kernel().split(";")
        assert "spmm" in toks and "write=dense" in toks, toks
        assert status(M) in (lib.GxB_FULL, lib.GxB_BITMAP)
        d = dict(zip(zip(want.I.tolist(), want.J.tolist()), want.X))
    elif op == "dense_round_trip":
        x, p = M.to_numpy()
        M = Matrix.from_numpy(x, None if p.all() else p, g)
        assert status(M) == (lib.GxB_FULL if p.all() else lib.GxB_BITMAP)
    elif op == "csr_round_trip":
        Ap, Aj, Ax = M.to_csr()
        M = Matrix.from_csr(Ap, Aj, Ax, n, n, g)
    else:
        raise AssertionError(op)
    return M, d


def walk_plan(seed, reached):
    """(matrix, form, op) for each step: the least reached (form, op) pair first, ties broken by the seed."""
    rng = np.random.default_rng(1000 + seed)
    steps = []
    for _ in range(WALK_STEPS):
        low = min(reached.values())
        cand = [k for k, c in reached.items() if c == low]
        f, o = cand[int(rng.integers(len(cand)))]
        steps.append((int(rng.integers(len(MTYPES))), f, o))
        reached[(f, o)] += 1
    return steps


@functools.lru_cache(maxsize=None)
def _plans():
    reached = {(f, o): 0 for f in MFORMS for o in MOPS}
    return {s: walk_plan(s, reached) for s in WALK_SEEDS}


@pytest.mark.parametrize("seed", WALK_SEEDS)
def test_matrix_state_walk(seed):
    """Pool of four square matrices of mixed types (one dense enough for the run kernels of mxv).  Each step puts the chosen
    matrix into the step's form -- "as_left" keeps whatever the previous steps and their checks left -- applies the
    operation, and checks the matrix against its model and four products against the oracle."""
    rng = np.random.default_rng(seed)
    n = 120 + 10 * seed
    pool = []
    for k, typ in enumerate(MTYPES):
        m = util.rand_mat(rng, typ, n, n, 0.3 if k == 0 else 0.03)
        d = dict(zip(zip(m["I"], m["J"]), np.asarray(m["X"], orc.DTYPES[typ])))
        pool.append([form_matrix("host", typ, n, d, rng), d, typ])
    for step, (k, form, op) in enumerate(_plans()[seed]):
        M, d, typ = pool[k]
        label = f"seed {seed} step {step}: {op} on {typ} matrix {k} as {form}"
        if form != "as_left":
            M = form_matrix(form, typ, n, d, rng)
            if form in ("dense", "dense+csr"):
                assert status(M) in (lib.GxB_FULL, lib.GxB_BITMAP), label
            else:
                assert status(M) not in (lib.GxB_FULL, lib.GxB_BITMAP), label
        other = [j for j, e in enumerate(pool) if e[2] == typ and j != k]
        O, dO = (pool[other[0]][0], pool[other[0]][1]) if other and rng.random() < 0.5 else (M, dict(d))
        M, d = apply_mop(op, M, d, O, dO, typ, n, rng)
        pool[k][0], pool[k][1] = M, d
        check_mat(M, d, typ, label)
        check_products(M, d, typ, n, rng, label)
        REACHED.add((form, op))
    lib.B200_device_synchronize()


def test_every_form_and_operation_of_the_walk_was_reached(request):
    mine = [it for it in request.session.items if it.module is request.module and it is not request.node]
    if len(mine) < kc.full_count(request.module, "test_every_form_and_operation_of_the_walk_was_reached"):
        pytest.skip("only part of the module was selected")
    missing = {(f, o) for f in MFORMS for o in MOPS} - REACHED
    assert not missing, f"(form, operation) pairs no step reached: {sorted(missing)}"
