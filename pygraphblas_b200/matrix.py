"""Matrix: host-side mirror of reference: pygraphblas/matrix.py for the hot path.

Same names, argument meaning and error behaviour as the reference for
`Matrix.mxm` (matrix.py:2401-2584), `Matrix.mxv` (matrix.py:2586-2726), `@` / `@=`
(matrix.py:2728-2737), `**` (matrix.py:1722-1730), `_get_args` (matrix.py:2380-2399)
and the handle plumbing around them (sparse / from_lists / dup / nvals / to_lists /
element access / transpose / iseq / wait).  Every numeric operation is one call through
the C ABI of libb200grb.so (`lib.GrB_mxm`, `lib.GrB_mxv`); nothing is computed in Python.
"""
from functools import partial
import numpy as np

from .base import lib, ffi, NULL, _check, NoValue
from . import types
from .ops import current_semiring, current_accum, current_binop, current_monoid, get_bin_op
from .descriptor import current_desc, T0 as _T0

GxB_INDEX_MAX = 1 << 60


class Matrix:
    __slots__ = ("_matrix", "_keep", "_mask_alive", "_desc_alive", "__weakref__")

    def __init__(self, handle):
        """Wrap a raw GrB_Matrix* (ffi.new("GrB_Matrix*")); the type is read back from the
        library (matrix.py:99-107)."""
        self._matrix = handle
        self._keep = None

    def __del__(self):
        try:        # at interpreter shutdown the binding may already be torn down
            if lib is not None and getattr(self, "_matrix", None) is not None:
                lib.GrB_Matrix_free(self._matrix)
        except Exception:
            pass

    # ------------------------------------------------------------------ construction
    @classmethod
    def sparse(cls, typ, nrows=None, ncols=None):
        """Empty matrix; dimensions default to GxB_INDEX_MAX (matrix.py:120-180)."""
        nrows = GxB_INDEX_MAX if nrows is None else nrows
        ncols = GxB_INDEX_MAX if ncols is None else ncols
        m = ffi.new("GrB_Matrix*")
        _check(lib.GrB_Matrix_new(m, typ.gb_type, nrows, ncols))
        return cls(m)

    @classmethod
    def from_lists(cls, I, J, V=None, nrows=None, ncols=None, typ=None):
        """Build from coordinate lists; later duplicates win, as with the reference's
        setElement loop (matrix.py:269-331)."""
        I = np.ascontiguousarray(I, dtype=np.uint64)
        J = np.ascontiguousarray(J, dtype=np.uint64)
        if V is None:
            V = [True] * len(I)
            typ = typ or types.BOOL
        if typ is None:
            typ = types.from_python(V[0]) if len(V) else types.FP64
        if nrows is None:
            nrows = int(I.max()) + 1 if len(I) else 1
        if ncols is None:
            ncols = int(J.max()) + 1 if len(J) else 1
        X = np.ascontiguousarray(V, dtype=typ.dtype)
        if not (len(I) == len(J) == len(X)):
            raise ValueError("I, J and V must have the same length")
        m = cls.sparse(typ, nrows, ncols)
        _check(typ._Matrix_build(m._matrix[0], ffi.cast("GrB_Index*", I.ctypes.data), ffi.cast("GrB_Index*", J.ctypes.data),
                                 ffi.cast(typ.ptr, X.ctypes.data), len(I), NULL))
        return m

    @classmethod
    def from_csr(cls, indptr, indices, data, nrows, ncols, typ=None):
        """Bulk CSR ingest straight into HBM (B200 extension `B200_Matrix_import_CSR`; the
        reference has no bulk build, matrix.py:325).  `data=None` imports the pattern (all 1)."""
        Ap = np.ascontiguousarray(indptr, dtype=np.int64)
        Aj = np.ascontiguousarray(indices, dtype=np.uint32)
        if typ is None:
            typ = types._dtype_lookup(np.asarray(data).dtype) if data is not None else types.BOOL
        m = ffi.new("GrB_Matrix*")
        if data is None:
            ax = NULL
        else:
            Ax = np.ascontiguousarray(data, dtype=typ.dtype)
            ax = ffi.cast("void*", Ax.ctypes.data)
        _check(lib.B200_Matrix_import_CSR(m, typ.gb_type, nrows, ncols, ffi.cast("int64_t*", Ap.ctypes.data),
                                          ffi.cast("uint32_t*", Aj.ctypes.data), ax, len(Aj), 0))
        return cls(m)

    @classmethod
    def from_numpy(cls, x, present=None, typ=None):
        """Dense import of a 2-D array straight into HBM (B200 extension `B200_Matrix_import_dense`).  `present`
        (same shape, nonzero = present) marks the entries; None means every entry is present.

        Two dense forms under a sparse mask multiply one dot product per entry of the mask, and a sparse matrix times a dense
        form is the SpMM: the two halves of a GNN layer on a graph A (n x n) with features H (n x d), on the device throughout
        (`mxm` sizes a missing `out` without looking at T1, so the scores get theirs passed):

        >>> H = Matrix.from_numpy(h)                                         # doctest: +SKIP
        >>> S = Matrix.sparse(FP32, n, n)                                    # doctest: +SKIP
        >>> H.mxm(H, mask=A, desc=descriptor.ST1, out=S)    # S<A> = H H'    # doctest: +SKIP
        >>> Z = S.mxm(H)                                    # Z = S H        # doctest: +SKIP
        """
        x = np.asarray(x)
        if x.ndim != 2:
            raise ValueError("from_numpy expects a 2-D array")
        typ = typ or types._dtype_lookup(x.dtype)
        x = np.ascontiguousarray(x, dtype=typ.dtype)
        p = NULL
        if present is not None:
            present = np.ascontiguousarray(present, dtype=np.uint8)
            if present.shape != x.shape:
                raise ValueError("present must have the shape of x")
            p = ffi.cast("uint8_t*", present.ctypes.data)
        m = ffi.new("GrB_Matrix*")
        _check(lib.B200_Matrix_import_dense(m, typ.gb_type, x.shape[0], x.shape[1], ffi.cast("void*", x.ctypes.data), p, 0))
        return cls(m)

    def to_numpy(self, out=None, present_out=None):
        """(values, present) dense 2-D host arrays of any matrix (B200 extension `B200_Matrix_export_dense`); absent
        entries read 0.  `out` / `present_out` are C-contiguous arrays of the matrix's shape to fill."""
        shape = (self.nrows, self.ncols)
        x = np.empty(shape, self.type.dtype) if out is None else out
        p = np.empty(shape, np.uint8) if present_out is None else present_out
        for a, dt in ((x, self.type.dtype), (p, np.uint8)):
            if a.shape != shape or a.dtype != dt or not a.flags.c_contiguous:
                raise ValueError(f"output arrays must be C-contiguous {dt} of shape {shape}")
        _check(lib.B200_Matrix_export_dense(self._matrix[0], ffi.cast("void*", x.ctypes.data), ffi.cast("uint8_t*", p.ctypes.data), 0))
        return x, p

    @classmethod
    def from_mm(cls, mm_file):
        """Create a matrix from a Matrix-Market file (matrix.py:377-409 of the reference), parsed in bulk."""
        from .io import mm_read
        I, J, V, nrows, ncols, typ = mm_read(mm_file)
        return cls.from_lists(I, J, V, nrows, ncols, typ)

    def to_mm(self, fileobj):
        """Write the matrix as a Matrix-Market file (tests/test_matrix.py:329-346 of the reference)."""
        from .io import mm_write
        mm_write(self, fileobj)

    @classmethod
    def from_tsv(cls, tsv_file, typ, nrows, ncols, one_based=True, delimiter="\t"):
        """(matrix.py:411-475)"""
        from .io import delimited_read
        I, J, V = delimited_read(tsv_file, typ, one_based, delimiter)
        return cls.from_lists(I, J, V, nrows, ncols, typ)

    @classmethod
    def identity(cls, typ, nrows, value=None):
        """Square matrix with `value` (default one) on the diagonal (matrix.py:574-594 of the reference), built in bulk."""
        d = np.arange(nrows, dtype=np.uint64)
        return cls.from_lists(d, d, np.full(nrows, 1 if value is None else value, dtype=typ.dtype), nrows, nrows, typ)

    @classmethod
    def from_scipy_sparse(cls, m):
        """Type inferred from m.dtype (matrix.py:3495-3514); goes through the host tuple form like the reference
        (`from_scipy` is the bulk route straight into HBM)."""
        ss = m.tocoo()
        return cls.from_lists(ss.row, ss.col, ss.data, ss.shape[0], ss.shape[1], types._dtype_lookup(m.dtype))

    def to_scipy_sparse(self, format="csr"):
        """(matrix.py:3516-3534)"""
        from scipy import sparse
        rows, cols, vals = self.to_arrays()
        s = sparse.coo_matrix((vals, (rows.astype(np.int64), cols.astype(np.int64))), shape=self.shape, dtype=self.type.dtype)
        if format == "coo":
            return s
        if format not in {"bsr", "csr", "csc", "coo", "lil", "dia", "dok"}:
            raise TypeError(f"Invalid format: {format}")
        return s.asformat(format)

    @classmethod
    def from_scipy(cls, A, typ=None):
        A = A.tocsr()
        A.sort_indices()
        return cls.from_csr(A.indptr, A.indices, A.data, A.shape[0], A.shape[1], typ)

    def dup(self):
        m = ffi.new("GrB_Matrix*")
        _check(lib.GrB_Matrix_dup(m, self._matrix[0]))
        return Matrix(m)

    # ------------------------------------------------------------------ properties
    @property
    def gb_type(self):
        t = ffi.new("GrB_Type*")
        _check(lib.GxB_Matrix_type(t, self._matrix[0]))
        return t[0]

    @property
    def type(self):
        return types.from_handle(self.gb_type)

    @property
    def nrows(self):
        n = ffi.new("GrB_Index*")
        _check(lib.GrB_Matrix_nrows(n, self._matrix[0]))
        return n[0]

    @property
    def ncols(self):
        n = ffi.new("GrB_Index*")
        _check(lib.GrB_Matrix_ncols(n, self._matrix[0]))
        return n[0]

    @property
    def shape(self):
        return (self.nrows, self.ncols)

    @property
    def nvals(self):
        n = ffi.new("GrB_Index*")
        _check(lib.GrB_Matrix_nvals(n, self._matrix[0]))
        return n[0]

    def __len__(self):
        return self.nvals

    def clear(self):
        _check(lib.GrB_Matrix_clear(self._matrix[0]))

    def wait(self):
        """Force completion of pending work (matrix.py:3348-3353)."""
        _check(lib.GrB_Matrix_wait(self._matrix))

    # ------------------------------------------------------------------ element access
    def to_arrays(self):
        """(I, J, X) numpy arrays in row-major order (matrix.py:1475-1492)."""
        typ = self.type
        n = self.nvals
        I = np.empty(n, np.uint64)
        J = np.empty(n, np.uint64)
        X = np.empty(n, typ.dtype)
        nv = ffi.new("GrB_Index*", n)
        _check(typ._Matrix_extractTuples(ffi.cast("GrB_Index*", I.ctypes.data), ffi.cast("GrB_Index*", J.ctypes.data),
                                         ffi.cast(typ.ptr, X.ctypes.data), nv, self._matrix[0]))
        return I, J, X

    def to_lists(self):
        I, J, X = self.to_arrays()
        return [I.tolist(), J.tolist(), X.tolist()]

    def __iter__(self):
        I, J, X = self.to_lists()
        return iter(zip(I, J, X))

    def to_csr(self):
        """(indptr int64, indices uint32, data) numpy arrays (B200 extension)."""
        typ = self.type
        n = self.nvals
        Ap = np.empty(self.nrows + 1, np.int64)
        Aj = np.empty(n, np.uint32)
        Ax = np.empty(n, typ.dtype)
        _check(lib.B200_Matrix_export_CSR(self._matrix[0], ffi.cast("int64_t*", Ap.ctypes.data),
                                          ffi.cast("uint32_t*", Aj.ctypes.data), ffi.cast("void*", Ax.ctypes.data), 0))
        return Ap, Aj, Ax

    def __getitem__(self, index):
        i, j = index
        typ = self.type
        x = ffi.new(typ.ptr)
        res = typ._Matrix_extractElement(x, self._matrix[0], i, j)
        if res == lib.GrB_NO_VALUE:
            raise NoValue(f"no value at ({i},{j})")
        _check(res)
        return typ.from_value(x[0])

    def get(self, i, j, default=None):
        try:
            return self[i, j]
        except NoValue:
            return default

    def __setitem__(self, index, value):
        i, j = index
        typ = self.type
        _check(typ._Matrix_setElement(self._matrix[0], typ.from_value(value), i, j))

    def __delitem__(self, index):
        i, j = index
        _check(lib.GrB_Matrix_removeElement(self._matrix[0], i, j))

    def __contains__(self, index):
        return self.get(*index) is not None

    def iseq(self, other):
        """Same type, shape, pattern and values (matrix.py:1436-1453)."""
        if not isinstance(other, Matrix) or self.type is not other.type or self.shape != other.shape:
            return False
        a, b = self.to_arrays(), other.to_arrays()
        return all(np.array_equal(x, y) for x, y in zip(a, b))

    def isne(self, other):
        return not self.iseq(other)

    def transpose(self, cast=None, out=None, mask=None, accum=None, desc=None):
        """New matrix holding the transpose (matrix.py:1003-1061)."""
        if out is None:
            out = Matrix.sparse(cast or self.type, self.ncols, self.nrows)
        mask, accum, desc = self._get_args(mask, accum, desc)
        _check(lib.GrB_transpose(out._matrix[0], mask, accum, self._matrix[0], desc))
        return out

    @property
    def T(self):
        return self.transpose()

    # ------------------------------------------------------------------ the hot path
    def _get_args(self, mask=None, accum=None, desc=None):
        """Resolve mask handle, accumulator and descriptor incl. the context-manager
        defaults (matrix.py:2380-2399)."""
        from .vector import Vector
        if isinstance(mask, Matrix):
            self._mask_alive = mask            # a temporary passed as mask= must outlive the call
            mask = mask._matrix[0]
        elif isinstance(mask, Vector):
            mask = mask._vector[0]
        else:
            mask = NULL
        if accum is None:
            accum = current_accum.get(NULL)
        if accum is not NULL:
            accum = accum.get_op()
        if desc is None:
            desc = current_desc.get(NULL)
        if desc is not NULL:
            self._desc_alive = desc            # a temporary descriptor (desc & other) must outlive the call
            desc = desc.get_desc()
        return mask, accum, desc

    def mxm(self, other, semiring=None, cast=None, out=None, mask=None, accum=None, desc=None):
        """Matrix-matrix multiply C<mask> = accum(C, A (+).(x) B)  (matrix.py:2401-2584)."""
        if not isinstance(other, Matrix):
            raise TypeError("Right argument to mxm must be a Matrix.")
        if semiring is None:
            semiring = current_semiring.get(NULL)
        if out is None:
            if cast is not None:
                typ = cast
            elif semiring is not NULL:
                typ = semiring.ztype
            else:
                typ = types.promote(self.type, other.type)
            out = Matrix.sparse(typ, self.nrows, other.ncols)      # matrix.py:2563 (ignores T0/T1)
        else:
            typ = out.type
        if semiring is NULL:
            semiring = out.type._default_semiring()
        mask, accum, desc = self._get_args(mask, accum, desc)
        _check(lib.GrB_mxm(out._matrix[0], mask, accum, semiring.get_op(), self._matrix[0], other._matrix[0], desc))
        return out

    def mxv(self, other, semiring=None, cast=None, out=None, mask=None, accum=None, desc=None):
        """Matrix-vector multiply w<mask> = accum(w, A (+).(x) u)  (matrix.py:2586-2726)."""
        from .vector import Vector
        if not isinstance(other, Vector):
            raise TypeError("Right argument to mxv must be a Vector.")
        if semiring is None:
            semiring = current_semiring.get(NULL)
        if out is None:
            d = desc if desc is not None else current_desc.get(None)
            new_dimension = self.ncols if (d is not None and _T0 in d) else self.nrows
            if cast is not None:
                typ = cast
            elif semiring is not NULL:
                typ = semiring.ztype
            else:
                typ = types.promote(self.type, other.type)
            out = Vector.sparse(typ, new_dimension)
        if semiring is NULL:
            semiring = out.type._default_semiring()
        mask, accum, desc = self._get_args(mask, accum, desc)
        _check(lib.GrB_mxv(out._vector[0], mask, accum, semiring.get_op(), self._matrix[0], other._vector[0], desc))
        return out

    # ------------------------------------------------------------------ consumers of the hot path (matrix_ops.cu)
    _SELECT = {">": "GT_THUNK", "<": "LT_THUNK", ">=": "GE_THUNK", "<=": "LE_THUNK", "!=": "NE_THUNK", "==": "EQ_THUNK",
               ">0": "GT_ZERO", "<0": "LT_ZERO", ">=0": "GE_ZERO", "<=0": "LE_ZERO", "!=0": "NONZERO", "==0": "EQ_ZERO"}

    def select(self, op, thunk=None, out=None, mask=None, accum=None, desc=None):
        """C<mask> = accum(C, select(A, thunk))  (matrix.py:2042-2140 of the reference)."""
        from .scalar import Scalar
        if out is None:
            out = Matrix.sparse(self.type, self.nrows, self.ncols)
        if isinstance(op, str):
            op = getattr(lib, "GxB_" + self._SELECT[op])
        keep = None
        if thunk is None:
            thunk = NULL
        elif isinstance(thunk, (bool, int, float)):
            keep = Scalar.from_value(thunk); thunk = keep._scalar[0]
        elif isinstance(thunk, Scalar):
            keep = thunk; thunk = keep._scalar[0]
        mask, accum, desc = self._get_args(mask, accum, desc)
        _check(lib.GxB_Matrix_select(out._matrix[0], mask, accum, op, self._matrix[0], thunk, desc))
        return out

    def tril(self, offset=None):
        """(matrix.py:2142-2170)"""
        return self.select(lib.GxB_TRIL, offset)

    def triu(self, offset=None):
        """(matrix.py:2172-2200)"""
        return self.select(lib.GxB_TRIU, offset)

    def diag(self, offset=None):
        return self.select(lib.GxB_DIAG, offset)

    def offdiag(self, offset=None):
        """(matrix.py:2279-2307)"""
        return self.select(lib.GxB_OFFDIAG, offset)

    def nonzero(self):
        """(matrix.py:2309-2311)"""
        return self.select(lib.GxB_NONZERO)

    def apply(self, op, out=None, mask=None, accum=None, desc=None):
        """(matrix.py:1934-1963)"""
        if out is None:
            out = Matrix.sparse(self.type, self.nrows, self.ncols)
        mask, accum, desc = self._get_args(mask, accum, desc)
        _check(lib.GrB_Matrix_apply(out._matrix[0], mask, accum, op.get_op(), self._matrix[0], desc))
        return out

    def apply_first(self, first, op, out=None, mask=None, accum=None, desc=None):
        """(matrix.py:1965-2005)"""
        if out is None:
            out = Matrix.sparse(self.type, self.nrows, self.ncols)
        from .scalar import Scalar
        mask, accum, desc = self._get_args(mask, accum, desc)
        if isinstance(first, Scalar):
            self._keep = first
            _check(lib.GxB_Matrix_apply_BinaryOp1st(out._matrix[0], mask, accum, op.get_op(), first._scalar[0], self._matrix[0], desc))
        else:           # the typed entry point of the matrix's own type (matrix.py:1992-2005)
            _check(self.type._Matrix_apply_BinaryOp1st(out._matrix[0], mask, accum, op.get_op(), first, self._matrix[0], desc))
        return out

    def apply_second(self, op, second, out=None, mask=None, accum=None, desc=None):
        """(matrix.py:2007-2040)"""
        if out is None:
            out = Matrix.sparse(self.type, self.nrows, self.ncols)
        from .scalar import Scalar
        mask, accum, desc = self._get_args(mask, accum, desc)
        if isinstance(second, Scalar):
            self._keep = second
            _check(lib.GxB_Matrix_apply_BinaryOp2nd(out._matrix[0], mask, accum, op.get_op(), self._matrix[0], second._scalar[0], desc))
        else:           # matrix.py:2027-2040
            _check(self.type._Matrix_apply_BinaryOp2nd(out._matrix[0], mask, accum, op.get_op(), self._matrix[0], second, desc))
        return out

    def pattern(self, typ=types.BOOL, out=None):
        """(matrix.py:887-902)"""
        if out is None:
            out = Matrix.sparse(typ, self.nrows, self.ncols)
        return self.apply(typ.ONE, out=out)

    def eadd(self, other, add_op=None, cast=None, out=None, mask=None, accum=None, desc=None):
        """Element-wise union (matrix.py:1103-1264; also `|`, `+`, `-`)."""
        from .ops import Monoid, Semiring
        func = lib.GrB_Matrix_eWiseAdd_BinaryOp
        if isinstance(add_op, Monoid):
            func = lib.GrB_Matrix_eWiseAdd_Monoid
        elif isinstance(add_op, Semiring):
            func = lib.GrB_Matrix_eWiseAdd_Semiring
        if out is None:
            out = Matrix.sparse(cast or types.promote(self.type, other.type), self.nrows, self.ncols)
        if add_op is None:
            add_op = current_binop.get(None) or out.type._default_addop()
        mask, accum, desc = self._get_args(mask, accum, desc)
        _check(func(out._matrix[0], mask, accum, add_op.get_op(), self._matrix[0], other._matrix[0], desc))
        return out

    def emult(self, other, mult_op=None, cast=None, out=None, mask=None, accum=None, desc=None):
        """Element-wise intersection (matrix.py:1266-1415; also `&`, `*`, `/`)."""
        if out is None:
            out = Matrix.sparse(cast or types.promote(self.type, other.type), self.nrows, self.ncols)
        if mult_op is None:
            mult_op = current_binop.get(None) or out.type._default_multop()
        elif isinstance(mult_op, str):
            mult_op = get_bin_op(mult_op, self.type)
        mask, accum, desc = self._get_args(mask, accum, desc)
        _check(lib.GrB_Matrix_eWiseMult_BinaryOp(out._matrix[0], mask, accum, mult_op.get_op(), self._matrix[0], other._matrix[0], desc))
        return out

    def _reduce(self, typ, mon, accum=None):
        if mon is None:
            mon = current_monoid.get(None) or getattr(typ, "LOR_MONOID" if typ is types.BOOL else "PLUS_MONOID")
        x = ffi.new(typ.ptr)
        _, accum, desc = self._get_args(None, accum, None)
        _check(typ._Matrix_reduce(x, accum, mon.get_op(), self._matrix[0], desc))
        return typ.from_value(x[0])

    def reduce_bool(self, mon=None, **kw):
        """(matrix.py:1759-1780)"""
        return self._reduce(types.BOOL, mon, **kw)

    def reduce_int(self, mon=None, **kw):
        """(matrix.py:1782-1804)"""
        return self._reduce(types.INT64, mon, **kw)

    def reduce_float(self, mon=None, **kw):
        """(matrix.py:1806-1828)"""
        return self._reduce(types.FP64, mon, **kw)

    def reduce_vector(self, mon=None, out=None, mask=None, accum=None, desc=None):
        """w<mask> = accum(w, reduce rows of op(A))  (matrix.py:1861-1932)."""
        from .vector import Vector
        if mon is None:
            mon = getattr(self.type, "LOR_MONOID" if self.type is types.BOOL else "PLUS_MONOID")
        if out is None:
            d = desc if desc is not None else current_desc.get(None)
            out = Vector.sparse(self.type, self.ncols if (d is not None and _T0 in d) else self.nrows)
        mask, accum, desc = self._get_args(mask, accum, desc)
        _check(lib.GrB_Matrix_reduce_Monoid(out._vector[0], mask, accum, mon.get_op(), self._matrix[0], desc))
        return out

    # arithmetic operators: exactly the calls the reference makes (matrix.py:1625-1720), including the default
    # operator taken from the `with <BinaryOp>:` context and the operand order of the in-place forms
    def __and__(self, other):
        return self.emult(other, current_binop.get(self.type.SECOND))

    def __iand__(self, other):
        return self.emult(other, current_binop.get(self.type.SECOND), out=self)

    def __or__(self, other):
        return self.eadd(other, current_binop.get(self.type.SECOND))

    def __ior__(self, other):
        return self.eadd(other, current_binop.get(self.type.SECOND), out=self)

    def __add__(self, other):
        op = current_binop.get(self.type.PLUS)
        if not isinstance(other, Matrix):
            return self.apply_second(op, other)
        return self.eadd(other, op)

    def __radd__(self, other):
        return self.apply_first(other, current_binop.get(self.type.PLUS))

    def __iadd__(self, other):
        op = current_binop.get(self.type.PLUS)
        if not isinstance(other, Matrix):
            return self.apply_second(op, other, out=self)
        return self.eadd(other, op, out=self)

    def __sub__(self, other):
        op = current_binop.get(self.type.MINUS)
        if not isinstance(other, Matrix):
            return self.apply_second(op, other)
        return self.eadd(other, op)

    def __rsub__(self, other):
        return self.apply_first(other, current_binop.get(self.type.MINUS))

    def __isub__(self, other):
        op = current_binop.get(self.type.MINUS)
        if not isinstance(other, Matrix):
            return self.apply_second(op, other, out=self)
        return other.eadd(self, op, out=self)

    def __mul__(self, other):
        op = current_binop.get(self.type.TIMES)
        if not isinstance(other, Matrix):
            return self.apply_second(op, other)
        return self.emult(other, op)

    def __rmul__(self, other):
        return self.apply_first(other, current_binop.get(self.type.TIMES))

    def __imul__(self, other):
        op = current_binop.get(self.type.TIMES)
        if not isinstance(other, Matrix):
            return self.apply_second(op, other)
        return other.emult(self, op, out=self)

    def __truediv__(self, other):
        op = current_binop.get(self.type.DIV)
        if not isinstance(other, Matrix):
            return self.apply_second(op, other)
        return self.emult(other, op)

    def __rtruediv__(self, other):
        return self.apply_first(other, current_binop.get(self.type.DIV))

    def __itruediv__(self, other):
        op = current_binop.get(self.type.DIV)
        if not isinstance(other, Matrix):
            return self.apply_second(op, other)
        return other.emult(self, op, out=self)

    def __invert__(self):
        return self.apply(self.type.MINV)

    def __neg__(self):
        return self.apply(self.type.AINV)

    def __abs__(self):
        return self.apply(self.type.ABS)

    def __matmul__(self, other):
        from .vector import Vector
        if isinstance(other, Matrix):
            return self.mxm(other)
        if isinstance(other, Vector):
            return self.mxv(other)
        raise TypeError("Right argument to @ must be Matrix or Vector.")

    def __imatmul__(self, other):
        return self.mxm(other, out=self)

    def __pow__(self, exponent):
        """A ** k by repeated mxm into a copy (matrix.py:1722-1730)."""
        if exponent == 0:
            raise ValueError("exponent must be >= 1")
        if exponent == 1:
            return self.dup()
        result = self.dup()
        for _ in range(1, exponent):
            result.mxm(self, out=result)
        return result

    def __getattr__(self, name):
        """`A.min_plus(B)`: look the operator up on the type (matrix.py:1607-1613)."""
        if name.startswith("_"):
            raise AttributeError(name)
        try:
            attr = getattr(self.type, name)
        except AttributeError:
            raise AttributeError(f"Matrix has no attribute or type operator {name}")
        return partial(attr, self)

    def __repr__(self):
        return f"<Matrix ({self.nrows}x{self.ncols} : {self.nvals}:{self.type.name})>"
