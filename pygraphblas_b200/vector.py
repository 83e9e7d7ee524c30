"""Vector: host-side mirror of reference: pygraphblas/vector.py for the hot path:
`Vector.vxm` (vector.py:835-971), `@` / `@=` (vector.py:973-977), `_get_args`
(vector.py:1078-1099) and the plumbing around it (sparse / from_lists / dup / nvals /
to_lists / element access / iseq / wait), plus dense import/export for bulk transfers."""
from functools import partial
import numpy as np

from .base import lib, ffi, NULL, _check, NoValue
from . import types
from .ops import current_semiring, current_accum, current_binop, current_monoid, get_bin_op
from .descriptor import current_desc, T1 as _T1

GxB_INDEX_MAX = 1 << 60


class Vector:
    __slots__ = ("_vector", "_mask_alive", "_desc_alive", "_keep_scalar", "_owner", "__weakref__")

    def __init__(self, handle, owner=None):
        self._vector = handle
        self._owner = owner          # set for views whose handle belongs to another object (distributed.Comm): not freed here

    def __del__(self):
        try:        # at interpreter shutdown the binding may already be torn down
            if lib is not None and getattr(self, "_vector", None) is not None and getattr(self, "_owner", None) is None:
                lib.GrB_Vector_free(self._vector)
        except Exception:
            pass

    # ------------------------------------------------------------------ construction
    @classmethod
    def sparse(cls, typ, size=None):
        """Empty vector; size defaults to GxB_INDEX_MAX (vector.py:250-286)."""
        v = ffi.new("GrB_Vector*")
        _check(lib.GrB_Vector_new(v, typ.gb_type, GxB_INDEX_MAX if size is None else size))
        return cls(v)

    @classmethod
    def from_lists(cls, I, V, size=None, typ=None):
        """(vector.py:330-356); later duplicates win."""
        I = np.ascontiguousarray(I, dtype=np.uint64)
        if typ is None:
            typ = types.from_python(V[0]) if len(V) else types.FP64
        if size is None:
            size = int(I.max()) + 1 if len(I) else 1
        X = np.ascontiguousarray(V, dtype=typ.dtype)
        v = cls.sparse(typ, size)
        _check(typ._Vector_build(v._vector[0], ffi.cast("GrB_Index*", I.ctypes.data), ffi.cast(typ.ptr, X.ctypes.data), len(I), NULL))
        return v

    @classmethod
    def from_1_to_n(cls, n):
        """(vector.py:370-382)"""
        return cls.from_lists(np.arange(n, dtype=np.uint64), np.arange(1, n + 1, dtype=np.int64), n, types.INT64)

    @classmethod
    def from_list(cls, V, typ=None):
        return cls.from_lists(list(range(len(V))), V, len(V), typ)

    @classmethod
    def from_numpy(cls, x, present=None, typ=None):
        """Dense import straight into HBM (B200 extension `B200_Vector_import_dense`)."""
        x = np.ascontiguousarray(x)
        typ = typ or types._dtype_lookup(x.dtype)
        x = np.ascontiguousarray(x, dtype=typ.dtype)
        p = NULL
        if present is not None:
            present = np.ascontiguousarray(present, dtype=np.uint8)
            p = ffi.cast("uint8_t*", present.ctypes.data)
        v = ffi.new("GrB_Vector*")
        _check(lib.B200_Vector_import_dense(v, typ.gb_type, len(x), ffi.cast("void*", x.ctypes.data), p, 0))
        return cls(v)

    def set_numpy(self, x, present=None):
        """Refill this vector from a dense host array without reallocating in HBM."""
        typ = self.type
        x = np.ascontiguousarray(x, dtype=typ.dtype)
        p = NULL
        if present is not None:
            present = np.ascontiguousarray(present, dtype=np.uint8)
            p = ffi.cast("uint8_t*", present.ctypes.data)
        _check(lib.B200_Vector_set_dense(self._vector[0], ffi.cast("void*", x.ctypes.data), p, 0))

    def to_numpy(self, out=None, present_out=None):
        """(values, present) dense host arrays (B200 extension `B200_Vector_export_dense`)."""
        typ = self.type
        n = self.size
        x = np.empty(n, typ.dtype) if out is None else out
        p = np.empty(n, np.uint8) if present_out is None else present_out
        _check(lib.B200_Vector_export_dense(self._vector[0], ffi.cast("void*", x.ctypes.data), ffi.cast("uint8_t*", p.ctypes.data), 0))
        return x, p

    def device_ptrs(self):
        """(values_ptr, present_ptr or 0): raw CUDA device pointers of the dense HBM form."""
        vals = ffi.new("void**")
        pres = ffi.new("uint8_t**")
        _check(lib.B200_Vector_device_ptrs(self._vector[0], vals, pres))
        return int(ffi.cast("uintptr_t", vals[0])), int(ffi.cast("uintptr_t", pres[0]))

    def dup(self):
        v = ffi.new("GrB_Vector*")
        _check(lib.GrB_Vector_dup(v, self._vector[0]))
        return Vector(v)

    # ------------------------------------------------------------------ properties
    @property
    def gb_type(self):
        t = ffi.new("GrB_Type*")
        _check(lib.GxB_Vector_type(t, self._vector[0]))
        return t[0]

    @property
    def type(self):
        return types.from_handle(self.gb_type)

    @property
    def size(self):
        n = ffi.new("GrB_Index*")
        _check(lib.GrB_Vector_size(n, self._vector[0]))
        return n[0]

    @property
    def shape(self):
        return (self.size,)

    @property
    def nvals(self):
        n = ffi.new("GrB_Index*")
        _check(lib.GrB_Vector_nvals(n, self._vector[0]))
        return n[0]

    def __len__(self):
        return self.nvals

    def clear(self):
        _check(lib.GrB_Vector_clear(self._vector[0]))

    def wait(self):
        _check(lib.GrB_Vector_wait(self._vector))

    # ------------------------------------------------------------------ element access
    def to_arrays(self):
        typ = self.type
        n = self.nvals
        I = np.empty(n, np.uint64)
        X = np.empty(n, typ.dtype)
        nv = ffi.new("GrB_Index*", n)
        _check(typ._Vector_extractTuples(ffi.cast("GrB_Index*", I.ctypes.data), ffi.cast(typ.ptr, X.ctypes.data), nv, self._vector[0]))
        return I, X

    def to_lists(self):
        I, X = self.to_arrays()
        return [I.tolist(), X.tolist()]

    def __iter__(self):
        I, X = self.to_lists()
        return iter(zip(I, X))

    def __getitem__(self, i):
        if not isinstance(i, (int, np.integer)):
            return self.extract(i)
        typ = self.type
        x = ffi.new(typ.ptr)
        res = typ._Vector_extractElement(x, self._vector[0], i)
        if res == lib.GrB_NO_VALUE:
            raise NoValue(f"no value at {i}")
        _check(res)
        return typ.from_value(x[0])

    def get(self, i, default=None):
        try:
            return self[i]
        except NoValue:
            return default

    def __setitem__(self, i, value):
        if isinstance(i, Vector):                            # v[mask] = x  (vector.py:1449-1457)
            if isinstance(value, Vector):
                return self.assign(value, None, mask=i)
            return self.assign_scalar(value, None, mask=i)
        if not isinstance(i, (int, np.integer)):
            if isinstance(value, Vector):
                return self.assign(value, i)
            return self.assign_scalar(value, i)
        typ = self.type
        _check(typ._Vector_setElement(self._vector[0], typ.from_value(value), i))

    def __delitem__(self, i):
        _check(lib.GrB_Vector_removeElement(self._vector[0], i))

    def __contains__(self, i):
        return self.get(i) is not None

    def iseq(self, other):
        """(vector.py:213-235)"""
        if not isinstance(other, Vector) or self.type is not other.type or self.size != other.size:
            return False
        a, b = self.to_arrays(), other.to_arrays()
        return all(np.array_equal(x, y) for x, y in zip(a, b))

    def isne(self, other):
        return not self.iseq(other)

    # ------------------------------------------------------------------ the hot path
    def _get_args(self, mask=None, accum=None, desc=None):
        """(vector.py:1078-1099)"""
        if isinstance(mask, Vector):
            self._mask_alive = mask            # a temporary passed as mask= must outlive the call
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

    def vxm(self, other, semiring=None, cast=None, out=None, mask=None, accum=None, desc=None):
        """Vector-matrix multiply w'<mask'> = accum(w', u' (+).(x) A)  (vector.py:835-971)."""
        from .matrix import Matrix
        if not isinstance(other, Matrix):
            raise TypeError("Right argument to vxm must be a Matrix.")
        if semiring is None:
            semiring = current_semiring.get(NULL)
        if out is None:
            d = desc if desc is not None else current_desc.get(None)
            new_dimension = other.nrows if (d is not None and _T1 in d) else other.ncols   # vector.py:946
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
        _check(lib.GrB_vxm(out._vector[0], mask, accum, semiring.get_op(), self._vector[0], other._matrix[0], desc))
        return out

    # ------------------------------------------------------------------ loop glue (vector_ops.cu)
    def _out_like(self, out, typ=None):
        return out if out is not None else Vector.sparse(typ or self.type, self.size)

    def eadd(self, other, add_op=None, cast=None, out=None, mask=None, accum=None, desc=None):
        """Element-wise union w<mask> = accum(w, u (+) v)  (vector.py:604-735 of the reference; also `|`, `+`, `-`)."""
        from .ops import Monoid, Semiring
        func = lib.GrB_Vector_eWiseAdd_BinaryOp
        if isinstance(add_op, Monoid):
            func = lib.GrB_Vector_eWiseAdd_Monoid
        elif isinstance(add_op, Semiring):
            func = lib.GrB_Vector_eWiseAdd_Semiring
        out = self._out_like(out, cast or types.promote(self.type, other.type))
        if add_op is None:
            add_op = current_binop.get(None) or out.type._default_addop()
        mask, accum, desc = self._get_args(mask, accum, desc)
        _check(func(out._vector[0], mask, accum, add_op.get_op(), self._vector[0], other._vector[0], desc))
        return out

    def emult(self, other, mult_op=None, cast=None, out=None, mask=None, accum=None, desc=None):
        """Element-wise intersection w<mask> = accum(w, u (x) v)  (vector.py:737-833; also `&`, `*`, `/`)."""
        out = self._out_like(out, cast or types.promote(self.type, other.type))
        if mult_op is None:
            mult_op = current_binop.get(None) or out.type._default_multop()
        elif isinstance(mult_op, str):
            mult_op = get_bin_op(mult_op, self.type)
        mask, accum, desc = self._get_args(mask, accum, desc)
        _check(lib.GrB_Vector_eWiseMult_BinaryOp(out._vector[0], mask, accum, mult_op.get_op(), self._vector[0], other._vector[0], desc))
        return out

    def apply(self, op, out=None, mask=None, accum=None, desc=None):
        """w<mask> = accum(w, f(u))  (vector.py:1101-1129)."""
        out = self._out_like(out)
        mask, accum, desc = self._get_args(mask, accum, desc)
        _check(lib.GrB_Vector_apply(out._vector[0], mask, accum, op.get_op(), self._vector[0], desc))
        return out

    def apply_first(self, first, op, out=None, mask=None, accum=None, desc=None):
        """w = op(first, u)  (vector.py:1131-1153)."""
        from .scalar import Scalar
        out = self._out_like(out)
        mask, accum, desc = self._get_args(mask, accum, desc)
        if isinstance(first, Scalar):
            self._keep_scalar = first
            _check(lib.GxB_Vector_apply_BinaryOp1st(out._vector[0], mask, accum, op.get_op(), first._scalar[0], self._vector[0], desc))
        else:           # the typed entry point of the vector's own type, as the reference picks it (vector.py:1293-1299)
            _check(self.type._Vector_apply_BinaryOp1st(out._vector[0], mask, accum, op.get_op(), first, self._vector[0], desc))
        return out

    def apply_second(self, op, second, out=None, mask=None, accum=None, desc=None):
        """w = op(u, second)  (vector.py:1155-1178)."""
        from .scalar import Scalar
        out = self._out_like(out)
        mask, accum, desc = self._get_args(mask, accum, desc)
        if isinstance(second, Scalar):
            self._keep_scalar = second
            _check(lib.GxB_Vector_apply_BinaryOp2nd(out._vector[0], mask, accum, op.get_op(), self._vector[0], second._scalar[0], desc))
        else:           # vector.py:1345-1351
            _check(self.type._Vector_apply_BinaryOp2nd(out._vector[0], mask, accum, op.get_op(), self._vector[0], second, desc))
        return out

    def _index(self, index, dim):
        """(I, ni, length) of a slice / list / None, exactly as base.py:216-252 (_build_range) of the reference
        builds it: GrB_ALL, an explicit list, or GxB_RANGE / GxB_STRIDE / GxB_BACKWARDS with an INCLUSIVE stop."""
        if isinstance(index, (list, tuple, np.ndarray)):
            idx = [int(i) for i in index]
            return ffi.new("GrB_Index[]", idx if idx else [0]), len(idx), len(idx)
        if index is None or index == slice(None, None, None):
            return lib.GrB_ALL, 0, dim
        start = 0 if index.start is None else index.start
        stop = dim - 1 if index.stop is None else index.stop
        step = index.step
        if step is None:
            return ffi.new("GrB_Index[2]", [start, stop]), lib.GxB_RANGE, (stop - start) + 1
        if step < 0:
            step = abs(step)
            size = 0 if start < stop else int((start - stop) / step) + 1
            return ffi.new("GrB_Index[3]", [start, stop, step]), lib.GxB_BACKWARDS, size
        size = 0 if (start > stop or step == 0) else int((stop - start) / step) + 1
        return ffi.new("GrB_Index[3]", [start, stop, step]), lib.GxB_STRIDE, size

    def assign_scalar(self, value, index=None, mask=None, accum=None, desc=None):
        """w<mask>(I) = accum(w(I), x)  (vector.py:1494-1524)."""
        typ = types.from_python(value)
        I, ni, _ = self._index(index, self.size)
        mask, accum, desc = self._get_args(mask, accum, desc)
        _check(typ._Vector_assignScalar(self._vector[0], mask, accum, typ.from_value(value), I, ni, desc))

    def assign(self, value, index=None, mask=None, accum=None, desc=None):
        """w<mask>(I) = accum(w(I), u)  (vector.py:1461-1492)."""
        I, ni, _ = self._index(index, self.size)
        mask, accum, desc = self._get_args(mask, accum, desc)
        _check(lib.GrB_Vector_assign(self._vector[0], mask, accum, value._vector[0], I, ni, desc))

    def extract(self, index=None, out=None, mask=None, accum=None, desc=None):
        """w<mask> = accum(w, u(I))  (vector.py:1526-1560)."""
        I, ni, length = self._index(index, self.size)
        if out is None:
            out = Vector.sparse(self.type, length)
        mask, accum, desc = self._get_args(mask, accum, desc)
        _check(lib.GrB_Vector_extract(out._vector[0], mask, accum, self._vector[0], I, ni, desc))
        return out

    def _reduce(self, typ, mon, accum=None):
        if mon is None:
            mon = current_monoid.get(None) or getattr(typ, "LOR_MONOID" if typ is types.BOOL else "PLUS_MONOID")
        x = ffi.new(typ.ptr)
        mask, accum, desc = self._get_args(None, accum, None)
        _check(typ._Vector_reduce(x, accum, mon.get_op(), self._vector[0], desc))
        return typ.from_value(x[0])

    def reduce_bool(self, mon=None, **kw):
        """(vector.py:533-552)"""
        return self._reduce(types.BOOL, mon, **kw)

    def reduce_int(self, mon=None, **kw):
        """(vector.py:554-572)"""
        return self._reduce(types.INT64, mon, **kw)

    def reduce_float(self, mon=None, **kw):
        """(vector.py:574-593)"""
        return self._reduce(types.FP64, mon, **kw)

    def pattern(self, typ=types.BOOL):
        """(vector.py:1405-1414)"""
        out = Vector.sparse(typ, self.size)
        self.apply(types.BOOL.ONE, out=out)
        return out

    # arithmetic operators: exactly the calls the reference makes (vector.py:991-1063), operand order of the
    # in-place forms included (`a -= b` evaluates MINUS(b, a) on the intersection there, :1016-1019)
    def __add__(self, other):
        if not isinstance(other, Vector):
            return self.apply_second(self.type.PLUS, other)
        return self.eadd(other)

    def __radd__(self, other):
        return self.apply_first(other, self.type.PLUS)

    def __iadd__(self, other):
        if not isinstance(other, Vector):
            return self.apply_second(self.type.PLUS, other, out=self)
        return self.eadd(other, out=self)

    def __sub__(self, other):
        if not isinstance(other, Vector):
            return self.apply_second(self.type.MINUS, other)
        return self.eadd(other, self.type.MINUS)

    def __rsub__(self, other):
        return self.apply_first(other, self.type.MINUS)

    def __isub__(self, other):
        if not isinstance(other, Vector):
            return self.apply_second(self.type.MINUS, other)
        return other.eadd(self, self.type.MINUS, out=self)

    def __mul__(self, other):
        if not isinstance(other, Vector):
            return self.apply_second(self.type.TIMES, other)
        return self.emult(other, self.type.TIMES)

    def __rmul__(self, other):
        return self.apply_first(other, self.type.TIMES)

    def __imul__(self, other):
        if not isinstance(other, Vector):
            return self.apply_second(self.type.TIMES, other, out=self)
        return other.emult(self, self.type.TIMES, out=self)

    def __truediv__(self, other):
        if not isinstance(other, Vector):
            return self.apply_second(self.type.DIV, other)
        return self.emult(other, self.type.DIV)

    def __rtruediv__(self, other):
        return self.apply_first(other, self.type.DIV)

    def __itruediv__(self, other):
        if not isinstance(other, Vector):
            return self.apply_second(self.type.DIV, other, out=self)
        return other.emult(self, self.type.DIV, out=self)

    def __and__(self, other):
        return self.emult(other)

    def __iand__(self, other):
        return self.emult(other, out=self)

    def __or__(self, other):
        return self.eadd(other)

    def __ior__(self, other):
        return self.eadd(other, out=self)

    def __invert__(self):
        return self.apply(self.type.MINV)

    def __neg__(self):
        return self.apply(self.type.AINV)

    def __abs__(self):
        return self.apply(self.type.ABS)

    _SELECT = {">": "GT_THUNK", "<": "LT_THUNK", ">=": "GE_THUNK", "<=": "LE_THUNK", "!=": "NE_THUNK", "==": "EQ_THUNK",
               ">0": "GT_ZERO", "<0": "LT_ZERO", ">=0": "GE_ZERO", "<=0": "LE_ZERO", "!=0": "NONZERO", "==0": "EQ_ZERO"}

    def select(self, op, thunk=None, out=None, mask=None, accum=None, desc=None):
        """w<mask> = accum(w, select(u, thunk))  (vector.py:1361-1403)."""
        from .scalar import Scalar
        if out is None:
            out = Vector.sparse(self.type, self.size)
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
        _check(lib.GxB_Vector_select(out._vector[0], mask, accum, op, self._vector[0], thunk, desc))
        return out

    def nonzero(self):
        """(vector.py:1426-1428)"""
        return self.select(lib.GxB_NONZERO)

    def __matmul__(self, other):
        from .matrix import Matrix
        if isinstance(other, Matrix):
            return self.vxm(other)
        raise TypeError("Right argument to @ must be a Matrix.")

    def __imatmul__(self, other):
        return self.vxm(other, out=self)

    def __getattr__(self, name):
        if name.startswith("_"):
            raise AttributeError(name)
        try:
            attr = getattr(self.type, name)
        except AttributeError:
            raise AttributeError(f"Vector has no attribute or type operator {name}")
        return partial(attr, self)

    def __repr__(self):
        return f"<Vector ({self.size} : {self.nvals}:{self.type.name})>"
