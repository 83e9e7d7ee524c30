"""Binary operators, accumulators, monoids and semirings.

Mirrors reference: pygraphblas/binaryop.py:28-101 (BinaryOp, Accum),
monoid.py:37-78 (Monoid) and semiring.py:29-84 (Semiring incl. call dispatch,
context manager and ztype).  As in the reference the objects are discovered from the
names `lib` exports (semiring.py:87-129) and attached to their type as attributes.
"""
import contextvars
import re
from .base import lib, ffi, _check, NULL
from . import types

current_semiring = contextvars.ContextVar("current_semiring")
current_accum = contextvars.ContextVar("current_accum")
current_binop = contextvars.ContextVar("current_binop")        # binaryop.py:18 of the reference
current_monoid = contextvars.ContextVar("current_monoid")      # monoid.py:16

_T = "BOOL|UINT8|UINT16|UINT32|UINT64|INT8|INT16|INT32|INT64|FP32|FP64"


class BinaryOp:
    def __init__(self, op, typ, handle):
        self.op, self.type, self.binaryop = op, typ, handle
        self.name = f"{op}_{typ}"

    def __enter__(self):                            # `with INT64.MAX: c = a | b`  (binaryop.py:51-57)
        self.token = current_binop.set(self)
        return self

    def __exit__(self, *errors):
        current_binop.reset(self.token)
        return False

    def __call__(self, A, B, *args, **kwargs):      # binaryop.py:59-60
        return A.emult(B, self, *args, **kwargs)

    def get_op(self):
        return self.binaryop

    def __repr__(self):
        return f"<BinaryOp {self.name}>"


class UnaryOp:
    """Builtin unary operator (unaryop.py:21-50): `FP32.ABS(v)` = `v.apply(FP32.ABS)`."""

    def __init__(self, op, typ, handle):
        self.op, self.type, self.unaryop = op, typ, handle
        self.name = f"{op}_{typ}"

    def __call__(self, A, *args, **kwargs):
        return A.apply(self, *args, **kwargs)

    def get_op(self):
        return self.unaryop

    def __repr__(self):
        return f"<UnaryOp {self.name}>"


class Accum:
    """`with Accum(INT64.min): o @= n`  (binaryop.py:80-101)."""

    def __init__(self, binaryop):
        self.binaryop = binaryop

    def __enter__(self):
        self.token = current_accum.set(self.binaryop)
        return self

    def __exit__(self, *errors):
        current_accum.reset(self.token)
        return False


class Monoid:
    def __init__(self, op, typ, handle):
        self.op, self.type, self.monoid = op, typ, handle
        self.name = f"{op}_{typ}_MONOID"

    def __enter__(self):                            # `with INT8.TIMES_MONOID: m.reduce_int()`  (monoid.py:60-66)
        self.token = current_monoid.set(self)
        return self

    def __exit__(self, *errors):
        current_monoid.reset(self.token)
        return False

    def get_op(self):
        return self.monoid

    def __repr__(self):
        return f"<Monoid {self.name}>"


class Semiring:
    def __init__(self, pls, mul, typ, handle):
        self.pls, self.mul, self.type, self.semiring = pls, mul, typ, handle
        self.name = f"{pls}_{mul}_{typ}"
        self.token = None

    def __call__(self, A, B, *args, **kwargs):     # semiring.py:47-56
        from .vector import Vector
        if isinstance(A, Vector):
            op = A.vxm
        elif isinstance(B, Vector):
            op = A.mxv
        else:
            op = A.mxm
        return op(B, self, *args, **kwargs)

    def __enter__(self):
        self.token = current_semiring.set(self)
        return self

    def __exit__(self, *errors):
        current_semiring.reset(self.token)
        return False

    def get_op(self):
        return self.semiring

    @property
    def ztype(self):                                # types.py:442-461
        m = ffi.new("GrB_Monoid*")
        _check(lib.GxB_Semiring_add(m, self.semiring))
        o = ffi.new("GrB_BinaryOp*")
        _check(lib.GxB_Monoid_operator(o, m[0]))
        t = ffi.new("GrB_Type*")
        _check(lib.GxB_BinaryOp_ztype(t, o[0]))
        return types.from_handle(t[0])

    def __repr__(self):
        return f"<Semiring {self.name}>"


_STR_BINOP = {">": "GT", "<": "LT", ">=": "GE", "<=": "LE", "!=": "NE", "==": "EQ", "+": "PLUS", "-": "MINUS", "*": "TIMES", "/": "DIV"}


def get_bin_op(op, typ):
    """'+', '>=' ... -> the operator of `typ` (base.py:270-282)."""
    return getattr(typ, _STR_BINOP[op])


_binop_re = re.compile(rf"^(?:GrB|GxB)_([A-Z0-9]+)_({_T})$")
_monoid_res = (re.compile(rf"^GxB_([A-Z]+)_({_T})_MONOID$"), re.compile(rf"^GrB_([A-Z]+)_MONOID_({_T})$"))
# the multiply may carry a digit: the positional semirings MIN_FIRSTI1 ... TIMES_SECONDJ1 (semiring.py:87-93 of the reference)
_semiring_re = re.compile(rf"^(?:GrB|GxB)_([A-Z]+)_([A-Z][A-Z0-9]*)_(?:SEMIRING_)?({_T})$")
_skip_binop_prefix = ("Matrix", "Vector", "Monoid", "DESC", "ONEB")

binaryops, monoids, semirings, unaryops = {}, {}, {}, {}


def _attach(typ_name, attr, obj):
    t = types.by_name(typ_name)
    setattr(t, attr, obj)
    setattr(t, attr.lower(), obj)


def _discover():
    names = dir(lib)
    for n in names:
        m = _binop_re.match(n)
        if m and not m.group(1).startswith(_skip_binop_prefix):
            obj = getattr(lib, n)
            if ffi.typeof(obj).cname != "struct GB_BinaryOp_opaque *":
                continue
            b = BinaryOp(m.group(1), m.group(2), obj)
            binaryops[b.name] = b
            _attach(m.group(2), m.group(1), b)
    for n in names:
        m = _binop_re.match(n)
        if m and ffi.typeof(getattr(lib, n)).cname == "struct GB_UnaryOp_opaque *":
            u = UnaryOp(m.group(1), m.group(2), getattr(lib, n))
            unaryops[u.name] = u
            _attach(m.group(2), m.group(1), u)
    for n in names:
        for r in _monoid_res:
            m = r.match(n)
            if m:
                op = "EQ" if m.group(1) == "LXNOR" else m.group(1)
                mo = Monoid(op, m.group(2), getattr(lib, n))
                monoids[mo.name] = mo
                _attach(m.group(2), m.group(1) + "_MONOID", mo)
    for n in names:
        m = _semiring_re.match(n)
        if m and ffi.typeof(getattr(lib, n)).cname == "struct GB_Semiring_opaque *":
            pls = "EQ" if m.group(1) == "LXNOR" else m.group(1)
            s = Semiring(pls, m.group(2), m.group(3), getattr(lib, n))
            semirings[s.name] = s
            _attach(m.group(3), f"{m.group(1)}_{m.group(2)}", s)


_discover()
