"""Descriptors.  Mirrors reference: pygraphblas/descriptor.py:10-182: the 27 builtin
combinations of T0/T1 (transpose input), C (complement mask), S (structural mask),
R (replace output), usable as arguments, context managers and combinable with `&`.  GxB_AxB_METHOD set on a
descriptor (GxB_AxB_DOT: the pull route of a complemented-mask mxm, DESIGN.md section 3.2) is combined the same way."""
import contextvars
from .base import lib, ffi, _check, NULL

current_desc = contextvars.ContextVar("current_desc")

_FIELDS = ("GrB_INP0", "GrB_INP1", "GrB_MASK", "GrB_OUTP", "GxB_AxB_METHOD")


class Descriptor:
    def __init__(self, desc=None, name=""):
        self._desc = ffi.new("GrB_Descriptor*")
        self._owned = desc is None
        if desc is None:
            _check(lib.GrB_Descriptor_new(self._desc))
        else:
            self._desc[0] = desc
        self.name = name
        self.token = None

    def get_desc(self):
        return self._desc[0]

    def __del__(self):
        try:
            if getattr(self, "_owned", False) and lib is not None:
                lib.GrB_Descriptor_free(self._desc)
        except Exception:
            pass

    def __getitem__(self, field):
        val = ffi.new("GrB_Desc_Value*")
        _check(lib.GxB_Desc_get(self._desc[0], field, val))
        return val[0]

    def __setitem__(self, field, value):
        _check(lib.GrB_Descriptor_set(self._desc[0], field, value))

    def __and__(self, other):
        d = Descriptor(name=self.name + other.name)
        for f in _FIELDS:
            f = getattr(lib, f)
            for src in (self, other):
                v = src[f]
                if v != lib.GxB_DEFAULT:
                    d[f] = v
        return d

    def __eq__(self, other):
        return all(self[getattr(lib, f)] == other[getattr(lib, f)] for f in _FIELDS)

    def __hash__(self):
        return hash(tuple(self[getattr(lib, f)] for f in _FIELDS))

    def __contains__(self, other):
        """True when every non-default field of `other` is set identically here.
        (The reference's version always returns True, descriptor.py:126-142; the only use on
        the hot path is `T0 in desc` for sizing mxv's output, matrix.py:2697.)"""
        for f in _FIELDS:
            f = getattr(lib, f)
            o = other[f]
            if o != lib.GxB_DEFAULT and (self[f] & o) != o and self[f] != o:
                return False
        return True

    def __enter__(self):
        self.token = current_desc.set(self)
        return self

    def __exit__(self, *errors):
        current_desc.reset(self.token)
        return False

    def __repr__(self):
        return f"<Descriptor {self.name}>"


Default = Descriptor(NULL, "Default")
__all__ = ["Descriptor", "Default", "current_desc"]
for _n in ("T1 T0 T0T1 C CT1 CT0 CT0T1 S ST1 ST0 ST0T1 SC SCT1 SCT0 SCT0T1 R RT1 RT0 RT0T1 "
           "RC RCT1 RCT0 RCT0T1 RS RST1 RST0 RST0T1 RSC RSCT1 RSCT0 RSCT0T1").split():
    globals()[_n] = Descriptor(getattr(lib, "GrB_DESC_" + _n), _n)
    __all__.append(_n)
