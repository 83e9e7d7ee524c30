"""Model of the positional operators -- TEST INFRASTRUCTURE ONLY.

What GrB_mxm / GrB_mxv / GrB_vxm compute with a positional semiring ({MIN,MAX,ANY,PLUS,TIMES}_{FIRSTI ... SECONDJ1}) and
what apply computes with POSITIONI ... POSITIONJ1 or a bound FIRSTI ... SECONDJ1, restated from the definitions on dict
containers ({(i, j): value} for matrices, {k: value} for vectors).  mxv and vxm are the mxm of an n x 1 / 1 x n operand:

    call                     x is at          y is at         FIRSTI  FIRSTJ  SECONDI  SECONDJ
    C = op(A) op(B)          op(A)(i,k)       op(B)(k,j)      i       k       k        j
    w = op(A) u              op(A)(i,k)       u(k) = (k,0)    i       k       k        0
    w' = u' op(A)            u(k) = (0,k)     op(A)(k,j)      0       k       k        j

The ...1 forms add 1; INT32 keeps the low 32 bits of the index (a C cast); PLUS and TIMES wrap.  Mask, accumulator and
GrB_REPLACE act on T as for every other semiring: the write-back is oracle/pymodel.py's own (see `writeback`).
"""
from oracle import pymodel

POSITIONAL = ["FIRSTI", "FIRSTI1", "FIRSTJ", "FIRSTJ1", "SECONDI", "SECONDI1", "SECONDJ", "SECONDJ1"]
UNARY = ["POSITIONI", "POSITIONI1", "POSITIONJ", "POSITIONJ1"]
MONOIDS = ["MIN", "MAX", "ANY", "PLUS", "TIMES"]
TYPES = ["INT32", "INT64"]


def trunc(v, typ):
    """The Python int v as a value of typ: its low 32 / 64 bits in two's complement."""
    bits = 32 if typ == "INT32" else 64
    v &= (1 << bits) - 1
    return v - (1 << bits) if v >> (bits - 1) else v


def _split(op):
    return (op[:-1], 1) if op.endswith("1") else (op, 0)


def position(mul, i, k, j):
    """The product of mul for x at (i, k) and y at (k, j)."""
    base, off = _split(mul)
    return {"FIRSTI": i, "FIRSTJ": k, "SECONDI": k, "SECONDJ": j}[base] + off


def fold(add, typ, vals):
    vals = [trunc(v, typ) for v in vals]
    if add == "MIN":
        return min(vals)
    if add == "MAX":
        return max(vals)
    if add == "ANY":
        return vals[0]
    r = 0 if add == "PLUS" else 1
    for v in vals:
        r = trunc(r + v if add == "PLUS" else r * v, typ)
    return r


def product(add, mul, typ, A, B, tran0=False, tran1=False):
    """T = op(A) add.mul op(B) on dict matrices (values never read): T and, per entry, the set of its products (what an
    ANY fold may return)."""
    if tran0:
        A = {(j, i): v for (i, j), v in A.items()}
    if tran1:
        B = {(j, i): v for (i, j), v in B.items()}
    brows = {}
    for (k, j) in sorted(B):
        brows.setdefault(k, []).append(j)
    prods = {}
    for (i, k) in sorted(A):
        for j in brows.get(k, ()):
            prods.setdefault((i, j), []).append(position(mul, i, k, j))
    return {e: fold(add, typ, p) for e, p in prods.items()}, {e: {trunc(v, typ) for v in p} for e, p in prods.items()}


def writeback(C, ctype, M, accum, T, ttype, desc):
    """C<M> = accum(C, T) on dict matrices: pymodel.mxm's own write-back (steps 4-6), handed T as the product T . I under
    ttype's PLUS.FIRST (one product per entry, so the product is T itself).  desc: dict(replace, mask_comp, mask_struct)."""
    d = dict(replace=False, mask_comp=False, mask_struct=False)
    d.update({k: desc[k] for k in d if k in desc})
    d.update(tran0=False, tran1=False)
    eye = {(j, j): 1 for (_, j) in T}
    return pymodel.mxm(C, ctype, M, "BOOL", accum, ("PLUS", "FIRST", ttype), T, ttype, eye, ttype, d)


def _as_col(v):
    return None if v is None else {(k, 0): x for k, x in v.items()}


def _vec_writeback(w, wtype, mask, accum, T, ttype, desc):
    out = writeback(_as_col(w), wtype, _as_col(mask), accum, _as_col(T), ttype, desc)
    return {i: x for (i, _), x in out.items()}


def _desc(desc):
    d = dict(replace=False, mask_comp=False, mask_struct=False, tran0=False, tran1=False)
    d.update(desc or {})
    return d


def mxm(C, ctype, M, accum, semiring, A, B, desc=None):
    add, mul, typ = semiring
    d = _desc(desc)
    T, cands = product(add, mul, typ, A, B, d["tran0"], d["tran1"])
    return writeback(C, ctype, M, accum, T, typ, d), cands


def mxv(w, wtype, mask, accum, semiring, A, u, desc=None):
    """w<mask> = accum(w, op(A) (+).(x) u), u as an n x 1 matrix."""
    add, mul, typ = semiring
    d = _desc(desc)
    T, cands = product(add, mul, typ, A, {(k, 0): v for k, v in u.items()}, d["tran0"], False)
    T = {i: v for (i, _), v in T.items()}
    return _vec_writeback(w, wtype, mask, accum, T, typ, d), {i: c for (i, _), c in cands.items()}


def vxm(w, wtype, mask, accum, semiring, u, A, desc=None):
    """w'<mask'> = accum(w', u' (+).(x) op(A)), u' as a 1 x n matrix."""
    add, mul, typ = semiring
    d = _desc(desc)
    T, cands = product(add, mul, typ, {(0, k): v for k, v in u.items()}, A, False, d["tran1"])
    T = {j: v for (_, j), v in T.items()}
    return _vec_writeback(w, wtype, mask, accum, T, typ, d), {j: c for (_, j), c in cands.items()}


def apply_index(op, typ, i, j):
    """POSITIONI / J (unary) or FIRSTI ... SECONDJ1 bound to a scalar (ignored): the row or the column of the entry."""
    base, off = _split(op)
    return trunc((j if base.endswith("J") else i) + off, typ)


def apply(op, typ, A, tran=False):
    """T = op(op(A)) on a dict matrix, before the write-back."""
    if tran:
        A = {(j, i): v for (i, j), v in A.items()}
    return {(i, j): apply_index(op, typ, i, j) for (i, j) in A}


def apply_vector(op, typ, u):
    """A vector is a column: position k is (k, 0)."""
    return {k: apply_index(op, typ, k, 0) for k in u}
