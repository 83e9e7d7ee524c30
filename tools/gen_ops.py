#!/usr/bin/env python
"""Generate the builtin-operator tables of libb200grb.

GraphBLAS exposes its builtin binary ops / monoids / semirings as *global
handles* (``extern GrB_Semiring GrB_PLUS_TIMES_SEMIRING_FP32;`` ...).  The
reference discovers them by regex over ``dir(lib)``
(reference: pygraphblas/semiring.py:87-129, monoid.py:81-102,
binaryop.py:104-121), so the C-ABI must export one symbol per operator.
There are ~2000 of them; all are (opcode, type) pairs, so both the header
declarations and the definitions are generated here:

    include/b200grb_ops.h                    extern declarations (C ABI)
    pygraphblas_b200/csrc/ops_table.inc      definitions (included by objects.cu)

Run:  python tools/gen_ops.py
"""
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

INTS = ["INT8", "INT16", "INT32", "INT64"]
UINTS = ["UINT8", "UINT16", "UINT32", "UINT64"]
FLOATS = ["FP32", "FP64"]
NONBOOL = INTS + UINTS + FLOATS
ALL = ["BOOL"] + NONBOOL

# binary ops with z type == x type, for every type
GRB_ARITH = ["FIRST", "SECOND", "MIN", "MAX", "PLUS", "MINUS", "TIMES", "DIV"]
GXB_ARITH = ["PAIR", "ANY", "RMINUS", "RDIV", "POW", "ISEQ", "ISNE", "ISGT",
             "ISLT", "ISGE", "ISLE", "LOR", "LAND", "LXOR"]
CMP = ["EQ", "NE", "GT", "LT", "GE", "LE"]          # z = BOOL
BITWISE = ["BOR", "BAND", "BXOR", "BXNOR"]            # integer types only

binops = []      # (symbol, opcode, xtype, ztype)
binop_sym = {}   # (op, type) -> canonical symbol


def add_binop(sym, op, xt, zt):
    binops.append((sym, op, xt, zt))
    binop_sym.setdefault((op, xt), sym)


for t in ALL:
    for op in GRB_ARITH:
        add_binop(f"GrB_{op}_{t}", op, t, t)
    for op in GXB_ARITH:
        add_binop(f"GxB_{op}_{t}", op, t, t)
    for op in CMP:
        add_binop(f"GrB_{op}_{t}", op, t, "BOOL")
for t in INTS + UINTS:
    for op in BITWISE:
        add_binop(f"GrB_{op}_{t}", op, t, t)
# un-suffixed boolean ops of the C API
for op in ["LOR", "LAND", "LXOR"]:
    add_binop(f"GrB_{op}", op, "BOOL", "BOOL")
add_binop("GrB_LXNOR", "EQ", "BOOL", "BOOL")
for t in ALL:  # v2.0 name of PAIR; harmless extra
    add_binop(f"GrB_ONEB_{t}", "PAIR", t, t)
# positional operators (SuiteSparse v4 names, INT32 / INT64 only): z is an index of where x / y sit, their values are never
# read.  x = y = z = the index type, so that the object has no NULL type (the reference prints only the ztype).
POSITIONAL = ["FIRSTI", "FIRSTI1", "FIRSTJ", "FIRSTJ1", "SECONDI", "SECONDI1", "SECONDJ", "SECONDJ1"]
POS_T = ["INT32", "INT64"]
for t in POS_T:
    for op in POSITIONAL:
        add_binop(f"GxB_{op}_{t}", op, t, t)

monoids = []     # (symbol, op, type)
monoid_sym = {}  # (op, type) -> canonical symbol


def add_monoid(sym, op, t):
    monoids.append((sym, op, t))
    monoid_sym.setdefault((op, t), sym)


for t in NONBOOL:
    for op in ["MIN", "MAX", "PLUS", "TIMES"]:
        add_monoid(f"GrB_{op}_MONOID_{t}", op, t)
        add_monoid(f"GxB_{op}_{t}_MONOID", op, t)
    add_monoid(f"GxB_ANY_{t}_MONOID", "ANY", t)
for t in UINTS:
    for op in BITWISE:
        add_monoid(f"GxB_{op}_{t}_MONOID", op, t)
for op, code in [("LOR", "LOR"), ("LAND", "LAND"), ("LXOR", "LXOR"), ("LXNOR", "EQ")]:
    add_monoid(f"GrB_{op}_MONOID_BOOL", code, "BOOL")
for op, code in [("ANY", "ANY"), ("LOR", "LOR"), ("LAND", "LAND"), ("LXOR", "LXOR"), ("EQ", "EQ")]:
    add_monoid(f"GxB_{op}_BOOL_MONOID", code, "BOOL")

# unary operators (apply): reference: pygraphblas/unaryop.py:57-66 discovers them by regex
unops = []       # (symbol, opcode, xtype, ztype)
for t in ALL:
    for op in ["IDENTITY", "AINV", "MINV"]:
        unops.append((f"GrB_{op}_{t}", op, t, t))
    for op in ["LNOT", "ONE", "ABS"]:
        unops.append((f"GxB_{op}_{t}", op, t, t))
    unops.append((f"GrB_ABS_{t}", "ABS", t, t))
for t in INTS + UINTS:
    unops.append((f"GrB_BNOT_{t}", "BNOT", t, t))
unops.append(("GrB_LNOT", "LNOT", "BOOL", "BOOL"))
FP_UNARY = ["SQRT", "LOG", "EXP", "LOG2", "SIN", "COS", "TAN", "ACOS", "ASIN", "ATAN", "SINH", "COSH", "TANH", "ACOSH",
            "ASINH", "ATANH", "SIGNUM", "CEIL", "FLOOR", "ROUND", "TRUNC", "EXP2", "EXPM1", "LOG10", "LOG1P", "LGAMMA",
            "TGAMMA", "ERF", "ERFC"]
for t in FLOATS:
    for op in FP_UNARY:
        unops.append((f"GxB_{op}_{t}", op, t, t))
    for op in ["ISINF", "ISNAN", "ISFINITE"]:
        unops.append((f"GxB_{op}_{t}", op, t, "BOOL"))
for t in POS_T:
    for op in ["POSITIONI", "POSITIONI1", "POSITIONJ", "POSITIONJ1"]:
        unops.append((f"GxB_{op}_{t}", op, t, t))

semirings = []   # (symbol, add op, add type, mul op, mul xtype)


def add_semiring(sym, aop, atype, mop, mtype):
    semirings.append((sym, aop, atype, mop, mtype))


MULS = ["FIRST", "SECOND", "PAIR", "MIN", "MAX", "PLUS", "MINUS", "RMINUS", "TIMES",
        "DIV", "RDIV", "ISEQ", "ISNE", "ISGT", "ISLT", "ISGE", "ISLE", "LOR", "LAND", "LXOR"]
for t in NONBOOL:
    for a in ["MIN", "MAX", "PLUS", "TIMES", "ANY"]:
        for m in MULS:
            add_semiring(f"GxB_{a}_{m}_{t}", a, t, m, t)
    for a in ["LOR", "LAND", "LXOR", "EQ", "ANY"]:
        for m in CMP:
            add_semiring(f"GxB_{a}_{m}_{t}", a, "BOOL", m, t)
for a in ["LOR", "LAND", "LXOR", "EQ", "ANY"]:
    for m in ["FIRST", "SECOND", "PAIR", "LOR", "LAND", "LXOR", "EQ", "GT", "LT", "GE", "LE"]:
        add_semiring(f"GxB_{a}_{m}_BOOL", a, "BOOL", m, "BOOL")
for t in UINTS:
    for a in BITWISE:
        for m in BITWISE:
            add_semiring(f"GxB_{a}_{m}_{t}", a, t, m, t)
# C API 1.3 named semirings
for t in NONBOOL:
    for a, m in [("PLUS", "TIMES"), ("MIN", "PLUS"), ("MAX", "PLUS"), ("MIN", "TIMES"),
                 ("MIN", "MAX"), ("MAX", "MIN"), ("MAX", "TIMES"), ("PLUS", "MIN"),
                 ("MIN", "FIRST"), ("MIN", "SECOND"), ("MAX", "FIRST"), ("MAX", "SECOND")]:
        add_semiring(f"GrB_{a}_{m}_SEMIRING_{t}", a, t, m, t)
for name, a, m in [("LOR_LAND", "LOR", "LAND"), ("LAND_LOR", "LAND", "LOR"),
                   ("LXOR_LAND", "LXOR", "LAND"), ("LXNOR_LOR", "EQ", "LOR")]:
    add_semiring(f"GrB_{name}_SEMIRING_BOOL", a, "BOOL", m, "BOOL")
for t in POS_T:
    for a in ["MIN", "MAX", "ANY", "PLUS", "TIMES"]:
        for m in POSITIONAL:
            add_semiring(f"GxB_{a}_{m}_{t}", a, t, m, t)


def main():
    hdr = ["/* GENERATED by tools/gen_ops.py -- do not edit.",
           " * Builtin operator handles of the GraphBLAS C API (global objects, read as",
           " * lib.NAME by reference: pygraphblas/{binaryop,monoid,semiring}.py). */",
           "#ifndef B200GRB_OPS_H", "#define B200GRB_OPS_H"]
    for sym, *_ in binops:
        hdr.append(f"extern GrB_BinaryOp {sym};")
    for sym, *_ in monoids:
        hdr.append(f"extern GrB_Monoid {sym};")
    for sym, *_ in semirings:
        hdr.append(f"extern GrB_Semiring {sym};")
    for sym, *_ in unops:
        hdr.append(f"extern GrB_UnaryOp {sym};")
    hdr.append("#endif")
    with open(os.path.join(ROOT, "include", "b200grb_ops.h"), "w") as f:
        f.write("\n".join(hdr) + "\n")

    CT = {"BOOL": "bool", "INT8": "int8_t", "INT16": "int16_t", "INT32": "int32_t",
          "INT64": "int64_t", "UINT8": "uint8_t", "UINT16": "uint16_t", "UINT32": "uint32_t",
          "UINT64": "uint64_t", "FP32": "float", "FP64": "double"}
    th = ["/* GENERATED by tools/gen_ops.py -- do not edit.",
          " * Per-type entry points (the 17-per-type family resolved by",
          " * reference: pygraphblas/types.py:87-110, plus build). */",
          "#ifndef B200GRB_TYPED_H", "#define B200GRB_TYPED_H"]
    for t in ALL:
        c = CT[t]
        th += [
            f"GrB_Info GrB_Matrix_setElement_{t}(GrB_Matrix C, {c} x, GrB_Index i, GrB_Index j);",
            f"GrB_Info GrB_Matrix_extractElement_{t}({c} *x, const GrB_Matrix A, GrB_Index i, GrB_Index j);",
            f"GrB_Info GrB_Matrix_extractTuples_{t}(GrB_Index *I, GrB_Index *J, {c} *X, GrB_Index *nvals, const GrB_Matrix A);",
            f"GrB_Info GrB_Matrix_build_{t}(GrB_Matrix C, const GrB_Index *I, const GrB_Index *J, const {c} *X, GrB_Index nvals, const GrB_BinaryOp dup);",
            f"GrB_Info GrB_Vector_setElement_{t}(GrB_Vector w, {c} x, GrB_Index i);",
            f"GrB_Info GrB_Vector_extractElement_{t}({c} *x, const GrB_Vector v, GrB_Index i);",
            f"GrB_Info GrB_Vector_extractTuples_{t}(GrB_Index *I, {c} *X, GrB_Index *nvals, const GrB_Vector v);",
            f"GrB_Info GrB_Vector_build_{t}(GrB_Vector w, const GrB_Index *I, const {c} *X, GrB_Index nvals, const GrB_BinaryOp dup);",
            f"GrB_Info GrB_Monoid_new_{t}(GrB_Monoid *monoid, GrB_BinaryOp op, {c} identity);",
        ]
    th.append("#endif")
    with open(os.path.join(ROOT, "include", "b200grb_typed.h"), "w") as f:
        f.write("\n".join(th) + "\n")

    inc = ["// GENERATED by tools/gen_ops.py -- do not edit."]
    done = {}
    for sym, op, xt, zt in binops:
        key = (op, xt)
        if key not in done:
            done[key] = f"bop_{op}_{xt}"
            inc.append(f"static GB_BinaryOp_opaque bop_{op}_{xt} = "
                       f"{{GB_MAGIC, OP_{op}, &type_{xt}, &type_{xt}, &type_{zt}, \"{sym}\", nullptr}};")
        inc.append(f"GrB_BinaryOp {sym} = &{done[key]};")
    mdone = {}
    for sym, op, t in monoids:
        key = (op, t)
        if key not in mdone:
            mdone[key] = f"mon_{op}_{t}"
            inc.append(f"static GB_Monoid_opaque mon_{op}_{t} = "
                       f"{{GB_MAGIC, &bop_{op}_{t}, \"{sym}\", true}};")
        inc.append(f"GrB_Monoid {sym} = &{mdone[key]};")
    sdone = {}
    for sym, aop, at, mop, mt in semirings:
        key = (aop, at, mop, mt)
        if key not in sdone:
            sdone[key] = f"sr_{aop}_{mop}_{mt}"
            assert (aop, at) in mdone, (sym, aop, at)
            assert (mop, mt) in done, (sym, mop, mt)
            inc.append(f"static GB_Semiring_opaque sr_{aop}_{mop}_{mt} = "
                       f"{{GB_MAGIC, &mon_{aop}_{at}, &bop_{mop}_{mt}, \"{sym}\", true}};")
        inc.append(f"GrB_Semiring {sym} = &{sdone[key]};")
    udone = {}
    for sym, op, xt, zt in unops:
        key = (op, xt)
        if key not in udone:
            udone[key] = f"uop_{op}_{xt}"
            inc.append(f"static GB_UnaryOp_opaque uop_{op}_{xt} = {{GB_MAGIC, UOP_{op}, &type_{xt}, &type_{zt}, \"{sym}\"}};")
        inc.append(f"GrB_UnaryOp {sym} = &{udone[key]};")
    # name lookup table (B200_lookup)
    inc.append("struct GB_named { const char *name; int kind; void *obj; };")
    inc.append("static const GB_named gb_named_objects[] = {")
    for sym, op, xt, zt in binops:
        inc.append(f"  {{\"{sym}\", 0, (void*)&{done[(op, xt)]}}},")
    for sym, op, t in monoids:
        inc.append(f"  {{\"{sym}\", 1, (void*)&{mdone[(op, t)]}}},")
    for sym, aop, at, mop, mt in semirings:
        inc.append(f"  {{\"{sym}\", 2, (void*)&{sdone[(aop, at, mop, mt)]}}},")
    for sym, op, xt, zt in unops:
        inc.append(f"  {{\"{sym}\", 3, (void*)&{udone[(op, xt)]}}},")
    inc.append("  {nullptr, 0, nullptr}};")
    with open(os.path.join(ROOT, "pygraphblas_b200", "csrc", "ops_table.inc"), "w") as f:
        f.write("\n".join(inc) + "\n")
    print(f"binops={len(binops)} monoids={len(monoids)} semirings={len(semirings)} unops={len(unops)}")


if __name__ == "__main__":
    main()
