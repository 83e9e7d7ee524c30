"""CPU: GrB_mxm with two full dense-form operands, the tiled semiring GEMM (DESIGN.md section 3.6, "Two full dense operands").
The routing rule restated (the SDDMM rule of test_sddmm.py, then the gemm branch), the call shapes C = X (+).(x) Y and
C = X (+).(x) Y' keeping every argument check ahead of the device check and ending in GrB_PANIC without a device, and the SASS
of the kernels: the specialised instantiations are exactly the SpMV fast list, never contract the multiply into the fold's add,
and keep nothing in local memory."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import pygraphblas_b200 as gb
from pygraphblas_b200 import Matrix, descriptor, ffi, lib
from test_sddmm import route as sddmm_route

NULL = ffi.NULL
INT32_MAX = (1 << 31) - 1
LIB = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pygraphblas_b200", "libb200grb.so")


# ------------------------------------------------------------------ the routing rule
def route(a_dense, b_dense, mask, mask_comp=False, mask_dense=False, positional=False, a_pres=False, b_pres=False, am=8, bn=8):
    """The route GrB_mxm takes for a builtin semiring on non-hypersparse operands, as far as the dense forms decide it: SDDMM
    first (a sparse non-complemented mask), then the GEMM for two dense forms without presence bytes and a result of at most
    2^31-1 positions."""
    r = sddmm_route(a_dense, b_dense, mask, mask_comp, mask_dense, positional)
    if r != "other" or (a_dense and b_dense and mask and not mask_comp and not mask_dense):
        return r
    if a_dense and b_dense and not a_pres and not b_pres and am * bn <= INT32_MAX:
        return "gemm"
    return "other"


def test_routing_rule():
    full = {"a_dense": True, "b_dense": True}
    assert route(**full, mask=False) == "gemm"
    # presence bytes on A, on B, on both
    for kw in ({"a_pres": True}, {"b_pres": True}, {"a_pres": True, "b_pres": True}):
        assert route(**full, mask=False, **kw) == "other", kw
    # every kind of mask: a sparse non-complemented one stays on SDDMM, the others take the GEMM
    assert route(**full, mask=True) == "sddmm"
    assert route(**full, mask=True, mask_comp=True) == "gemm"
    assert route(**full, mask=True, mask_dense=True) == "gemm"
    assert route(**full, mask=True, mask_dense=True, mask_comp=True) == "gemm"
    # positional semirings are rewritten first
    assert route(**full, mask=False, positional=True) == "positional"
    # the size of the result: 2^31-1 positions fit a dense form, 2^31 do not
    assert route(**full, mask=False, am=INT32_MAX, bn=1) == "gemm"
    assert route(**full, mask=False, am=1 << 16, bn=(1 << 15)) == "other"
    assert route(**full, mask=False, am=1 << 31, bn=1) == "other"
    # one CSR operand
    assert route(True, False, False) == "other" and route(False, True, False) == "other"


# ------------------------------------------------------------------ the call shapes without a device
@ffi.callback("void(void*, const void*, const void*)")
def _user_fn(z, x, y):
    pass


def _call(C, M, A, B, semiring=None, accum=NULL, desc=None):
    return lib.GrB_mxm(C._matrix[0] if C is not None else NULL, M._matrix[0] if M is not None else NULL, accum,
                       semiring if semiring is not None else gb.FP32.MIN_PLUS.get_op(),
                       A._matrix[0] if A is not None else NULL, B._matrix[0] if B is not None else NULL,
                       desc.get_desc() if desc is not None else NULL)


@pytest.mark.parametrize("tran1", [False, True])
def test_every_check_comes_before_the_device_check(tran1):
    m, n, k = 5, 7, 3
    X = Matrix.from_lists([0, 4], [0, 2], [1.0, 2.0], m, k, gb.FP32)
    Y = Matrix.from_lists([0, 6], [1, 2], [1.0, 2.0], n, k, gb.FP32) if tran1 else \
        Matrix.from_lists([0, 2], [1, 6], [1.0, 2.0], k, n, gb.FP32)
    d = descriptor.T1 if tran1 else None
    C = Matrix.sparse(gb.FP32, m, n)
    assert _call(None, None, X, Y, desc=d) == lib.GrB_NULL_POINTER
    assert _call(C, None, None, Y, desc=d) == lib.GrB_NULL_POINTER
    assert _call(C, None, X, None, desc=d) == lib.GrB_NULL_POINTER
    assert _call(C, None, X, Y, desc=descriptor.T0 if tran1 else descriptor.T1) == lib.GrB_DIMENSION_MISMATCH
    assert _call(Matrix.sparse(gb.FP32, m, k), None, X, Y, desc=d) == lib.GrB_DIMENSION_MISMATCH
    assert _call(C, Matrix.sparse(gb.BOOL, n, m), X, Y, desc=descriptor.C & d if d else descriptor.C) == lib.GrB_DIMENSION_MISMATCH
    op = ffi.new("GrB_BinaryOp*")
    assert lib.GrB_BinaryOp_new(op, _user_fn, lib.GrB_FP32, lib.GrB_FP32, lib.GrB_FP32) == lib.GrB_SUCCESS
    sr = ffi.new("GrB_Semiring*")
    assert lib.GrB_Semiring_new(sr, lib.GrB_MIN_MONOID_FP32, op[0]) == lib.GrB_SUCCESS
    try:
        assert _call(C, None, X, Y, semiring=sr[0], desc=d) == lib.GrB_INVALID_VALUE
        assert _call(C, None, X, Y, accum=op[0], desc=d) == lib.GrB_INVALID_VALUE
        assert _call(Matrix.sparse(gb.INT64, m, n), None, X, Y, accum=lib.GxB_FIRSTI_INT64, desc=d) == lib.GrB_DOMAIN_MISMATCH
    finally:
        lib.GrB_Semiring_free(sr); lib.GrB_BinaryOp_free(op)
    assert C.nvals == 0


def test_the_valid_call_panics_without_a_device():
    if gb.have_device():
        pytest.skip("a GPU is present: the call computes (tests/test_gemm_gpu.py)")
    X = Matrix.from_lists([0, 4], [0, 2], [1.0, 2.0], 5, 3, gb.FP32)
    Y = Matrix.from_lists([0, 6], [1, 2], [1.0, 2.0], 7, 3, gb.FP32)
    for desc, mask in ((descriptor.T1, None), (descriptor.CT1, Matrix.from_lists([0], [0], [True], 5, 7, gb.BOOL))):
        with pytest.raises(gb.base.Panic) as e:
            X.mxm(Y, semiring=gb.FP32.MIN_PLUS, mask=mask, desc=desc, out=Matrix.sparse(gb.FP32, 5, 7))
        assert "no CPU fallback" in str(e.value)


# ------------------------------------------------------------------ the SASS of the kernels
@pytest.fixture(scope="module")
def gemm_sass():
    """{demangled name: SASS lines} of every gemm_kernel and sddmm_kernel instantiation in the built library."""
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    filt = shutil.which("c++filt")
    if not os.path.exists(exe) or not os.path.exists(LIB) or not filt:
        pytest.skip("cuobjdump, c++filt or the built library is not available")
    text = subprocess.run([exe, "-sass", LIB], capture_output=True, text=True, timeout=600).stdout
    funcs, name = {}, None
    for line in text.splitlines():
        f = re.search(r"Function : (\S+)", line)
        if f:
            name = f.group(1) if re.match(r"_Z\d+(gemm|sddmm)_kernelI", f.group(1)) else None
            if name:
                funcs[name] = []
            continue
        if name:
            funcs[name].append(line)
    if not funcs:
        pytest.skip("no SASS found in the library")
    names = list(funcs)
    dem = subprocess.run([filt], input="\n".join(names), capture_output=True, text=True).stdout.split("\n")
    return {d: funcs[n] for n, d in zip(names, dem)}


def _inst(name):
    """(kernel, x type, z type, add, mul) of a demangled instantiation."""
    m = re.match(r"void (\w+)<([\w ]+), ([\w ]+), (-?\d+), (-?\d+)>", name)
    return m.group(1), m.group(2), m.group(3), int(m.group(4)), int(m.group(5))


def test_specialised_instantiations_are_the_fast_list(gemm_sass):
    insts = [_inst(n) for n in gemm_sass]
    gemm = {(x, a, m) for k, x, z, a, m in insts if k == "gemm_kernel" and a >= 0}
    sddmm = {(x, a, m) for k, x, z, a, m in insts if k == "sddmm_kernel" and a >= 0}
    assert len(gemm) == 47 and gemm == sddmm
    by_type = {}
    for x, a, m in gemm:
        by_type.setdefault(x, set()).add((a, m))
    assert sorted(len(v) for v in by_type.values()) == [5] + [7] * 6
    numeric = [v for t, v in by_type.items() if t != "bool"]
    assert all(v == numeric[0] for v in numeric)
    # the run-time operator codes: one instantiation per domain of GB_FOR_DOMAINS
    assert len({(x, z) for k, x, z, a, m in insts if k == "gemm_kernel" and a < 0}) == 21


def test_no_contraction_in_the_specialised_fp_kernels(gemm_sass):
    """FP32 / FP64 products are rounded before they are folded: no FFMA / DFMA.  (The run-time instantiations fold with the
    same explicitly rounded add; their divide and pow are FFMA sequences of their own, so only the specialised ones are
    scanned.)"""
    seen = 0
    for name, lines in gemm_sass.items():
        k, x, z, a, m = _inst(name)
        if k != "gemm_kernel" or a < 0 or x not in ("float", "double"):
            continue
        seen += 1
        op = "FFMA" if x == "float" else "DFMA"
        bad = [ln.strip() for ln in lines if re.search(rf"\b{op}\b", ln)]
        assert not bad, f"{name}: {bad[:3]}"
    assert seen == 14


def test_no_local_memory_in_the_specialised_kernels(gemm_sass):
    bad = [f"{n}: {ln.strip()}" for n, lines in gemm_sass.items() if _inst(n)[0] == "gemm_kernel" and _inst(n)[3] >= 0
           for ln in lines if re.search(r"\b(LDL|STL)\b", ln)]
    assert not bad, "\n".join(bad[:10])
