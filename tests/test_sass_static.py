"""Static checks on the SASS of the built library (no GPU needed: cuobjdump reads the cubin in libb200grb.so).

1. The TMA-staged SpMV kernel (spmv_run.cuh) must keep its WAR guard: in every instantiation, between the mbarrier wait of a run
   (SYNCS.PHASECHK...TRYWAIT) and the bulk copy of the NEXT run into the same stage (UBLKCP) there is a warp vote that reads the
   words just loaded from the stage -- without it the copy can overtake shared-memory loads that were only issued (DESIGN.md 3.1).
2. The library is sm_90a code using the bulk-copy / mbarrier instructions DESIGN.md claims (UBLKCP, SYNCS.ARRIVE.TRANS64).
3. No floating-point atomic or reduction flushes a subnormal: on sm_90 atomicAdd(float *) on a global address compiles to
   RED.E.ADD.F32.FTZ, which turns a subnormal product or partial sum into 0 where every other path (and the CPU) keeps it.
   The library issues that reduction only behind a magnitude test, |v| >= 2^-100, where the flush provably cannot change
   the sum (spgemm.cu, atomic_combine), and falls back to a compare-and-swap loop otherwise.  So every FP32 FTZ atomic
   must be preceded in its function by that test and the function must hold the CAS loop; FTZ atomics of other widths
   are not allowed at all.  Only atomics are checked: the cubin has many legitimate .FTZ opcodes (F2I.FTZ in integer
   division, FSETP.*.FTZ).
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pygraphblas_b200", "libb200grb.so")


@pytest.fixture(scope="module")
def sass_text():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe) or not os.path.exists(LIB):
        pytest.skip("cuobjdump or the built library is not available")
    out = subprocess.run([exe, "-sass", LIB], capture_output=True, text=True, timeout=600).stdout
    if "Function : " not in out:
        pytest.skip("no SASS found in the library")
    return out


@pytest.fixture(scope="module")
def hot2_sass(sass_text):
    funcs, name = {}, None
    for line in sass_text.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            continue
        if name and "spmv_run_hot2_kernel" in name:
            m = re.search(r"/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_.]*)", line)
            if m:
                funcs.setdefault(name, []).append(m.group(1))
    if not funcs:
        pytest.skip("no SASS found in the library")
    return funcs


def test_every_hot2_instantiation_keeps_the_stage_guard(hot2_sass):
    assert len(hot2_sass) == 47                       # the specialised semirings: 7 on each of the 6 numeric types, 5 on BOOL
    for name, ops in hot2_sass.items():
        waits = [i for i, o in enumerate(ops) if o.startswith("SYNCS.PHASECHK")]
        copies = [i for i, o in enumerate(ops) if o.startswith("UBLKCP")]
        votes = [i for i, o in enumerate(ops) if o.startswith("VOTE.")]
        assert waits and copies, name
        guarded = 0
        for u in copies:
            before = [w for w in waits if w < u]
            if not before:
                continue                              # prologue: the table and the first run, nothing has been read yet
            w = before[-1]
            assert any(w < v < u for v in votes), f"{name}: bulk copy at instruction {u} follows the wait at {w} without the vote"
            guarded += 1
        assert guarded >= 1, name


def test_the_kernel_uses_bulk_copies_and_transaction_barriers(hot2_sass):
    for name, ops in hot2_sass.items():
        assert any(o.startswith("UBLKCP") for o in ops) and any(o.startswith("SYNCS.ARRIVE.TRANS64") for o in ops), name


FP_ATOMIC_FTZ = re.compile(r"\b(?:RED|ATOM)[A-Z]*\.[A-Z0-9_.]*\bF(16|32|64)\b[A-Z0-9_.]*\.FTZ\b|\b(?:RED|ATOM)[A-Z]*\.[A-Z0-9_.]*\.FTZ\.[A-Z0-9_.]*\bF(16|32|64)\b")
FP_ATOMIC = re.compile(r"\b(?:RED|ATOM)[A-Z]*\.[A-Z0-9_.]*\.F(?:32|64)\b")
GUARD_2M100 = re.compile(r"FSETP\.[A-Z.]+ P\d+, PT, \|R\d+\|(?:\.reuse)?, 7\.88860905221011\d*e-31")     # |v| >= 2^-100
CAS = re.compile(r"\bATOMG?\.E\.CAS\b")


def test_no_floating_point_atomic_flushes_subnormals(sass_text):
    funcs, name = {}, None
    for line in sass_text.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            continue
        if name:
            funcs.setdefault(name, []).append(line)
    bad, fp_atomics, guarded = [], 0, 0
    for name, lines in funcs.items():
        guards = [i for i, ln in enumerate(lines) if GUARD_2M100.search(ln)]
        has_cas = any(CAS.search(ln) for ln in lines)
        for i, ln in enumerate(lines):
            if FP_ATOMIC.search(ln):
                fp_atomics += 1
            m = FP_ATOMIC_FTZ.search(ln)
            if not m:
                continue
            width = m.group(1) or m.group(2)
            if width == "32" and has_cas and any(g < i for g in guards):
                guarded += 1
                continue
            bad.append(f"{name}: {ln.strip()}")
    assert fp_atomics > 0                             # the pattern sees the atomics (FP64 PLUS combines: RED.E.ADD.F64.RN)
    assert not bad, "floating-point atomics that can flush subnormals to zero:\n" + "\n".join(bad[:20])
    assert guarded > 0                                # the guarded FP32 reductions of the dense accumulator and the streamed masked kernel
