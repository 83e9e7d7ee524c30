"""CPU: the pull route of a complemented-mask mxm (DESIGN.md section 3.2) -- GxB_AxB_METHOD on descriptors, the no-device
refusal of a GxB_AxB_DOT call, the per-row rule restated, and the compiled pull kernels (no local memory)."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import pygraphblas_b200 as gb
from pygraphblas_b200 import Matrix, descriptor, lib
from pygraphblas_b200.descriptor import Descriptor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pygraphblas_b200", "libb200grb.so")
PULL_MONOIDS = ("LOR", "LAND", "ANY")
MXM_PULL_LONG = 128                 # op(B)' rows longer than this are walked by a warp, shorter ones by a lane


def pull_rows(flops, blocked, ncols, bnnz, method="DEFAULT", alpha=0.0):
    """The rows of an eligible call that pull (spgemm_pull.cu, pull_pick_kernel): with GxB_AxB_DOT every row with products;
    with the default descriptor the rows where alpha > 0 and alpha * flops_i * ncols >= open_i * nnz(op(B)), open_i the
    columns M'(i,:) leaves open -- Beamer's m_f > m_u / alpha with m_u estimated per row; never under another method."""
    flops = np.asarray(flops, np.int64)
    open_ = ncols - np.asarray(blocked, np.int64)
    if method == "DOT":
        return flops > 0
    if method != "DEFAULT" or alpha <= 0:
        return np.zeros(len(flops), bool)
    return (flops > 0) & (alpha * flops.astype(np.float64) * float(ncols) >= open_.astype(np.float64) * float(bnnz))


def axb(method):
    """A descriptor with only GxB_AxB_METHOD set (None: the default descriptor)."""
    d = Descriptor()
    if method != "DEFAULT":
        d[lib.GxB_AxB_METHOD] = getattr(lib, f"GxB_AxB_{method}")
    return d


def test_axb_method_set_get_and_combine():
    d = axb("DOT")
    assert d[lib.GxB_AxB_METHOD] == lib.GxB_AxB_DOT
    for name in ("RSC", "C", "SCT1"):
        base = getattr(descriptor, name)
        for both in (base & d, d & base):
            assert both[lib.GxB_AxB_METHOD] == lib.GxB_AxB_DOT
            for f in (lib.GrB_INP0, lib.GrB_INP1, lib.GrB_MASK, lib.GrB_OUTP):
                assert both[f] == base[f]
        assert (base & d) != base and (base & axb("DEFAULT")) == base
    assert (axb("SAXPY") & d)[lib.GxB_AxB_METHOD] == lib.GxB_AxB_DOT        # the right operand's setting wins
    assert (d & axb("HASH"))[lib.GxB_AxB_METHOD] == lib.GxB_AxB_HASH
    assert descriptor.RSC[lib.GxB_AxB_METHOD] == lib.GxB_DEFAULT


@pytest.mark.skipif(gb.have_device(), reason="checks the no-device refusal")
def test_dot_calls_without_a_device_panic():
    F = Matrix.from_lists([0, 1], [1, 2], [True, True], 2, 4, gb.BOOL)
    A = Matrix.from_lists([1, 2], [2, 3], [True, True], 4, 4, gb.BOOL)
    V = F.dup()
    for sr in (gb.BOOL.ANY_PAIR, gb.BOOL.LOR_LAND):
        with pytest.raises(gb.base.Panic):
            F.mxm(A, semiring=sr, out=F, mask=V, desc=descriptor.RSC & axb("DOT"))


def test_the_rule_on_hand_made_rows():
    # ncols 100 and nnz(op(B)) 400: an open column costs about 4 probes
    flops = [0, 99, 100, 100, 10, 9, 5000, 1]
    blocked = [0, 0, 0, 0, 90, 90, 100, 99]
    got = pull_rows(flops, blocked, 100, 400, "DEFAULT", 4.0)
    # 4 * 100 * 100 >= 100 * 400 (equality pulls); 4 * 10 * 100 >= 10 * 400; a fully blocked row with products pulls
    assert got.tolist() == [False, False, True, True, True, False, True, True]
    assert pull_rows(flops, blocked, 100, 400, "DEFAULT", 0.0).tolist() == [False] * 8
    assert pull_rows(flops, blocked, 100, 400, "DOT").tolist() == [f > 0 for f in flops]
    for m in ("SAXPY", "GUSTAVSON", "HASH"):
        assert not pull_rows(flops, blocked, 100, 400, m, 4.0).any()
    # a larger alpha takes more rows
    assert pull_rows(flops, blocked, 100, 400, "DEFAULT", 8.0).tolist() == [False, True, True, True, True, True, True, True]


@pytest.fixture(scope="module")
def pull_sass():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe) or not os.path.exists(LIB):
        pytest.skip("cuobjdump or the built library is not available")
    out = subprocess.run([exe, "-sass", LIB], capture_output=True, text=True, timeout=600).stdout
    funcs, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            continue
        if name and re.search(r"pull_(pick|bits|count|fill|fill_pair)_kernel", name):
            funcs.setdefault(name, []).append(line)
    if not funcs:
        pytest.skip("no SASS found in the library")
    return funcs


def test_pull_kernels_use_no_local_memory(pull_sass):
    fills = [n for n in pull_sass if "pull_fill_kernel" in n]
    assert len(fills) == 21                         # the (x, z) domains: z = x on the 11 types, z = BOOL on the 10 others
    assert any("pull_fill_pair_kernel" in n for n in pull_sass) and any("pull_count_kernel" in n for n in pull_sass)
    for name, lines in pull_sass.items():
        bad = [ln.strip() for ln in lines if re.search(r"\b(LDL|STL)\b", ln)]
        assert not bad, f"{name} uses local memory: {bad[:3]}"
