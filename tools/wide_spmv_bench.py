#!/usr/bin/env python
"""mxv on matrices with 2^32 or more entries (the wide route: 64-bit entry offsets), in one command.

1. A Kronecker graph A = kron(G, J) of 2^32 + 2^26 entries, formed on the device: FP32 PLUS_TIMES when the card has the
   free memory for it, else BOOL LOR_LAND.  Reports GEdge/s and algorithmic bytes over time.
2. The s22 benchmark graph on the narrow route and on the wide route (forced with B200_debug_wide), alternating, medians
   over repeated calls, outputs compared bit for bit: the cost of 64-bit offsets where both routes run.

    python tools/wide_spmv_bench.py [--reps 20] [--skip-large]

Prints one JSON line per measurement, with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import scipy.sparse as sp
import pygraphblas_b200 as gb
from pygraphblas_b200 import Matrix, Vector, ffi, lib
from bench import cached_graph, spmv_inputs


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
    except Exception:
        name, power = torch.cuda.get_device_name(), "not measured"
    return {"gpu": name, "power_limit": power}


def stream():
    p = ffi.new("void**")
    lib.B200_get_stream(p)
    return torch.cuda.ExternalStream(int(ffi.cast("uintptr_t", p[0])))


def timed(fn, reps, s):
    """Per-call device times (ms) of fn, each call between CUDA events on the library's stream."""
    out = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(s)
        fn()
        e1.record(s)
        lib.B200_device_synchronize()
        out.append(e0.elapsed_time(e1))
    return out


def factor(seed, n, nnz):
    rng = np.random.default_rng(seed)
    first = np.arange(n, dtype=np.int64) * n + rng.integers(0, n, n)
    rest = np.setdiff1d(rng.choice(n * n, nnz * 2, replace=False), first)
    keys = np.sort(np.concatenate([first, rng.choice(rest, nnz - n, replace=False)]))
    S = sp.csr_matrix((np.ones(nnz, np.float32), (keys // n, keys % n)), shape=(n, n))
    S.sort_indices()
    return S


def large(reps, s, info):
    NG = NJ = 4096
    G, J = factor(1, NG, (1 << 16) + (1 << 10)), factor(2, NJ, 1 << 16)
    nnz = G.nnz * J.nnz
    n = NG * NJ
    free = torch.cuda.mem_get_info()[0]
    # FP32: A 8 B per entry, its run plan ~0.5 and hot plan 4; BOOL: 5 + 0.5 + 4
    fp32 = free > nnz * 12.5 + 4e9
    typ = gb.FP32 if fp32 else gb.BOOL
    if not fp32 and free < nnz * 9.5 + 4e9:
        print(json.dumps({**info, "case": "wide-kron", "nnz": nnz, "result": "not measured",
                          "reason": f"{free / 1e9:.1f} GB free"}), flush=True)
        return
    mk = lambda S: Matrix.from_csr(S.indptr, S.indices, S.data.astype(typ.dtype), S.shape[0], S.shape[1], typ)
    A = Matrix.sparse(typ, n, n)
    op = (gb.FP32.TIMES if fp32 else gb.BOOL.LAND).get_op()
    Gm, Jm = mk(G), mk(J)
    gb.base._check(lib.GrB_Matrix_kronecker_BinaryOp(A._matrix[0], ffi.NULL, ffi.NULL, op, Gm._matrix[0], Jm._matrix[0], ffi.NULL))
    del Gm, Jm
    u = Vector.from_numpy(np.ones(n, typ.dtype), typ=typ)
    w = Vector.sparse(typ, n)
    sr = gb.FP32.PLUS_TIMES if fp32 else gb.BOOL.LOR_LAND
    for _ in range(3):
        A.mxv(u, semiring=sr, out=w)
    lib.B200_device_synchronize()
    kern = ffi.string(lib.B200_debug_last_kernel()).decode()
    ms = float(np.median(timed(lambda: A.mxv(u, semiring=sr, out=w), reps, s)))
    vs = 4 if fp32 else 1
    nbytes = nnz * (4 + vs) + (n + 1) * 8 + n * vs + n * (vs + 1)
    I, X = w.to_arrays()
    want = np.outer(np.diff(G.indptr), np.diff(J.indptr)).ravel()
    ok = bool(np.array_equal(I, np.arange(n)) and (np.array_equal(X, want.astype(np.float32)) if fp32 else X.all()))
    print(json.dumps({**info, "case": "wide-kron", "semiring": "FP32 PLUS_TIMES" if fp32 else "BOOL LOR_LAND", "n": n, "nnz": nnz,
                      "median_ms": round(ms, 3), "GEdge_per_s": round(nnz / ms / 1e6, 2),
                      "alg_GB_per_s": round(nbytes / ms / 1e6, 1), "kernels": kern, "result_ok": ok}), flush=True)


def s22(reps, s, info):
    n, indptr, indices = cached_graph(22)
    vals, u0 = spmv_inputs(len(indices), n)
    u = Vector.from_numpy(u0)
    A = {False: Matrix.from_csr(indptr, indices, vals, n, n, gb.FP32), True: Matrix.from_csr(indptr, indices, vals, n, n, gb.FP32)}
    W = {k: Vector.sparse(gb.FP32, n) for k in A}
    times = {False: [], True: []}
    kern = {}

    def call(wide):
        lib.B200_debug_wide(1 << 30 if wide else 0)
        A[wide].mxv(u, semiring=gb.FP32.PLUS_TIMES, out=W[wide])

    for wide in (False, True):
        for _ in range(3):
            call(wide)
        lib.B200_device_synchronize()
        kern[wide] = ffi.string(lib.B200_debug_last_kernel()).decode()
    for _ in range(reps):
        for wide in (False, True):
            times[wide] += timed(lambda: call(wide), 1, s)
    lib.B200_debug_wide(0)
    (I0, X0), (I1, X1) = W[False].to_arrays(), W[True].to_arrays()
    same = bool(np.array_equal(I0, I1) and np.array_equal(X0.view(np.uint32), X1.view(np.uint32)))
    nnz = len(indices)
    for wide in (False, True):
        ms = float(np.median(times[wide]))
        print(json.dumps({**info, "case": "s22-wide" if wide else "s22-narrow", "nnz": nnz, "median_ms": round(ms, 4),
                          "GEdge_per_s": round(nnz / ms / 1e6, 2), "kernels": kern[wide], "outputs_bit_identical": same}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--skip-large", action="store_true")
    a = ap.parse_args()
    if not gb.have_device():
        sys.exit("wide_spmv_bench: no CUDA device")
    s = stream()
    info = card()
    s22(a.reps, s, info)
    if not a.skip_large:
        large(a.reps, s, info)


if __name__ == "__main__":
    main()
