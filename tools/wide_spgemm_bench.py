#!/usr/bin/env python
"""Masked mxm on matrices with 2^32 or more entries (the wide route: row panels of A and M, B's 64-bit offsets), in one command.

1. bench.py's masked leg, C<L> = L (+.pair) L at R-MAT scale 20, on the narrow route and on the wide route (forced with
   B200_debug_wide(2^27)), alternating on the same inputs, medians over repeated calls, outputs compared bit for bit: the
   cost of the wide route where both run.
2. The Kronecker graph A = kron(G, J) of tests/test_wide_spgemm_gpu.py (2^28 rows, 2^32 + 2^26 entries, cliques planted in
   the factors), in the triangle form C<A> = A (+.pair) A in UINT32: time, products per second and the observed peak of
   device memory.

    python tools/wide_spgemm_bench.py [--reps 10] [--skip-large]

Prints one JSON line per measurement, with the card's name and power limit."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
import pygraphblas_b200 as gb
from pygraphblas_b200 import Matrix, descriptor, ffi, lib
from bench import lower_triangle
from wide_spmv_bench import card, stream, timed


def s20(reps, s, info):
    n, lp, lj = lower_triangle(20)
    L = Matrix.from_csr(lp, lj, np.ones(len(lj), np.int64), n, n, gb.INT64)
    out, times, kern = {}, {False: [], True: []}, {}

    def call(wide):
        lib.B200_debug_wide((1 << 27) if wide else 0)
        out[wide] = L.mxm(L, mask=L, semiring=gb.INT64.PLUS_PAIR, desc=descriptor.S)

    for wide in (False, True):
        for _ in range(2):
            call(wide)
        lib.B200_device_synchronize()
        kern[wide] = ffi.string(lib.B200_debug_last_kernel()).decode()
    for _ in range(reps):
        for wide in (False, True):
            times[wide] += timed(lambda: call(wide), 1, s)
    lib.B200_debug_wide(0)
    flops, nout = ffi.new("uint64_t*"), ffi.new("uint64_t*")
    lib.B200_last_mxm_stats(flops, nout)
    a, b = out[False].to_csr(), out[True].to_csr()
    same = all(np.array_equal(x, y) for x, y in zip(a, b))
    for wide in (False, True):
        ms = float(np.median(times[wide]))
        print(json.dumps({**info, "case": "s20-triangle-wide" if wide else "s20-triangle-narrow", "nnz_L": len(lj),
                          "products": int(flops[0]), "median_ms": round(ms, 3), "min_ms": round(min(times[wide]), 3),
                          "max_ms": round(max(times[wide]), 3), "Gproducts_per_s": round(flops[0] / ms / 1e6, 2),
                          "kernels": kern[wide], "outputs_bit_identical": same}), flush=True)


def large(reps, s, info):
    import test_wide_spgemm_gpu as t
    free0 = torch.cuda.mem_get_info()[0]
    if free0 < t.PLANNED + 2e9:
        print(json.dumps({**info, "case": "wide-kron-triangle", "result": "not measured", "reason": f"{free0 / 1e9:.1f} GB free"}), flush=True)
        return
    G, J = t.factor_cliques(1, t.NG, t.NNZ_G), t.factor_cliques(2, t.NJ, t.NNZ_J)
    A = t.kron(G, J, "UINT8")
    low = torch.cuda.mem_get_info()[0]
    C = Matrix.sparse(gb.UINT32, t.n, t.n)

    def call():
        A.mxm(A, mask=A, semiring=gb.UINT32.PLUS_PAIR, out=C, desc=descriptor.S)

    call()
    lib.B200_device_synchronize()
    low = min(low, torch.cuda.mem_get_info()[0])
    kern = ffi.string(lib.B200_debug_last_kernel()).decode()
    times = timed(call, reps, s)
    low = min(low, torch.cuda.mem_get_info()[0])
    flops, nout = ffi.new("uint64_t*"), ffi.new("uint64_t*")
    lib.B200_last_mxm_stats(flops, nout)
    ms = float(np.median(times))
    print(json.dumps({**info, "case": "wide-kron-triangle", "n": t.n, "nnz": t.NNZ, "products": int(flops[0]), "nnz_C": int(nout[0]),
                      "median_ms": round(ms, 1), "min_ms": round(min(times), 1), "max_ms": round(max(times), 1),
                      "Gproducts_per_s": round(flops[0] / ms / 1e6, 2), "observed_peak_GB": round((free0 - low) / 1e9, 1),
                      "planned_peak_GB": round(t.PLANNED / 1e9, 1), "kernels": kern}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--skip-large", action="store_true")
    a = ap.parse_args()
    if not gb.have_device():
        sys.exit("wide_spgemm_bench: no CUDA device")
    s = stream()
    info = card()
    s20(a.reps, s, info)
    if not a.skip_large:
        large(max(1, a.reps // 3), s, info)


if __name__ == "__main__":
    main()
