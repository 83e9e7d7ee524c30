#!/usr/bin/env python
"""Unmasked and complemented-mask mxm on matrices with 2^32 or more entries (the wide route of the esc / spa / spa-split bins:
row panels of A and M', B's 64-bit offsets), in one command.

1. The cost of the wide route where both routes run, on R-MAT graphs, narrow and forced wide (B200_debug_wide_gemm(2^27))
   alternated on the same inputs, medians over repeated calls, outputs compared: the unmasked C = A (+.second) A in FP32 at
   scale 17, and the mxm calls of the multi-source BFS sweep F<!V, R> = F any.pair A with k = 64 sources at scale 22 (device
   time of the mxm calls alone, summed over the levels, as tools/msbfs_bench.py has it).
2. The three calls of tests/test_wide_gemm_gpu.py on A = kron(G, J) (2^24 rows, 2^32 + 2^26 entries, UINT8): the coarsening
   product A (+.times) P, the wide right operand P' (+.times) A, and the mxm calls of the 16-source BFS sweep to its last level:
   time, products per second and the observed peak of device memory.

    python tools/wide_gemm_bench.py [--reps 5] [--skip-rmat] [--skip-large]

Prints one JSON line per measurement, with the card's name and power limit."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch
import pygraphblas_b200 as gb
from pygraphblas_b200 import Matrix, descriptor, ffi, lib
from pygraphblas_b200.generators import rmat_csr
from wide_spmv_bench import card, stream, timed


def stats():
    f, o = ffi.new("uint64_t*"), ffi.new("uint64_t*")
    lib.B200_last_mxm_stats(f, o)
    return int(f[0]), int(o[0])


def kernels():
    return ffi.string(lib.B200_debug_last_kernel()).decode()


def msbfs(A, n, sources, s):
    """F<!V, R> = F any.pair A from the sources to the last level; returns (V, summed products, summed device time of the mxm
    calls alone in ms: the V updates and the F.nvals reads are not the route under test)"""
    k = len(sources)
    F = Matrix.from_lists(list(range(k)), [int(x) for x in sources], [True] * k, k, n, gb.BOOL)
    V = F.dup()
    products, ms = 0, 0.0
    while True:
        Fn = Matrix.sparse(gb.BOOL, k, n)
        ms += timed(lambda: F.mxm(A, semiring=gb.BOOL.ANY_PAIR, out=Fn, mask=V, desc=descriptor.RSC), 1, s)[0]
        products += stats()[0]
        F = Fn
        if F.nvals == 0:
            return V, products, ms
        V.eadd(F, gb.BOOL.LOR, out=V)


def narrow_vs_wide(name, call, reps, s, info):
    """call() returns (result, products, device ms of the mxm calls or None: then the whole call is timed)"""
    out, times, kern, prod = {}, {False: [], True: []}, {}, {}

    def run(wide):
        lib.B200_debug_wide_gemm((1 << 27) if wide else 0, 0, 0)
        out[wide], prod[wide], ms = call()
        return ms

    for wide in (False, True):
        run(wide)
        lib.B200_device_synchronize()
        kern[wide] = kernels()
    for _ in range(reps):
        for wide in (False, True):
            box = {}
            whole = timed(lambda: box.update(ms=run(wide)), 1, s)
            times[wide].append(box["ms"] if box["ms"] is not None else whole[0])
    lib.B200_debug_wide_gemm(0, 0, 0)
    same = all(np.array_equal(x, y) for x, y in zip(out[False].to_arrays(), out[True].to_arrays()))
    for wide in (False, True):
        ms = float(np.median(times[wide]))
        print(json.dumps({**info, "case": f"{name}-{'wide' if wide else 'narrow'}", "products": prod[wide], "median_ms": round(ms, 3),
                          "min_ms": round(min(times[wide]), 3), "max_ms": round(max(times[wide]), 3),
                          "Gproducts_per_s": round(prod[wide] / ms / 1e6, 2), "kernels_last_call": kern[wide],
                          "outputs_identical": same}), flush=True)


def rmat(reps, s, info):
    n, indptr, indices = rmat_csr(17, 16, seed=1)
    A = Matrix.from_csr(indptr, indices, np.ones(len(indices), np.float32), n, n, gb.FP32)

    def second():
        C = A.mxm(A, semiring=gb.FP32.PLUS_SECOND)
        return C, stats()[0], None
    narrow_vs_wide("s17-plus-second", second, reps, s, info)
    del A
    n, indptr, indices = rmat_csr(22, 16, seed=1)
    Ab = Matrix.from_csr(indptr, indices, np.ones(len(indices), bool), n, n, gb.BOOL)
    sources = np.argsort(-np.diff(indptr), kind="stable")[:64]
    narrow_vs_wide("s22-msbfs-k64", lambda: msbfs(Ab, n, sources, s), reps, s, info)


def large(s, info):
    import test_wide_gemm_gpu as t
    free0 = torch.cuda.mem_get_info()[0]
    if free0 < t.PLANNED + 2e9:
        print(json.dumps({**info, "case": "wide-kron", "result": "not measured", "reason": f"{free0 / 1e9:.1f} GB free"}), flush=True)
        return
    G, J = t.factor(1, t.NG, t.NNZ_G), t.factor(2, t.NJ, t.NNZ_J)
    A = t.kron(G, J, "UINT8")
    low = [torch.cuda.mem_get_info()[0]]
    PG, PJ = t.one_hot(3, t.NG), t.one_hot(4, t.NJ)
    P = t.kron(PG, PJ, "UINT8")
    PGt, PJt = PG.T.tocsr(), PJ.T.tocsr()
    PGt.sort_indices(); PJt.sort_indices()
    Pt = t.kron(PGt, PJt, "UINT8")
    rng = np.random.default_rng(9)
    sources = rng.integers(0, t.NG, t.SOURCES).astype(np.int64) * t.NJ + rng.integers(0, t.NJ, t.SOURCES)
    box = {}

    def ap():
        box["C"] = A.mxm(P, semiring=gb.UINT8.PLUS_TIMES)
        box["p"] = stats()[0]

    def pta():
        box["C"] = Pt.mxm(A, semiring=gb.UINT8.PLUS_TIMES)
        box["p"] = stats()[0]

    def bfs():
        box["C"], box["p"], box["mxm_ms"] = msbfs(A, t.n, sources, s)

    for name, fn in (("wide-kron-a-p", ap), ("wide-kron-pt-a", pta), ("wide-kron-msbfs16", bfs)):
        ms = timed(fn, 1, s)[0]
        low.append(torch.cuda.mem_get_info()[0])
        nvals, products, kern = box["C"].nvals, box["p"], kernels()
        ms = box.get("mxm_ms", ms)                  # the BFS: its mxm calls alone
        box.clear()
        print(json.dumps({**info, "case": name, "n": t.n, "nnz": t.NNZ, "products": products, "ms": round(ms, 1),
                          "Gproducts_per_s": round(products / ms / 1e6, 2), "nvals_C": nvals, "kernels_last_call": kern,
                          "observed_peak_GB": round((free0 - min(low)) / 1e9, 1), "planned_peak_GB": round(t.PLANNED / 1e9, 1)}),
              flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--skip-large", action="store_true")
    ap.add_argument("--skip-rmat", action="store_true")
    a = ap.parse_args()
    if not gb.have_device():
        sys.exit("wide_gemm_bench: no CUDA device")
    s = stream()
    info = card()
    if not a.skip_rmat:
        rmat(a.reps, s, info)
    if not a.skip_large:
        large(s, info)


if __name__ == "__main__":
    main()
