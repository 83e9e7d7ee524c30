#!/usr/bin/env python
"""Which part of the SpMV tile kernel costs what: same graph, semirings that drop the gather / the value stream."""
import os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import pygraphblas_b200 as gb
from pygraphblas_b200 import Matrix, Vector, FP32
from bench import cached_graph, spmv_inputs

scale = int(sys.argv[1]) if len(sys.argv) > 1 else 22
n, indptr, indices = cached_graph(scale)
vals, u0 = spmv_inputs(len(indices), n)
A = Matrix.from_csr(indptr, indices, vals, n, n, FP32)
u = Vector.from_numpy(u0)
w = Vector.sparse(FP32, n)
sp_ = gb.ffi.new("void**"); gb.lib.B200_get_stream(sp_)
stream = torch.cuda.ExternalStream(int(gb.ffi.cast("uintptr_t", sp_[0])))

def run(label, sr, env):
    keep_run = os.environ.get("B200GRB_SPMV_RUN")
    for k in ("B200GRB_SPMV_ITEMS", "B200GRB_SPMV_HOT", "B200GRB_HOT_GROUPS", "B200GRB_SPMV_DEBUG", "B200GRB_SPMV_RUN", "B200GRB_SPMV_PIPE",
              "B200GRB_SPMV_CLUSTER", "B200GRB_SPMV_HOT_REPL"):
        os.environ.pop(k, None)
    if keep_run is not None and "B200GRB_SPMV_RUN" not in env:
        os.environ["B200GRB_SPMV_RUN"] = keep_run
    os.environ.update(env)
    gb.lib.B200_reload_tunables()
    for _ in range(5):
        A.mxv(u, semiring=sr, out=w)
    gb.lib.B200_device_synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(30):
        A.mxv(u, semiring=sr, out=w)
    e1.record(stream)
    gb.lib.B200_device_synchronize(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 30
    print(f"{label:44s} {ms*1e3:8.1f} us", flush=True)
    return ms * 1e3

if len(sys.argv) > 2 and sys.argv[2] == "cluster":
    # hot-table kernel as clusters of C CTAs (C x T0 replicated KB x PIPE), three repetitions each; the route names the C launched
    rows = {}
    for rep in range(3):
        for C in (1, 2, 4, 8, 16):
            for t0kb in ((0, 32, 64, 96) if C > 1 else (128,)):
                for pipe in ("0", "1"):
                    us = run(f"rep {rep} C={C:2d} T0={t0kb:3d}KB pipe={pipe}", FP32.PLUS_TIMES,
                             {"B200GRB_SPMV_CLUSTER": str(C), "B200GRB_SPMV_HOT_REPL": str(t0kb), "B200GRB_SPMV_PIPE": pipe})
                    tok = dict(t.split("=", 1) for t in gb.ffi.string(gb.lib.B200_debug_last_kernel()).decode().split(";") if "=" in t)
                    rows.setdefault((C, t0kb, pipe), []).append((us, tok.get("hot-cluster", "-"), tok.get("hot-ctas", "-")))
    # launched C and the clusters of its grid.  The grid is min(cudaOccupancyMaxActiveClusters, clusters the runs fill) x C;
    # the bench graph fills far more, so on it the launched clusters are the device's co-scheduling limit
    print(" C T0KB pipe  launched  grid_ctas  clusters_launched   min_us   max_us  mean_us")
    for (C, t0kb, pipe), v in sorted(rows.items()):
        us = [x for x, _, _ in v]
        lc, ctas = v[0][1], v[0][2]
        ncl = int(ctas) // int(lc) if lc != "-" else "-"
        print(f"{C:2d} {t0kb:4d} {pipe:>4s}  {lc:>8s}  {ctas:>9s}  {ncl!s:>17s}  {min(us):7.1f}  {max(us):7.1f}  {sum(us)/len(us):7.1f}", flush=True)
    sys.exit(0)

if len(sys.argv) > 2 and sys.argv[2] == "sweep":
    for rep in range(3):
        for pipe in ("0", "1"):
            for kb in ("64", "96", "128"):
                run(f"rep {rep} pipe={pipe} table cap {kb}KB PLUS_TIMES", FP32.PLUS_TIMES, {"B200GRB_SPMV_HOT": kb, "B200GRB_SPMV_PIPE": pipe})
    run("plain run kernel (no table, no staging)", FP32.PLUS_TIMES, {"B200GRB_SPMV_HOT": "0"})
    run("default MIN_PLUS", FP32.MIN_PLUS, {})
    run("default PLUS_SECOND", FP32.PLUS_SECOND, {})
    run("PLUS_FIRST (no gather)", FP32.PLUS_FIRST, {})
    sys.exit(0)
run("default (hot table, TMA staged) PLUS_TIMES", FP32.PLUS_TIMES, {})
run("run kernel PLUS_SECOND", FP32.PLUS_SECOND, {})
run("run kernel PLUS_FIRST (no gather)", FP32.PLUS_FIRST, {})
run("run kernel PLUS_PAIR (col only)", FP32.PLUS_PAIR, {})
run("run kernel MIN_PLUS", FP32.MIN_PLUS, {})
for kb in ("0", "32", "64", "96", "128", "160"):
    run(f"run kernel + hot table {kb}KB PLUS_TIMES", FP32.PLUS_TIMES, {"B200GRB_SPMV_HOT": kb})
run("run-time operators: PLUS_MINUS", FP32.PLUS_MINUS, {})
