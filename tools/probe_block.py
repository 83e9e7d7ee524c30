#!/usr/bin/env python
"""Local SpMV of ONE rank's block of an N-way partition, on one GPU: which kernel shape suits a 1/N-sized matrix.
    python tools/probe_block.py [world]"""
import os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import pygraphblas_b200 as gb
from pygraphblas_b200 import Matrix, Vector, FP32
from pygraphblas_b200.distributed import local_block_scattered, to_scattered
from bench import cached_graph, spmv_inputs

world = int(sys.argv[1]) if len(sys.argv) > 1 else 8
n, indptr, indices = cached_graph(22)
vals, u0 = spmv_inputs(len(indices), n)
newid, lb, lptr, lidx, lval = local_block_scattered(indptr, indices, vals, world, 0)
A = Matrix.from_csr(lptr, lidx, lval, lb, world * lb, FP32)
u = Vector.from_numpy(to_scattered(u0, newid, world * lb))
w = Vector.sparse(FP32, lb)
sp_ = gb.ffi.new("void**"); gb.lib.B200_get_stream(sp_)
stream = torch.cuda.ExternalStream(int(gb.ffi.cast("uintptr_t", sp_[0])))
print(f"block of a {world}-way partition: {lb} rows, {len(lidx)} entries")
for label, env in (("default", {}), ("plain run kernel", {"B200GRB_SPMV_HOT": "0"}), ("table 32KB", {"B200GRB_SPMV_HOT": "32"}), ("table 64KB", {"B200GRB_SPMV_HOT": "64"})):
    os.environ.pop("B200GRB_SPMV_HOT", None)
    os.environ.update(env); gb.lib.B200_reload_tunables()
    for _ in range(10):
        A.mxv(u, semiring=FP32.PLUS_TIMES, out=w)
    gb.lib.B200_device_synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(100):
        A.mxv(u, semiring=FP32.PLUS_TIMES, out=w)
    e1.record(stream)
    gb.lib.B200_device_synchronize(); torch.cuda.synchronize()
    print(f"{label:28s} {e0.elapsed_time(e1) / 100 * 1e3:8.1f} us per local mxv", flush=True)
