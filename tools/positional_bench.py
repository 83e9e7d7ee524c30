#!/usr/bin/env python
"""Cost of the positional semirings against the value semirings they are rewritten onto, on the R-MAT graph of bench.py:

    mxv MIN_SECONDI_INT64   vs  MIN_SECOND_INT64    (inner form: u's values replaced by an iota, then MIN.SECOND)
    mxv PLUS_FIRSTI_INT64   vs  PLUS_PAIR_INT64     (count form: PLUS.PAIR, then one kernel turns counts into count * i)
    BFS with parents        vs  level BFS           (q'<!pi> = q' ANY.SECONDI A  against  q'<!v> = q' LOR.LAND A, BOOL A)

plus one torch.profiler split of a positional call.  Device times from CUDA events on the library's stream, medians of
--reps calls after --warmup.  python tools/positional_bench.py [--scale 22] [--reps 20] [--warmup 3]"""
import argparse
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import pygraphblas_b200 as gb
from pygraphblas_b200 import BOOL, INT64, Matrix, Vector, descriptor
from bench import cached_graph


def lib_stream():
    sp_ = gb.ffi.new("void**")
    gb.lib.B200_get_stream(sp_)
    return torch.cuda.ExternalStream(int(gb.ffi.cast("uintptr_t", sp_[0])))


def timed(stream, f, reps, warmup):
    for _ in range(warmup):
        f()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        f()
        e1.record(stream)
        gb.lib.B200_device_synchronize()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def last_kernel():
    return gb.ffi.string(gb.lib.B200_debug_last_kernel()).decode()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=int, default=22)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    n, indptr, indices = cached_graph(a.scale)
    nnz = len(indices)
    print(f"card: {card}; R-MAT scale {a.scale}: n={n} nnz={nnz}")
    stream = lib_stream()

    A = Matrix.from_csr(indptr, indices, np.ones(nnz, np.int64), n, n, INT64)
    u = Vector.from_numpy(np.ones(n, np.int64), typ=INT64)
    w = Vector.sparse(INT64, n)
    for pos, val in [(INT64.MIN_SECONDI, INT64.MIN_SECOND), (INT64.PLUS_FIRSTI, INT64.PLUS_PAIR)]:
        tp = timed(stream, lambda: A.mxv(u, semiring=pos, out=w), a.reps, a.warmup)
        kp = last_kernel()
        tv = timed(stream, lambda: A.mxv(u, semiring=val, out=w), a.reps, a.warmup)
        kv = last_kernel()
        print(f"mxv {pos.name:20s} {tp * 1e3:9.1f} us  [{kp}]")
        print(f"mxv {val.name:20s} {tv * 1e3:9.1f} us  [{kv}]   positional / value = {tp / tv:.3f}")

    # BFS: parents (ANY.SECONDI on the BOOL graph) against levels (LOR.LAND), the same source and graph
    Ab = Matrix.from_csr(indptr, indices, None, n, n, BOOL)
    src = int(np.argmax(np.diff(indptr)))

    def bfs_parents():
        parent = Vector.from_lists([src], [src], n, INT64)
        q = Vector.from_lists([src], [src], n, INT64)
        while q.nvals:
            q = q.vxm(Ab, semiring=INT64.ANY_SECONDI, mask=parent, desc=descriptor.RSC)
            parent.eadd(q, INT64.FIRST, out=parent)
        return parent

    def bfs_levels():
        q = Vector.sparse(BOOL, n); q[src] = True
        visited = Vector.sparse(BOOL, n); visited[src] = True
        while q.nvals:
            q = q.vxm(Ab, mask=visited, desc=descriptor.RC, semiring=BOOL.LOR_LAND)
            visited.eadd(q, BOOL.LOR, out=visited)
        return visited

    tp = timed(stream, bfs_parents, max(3, a.reps // 4), 1)
    tl = timed(stream, bfs_levels, max(3, a.reps // 4), 1)
    print(f"BFS with parents (ANY.SECONDI) {tp:9.2f} ms; level BFS (LOR.LAND) {tl:9.2f} ms; ratio {tp / tl:.3f}; "
          f"reached {bfs_parents().nvals} / {bfs_levels().nvals}")

    # where the time of one positional call goes
    from torch.profiler import ProfilerActivity, profile
    A.mxv(u, semiring=INT64.MIN_SECONDI, out=w)
    gb.lib.B200_device_synchronize()
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        A.mxv(u, semiring=INT64.MIN_SECONDI, out=w)
        gb.lib.B200_device_synchronize()
    print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=8))


if __name__ == "__main__":
    main()
