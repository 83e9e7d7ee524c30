#!/usr/bin/env python
"""torch.profiler split of the benchmarked mxv step (FP32 PLUS_TIMES, w formed in place): the mean device time of every
kernel of a step and the gap between consecutive kernels (start of one minus end of the one before; negative when
they overlap, as programmatic dependent launches may).

    python tools/prof_spmv_split.py [--graph rmat|uniform] [--scale 22] [--steps 30] [--out DIR]

rmat is the bench graph (R-MAT, edge factor 16, seed 1: hub rows that span hundreds of runs); uniform has 16 entries in
every row (no hub rows), so the fix-up there shows the cost of its 8-lane path alone.  The trace is written to DIR."""
import argparse
import json
import os
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import pygraphblas_b200 as gb
from pygraphblas_b200 import Matrix, Vector, FP32
from bench import cached_graph, spmv_inputs

KNOWN = ("spmv_hot2_prep_kernel", "spmv_run_hot2_kernel", "spmv_run_fixup_kernel", "spmv_run_kernel")


def short(name):
    for k in KNOWN:                      # no name in KNOWN is a substring of another
        if k in name:
            return k
    return name[:48]


def uniform_graph(scale, deg=16, seed=5):
    """16 entries per row, columns spread over the whole range (one per n/16 block, jittered): sorted and unique."""
    n = 1 << scale
    rng = np.random.default_rng(seed)
    block = n // deg
    base = rng.integers(0, n, n, dtype=np.int64)
    cols = (base[:, None] + np.arange(deg, dtype=np.int64)[None, :] * block + rng.integers(0, block, (n, deg))) % n
    cols.sort(axis=1)
    ok = (np.diff(cols, axis=1) > 0).all(axis=1)
    cols[~ok] = np.arange(deg, dtype=np.int64)[None, :] * block         # a rare collision: an evenly spaced row instead
    return n, np.arange(n + 1, dtype=np.int64) * deg, cols.reshape(-1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--graph", choices=("rmat", "uniform"), default="rmat")
    ap.add_argument("--scale", type=int, default=22)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--out", default=tempfile.gettempdir())
    args = ap.parse_args()
    if not gb.have_device():
        raise SystemExit("no CUDA device")
    n, indptr, indices = cached_graph(args.scale) if args.graph == "rmat" else uniform_graph(args.scale)
    vals, u0 = spmv_inputs(len(indices), n)
    A = Matrix.from_csr(indptr, indices, vals, n, n, FP32)
    u = Vector.from_numpy(u0)
    w = Vector.sparse(FP32, n)
    for _ in range(10):
        A.mxv(u, semiring=FP32.PLUS_TIMES, out=w)
    gb.lib.B200_device_synchronize()
    print("route:", gb.ffi.string(gb.lib.B200_debug_last_kernel()).decode(), flush=True)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            A.mxv(u, semiring=FP32.PLUS_TIMES, out=w)
        gb.lib.B200_device_synchronize()
        torch.cuda.synchronize()
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, f"spmv_split_{args.graph}_s{args.scale}.pt.trace.json")
    prof.export_chrome_trace(path)
    with open(path) as f:
        ev = [e for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel" and e.get("ph") == "X"]
    ev.sort(key=lambda e: e["ts"])
    dur, gaps = {}, {}
    for e in ev:
        dur.setdefault(short(e["name"]), []).append(e["dur"])
    for a, b in zip(ev, ev[1:]):
        gaps.setdefault((short(a["name"]), short(b["name"])), []).append(b["ts"] - (a["ts"] + a["dur"]))
    print(f"graph {args.graph} s{args.scale}, nnz {len(indices)}, {args.steps} steps, {len(ev)} kernels; device "
          f"{torch.cuda.get_device_name(0)}", flush=True)
    for k, v in dur.items():
        print(f"  kernel {k:28s} n={len(v):4d}  median {np.median(v):8.2f} us  mean {np.mean(v):8.2f}  min {np.min(v):8.2f}  max {np.max(v):8.2f}")
    for (a, b), v in gaps.items():
        print(f"  gap {a} -> {b}: n={len(v):4d}  median {np.median(v):7.2f} us  mean {np.mean(v):7.2f}  min {np.min(v):7.2f}  max {np.max(v):7.2f}")
    step = (ev[-1]["ts"] + ev[-1]["dur"] - ev[0]["ts"]) / args.steps
    print(f"  step (first kernel start to last kernel end, per step): {step:.1f} us", flush=True)


if __name__ == "__main__":
    main()
