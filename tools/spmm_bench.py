#!/usr/bin/env python
"""GrB_mxm with a dense right operand (the SpMM path, DESIGN.md section 3.6) on the R-MAT graph of bench.py, against

    (b) k back-to-back GrB_mxv calls of the same semiring, one per column of X
    (c) the CSR GrB_mxm on the same X imported as CSR (at --scale-csr only: at scale 22 it sorts nnz(A) * k products)

for FP32 PLUS_TIMES and MAX_PLUS and k in {8, 32, 128}.  Device times from CUDA events on the library's stream, medians of
--reps calls after --warmup, the arms alternated in one process.  Outputs are checked: bit-equal across the arms on
quarter-valued inputs, and within 1e-6 relative of an fp64 scipy reference on random FP32 (PLUS_TIMES).  The byte model is

    nnz(A) (4 + b_A) + (m + 1) 4 + n k (b_X [+ 1 with presence]) + m k (b_C + 1)

and the share of it is over the data sheet's 3.35 TB/s.  --profile prints one torch.profiler split of a call instead.

--left measures the dense left operand, C = X (+).(x) A with X a k x n dense form, against (b) k back-to-back GrB_vxm calls,
(c) the right route on X' stored n x k (A' (+).(x) X' with T0: the same kernel without the two transposes) and (d) the CSR
GrB_mxm (at --scale-csr and k = 8, one repetition), plus a k = 32 SSSP sweep D <- min(D, D min.+ A) against 32 single-source
GrB_vxm sweeps; --left --profile splits one call into x-transpose, kernel, combine, t-transpose and write-back.

--sddmm measures two dense-form operands under a sparse mask, C<M> = X (+).(x) Y' (DESIGN.md section 3.6): M = the R-MAT graph
as a structural mask, X and Y random FP32 (and quarter-valued) n x d, desc = ST1, against (b) the same call without T1 on Y
stored d x n (what y-transpose costs), (c) the CSR path on the same operands imported as CSR, at scale <= 14 and d = 8 only (above
2^18 entries of Y that path forms m d n products and does not finish), and (d) torch on the same device, (X[rows] * Y[cols]).sum(1)
in edge chunks (PLUS_TIMES only).  Checks: (a) = (b) bit for bit, (a) = (c) bit for bit on quarter values, (a) within 1e-6 relative
of fp64 numpy on 10^6 sampled edges plus the edges of the 16 longest mask rows.  Its byte model is

    nnz(M) 4 + (m + 1) 4 + m d b_X + n d b_Y + nnz(T) (4 + b_C) + (m + 1) 8   [+ 2 n d b_Y for y-transpose]

which leaves out the gather, nnz(M) d b_Y (reported beside it); --sddmm --profile splits one call into row ids, kernel,
transposes and write-back.

--wide measures the three routes on 64-bit row offsets (the wide route of matrices with 2^32 or more entries): (1) on the
Kronecker graph A = kron(G, J) of 2^32 + 2^26 entries (n = 2^24), A (+).(x) X at k = 8 and 32, X (+).(x) A at k = 32 and SDDMM
under A at d = 32, in FP32 when the card has the free memory for A and its transpose (8 B per entry each), else in UINT8 --
time and algorithmic bytes over time, with (m + 1) 8 bytes of row offsets in the byte models; (2) the same three calls on the
R-MAT graph at --scale, on the narrow and the forced-wide route (B200_debug_wide) alternated, outputs compared bit for bit:
the cost of 64-bit offsets where both routes run.

    python tools/spmm_bench.py [--scale 22] [--scale-csr 20] [--reps 10] [--warmup 2] [--profile] [--left | --sddmm | --wide] [--ds 8,32,128]"""
import argparse
import os
import subprocess
import sys

import numpy as np
import scipy.sparse as sp

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import pygraphblas_b200 as gb
from pygraphblas_b200 import FP32, Matrix, Vector, descriptor
from bench import cached_graph

HBM_BPS = 3.35e12
KS = (8, 32, 128)


def lib_stream():
    sp_ = gb.ffi.new("void**")
    gb.lib.B200_get_stream(sp_)
    return torch.cuda.ExternalStream(int(gb.ffi.cast("uintptr_t", sp_[0])))


def time_once(stream, f):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    f()
    e1.record(stream)
    gb.lib.B200_device_synchronize()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def alternate(stream, arms, reps, warmup):
    """Median ms of each arm, the arms interleaved call by call."""
    for f in arms.values():
        for _ in range(warmup):
            f()
    ts = {k: [] for k in arms}
    for _ in range(reps):
        for k, f in arms.items():
            ts[k].append(time_once(stream, f))
    return {k: float(np.median(v)) for k, v in ts.items()}


def last_kernel():
    return gb.ffi.string(gb.lib.B200_debug_last_kernel()).decode()


def byte_model(nnz, m, n, k, b=4):
    return nnz * (4 + b) + (m + 1) * 4 + n * k * b + m * k * (b + 1)


def graph(scale, quarter, seed=2):
    n, indptr, indices = cached_graph(scale)
    rng = np.random.default_rng(seed)
    nnz = len(indices)
    vals = (rng.integers(1, 9, nnz) / 4.0).astype(np.float32) if quarter else (rng.random(nnz, dtype=np.float32) + np.float32(0.5))
    return n, indptr, indices, vals


def xblock(n, k, quarter, seed=3):
    rng = np.random.default_rng(seed + k)
    return (rng.integers(-4, 5, (n, k)) / 4.0).astype(np.float32) if quarter else rng.random((n, k), dtype=np.float32)


def run_scale(stream, scale, with_csr, reps, warmup, out):
    for quarter in (True, False):
        n, indptr, indices, vals = graph(scale, quarter)
        nnz = len(indices)
        A = Matrix.from_csr(indptr, indices, vals, n, n, FP32)
        S64 = sp.csr_matrix((vals.astype(np.float64), indices, indptr), shape=(n, n)) if not quarter else None
        for semi in (FP32.PLUS_TIMES, FP32.MAX_PLUS):
            if not quarter and semi is not FP32.PLUS_TIMES:
                continue
            for k in KS:
                x = xblock(n, k, quarter)
                X = Matrix.from_numpy(x)
                cols = [Vector.from_numpy(np.ascontiguousarray(x[:, j])) for j in range(k)]
                ws = [Vector.sparse(FP32, n) for _ in range(k)]
                C = Matrix.sparse(FP32, n, k)
                arms = {"spmm": lambda: A.mxm(X, semiring=semi, out=C),
                        "mxv": lambda: [A.mxv(cols[j], semiring=semi, out=ws[j]) for j in range(k)]}
                Xc = None
                if with_csr and k <= 32:
                    Xc = Matrix.from_csr(np.arange(0, n * k + 1, k, dtype=np.int64), np.tile(np.arange(k, dtype=np.uint32), n), x.reshape(-1), n, k, FP32)
                    Cc = Matrix.sparse(FP32, n, k)
                    arms["csr-mxm"] = lambda: A.mxm(Xc, semiring=semi, out=Cc)
                t = alternate(stream, arms, reps if k < 128 or not with_csr else max(3, reps // 2), warmup)
                A.mxm(X, semiring=semi, out=C)
                kern = last_kernel()
                # outputs
                got, pres = C.to_numpy()
                got = np.where(pres.astype(bool), got, np.float32(0))
                mxv = np.zeros((n, k), np.float32); mxv_p = np.zeros((n, k), np.uint8)
                for j in range(k):
                    v, p = ws[j].to_numpy()
                    mxv[:, j], mxv_p[:, j] = np.where(p.astype(bool), v, 0), p
                check = {"presence_equal_mxv": bool(np.array_equal(pres, mxv_p))}
                if quarter:
                    check["bits_equal_mxv"] = bool(np.array_equal(got.view(np.uint32), mxv.view(np.uint32)))
                    if Xc is not None:
                        cx, cp = Cc.to_numpy()
                        check["bits_equal_csr_mxm"] = bool(np.array_equal(cp, pres) and np.array_equal(np.where(cp.astype(bool), cx, 0).view(np.uint32), got.view(np.uint32)))
                else:
                    want = S64 @ x.astype(np.float64)
                    nz = pres.astype(bool)
                    rel = np.abs(got[nz] - want[nz]) / np.maximum(np.abs(want[nz]), 1e-300)
                    check["max_rel_err_fp64_spmm"] = float(rel.max()) if rel.size else 0.0
                    rel_b = np.abs(mxv[nz] - want[nz]) / np.maximum(np.abs(want[nz]), 1e-300)
                    check["max_rel_err_fp64_mxv"] = float(rel_b.max()) if rel_b.size else 0.0
                model = byte_model(nnz, n, n, k)
                rec = {"scale": scale, "n": n, "nnz": nnz, "semiring": semi.name, "k": k, "inputs": "quarter" if quarter else "random",
                       "ms": {a: round(v, 4) for a, v in t.items()}, "speedup_vs_mxv": round(t["mxv"] / t["spmm"], 2),
                       "byte_model": model, "gather_bytes": nnz * k * 4, "share_of_hbm_model": round(model / HBM_BPS / (t["spmm"] * 1e-3), 3),
                       "kernels": kern, "checks": check}
                if "csr-mxm" in t:
                    rec["speedup_vs_csr_mxm"] = round(t["csr-mxm"] / t["spmm"], 2)
                print(rec, flush=True)
                out.append(rec)
                del arms, X, cols, ws, C, Xc
        del A


def profile_split(scale):
    from torch.profiler import ProfilerActivity, profile
    n, indptr, indices, vals = graph(scale, False)
    A = Matrix.from_csr(indptr, indices, vals, n, n, FP32)
    X = Matrix.from_numpy(xblock(n, 32, False))
    M = Matrix.from_numpy((np.arange(n * 32).reshape(n, 32) % 3 == 0).astype(np.float32))
    C = Matrix.from_numpy(np.ones((n, 32), np.float32))
    f = lambda: A.mxm(X, semiring=FP32.PLUS_TIMES, out=C, mask=M, accum=FP32.PLUS)
    f(); gb.lib.B200_device_synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        f(); gb.lib.B200_device_synchronize()
    groups = {"prep": ("seg_", "scan_", "cast_", "narrow_"), "conversion": ("dense_", "csr_scatter"),
              "spmm": ("spmm_kernel", "spmm_combine"), "write-back": ("vec_finalize",)}
    split = {g: 0.0 for g in groups}; other = 0.0
    for ev in prof.key_averages():
        us = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        for g, keys in groups.items():
            if any(k in ev.key for k in keys):
                split[g] += us
                break
        else:
            other += us
    print({"profile": f"scale {scale} k=32 FP32 PLUS_TIMES, dense mask and PLUS accumulator", "device_us": {**{g: round(v, 1) for g, v in split.items()}, "other": round(other, 1)},
           "kernels": last_kernel()})
    print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=12))


def stack_vectors(ws, k, m):
    v, p = np.zeros((k, m), np.float32), np.zeros((k, m), np.uint8)
    for r in range(k):
        x, q = ws[r].to_numpy()
        v[r], p[r] = np.where(q.astype(bool), x, 0), q
    return v, p


def run_scale_left(stream, scale, with_csr, reps, warmup, out):
    """--left: C = X (+).(x) A with X a k x n dense form (the left route) against (b) k GrB_vxm calls, (c) the right route on X'
    stored n x k (A' (+).(x) X' with T0: the same kernel without the two transposes) and (d) the CSR GrB_mxm at --scale-csr, k = 8."""
    for quarter in (True, False):
        n, indptr, indices, vals = graph(scale, quarter)
        nnz = len(indices)
        A = Matrix.from_csr(indptr, indices, vals, n, n, FP32)
        S64t = sp.csr_matrix((vals.astype(np.float64), indices, indptr), shape=(n, n)).T.tocsr() if not quarter else None
        for semi in (FP32.PLUS_TIMES, FP32.MAX_PLUS):
            if not quarter and semi is not FP32.PLUS_TIMES:
                continue
            for k in KS:
                xt = xblock(n, k, quarter)                     # n x k
                x = np.ascontiguousarray(xt.T)                 # k x n: the rows are the vectors
                X, Xt = Matrix.from_numpy(x), Matrix.from_numpy(xt)
                rows = [Vector.from_numpy(x[r]) for r in range(k)]
                ws = [Vector.sparse(FP32, n) for _ in range(k)]
                C, R = Matrix.sparse(FP32, k, n), Matrix.sparse(FP32, n, k)
                arms = {"left": lambda: X.mxm(A, semiring=semi, out=C),
                        "vxm": lambda: [rows[r].vxm(A, semiring=semi, out=ws[r]) for r in range(k)],
                        "right-on-Xt": lambda: A.mxm(Xt, semiring=semi, out=R, desc=gb.descriptor.T0)}
                t = alternate(stream, arms, reps, warmup)
                Xc = None
                if with_csr and k == 8:
                    Xc = Matrix.from_csr(np.arange(0, n * k + 1, n, dtype=np.int64), np.tile(np.arange(n, dtype=np.uint32), k), x.reshape(-1), k, n, FP32)
                    Cc = Matrix.sparse(FP32, k, n)
                    t.update(alternate(stream, {"csr-mxm": lambda: Xc.mxm(A, semiring=semi, out=Cc)}, 1, 0))
                X.mxm(A, semiring=semi, out=C)
                kern = last_kernel()
                got, pres = C.to_numpy()
                got = np.where(pres.astype(bool), got, np.float32(0))
                vx, vp = stack_vectors(ws, k, n)
                rv, rp = R.to_numpy()
                rv, rp = np.where(rp.astype(bool), rv, np.float32(0)).T, rp.T
                check = {"presence_equal_vxm": bool(np.array_equal(pres, vp)), "presence_equal_right": bool(np.array_equal(pres, rp))}
                if quarter:
                    check["bits_equal_vxm"] = bool(np.array_equal(got.view(np.uint32), vx.view(np.uint32)))
                    check["bits_equal_right"] = bool(np.array_equal(got.view(np.uint32), rv.view(np.uint32)))
                    if Xc is not None:
                        cx, cp = Cc.to_numpy()
                        check["bits_equal_csr_mxm"] = bool(np.array_equal(cp, pres) and np.array_equal(np.where(cp.astype(bool), cx, 0).view(np.uint32), got.view(np.uint32)))
                else:
                    want = (S64t @ xt.astype(np.float64)).T
                    nz = pres.astype(bool)
                    for name, g in (("left", got), ("vxm", vx), ("right", rv)):
                        rel = np.abs(g[nz] - want[nz]) / np.maximum(np.abs(want[nz]), 1e-300)
                        check[f"max_rel_err_fp64_{name}"] = float(rel.max()) if rel.size else 0.0
                # the right route's bytes plus the two transposes (X' read and written, T' read and written)
                model = byte_model(nnz, n, n, k) + 2 * n * k * 4 + 2 * n * k * 5
                rec = {"mode": "left", "scale": scale, "n": n, "nnz": nnz, "semiring": semi.name, "k": k, "inputs": "quarter" if quarter else "random",
                       "ms": {a: round(v, 4) for a, v in t.items()}, "left_vs_vxm": round(t["vxm"] / t["left"], 2),
                       "left_over_right": round(t["left"] / t["right-on-Xt"], 3), "byte_model": model,
                       "share_of_hbm_model": round(model / HBM_BPS / (t["left"] * 1e-3), 3), "kernels": kern, "checks": check}
                print(rec, flush=True)
                out.append(rec)
                del arms, X, Xt, rows, ws, C, R, Xc
        del A


def sssp_left(stream, scale, reps, warmup, k=32):
    """k-source SSSP sweeps D <- min(D, D min.+ A) on the left route against k single-source sweeps w <- min(w, w min.+ A) of
    GrB_vxm, the same number of steps each (the steps the k-source sweep takes to converge)."""
    n, indptr, indices = cached_graph(scale)
    rng = np.random.default_rng(7)
    w = rng.integers(1, 10, len(indices)).astype(np.float32)
    A = Matrix.from_csr(indptr, indices, w, n, n, FP32)
    src = rng.choice(n, k, replace=False)
    d0, p0 = np.zeros((k, n), np.float32), np.zeros((k, n), np.uint8)
    p0[np.arange(k), src] = 1
    D = Matrix.from_numpy(d0, present=p0)
    steps, prev = 0, D.to_numpy()
    while True:
        D.mxm(A, semiring=FP32.MIN_PLUS, accum=FP32.MIN, out=D)
        steps += 1
        cur = D.to_numpy()
        if np.array_equal(cur[1], prev[1]) and np.array_equal(cur[0], prev[0]):
            break
        prev = cur
    kern = last_kernel()
    state = {}

    def prep_left():
        state["D"] = Matrix.from_numpy(d0, present=p0)

    def left():
        Dl = state["D"]
        for _ in range(steps):
            Dl.mxm(A, semiring=FP32.MIN_PLUS, accum=FP32.MIN, out=Dl)

    def prep_vxm():
        state["w"] = [Vector.from_numpy(d0[r], present=p0[r]) for r in range(k)]

    def vxm():
        for wr in state["w"]:
            for _ in range(steps):
                wr.vxm(A, semiring=FP32.MIN_PLUS, accum=FP32.MIN, out=wr)

    # the arms alternated, each from fresh distances prepared outside the timed region
    ts = {"left": [], "vxm": []}
    for rep in range(warmup + reps):
        for name, prep, f in (("left", prep_left, left), ("vxm", prep_vxm, vxm)):
            prep()
            gb.lib.B200_device_synchronize()
            ms = time_once(stream, f)
            if rep >= warmup:
                ts[name].append(ms)
    t = {a: float(np.median(v)) for a, v in ts.items()}
    got, pres = state["D"].to_numpy()
    vx, vp = stack_vectors(state["w"], k, n)
    rec = {"mode": "left-sssp", "scale": scale, "k": k, "steps": steps, "ms": {a: round(v, 3) for a, v in t.items()},
           "left_vs_vxm": round(t["vxm"] / t["left"], 2), "kernels": kern,
           "checks": {"equal_vxm": bool(np.array_equal(pres, vp) and np.array_equal(np.where(pres.astype(bool), got, 0), vx)),
                      "equal_converged": bool(np.array_equal(pres, cur[1]) and np.array_equal(got[pres == 1], cur[0][pres == 1]))}}
    print(rec, flush=True)


def profile_left(scale, k=32):
    """torch.profiler split of one unmasked left-route call: the two dense transposes told apart by their start times."""
    from torch.profiler import ProfilerActivity, profile
    n, indptr, indices, vals = graph(scale, False)
    A = Matrix.from_csr(indptr, indices, vals, n, n, FP32)
    X = Matrix.from_numpy(np.ascontiguousarray(xblock(n, k, False).T))
    C = Matrix.sparse(FP32, k, n)
    f = lambda: X.mxm(A, semiring=FP32.PLUS_TIMES, out=C)
    f(); gb.lib.B200_device_synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        f(); gb.lib.B200_device_synchronize()
    groups = {"spmm kernel": ("spmm_kernel",), "combine": ("spmm_combine",), "prep": ("seg_", "scan_", "cast_", "narrow_"),
              "write-back": ("vec_finalize",)}
    split = {"x-transpose": 0.0, "t-transpose": 0.0, **{g: 0.0 for g in groups}}
    other = 0.0
    kernels = [e for e in prof.events() if getattr(e, "device_type", None) is not None and e.device_type.name == "CUDA"]
    tr = sorted((e for e in kernels if "dense_transpose" in e.name), key=lambda e: e.time_range.start)
    for i, e in enumerate(tr):
        split["x-transpose" if i == 0 and len(tr) == 2 else "t-transpose"] += e.time_range.elapsed_us()
    for e in kernels:
        if "dense_transpose" in e.name:
            continue
        for g, keys in groups.items():
            if any(s in e.name for s in keys):
                split[g] += e.time_range.elapsed_us()
                break
        else:
            other += e.time_range.elapsed_us()
    print({"profile": f"left route, scale {scale} k={k} FP32 PLUS_TIMES, no mask", "device_us": {**{g: round(v, 1) for g, v in split.items()}, "other": round(other, 1)},
           "kernels": last_kernel()})
    print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=12))


def sddmm_byte_model(nnz, m, n, d, b=4, y_transposed=False):
    return nnz * 4 + (m + 1) * 4 + m * d * b + n * d * b + nnz * (4 + b) + (m + 1) * 8 + (2 * n * d * b if y_transposed else 0)


def sddmm_values(C):
    I, J, V = C.to_arrays()
    return np.asarray(I), np.asarray(J), np.asarray(V)


def edge_dots64(x, y, r, c, chunk=1 << 18):
    """Per edge (r, c): the fp64 dot product of x[r] and y[c], and that of their absolute values (the error scale)."""
    want, scale = np.empty(len(r)), np.empty(len(r))
    for s0 in range(0, len(r), chunk):
        a, b = x[r[s0:s0 + chunk]].astype(np.float64), y[c[s0:s0 + chunk]].astype(np.float64)
        want[s0:s0 + chunk] = np.einsum("ij,ij->i", a, b)
        scale[s0:s0 + chunk] = np.einsum("ij,ij->i", np.abs(a), np.abs(b))
    return want, scale


def run_scale_sddmm(stream, scale, with_csr, reps, warmup, ds, out):
    n, indptr, indices = cached_graph(scale)
    nnz = len(indices)
    rows = np.repeat(np.arange(n, dtype=np.int64), np.diff(indptr))
    M = Matrix.from_csr(indptr, indices, np.ones(nnz, np.bool_), n, n, gb.BOOL)
    rows_t, cols_t = torch.from_numpy(rows).cuda(), torch.from_numpy(indices.astype(np.int64)).cuda()
    rng = np.random.default_rng(11)
    longest = np.argsort(np.diff(indptr))[-16:]
    sample = np.unique(np.concatenate([rng.integers(0, nnz, 1 << 20)] + [np.arange(indptr[r], indptr[r + 1]) for r in longest]))
    ST1, S = gb.descriptor.ST1, gb.descriptor.S
    for quarter in (True, False):
        for semi in (FP32.PLUS_TIMES, FP32.MAX_PLUS):
            if not quarter and semi is not FP32.PLUS_TIMES:
                continue
            for d in ds:
                x, y = xblock(n, d, quarter, seed=3), xblock(n, d, quarter, seed=5)
                X, Y, Yt = Matrix.from_numpy(x), Matrix.from_numpy(y), Matrix.from_numpy(np.ascontiguousarray(y.T))
                # every call writes a fresh, empty C, so the result is T itself; a C that holds entries (without GrB_REPLACE) adds the
                # row-wise merge of T with C that every masked mxm shares ("merge-into-C", one arm, for scale)
                res = {}
                arms = {"sddmm": lambda: res.__setitem__("a", X.mxm(Y, semiring=semi, mask=M, desc=ST1, out=Matrix.sparse(FP32, n, n))),
                        "y-given-d-x-n": lambda: res.__setitem__("b", X.mxm(Yt, semiring=semi, mask=M, desc=S, out=Matrix.sparse(FP32, n, n)))}
                if d == 32 and semi is FP32.PLUS_TIMES:
                    Cm = Matrix.sparse(FP32, n, n)
                    arms["merge-into-C"] = lambda: X.mxm(Y, semiring=semi, mask=M, desc=ST1, out=Cm)
                if semi is FP32.PLUS_TIMES:
                    xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
                    td = torch.empty(nnz, dtype=torch.float32, device="cuda")
                    chunk = max(1, (1 << 28) // d)               # 1 GiB of gathered FP32 values per operand and chunk

                    def torch_arm():
                        with torch.cuda.stream(stream):
                            for s0 in range(0, nnz, chunk):
                                td[s0:s0 + chunk] = (xd[rows_t[s0:s0 + chunk]] * yd[cols_t[s0:s0 + chunk]]).sum(1)
                    arms["torch"] = torch_arm
                t = alternate(stream, arms, reps, warmup)
                arms["sddmm"]()
                kern = last_kernel()
                I, J, V = sddmm_values(res["a"])
                I2, J2, V2 = sddmm_values(res["b"])
                check = {"pattern_is_mask": bool(np.array_equal(I, rows) and np.array_equal(J, indices)),
                         "bits_equal_y_given_d_x_n": bool(np.array_equal(I, I2) and np.array_equal(J, J2) and np.array_equal(V.view(np.uint32), V2.view(np.uint32)))}
                if with_csr and d == 8:
                    ptr = np.arange(0, n * d + 1, d, dtype=np.int64); ids = np.tile(np.arange(d, dtype=np.uint32), n)
                    Xc, Yc = Matrix.from_csr(ptr, ids, x.reshape(-1), n, d, FP32), Matrix.from_csr(ptr, ids, y.reshape(-1), n, d, FP32)
                    Cc = Matrix.sparse(FP32, n, n)
                    t.update(alternate(stream, {"csr-mxm": lambda: Xc.mxm(Yc, semiring=semi, mask=M, desc=ST1, out=Cc)}, 3, 1))
                    check["csr_kernels"] = last_kernel()
                    Ic, Jc, Vc = sddmm_values(Cc)
                    if quarter:
                        check["bits_equal_csr_mxm"] = bool(np.array_equal(I, Ic) and np.array_equal(J, Jc) and np.array_equal(V.view(np.uint32), Vc.view(np.uint32)))
                if semi is FP32.PLUS_TIMES:
                    want, scale_ = edge_dots64(x, y, rows[sample], indices[sample])
                    check["max_rel_err_fp64_sampled"] = float((np.abs(V[sample] - want) / np.maximum(scale_, 1e-300)).max())
                    check["sampled_edges"] = int(len(sample))
                    tv = td.cpu().numpy()
                    check["max_rel_err_fp64_torch"] = float((np.abs(tv[sample] - want) / np.maximum(scale_, 1e-300)).max())
                model, gather = sddmm_byte_model(nnz, n, n, d), nnz * d * 4
                sec = t["sddmm"] * 1e-3
                rec = {"mode": "sddmm", "scale": scale, "n": n, "nnz": nnz, "semiring": semi.name, "d": d, "inputs": "quarter" if quarter else "random",
                       "ms": {a: round(v, 4) for a, v in t.items()}, "y_transpose_cost": round(t["y-given-d-x-n"] / t["sddmm"], 3),
                       "byte_model": model, "gather_bytes": gather, "share_of_hbm_model": round(model / HBM_BPS / sec, 3),
                       "share_of_hbm_with_gather": round((model + gather) / HBM_BPS / sec, 3), "kernels": kern, "checks": check}
                if "torch" in t:
                    rec["speedup_vs_torch"] = round(t["torch"] / t["sddmm"], 2)
                print(rec, flush=True)
                out.append(rec)
                del arms, res, X, Y, Yt
    del M


def profile_sddmm(scale, d=32):
    """torch.profiler split of one call with T1 and of one without (which builds y-transpose)."""
    from torch.profiler import ProfilerActivity, profile
    n, indptr, indices = cached_graph(scale)
    M = Matrix.from_csr(indptr, indices, np.ones(len(indices), np.bool_), n, n, gb.BOOL)
    x, y = xblock(n, d, False, seed=3), xblock(n, d, False, seed=5)
    X, Y, Yt = Matrix.from_numpy(x), Matrix.from_numpy(y), Matrix.from_numpy(np.ascontiguousarray(y.T))
    C = Matrix.sparse(FP32, n, n)
    fresh = lambda: Matrix.sparse(FP32, n, n)
    groups = {"row ids": ("sddmm_rowid",), "kernel": ("sddmm_kernel",), "transposes": ("dense_transpose",),
              "compaction": ("row_found", "scan", "Scan"), "write-back": ("mat_finalize", "cast_", "rowptr32")}
    for name, f in (("desc=ST1, empty C", lambda: X.mxm(Y, semiring=FP32.PLUS_TIMES, mask=M, desc=descriptor.ST1, out=fresh())),
                    ("desc=S, Y given d x n, empty C", lambda: X.mxm(Yt, semiring=FP32.PLUS_TIMES, mask=M, desc=gb.descriptor.S, out=fresh())),
                    ("desc=ST1, C holds the last result", lambda: X.mxm(Y, semiring=FP32.PLUS_TIMES, mask=M, desc=descriptor.ST1, out=C))):
        f(); gb.lib.B200_device_synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            f(); gb.lib.B200_device_synchronize()
        split = {g: 0.0 for g in groups}; other = 0.0
        for ev in prof.key_averages():
            us = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
            for g, keys in groups.items():
                if any(k in ev.key for k in keys):
                    split[g] += us
                    break
            else:
                other += us
        print({"profile": f"sddmm, scale {scale} d={d} FP32 PLUS_TIMES, structural mask, {name}",
               "device_us": {**{g: round(v, 1) for g, v in split.items()}, "other (copies of M's pattern, memsets)": round(other, 1)}, "kernels": last_kernel()})
        print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=8))


def _bits_equal(a, b):
    return all(np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8)) for x, y in zip(a, b))


def wide_kron(stream, reps, warmup):
    """The three routes on kron(G, J), 2^32 + 2^26 entries: every call takes the wide route (no rowptr32)."""
    from wide_spmv_bench import factor
    NG = NJ = 4096
    G, J = factor(1, NG, (1 << 16) + (1 << 10)), factor(2, NJ, 1 << 16)
    nnz, n = G.nnz * J.nnz, NG * NJ
    free = torch.cuda.mem_get_info()[0]
    # FP32: A and A' at 8 B per entry, the partials of the split rows at k = 32 (~2.5 B per entry), the transpose's scratch and
    # the dense blocks
    fp32 = free > nnz * 18.5 + 8e9
    typ, b = (FP32, 4) if fp32 else (gb.UINT8, 1)
    sr = typ.PLUS_TIMES
    print({"case": "wide-kron", "type": typ.name, "nnz": nnz, "n": n, "free_GB": round(free / 1e9, 1)}, flush=True)
    mk = lambda S: Matrix.from_csr(S.indptr, S.indices, S.data.astype(typ.dtype), S.shape[0], S.shape[1], typ)
    A, Gm, Jm = Matrix.sparse(typ, n, n), mk(G), mk(J)
    gb.base._check(gb.lib.GrB_Matrix_kronecker_BinaryOp(A._matrix[0], gb.ffi.NULL, gb.ffi.NULL, typ.TIMES.get_op(),
                                                        Gm._matrix[0], Jm._matrix[0], gb.ffi.NULL))
    del Gm, Jm
    rng = np.random.default_rng(5)
    held = []

    def report(name, ms, nbytes):
        print({"case": name, "type": typ.name, "median_ms": round(ms, 2), "GEdge_per_s": round(nnz / ms / 1e6, 1),
               "alg_GB_per_s": round(nbytes / ms / 1e6, 1), "kernels": last_kernel()}, flush=True)

    for k in (8, 32):
        X = Matrix.from_numpy(rng.integers(0, 4, (n, k)).astype(typ.dtype), typ=typ)
        call = lambda: (held.clear(), held.append(A.mxm(X, semiring=sr)))
        ms = alternate(stream, {"spmm": call}, reps, warmup)["spmm"]
        report(f"wide-kron spmm k={k}", ms, nnz * (4 + b) + (n + 1) * 8 + n * k * b + n * k * (b + 1))
        held.clear(); del X
    d = 32
    X = Matrix.from_numpy(rng.integers(0, 4, (n, d)).astype(typ.dtype), typ=typ)
    Y = Matrix.from_numpy(rng.integers(0, 4, (n, d)).astype(typ.dtype), typ=typ)

    def sddmm():
        held.clear()                             # the previous T (as large as A) is freed before the next is formed
        C = Matrix.sparse(typ, n, n)
        X.mxm(Y, semiring=sr, mask=A, out=C, desc=descriptor.ST1)
        held.append(C)
    ms = alternate(stream, {"sddmm": sddmm}, reps, warmup)["sddmm"]
    report(f"wide-kron sddmm d={d}", ms, nnz * 4 + (n + 1) * 8 + 2 * n * d * b + nnz * (4 + b) + (n + 1) * 8)
    held.clear(); del X, Y
    k = 32
    X = Matrix.from_numpy(rng.integers(0, 4, (k, n)).astype(typ.dtype), typ=typ)
    X.mxm(A, semiring=sr)                        # builds and caches A' (the chunked transpose), outside the timed calls
    call = lambda: (held.clear(), held.append(X.mxm(A, semiring=sr)))
    ms = alternate(stream, {"left": call}, reps, warmup)["left"]
    xb, tb = n * k * b, n * k * (b + 1)
    report(f"wide-kron left k={k}", ms, nnz * (4 + b) + (n + 1) * 8 + xb + tb + 2 * xb + 2 * tb)
    held.clear()


def wide_vs_narrow(stream, scale, reps, warmup):
    """The three routes on the R-MAT graph, narrow and forced wide, alternated call by call; outputs compared bit for bit."""
    n, indptr, indices, vals = graph(scale, quarter=False)
    nnz = len(indices)
    A = {w: Matrix.from_csr(indptr, indices, vals, n, n, FP32) for w in (False, True)}
    k = d = 32
    X = Matrix.from_numpy(xblock(n, k, False), typ=FP32)
    Xl = Matrix.from_numpy(np.ascontiguousarray(xblock(n, k, False, seed=7).T), typ=FP32)
    Y = Matrix.from_numpy(xblock(n, d, False, seed=9), typ=FP32)
    out, kern = {}, {}

    def arm(name, wide, f):
        def g():
            gb.lib.B200_debug_wide(1 << 30 if wide else 0)
            try:
                out[(name, wide)] = f(A[wide])
            finally:
                gb.lib.B200_debug_wide(0)
            kern[(name, wide)] = last_kernel()
        return g

    def sddmm(a):
        C = Matrix.sparse(FP32, n, n)
        X.mxm(Y, semiring=FP32.PLUS_TIMES, mask=a, out=C, desc=descriptor.ST1)
        return C
    # (call, its result's arrays: the dense form's values and presence, or the CSR tuples)
    calls = {"spmm k=32": (lambda a: a.mxm(X, semiring=FP32.PLUS_TIMES), Matrix.to_numpy),
             "left k=32": (lambda a: Xl.mxm(a, semiring=FP32.PLUS_TIMES), Matrix.to_numpy),
             "sddmm d=32": (sddmm, Matrix.to_arrays)}
    for name, (f, arrays) in calls.items():
        ms = alternate(stream, {w: arm(name, w, f) for w in (False, True)}, reps, warmup)
        same = _bits_equal(arrays(out[(name, False)]), arrays(out[(name, True)]))
        for w in (False, True):
            print({"case": f"s{scale} {name} {'wide' if w else 'narrow'}", "nnz": nnz, "median_ms": round(ms[w], 4),
                   "wide_over_narrow": round(ms[True] / ms[False], 4), "kernels": kern[(name, w)], "outputs_bit_identical": same},
                  flush=True)
        out.clear()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=int, default=22)
    ap.add_argument("--scale-csr", type=int, default=20)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--left", action="store_true", help="the dense left operand, X (+).(x) A (the batched vxm)")
    ap.add_argument("--sddmm", action="store_true", help="two dense operands under a sparse mask, C<M> = X (+).(x) Y'")
    ap.add_argument("--ds", default="8,32,128", help="--sddmm: the inner dimensions d")
    ap.add_argument("--wide", action="store_true", help="the three routes on 64-bit row offsets: a graph of 2^32 + 2^26 entries, "
                                                        "and the R-MAT graph narrow against forced wide")
    ap.add_argument("--skip-large", action="store_true", help="--wide: only the narrow / forced-wide comparison")
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print({"card": card})
    stream = lib_stream()
    if a.wide:
        wide_vs_narrow(stream, a.scale, a.reps, a.warmup)
        if not a.skip_large:
            wide_kron(stream, max(3, a.reps // 3), 1)
        return
    if a.sddmm:
        if a.profile:
            profile_sddmm(a.scale)
            return
        out, ds = [], tuple(int(v) for v in a.ds.split(","))
        run_scale_sddmm(stream, a.scale, False, a.reps, a.warmup, ds, out)
        if a.scale_csr:
            run_scale_sddmm(stream, min(a.scale_csr, 14), True, a.reps, a.warmup, (8,), out)
        return
    if a.profile:
        if a.left:
            for k in (8, 32):
                profile_left(a.scale, k)
        else:
            profile_split(a.scale)
        return
    if a.left:
        out = []
        run_scale_left(stream, a.scale, False, a.reps, a.warmup, out)
        if a.scale_csr:
            run_scale_left(stream, a.scale_csr, True, a.reps, a.warmup, out)
        sssp_left(stream, a.scale, max(2, a.reps // 3), 1)
        return
    out = []
    run_scale(stream, a.scale, False, a.reps, a.warmup, out)
    if a.scale_csr:
        run_scale(stream, a.scale_csr, True, a.reps, a.warmup, out)


if __name__ == "__main__":
    main()
