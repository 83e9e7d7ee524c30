#!/usr/bin/env python
"""GrB_mxm with two full dense-form operands (the tiled semiring GEMM, DESIGN.md section 3.6) against

    (b) the SpMM route on the same values, A given an all-ones presence array (what these calls ran on before the GEMM route);
        the one-time CSR build of A that route caches is timed on its own
    (c) torch on the same device, as context: torch.matmul with TF32 off for FP32 / FP64 PLUS_TIMES (fused FMA, which the
        library deliberately does not use), a chunked broadcast-min for MIN_PLUS

on the workloads

    gnn      2^22 x 128 . 128 x 128 FP32 PLUS_TIMES (the feature transform of a GNN layer)
    gram     16384 x 256 . (16384 x 256)' FP32 PLUS_TIMES with T1 (no SpMM form: the old CSR SpGEMM path is run once at
             1024 x 64, where it finishes, beside the GEMM at that size)
    minplus  8192^2 FP32 MIN_PLUS (one squaring of all-pairs shortest paths)
    lorland  8192^2 BOOL LOR_LAND (one squaring of a transitive closure)
    fp64     4096^2 FP64 PLUS_TIMES

Device times from CUDA events on the library's stream, medians of --reps calls after --warmup, the arms alternated in one
process.  (a) and (b) must be equal bit for bit.  Reported: time, products per second, and for FP PLUS_TIMES / MIN_PLUS the
share of the issue-rate ceiling of two FP instructions per product (FP32: 128 lanes per SM and clock; FP64: 64) at the SM
clock read right after the workload; device memory in use after the first call of each arm over what the operands take (the
allocator keeps its high-water mark, so this includes each arm's transient scratch and cached CSR).  The card's name and power
limit are printed with the numbers.

    python tools/gemm_bench.py [--reps 5] [--warmup 1] [--only gnn,gram,...] [--out results.jsonl]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch
import pygraphblas_b200 as gb
from pygraphblas_b200 import BOOL, FP32, FP64, Matrix, descriptor
from spmm_bench import alternate, last_kernel, lib_stream, time_once


def smi(fields):
    r = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader,nounits"], capture_output=True, text=True)
    return [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")] if r.returncode == 0 and r.stdout.strip() else None


def used_mb():
    free, total = torch.cuda.mem_get_info()
    return (total - free) / 2**20


def bits(C):
    x, p = C.to_numpy()
    return (x.view(np.uint8) if x.dtype == np.bool_ else x.view(f"u{x.itemsize}")), p


def operands(name, rng):
    if name == "gnn":
        return FP32.PLUS_TIMES, rng.random((1 << 22, 128), dtype=np.float32), rng.random((128, 128), dtype=np.float32), None
    if name == "gram":
        x = rng.random((16384, 256), dtype=np.float32)
        return FP32.PLUS_TIMES, x, x, descriptor.T1
    if name == "minplus":
        return FP32.MIN_PLUS, rng.integers(0, 1000, (8192, 8192)).astype(np.float32), rng.integers(0, 1000, (8192, 8192)).astype(np.float32), None
    if name == "lorland":
        return BOOL.LOR_LAND, rng.random((8192, 8192)) < 0.001, rng.random((8192, 8192)) < 0.001, None
    if name == "fp64":
        return FP64.PLUS_TIMES, rng.random((4096, 4096)), rng.random((4096, 4096)), None
    raise ValueError(name)


def torch_arm(name, a, b):
    if name in ("gnn", "gram", "fp64"):
        ta, tb = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
        tb = tb.t() if name == "gram" else tb
        return lambda: torch.matmul(ta, tb)
    if name == "minplus":
        ta, tb = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
        rows = 16

        def f():
            out = torch.empty((ta.shape[0], tb.shape[1]), device="cuda")
            for i in range(0, ta.shape[0], rows):
                out[i:i + rows] = (ta[i:i + rows, :, None] + tb[None]).amin(dim=1)
            return out
        return f
    return None


def run(name, stream, reps, warmup, nsm):
    rng = np.random.default_rng(7)
    sr, a, b, desc = operands(name, rng)
    m, k = a.shape
    n = b.shape[0] if desc is descriptor.T1 else b.shape[1]
    base = used_mb()
    A, B = Matrix.from_numpy(a), Matrix.from_numpy(b)
    C1 = Matrix.sparse(A.type, m, n)
    rec = {"workload": name, "m": m, "k": k, "n": n, "semiring": sr.name if hasattr(sr, "name") else str(sr)}
    f_a = lambda: A.mxm(B, semiring=sr, out=C1, desc=desc)
    f_a()
    rec["kernel_a"] = last_kernel()
    rec["mem_a_mb"] = round(used_mb() - base, 1)
    arms = {"a_gemm": f_a}
    if desc is None:
        Ab = Matrix.from_numpy(a, present=np.ones(a.shape, np.uint8))
        C2 = Matrix.sparse(A.type, m, n)
        base_b = used_mb()
        rec["b_csr_build_ms"] = time_once(stream, lambda: Ab.mxm(B, semiring=sr, out=C2))     # first call: builds and caches A's CSR
        rec["kernel_b"] = last_kernel()
        rec["mem_b_mb"] = round(used_mb() - base_b + (base_b - base), 1)
        arms["b_spmm"] = lambda: Ab.mxm(B, semiring=sr, out=C2)
    tf = torch_arm(name, a, b)
    if tf is not None:
        torch.backends.cuda.matmul.allow_tf32 = False

        def on_stream():
            with torch.cuda.stream(stream):
                tf()
        arms["c_torch"] = on_stream
    t = alternate(stream, arms, reps, warmup)
    clk = smi("clocks.sm")
    rec["sm_clock_mhz"] = float(clk[0]) if clk else None
    if "b_spmm" in arms:
        rec["b_csr_build_ms"] = round(rec["b_csr_build_ms"] - t["b_spmm"], 3)     # the first call less a steady one
        (x1, p1), (x2, p2) = bits(C1), bits(C2)
        rec["a_equals_b_bits"] = bool(np.array_equal(p1, p2) and np.array_equal(x1, x2))
    prods = m * n * k
    for arm, ms in t.items():
        rec[f"{arm}_ms"] = round(ms, 3)
        rec[f"{arm}_gprod_per_s"] = round(prods / (ms * 1e-3) / 1e9, 1)
    if name != "lorland" and rec["sm_clock_mhz"]:
        lanes = 64 if name == "fp64" else 128
        ceiling = nsm * lanes * rec["sm_clock_mhz"] * 1e6 / 2          # products per second at two FP instructions each
        rec["a_share_of_issue_ceiling"] = round(prods / (t["a_gemm"] * 1e-3) / ceiling, 3)
    if name == "gram":
        # the old path at a size where it finishes: X as CSR, X X' through the CSR SpGEMM, once, beside the GEMM
        xs = a[:1024, :64].copy()
        Xs = Matrix.from_numpy(xs)
        Xc = Matrix.from_csr(np.arange(0, 1024 * 64 + 1, 64, dtype=np.int64), np.tile(np.arange(64, dtype=np.uint32), 1024), xs.reshape(-1), 1024, 64, FP32)
        Cs, Cc = Matrix.sparse(FP32, 1024, 1024), Matrix.sparse(FP32, 1024, 1024)
        Xs.mxm(Xs, semiring=sr, out=Cs, desc=descriptor.T1)
        rec["small_gemm_ms"] = round(time_once(stream, lambda: Xs.mxm(Xs, semiring=sr, out=Cs, desc=descriptor.T1)), 3)
        rec["small_csr_spgemm_ms"] = round(time_once(stream, lambda: Xc.mxm(Xc, semiring=sr, out=Cc, desc=descriptor.T1)), 3)
        rec["small_csr_kernel"] = last_kernel()
        gx, _ = Cs.to_numpy()
        cx, cp = Cc.to_numpy()
        rec["small_max_rel_diff"] = float((np.abs(gx - cx) / np.abs(cx)).max()) if cp.all() else None
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--only", default="gnn,gram,fp64,minplus,lorland")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not gb.have_device():
        raise SystemExit("gemm_bench.py: no CUDA device")
    card = smi("name,power.limit,clocks.max.sm")
    head = {"card": card[0] if card else None, "power_limit_w": card[1] if card else None, "max_sm_clock_mhz": card[2] if card else None}
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    head["sms"] = nsm
    print(json.dumps(head), flush=True)
    stream = lib_stream()
    out = open(args.out, "w") if args.out else None
    if out:
        out.write(json.dumps(head) + "\n")
    for name in args.only.split(","):
        try:
            rec = run(name, stream, args.reps, args.warmup, nsm)
        except (gb.base.GraphBLASException, RuntimeError) as e:       # e.g. out of memory for arm (b) on a card with less free
            rec = {"workload": name, "error": repr(e)}
        print(json.dumps(rec), flush=True)
        if out:
            out.write(json.dumps(rec) + "\n"); out.flush()
        gb.lib.B200_device_synchronize()
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
