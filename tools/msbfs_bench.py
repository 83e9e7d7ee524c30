"""GrB_mxm under a complemented mask: the filtered route against the two steps the library used to take.

    python tools/msbfs_bench.py [--scales 20 22] [--ks 4 64] [--reps 3] [--out DIR]
    python tools/msbfs_bench.py --pull [--alphas 2 4 8 14 32] [--scales 20 22] [--ks 4 64] [--reps 3] [--out DIR]

new  C<!M, R> = A (+).(x) B in one call: the unmasked bins never form a blocked product.
old  T = A (+).(x) B unmasked, then C<!M, R> = IDENTITY(T) (GrB_Matrix_apply): the product formed whole, then filtered.

Workloads: multi-source BFS (k = 4 and 64 sources, BOOL ANY_PAIR, F<!V, R> = F any.pair A), the forward sweep of the BC rounds
of gap/bcmark.py (4 sources, FP32 PLUS_FIRST, a valued FP32 path-count mask), and C<!A, R> = A any.pair A at scale 16.  Old and
new run alternately on the same inputs; their results must be equal, and the BFS levels must match scipy.  Times are host clocks
around calls that end in a device synchronise, medians over --reps repetitions.

--pull compares the directions of the multi-source BFS step instead (DESIGN.md section 3.2): push (GxB_AxB_SAXPY: the bins on
every level), dot (GxB_AxB_DOT: every row pulls on every level) and auto (the default descriptor under B200GRB_MXM_PULL = alpha,
for each --alphas value).  It reports the per-level times of each arm, the traversal medians and the alpha of the fastest auto
arm; every arm's F must equal push's at every level and the levels must match scipy.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import scipy.sparse as sp
import scipy.sparse.csgraph as csgraph
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pygraphblas_b200 as gb  # noqa: E402
from pygraphblas_b200 import Matrix, descriptor, ffi, lib  # noqa: E402
from pygraphblas_b200.generators import rmat_csr  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:      # the numbers are still printed, without the card
        return f"unknown ({e})"


def timed(f):
    torch.cuda.synchronize()
    t = time.perf_counter()
    r = f()
    torch.cuda.synchronize()          # the library's stream included: a device-wide synchronise
    return time.perf_counter() - t, r


def step(route, F, B, mask, sr, desc_new, identity):
    """One masked product F<!mask, R> = F (+).(x) B by the named route; returns the new F."""
    if route == "new":
        out = Matrix.sparse(F.type, F.nrows, B.ncols)
        return F.mxm(B, semiring=sr, out=out, mask=mask, desc=desc_new)
    T = F.mxm(B, semiring=sr)
    out = Matrix.sparse(F.type, F.nrows, B.ncols)
    gb.base._check(lib.GrB_Matrix_apply(out._matrix[0], mask._matrix[0], ffi.NULL, identity.get_op(), T._matrix[0], desc_new.get_desc()))
    return out


def same(X, Y):
    a, b = X.to_arrays(), Y.to_arrays()
    return all(np.array_equal(p, q) for p, q in zip(a, b))


def msbfs(A, S, n, k, reps):
    deg = np.diff(S.indptr)
    sources = np.argsort(-deg, kind="stable")[:k]
    res = {}
    for route in ("old", "new") * reps:
        F = Matrix.from_lists(list(range(k)), list(sources), [True] * k, k, n, gb.BOOL)
        V = F.dup()
        lev = np.full((k, n), -1, np.int64)
        lev[np.arange(k), sources] = 0
        times, d = [], 0
        while True:
            d += 1
            dt, F = timed(lambda: step(route, F, A, V, gb.BOOL.ANY_PAIR, descriptor.RSC, gb.BOOL.IDENTITY))
            times.append(dt)
            if F.nvals == 0:
                break
            I, J, _ = F.to_arrays()
            lev[I, J] = d
            V.eadd(F, gb.BOOL.LOR, out=V)
        res.setdefault(route, []).append((sum(times), times, lev))
    want = csgraph.shortest_path(S, unweighted=True, indices=sources)
    want = np.where(np.isinf(want), -1, want).astype(np.int64)
    ok = all(np.array_equal(r[2], want) for rs in res.values() for r in rs)
    med = {r: statistics.median(x[0] for x in res[r]) * 1e3 for r in res}
    per_level = {r: [round(t * 1e3, 3) for t in min(res[r], key=lambda x: x[0])[1]] for r in res}
    return {"old_ms": med["old"], "new_ms": med["new"], "levels": len(per_level["new"]), "per_level_ms": per_level, "matches_scipy": ok}


def axb(method):
    d = descriptor.Descriptor()
    d[lib.GxB_AxB_METHOD] = getattr(lib, f"GxB_AxB_{method}")
    return d


def set_alpha(alpha):
    os.environ["B200GRB_MXM_PULL"] = str(alpha)
    lib.B200_reload_tunables()


def msbfs_pull(A, S, n, k, reps, alphas):
    """F<!V, R> = F any.pair A level by level under push, dot and auto(alpha); arms alternate within each repetition."""
    sources = np.argsort(-np.diff(S.indptr), kind="stable")[:k]
    arms = [("push", descriptor.RSC & axb("SAXPY"), 0), ("dot", descriptor.RSC & axb("DOT"), 0)]
    arms += [(f"auto{a:g}", descriptor.RSC, a) for a in alphas]
    res, fronts = {}, {}
    for _ in range(reps):
        for name, desc, alpha in arms:
            set_alpha(alpha)
            F = Matrix.from_lists(list(range(k)), list(sources), [True] * k, k, n, gb.BOOL)
            V = F.dup()
            lev = np.full((k, n), -1, np.int64)
            lev[np.arange(k), sources] = 0
            times, levels, d = [], [], 0
            while True:
                d += 1
                dt, F = timed(lambda: F.mxm(A, semiring=gb.BOOL.ANY_PAIR, out=Matrix.sparse(gb.BOOL, k, n), mask=V, desc=desc))
                times.append(dt)
                I, J, _ = F.to_arrays()
                levels.append(I.astype(np.int64) * n + J)
                if F.nvals == 0:
                    break
                lev[I, J] = d
                V.eadd(F, gb.BOOL.LOR, out=V)
            res.setdefault(name, []).append((sum(times), times, lev))
            fronts[name] = levels
    set_alpha(0)
    want = csgraph.shortest_path(S, unweighted=True, indices=sources)
    want = np.where(np.isinf(want), -1, want).astype(np.int64)
    ok = all(np.array_equal(r[2], want) for rs in res.values() for r in rs)
    equal = all(len(fronts[a]) == len(fronts["push"]) and all(np.array_equal(x, y) for x, y in zip(fronts[a], fronts["push"]))
                for a in fronts)
    med = {a: round(statistics.median(x[0] for x in res[a]) * 1e3, 3) for a in res}
    per_level = {a: [round(statistics.median(x[1][lv] for x in res[a]) * 1e3, 3) for lv in range(len(res[a][0][1]))] for a in res}
    autos = [a for a in med if a.startswith("auto")]
    best = min(autos, key=lambda a: med[a]) if autos else None
    return {"traversal_ms": med, "per_level_ms": per_level, "best_auto": best, "levels": len(per_level["push"]),
            "equal": equal, "matches_scipy": ok}


def bc_forward(A, S, n, reps):
    """The forward sweep of gap/bcmark.py's bc() for 4 sources: frontier<!paths, R> = frontier plus.first A, paths += frontier."""
    deg = np.diff(S.indptr)
    sources = np.argsort(-deg, kind="stable")[:4]
    ns = len(sources)
    res, outs = {}, {}
    for route in ("old", "new") * reps:
        paths = Matrix.from_lists(np.repeat(np.arange(ns), n), np.tile(np.arange(n), ns), np.zeros(ns * n, np.float32), ns, n, gb.FP32)
        frontier = Matrix.sparse(gb.FP32, ns, n)
        for i, s in enumerate(sources):
            paths[i, int(s)] = 1.0
            frontier[i, int(s)] = 1.0
        tot = 0.0
        while True:
            dt, frontier = timed(lambda: step(route, frontier, A, paths, gb.FP32.PLUS_FIRST, descriptor.RC, gb.FP32.IDENTITY))
            tot += dt
            if frontier.nvals == 0:
                break
            gb.base._check(lib.GrB_Matrix_assign(paths._matrix[0], ffi.NULL, gb.FP32.PLUS.get_op(), frontier._matrix[0],
                                                 lib.GrB_ALL, ns, lib.GrB_ALL, n, ffi.NULL))
        res.setdefault(route, []).append(tot)
        outs[route] = paths
    return {"old_ms": statistics.median(res["old"]) * 1e3, "new_ms": statistics.median(res["new"]) * 1e3, "equal": same(outs["old"], outs["new"])}


def two_hop(A, reps):
    res, outs = {}, {}
    for route in ("old", "new") * reps:
        dt, C = timed(lambda: step(route, A, A, A, gb.BOOL.ANY_PAIR, descriptor.RSC, gb.BOOL.IDENTITY))
        res.setdefault(route, []).append(dt)
        outs[route] = C
    return {"old_ms": statistics.median(res["old"]) * 1e3, "new_ms": statistics.median(res["new"]) * 1e3,
            "equal": same(outs["old"], outs["new"]), "nvals": outs["new"].nvals}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scales", type=int, nargs="+", default=[20, 22])
    ap.add_argument("--ks", type=int, nargs="+", default=[4, 64], help="BFS source counts")
    ap.add_argument("--two-hop-scale", type=int, default=16)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--pull", action="store_true", help="push / dot / auto arms of the multi-source BFS step")
    ap.add_argument("--alphas", type=float, nargs="+", default=[2, 4, 8, 14, 32])
    a = ap.parse_args()
    if not gb.have_device():
        raise SystemExit("msbfs_bench: no CUDA device")
    report = {"card": card(), "workloads": []}
    print("card (name, power limit, max SM clock):", report["card"], flush=True)
    for scale in a.scales:
        n, indptr, indices = rmat_csr(scale, 16, seed=1)
        S = sp.csr_matrix((np.ones(len(indices), np.float32), indices, indptr), shape=(n, n))
        Ab = Matrix.from_csr(indptr, indices, np.ones(len(indices), bool), n, n, gb.BOOL)
        Af = Matrix.from_csr(indptr, indices, np.ones(len(indices), np.float32), n, n, gb.FP32)
        for k in a.ks:
            if a.pull:
                r = {"workload": f"msbfs pull s{scale} k={k}", **msbfs_pull(Ab, S, n, k, a.reps, a.alphas)}
            else:
                r = {"workload": f"msbfs s{scale} k={k}", **msbfs(Ab, S, n, k, a.reps)}
            print(json.dumps(r), flush=True)
            report["workloads"].append(r)
        if a.pull:
            continue
        r = {"workload": f"bc-forward s{scale} 4 sources", **bc_forward(Af, S, n, a.reps)}
        print(json.dumps(r), flush=True)
        report["workloads"].append(r)
    if not a.pull:
        n, indptr, indices = rmat_csr(a.two_hop_scale, 16, seed=1)
        Ab = Matrix.from_csr(indptr, indices, np.ones(len(indices), bool), n, n, gb.BOOL)
        r = {"workload": f"C<!A,R> = A any.pair A s{a.two_hop_scale}", **two_hop(Ab, a.reps)}
        print(json.dumps(r), flush=True)
        report["workloads"].append(r)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "msbfs_bench.json"), "w") as f:
            json.dump(report, f, indent=1)
    bad = [w["workload"] for w in report["workloads"] if not w.get("equal", True) or not w.get("matches_scipy", True)]
    if bad:
        raise SystemExit(f"results differ: {bad}")


if __name__ == "__main__":
    main()
