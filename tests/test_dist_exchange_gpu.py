"""The exchange of csrc/dist.cu (B200_Comm_allgather, B200_Comm_allreduce, B200_Comm_barrier) run by real ranks and checked
against a restatement of what each collective computes.

Every rank is a process of its own (torch.multiprocessing.spawn; gloo carries the control plane), and rank r uses device
r % ndev through B200GRB_DEVICE.  Two modes:
  * shared: every rank on device 0.  CUDA IPC works between processes on one device, and the driver time-slices their
    contexts, so this mode runs on a single GPU;
  * spread: rank r on device r, when at least `world` devices are visible.
Each world size (1, 2, 3, 4) of each mode is spawned once per module.  Every rank runs the same fixed list of cases and keeps
each case's raw result: the view's values and presence (a digest of them for long vectors).  The parametrized tests below
check them case by case after the ranks have exited.  Each run records its mode and the device of every rank.

A rank that waits for a peer that never arrives traps after 20 s, which is a GPU fault.  So the ranks keep these rules:
  * No rank asserts, skips or branches on a result between collectives.  All ranks make the same sequence of collective
    calls, and all checking happens in the parent after join.
  * Before each case the ranks agree, over gloo, that every rank built its inputs on the host.  If one did not, no rank
    enqueues the case.  After each case they agree that every rank's calls were accepted; if one was not, all stop.
  * Every argument form a rank passes at world > 1 is first passed at world 1, in this module.  A world > 1 case is
    skipped, not run, when the world-1 run refused one of its forms.
  * Refusals are tested at world 1 only.
  * The ranks are joined with a timeout, after which they are terminated: no process outlives the module.

Models.  All-gather: position i holds exactly what the slice covering i holds; presence identical, values bit for bit where
present, any NaN matching any NaN.  All-reduce: position i holds the fold (oracle/vecmodel.reduce) of the partials present at
i, in rank order from the first present one, and is absent where none is; kernel_check.compare decides (bit for bit, +-0
matching under MIN / MAX, an ANY value one of the present values).  The order is fixed, so FP PLUS and TIMES are exact too.

This module imports the library only inside functions: a rank must set B200GRB_DEVICE before the library starts.
"""
import hashlib
import json
import os
import socket
import time
import traceback
import zlib
from datetime import timedelta

import numpy as np
import pytest

import util
from oracle import vecmodel as vm
from oracle.pymodel import DT

pytestmark = pytest.mark.gpu

WORLDS = (1, 2, 3, 4)
RUNS = [("shared", w) for w in WORLDS] + [("spread", w) for w in WORLDS if w > 1]
JOIN_TIMEOUT = 1200                      # seconds for one spawned world
AG_NS = (1, 15, 16, 17, 33, 255, 256, 257, 4099, (1 << 20) + 3)
AG_LAYOUTS = ("eq-full", "eq-pres", "eq-none", "cut-mixed")
AR_NS = (17, 1000)                       # 17 at world 4: ranks 2 and 3 own empty fold ranges; 1000: the last range ends inside a word
AR_VARIANTS = ("dense", "sparse", "mixed")
DIGEST_N = 1 << 16                       # results at least this long are kept as digests
SEQ_STEPS = 200
HOLD_CYCLES = 6_000_000                  # torch.cuda._sleep: a few ms
FRESH = [(1, 0), (10, 0), (17, 0), (1, 48), (10, 48), (16, 48)]     # (length, row0) of single slices into a fresh n = 64 communicator


def seed_of(*parts):
    return zlib.crc32(repr(parts).encode())


def esize(typ):
    return np.dtype(DT[typ]).itemsize


def ag_ns(typ):
    """The lengths of the all-gather cases: AG_NS and n with n * esize just below, at and just above 256 (the end of the
    value bytes in the region is rounded to 256, and the presence bytes start there)."""
    k = 256 // esize(typ)
    return sorted(set(AG_NS) | {k - 1, k, k + 1})


def equal_row_blocks(n, world):
    from pygraphblas_b200.distributed import equal_row_blocks as erb
    return erb(n, world)


def cut_bounds(n, world, seed):
    """Hand-cut bounds covering [0, n): uneven multiples of 16, and from world 3 on a zero-length slice in the middle."""
    if world == 1:
        return [0, n]
    inner = sorted(int(x) * 16 for x in np.random.default_rng(seed).integers(0, n // 16 + 1, world - 1))
    if world >= 3:
        inner[1] = inner[0]
    return [0] + inner + [n]


def monoids(typ):
    from test_glue_edges_gpu import monoids_for
    return monoids_for(typ)


# ------------------------------------------------------------------ case specs (pure data; the same in the parent and every rank)
def ag_spec(typ, n, layout, world):
    if layout.startswith("eq"):
        bounds = equal_row_blocks(n, world)
    else:
        bounds = cut_bounds(n, world, seed_of(typ, n, world))
    fills = {"eq-full": ["full"] * world, "eq-pres": ["pres"] * world, "eq-none": ["none"] * world,
             "cut-mixed": [("pres", "full", "none")[r % 3] for r in range(world)]}[layout]
    return {"name": f"ag-{typ}-{n}-{layout}", "group": f"ag-{typ}", "kind": "ag", "type": typ, "n": n, "bounds": bounds, "fills": fills}


def fresh_spec(typ, length, row0, fill):
    return {"name": f"fresh-{typ}-{length}-at{row0}-{fill}", "group": "fresh", "kind": "fresh", "type": typ, "n": 64,
            "row0": row0, "len": length, "fill": fill}


def ar_spec(typ, n, op, variant):
    return {"name": f"ar-{typ}-{n}-{op}-{variant}", "group": f"ar-{typ}", "kind": "ar", "type": typ, "n": n, "op": op, "variant": variant}


def slice_data(name, typ, m, fill, r):
    """(values, presence or None) of rank r's slice of length m."""
    rng = np.random.default_rng(seed_of("slice", name, r))
    x = util.rand_edge_values(rng, typ, m, 0.5)
    if fill == "full":
        return x, None
    return x, ((rng.random(m) < 0.6) if fill == "pres" else np.zeros(m, bool)).astype(np.uint8)


def ar_presence(spec, world):
    """[world, n] presence of the partials: position i follows pattern i % (world + 3): none present, only rank r (each r),
    all present, random.  Dense partials are all present; "mixed" makes rank 0's dense."""
    n = spec["n"]
    kind = np.arange(n) % (world + 3)
    P = np.zeros((world, n), bool)
    for r in range(world):
        P[r, kind == r + 1] = True
    P[:, kind == world + 1] = True
    rnd = kind == world + 2
    P[:, rnd] = np.random.default_rng(seed_of("pres", spec["name"], world)).random((world, int(rnd.sum()))) < 0.5
    if spec["variant"] == "dense":
        P[:] = True
    elif spec["variant"] == "mixed":
        P[0] = True
    return P


def ar_dense(spec, r):
    return spec["variant"] == "dense" or (spec["variant"] == "mixed" and r == 0)


def ar_values(spec, r):
    return util.rand_edge_values(np.random.default_rng(seed_of("part", spec["name"], r)), spec["type"], spec["n"], 0.5)


def forms_of(spec, world):
    """The argument forms every rank passes: what a world-1 run has to accept before this case may run at world > 1."""
    if spec["kind"] == "ag":
        b = spec["bounds"]
        return [("ag", spec["type"], spec["n"], b[r], b[r + 1] - b[r], spec["fills"][r] == "full") for r in range(world)]
    if spec["kind"] == "ar":
        return [("ar", spec["type"], spec["n"], spec["op"], ar_dense(spec, r)) for r in range(world)]
    return [tuple(f) for f in spec.get("forms", [])]


# the compound cases: sequences, views, free / re-create, and the forms bench.py --gpus N runs
SEQ_A, SEQ_B = ("FP32", 100), ("INT16", 77)
SEQ_B_MONOIDS = ("PLUS", "MIN", "MAX", "TIMES")


def seq_step(k):
    """Step k of the sequence: (what, communicator); rank k % world is held back before it."""
    return [("ag", "A"), ("ar", "B"), ("barrier", "A"), ("ag", "B"), ("ar-view", "A"), ("barrier", "B")][k % 6]


def seq_forms(world):
    fs = []
    for typ, n in (SEQ_A, SEQ_B):
        b = equal_row_blocks(n, world)
        fs += [("ag", typ, n, b[r], b[r + 1] - b[r], typ == SEQ_B[0]) for r in range(world)]
    fs += [("ar", SEQ_B[0], SEQ_B[1], op, False) for op in SEQ_B_MONOIDS] + [("ar", SEQ_A[0], SEQ_A[1], "MIN", False)]
    return fs


def views_forms(world):
    b = equal_row_blocks(32, world)
    return [("ag", "INT32", 32, b[r], b[r + 1] - b[r], False) for r in range(world)] + \
           [("ag", "INT32", 32 * world, 32 * r, 32, False) for r in range(world)] + [("ar", "INT32", 32, "MAX", False)]


BENCH_SCALE = 12


def bench_graph():
    from pygraphblas_b200.generators import rmat_csr
    n, indptr, indices = rmat_csr(BENCH_SCALE, 8, seed=5)
    rng = np.random.default_rng(11)
    vals = (rng.random(len(indices), dtype=np.float32) + np.float32(0.5)).astype(np.float32)
    u0 = rng.random(n, dtype=np.float32)
    return n, indptr, indices, vals, u0


def bench_forms(world, typ, n, pres):
    b = equal_row_blocks(n, world)
    return [("ag", typ, n, b[r], b[r + 1] - b[r], not pres) for r in range(world)]


def all_cases(world):
    cases = []
    for typ in util.ALL_T:
        for n in ag_ns(typ):
            cases += [ag_spec(typ, n, layout, world) for layout in AG_LAYOUTS]
    if world == 1:
        cases += [fresh_spec(typ, m, row0, fill) for typ in ("INT8", "FP32", "FP64") for m, row0 in FRESH for fill in ("full", "pres")]
    for typ in util.ALL_T:
        for n in AR_NS:
            cases += [ar_spec(typ, n, op, v) for op in monoids(typ) for v in AR_VARIANTS]
    n = 1 << BENCH_SCALE
    cases += [
        {"name": "seq", "group": "seq", "kind": "seq", "forms": seq_forms(world)},
        {"name": "views", "group": "views", "kind": "views", "forms": views_forms(world)},
        {"name": "recreate", "group": "recreate", "kind": "recreate",
         "forms": bench_forms(world, "INT64", 48, False) + bench_forms(world, "INT64", 48, True)},
        # mxv returns its slice in whatever form it chose: both forms are probed
        {"name": "mxv-PLUS_TIMES", "group": "bench-mxv", "kind": "mxv", "sr": "PLUS_TIMES",
         "forms": bench_forms(world, "FP32", n, False) + bench_forms(world, "FP32", n, True)},
        {"name": "mxv-MIN_PLUS", "group": "bench-mxv", "kind": "mxv", "sr": "MIN_PLUS",
         "forms": bench_forms(world, "FP32", n, False) + bench_forms(world, "FP32", n, True)},
        {"name": "bfs", "group": "bench-bfs", "kind": "bfs", "forms": bench_forms(world, "BOOL", n, True)},
        {"name": "sssp", "group": "bench-sssp", "kind": "sssp", "forms": [("ar", "FP32", n, "MIN", False), ("ar", "FP32", n, "MIN", True)]},
    ]
    return cases


# ------------------------------------------------------------------ the ranks
class Rank:
    def __init__(self, rank, world, gb):
        import torch
        self.rank, self.world, self.gb = rank, world, gb
        self.comms = {}
        p = gb.ffi.new("void**")
        gb.lib.B200_get_stream(p)
        self.stream = torch.cuda.ExternalStream(int(gb.ffi.cast("uintptr_t", p[0])))

    def comm(self, typ, n):
        """The communicator of (typ, n), shared by consecutive cases; creating one frees the others (collective: the ranks
        meet cases in the same order)."""
        from pygraphblas_b200.distributed import Comm
        if (typ, n) not in self.comms:
            self.close()
            self.comms[(typ, n)] = Comm(n, util.g_type(typ), self.rank, self.world)
        return self.comms[(typ, n)]

    def close(self):
        for c in self.comms.values():
            c.close()
        self.comms.clear()

    def hold(self):
        import torch
        with torch.cuda.stream(self.stream):
            torch.cuda._sleep(HOLD_CYCLES)

    def vec(self, typ, x, p):
        return self.gb.Vector.from_numpy(x, present=p, typ=util.g_type(typ))


def keep(v):
    """A view's (values, presence) as the parent checks them; a digest for long vectors."""
    x, p = v.to_numpy()
    if len(p) >= DIGEST_N:
        return {"digest": np.array(digest(x, p))}
    return {"x": x, "p": p}


def digest(x, p):
    x = np.where(p != 0, x, np.zeros((), x.dtype))
    return hashlib.sha256((p != 0).tobytes() + x.tobytes()).hexdigest()


def build_case(R, spec):
    """Host-side inputs of this rank (nothing is enqueued on a communicator here)."""
    k, r, W = spec["kind"], R.rank, R.world
    if k == "ag":
        b = spec["bounds"]
        x, p = slice_data(spec["name"], spec["type"], b[r + 1] - b[r], spec["fills"][r], r)
        return R.vec(spec["type"], x, p)
    if k == "fresh":
        x, p = slice_data(spec["name"], spec["type"], spec["len"], spec["fill"], r)
        return R.vec(spec["type"], x, p)
    if k == "ar":
        P = ar_presence(spec, W)
        return R.vec(spec["type"], ar_values(spec, r), None if ar_dense(spec, r) else P[r].astype(np.uint8))
    if k == "seq":
        return [seq_inputs(R, k2) for k2 in range(SEQ_STEPS)]
    if k == "views":
        b = equal_row_blocks(32, W)
        x, p = slice_data("views", "INT32", b[r + 1] - b[r], "pres", r)
        return R.vec("INT32", x, p)
    if k == "recreate":
        b = equal_row_blocks(48, W)
        return [R.vec("INT64", *slice_data(f"recreate{j}", "INT64", b[r + 1] - b[r], fill, r)) for j, fill in enumerate(("full", "pres"))]
    import scipy.sparse as sp
    n, indptr, indices, vals, u0 = bench_graph()
    b = equal_row_blocks(n, W)
    if k == "bfs":
        S = sp.csr_matrix((np.ones(len(indices), bool), indices, indptr), shape=(n, n)).T.tocsr()[b[r]:b[r + 1]]
        return R.gb.Matrix.from_csr(S.indptr, S.indices, S.data, b[r + 1] - b[r], n, R.gb.BOOL), n, b
    S = sp.csr_matrix((vals, indices, indptr), shape=(n, n))[b[r]:b[r + 1]]
    return R.gb.Matrix.from_csr(S.indptr, S.indices, S.data, b[r + 1] - b[r], n, R.gb.FP32), n, b, u0


def seq_inputs(R, k):
    what, which = seq_step(k)
    typ, n = SEQ_A if which == "A" else SEQ_B
    if what == "ag":
        b = equal_row_blocks(n, R.world)
        return R.vec(typ, *slice_data(f"seq{k}", typ, b[R.rank + 1] - b[R.rank], "pres" if which == "A" else "full", R.rank))
    if what == "ar":
        spec = {"name": f"seq{k}", "n": n, "variant": "sparse", "type": typ}
        return R.vec(typ, ar_values(spec, R.rank), ar_presence(spec, R.world)[R.rank].astype(np.uint8))
    return None


def monoid(typ, op):
    return getattr(util.g_type(typ), f"{op}_MONOID")


def run_case(R, spec, inp):
    """Enqueue the case's collectives; returns {key: array} to keep.  Makes the same collective calls on every rank."""
    gb, r, W, k = R.gb, R.rank, R.world, spec["kind"]
    if k == "ag":
        return keep(R.comm(spec["type"], spec["n"]).allgather(inp, spec["bounds"][r]))
    if k == "fresh":
        R.close()
        return keep(R.comm(spec["type"], spec["n"]).allgather(inp, spec["row0"]))
    if k == "ar":
        return keep(R.comm(spec["type"], spec["n"]).allreduce(inp, monoid(spec["type"], spec["op"])))
    if k == "seq":
        R.close()
        from pygraphblas_b200.distributed import Comm
        cs = {"A": Comm(SEQ_A[1], util.g_type(SEQ_A[0]), r, W), "B": Comm(SEQ_B[1], util.g_type(SEQ_B[0]), r, W)}
        bounds = {c: equal_row_blocks(cs[c].n, W) for c in cs}
        dups = []
        for step in range(SEQ_STEPS):                 # no host synchronisation until every step is enqueued
            what, which = seq_step(step)
            c = cs[which]
            if step % W == r:
                R.hold()
            if what == "ag":
                dups.append(c.allgather(inp[step], bounds[which][r]).dup())
            elif what == "ar":
                dups.append(c.allreduce(inp[step], monoid(c.type.name, SEQ_B_MONOIDS[(step // 6) % 4])).dup())
            elif what == "ar-view":
                dups.append(c.allreduce(c._view(), monoid(c.type.name, "MIN")).dup())
            else:
                c.barrier()
        out = {}
        for j, d in enumerate(dups):
            x, p = d.to_numpy()
            out[f"{j}x"], out[f"{j}p"] = x, p
        for c in cs.values():
            c.close()
        return out
    if k == "views":
        R.close()
        from pygraphblas_b200.distributed import Comm
        small, big = Comm(32, gb.INT32, r, W), Comm(32 * W, gb.INT32, r, W)
        fresh = small._view().dup()                   # B200_Comm_result before any collective
        s = small.allgather(inp, equal_row_blocks(32, W)[r])
        s_d = s.dup()
        g = big.allgather(s, 32 * r)                  # a view as the next slice
        a = small.allreduce(s, monoid("INT32", "MAX"))  # and as the next partial, of its own communicator
        out = {}
        for key, v in (("fresh", fresh), ("small", s_d), ("big", g), ("max", a)):
            x, p = v.to_numpy()
            out[key + "x"], out[key + "p"] = x, p
        small.close(); big.close()
        return out
    if k == "recreate":
        R.close()
        from pygraphblas_b200.distributed import Comm
        out = {}
        for j in range(2):                            # free and create again in the same processes
            c = Comm(48, gb.INT64, r, W)
            x, p = c._view().to_numpy()
            out[f"fresh{j}x"], out[f"fresh{j}p"] = x, p
            x, p = c.allgather(inp[j], c.bounds[r]).to_numpy()
            out[f"{j}x"], out[f"{j}p"] = x, p
            c.close()
        return out
    R.close()
    from pygraphblas_b200.distributed import Comm
    from pygraphblas_b200 import descriptor
    if k == "mxv":
        A, n, b, u0 = inp
        comm = Comm(n, gb.FP32, r, W)
        sr = getattr(gb.FP32, spec["sr"])
        u, dups = gb.Vector.from_numpy(u0), []
        for step in range(4):                          # chained: each step's view is the next step's u
            u = comm.allgather(A.mxv(u, semiring=sr), b[r])
            dups.append(u.dup())
        out = {}
        for j, d in enumerate(dups):
            out[f"{j}x"], out[f"{j}p"] = d.to_numpy()
        comm.close()
        return out
    if k == "bfs":
        A, n, b = inp
        comm = Comm(n, gb.BOOL, r, W)
        level = np.full(n, -1, np.int64)
        level[0] = 0
        visited = level >= 0
        q = gb.Vector.from_numpy(visited.copy(), present=visited.astype(np.uint8))
        for depth in range(1, BFS_LEVELS + 1):          # a fixed number of levels: no rank stops on what it found
            yx, yp = A.mxv(q, semiring=gb.BOOL.LOR_LAND).to_numpy()
            new = (yp != 0) & (yx != 0) & ~visited[b[r]:b[r + 1]]
            sl = gb.Vector.from_numpy(new, present=new.astype(np.uint8))
            q = comm.allgather(sl, b[r])
            qx, qp = q.to_numpy()
            f = qp != 0
            level[f & ~visited] = depth
            visited |= f
        comm.close()
        return {"level": level}
    A, n, b, u0 = inp                                   # sssp: the T0 partial of my rows, MIN all-reduce
    comm = Comm(n, gb.FP32, r, W)
    dx, dp = np.zeros(n, np.float32), np.zeros(n, bool)
    dp[0] = True
    for _ in range(SSSP_ITERS):
        part = A.mxv(gb.Vector.from_numpy(dx[b[r]:b[r + 1]], present=dp[b[r]:b[r + 1]].astype(np.uint8)), semiring=gb.FP32.MIN_PLUS, desc=descriptor.T0)
        rx, rp = comm.allreduce(part, gb.FP32.MIN_MONOID).to_numpy()
        dx, dp = sssp_update(dx, dp, rx, rp)
    comm.close()
    return {"x": dx, "p": dp.astype(np.uint8)}


BFS_LEVELS = 12
SSSP_ITERS = 10


def sssp_update(dx, dp, rx, rp):
    rp = rp != 0
    take = rp & (~dp | (rx < dx))
    return np.where(take, rx, dx).astype(np.float32), dp | rp


def probe(R, forms):
    """Run each form once at world 1; returns the refused ones with the library's message."""
    refused = []
    for f in sorted(set(forms), key=repr):
        kind, typ, n = f[0], f[1], f[2]
        try:
            c = R.comm(typ, n)
            if kind == "ag":
                row0, m, full = f[3], f[4], f[5]
                c.allgather(R.vec(typ, np.zeros(m, DT[typ]), None if full else np.ones(m, np.uint8)), row0)
            else:
                c.allreduce(R.vec(typ, np.zeros(n, DT[typ]), None if f[4] else np.ones(n, np.uint8)), monoid(typ, f[3]))
        except Exception as e:
            refused.append([list(f), f"{type(e).__name__}: {e}"])
    R.close()
    return refused


def _agree(flag):
    import torch
    import torch.distributed as dist
    t = torch.tensor([1 if flag else 0])
    dist.all_reduce(t, op=dist.ReduceOp.MIN)
    return bool(t.item())


def _rank_main(rank, world, mode, port, outdir, probe_forms, refused):
    import torch
    ndev = torch.cuda.device_count()
    dev = 0 if mode == "shared" else rank % max(ndev, 1)
    os.environ["B200GRB_DEVICE"] = str(dev)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=timedelta(seconds=300))
    t0 = time.monotonic()
    status = {"mode": mode, "world": world, "rank": rank, "device": dev, "cases": {}, "refused": []}
    results = {}
    try:
        err = ""
        try:
            torch.cuda.set_device(dev)
            torch.zeros(1, device=f"cuda:{dev}")          # a context of this process's own on the device
            import pygraphblas_b200 as gb
            if not gb.have_device():
                err = f"the library could not use device {dev}"
        except Exception as e:                            # e.g. the device admits one process only
            err = f"{type(e).__name__}: {e}"
        errs = [None] * world
        dist.all_gather_object(errs, err)
        if any(errs):
            status["no_context"] = [e for e in errs if e]
            return
        R = Rank(rank, world, gb)
        if world == 1 and probe_forms:
            status["refused"] = probe(R, [tuple(f) for f in probe_forms])
        bad = {tuple(f) for f in refused}
        stopped = None
        for spec in all_cases(world):
            name = spec["name"]
            if stopped:
                status["cases"][name] = stopped
                continue
            if world > 1 and any(f in bad for f in forms_of(spec, world)):
                status["cases"][name] = "skipped: the world-1 run refused one of its argument forms"
                continue
            inp, msg = None, ""
            try:
                inp = build_case(R, spec)
            except Exception:
                msg = traceback.format_exc(limit=4)
            if not _agree(not msg):
                status["cases"][name] = "host: " + (msg or "another rank could not build its inputs")
                continue
            out = None
            try:
                out = run_case(R, spec, inp)
            except Exception:
                msg = traceback.format_exc(limit=4)
            good = _agree(out is not None)
            if out is not None:
                status["cases"][name] = "ok"
                for key, a in out.items():
                    results[f"{name}@{key}"] = a
            else:
                status["cases"][name] = "error: " + (msg or "another rank's call failed")
            if not good and world > 1:
                stopped = f"not run: a rank's call failed in case {name}"
            del inp
        R.close()
    except Exception:
        status["fatal"] = traceback.format_exc()
    finally:
        status["seconds"] = time.monotonic() - t0
        np.savez(os.path.join(outdir, f"res.{rank}.npz"), **results)
        with open(os.path.join(outdir, f"status.{rank}.json"), "w") as f:
            json.dump(status, f)
        dist.destroy_process_group()


# ------------------------------------------------------------------ the parent: spawn once per (mode, world), then check
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _spawn(world, mode, outdir, probe_forms, refused):
    import torch.multiprocessing as mp
    ctx = mp.spawn(_rank_main, args=(world, mode, _free_port(), str(outdir), probe_forms, refused), nprocs=world, join=False)
    deadline, err = time.monotonic() + JOIN_TIMEOUT, None
    try:
        while not ctx.join(timeout=5):
            if time.monotonic() > deadline:
                err = f"the ranks did not finish within {JOIN_TIMEOUT} s"
                break
    except Exception as e:
        err = f"{type(e).__name__}: {e}"
    finally:
        for p in ctx.processes:
            if p.is_alive():
                p.terminate()
            p.join(30)
            if p.is_alive():
                p.kill()
                p.join()
    run = {"world": world, "mode": mode, "err": err, "status": [], "res": []}
    for r in range(world):
        try:
            with open(os.path.join(outdir, f"status.{r}.json")) as f:
                run["status"].append(json.load(f))
            run["res"].append(dict(np.load(os.path.join(outdir, f"res.{r}.npz"))))
        except OSError as e:
            run["err"] = (run["err"] or "") + f"; rank {r} left no result ({e})"
    run["specs"] = {s["name"]: s for s in all_cases(world)}
    return run


@pytest.fixture(scope="module")
def runs(tmp_path_factory):
    done = {}

    def get(mode, world):
        if (mode, world) not in done:
            if mode == "spread":
                import torch
                if torch.cuda.device_count() < world:
                    pytest.skip(f"spread mode at world {world} needs {world} GPUs; {torch.cuda.device_count()} visible")
            if world == 1:
                forms = sorted({f for w in WORLDS[1:] for s in all_cases(w) for f in forms_of(s, w)}, key=repr)
                done[(mode, world)] = _spawn(1, mode, tmp_path_factory.mktemp("w1"), forms, [])
            else:
                w1 = get("shared", 1)
                refused = [f for f, _ in w1["status"][0]["refused"]] if w1["status"] else []
                done[(mode, world)] = _spawn(world, mode, tmp_path_factory.mktemp(f"{mode}{world}"), [], refused)
        run = done[(mode, world)]
        assert run["status"] and len(run["status"]) == world, f"{mode} world {world}: {run['err']}"
        nc = run["status"][0].get("no_context")
        if nc:
            pytest.skip(f"a second process could not use the device: {nc[0]}")
        for s in run["status"]:
            assert "fatal" not in s, s["fatal"]
            assert s["mode"] == mode and s["device"] == (0 if mode == "shared" else s["rank"]), s
        return run
    return get


def check_group(run, group, check):
    """Run check(spec, results of every rank) on each case of the group; fail with all mismatches, then skip if cases were
    skipped."""
    fails, skips, n = [], [], 0
    for name, spec in run["specs"].items():
        if spec["group"] != group:
            continue
        sts = {s["cases"].get(name, "missing") for s in run["status"]}
        if sts != {"ok"}:
            st = sorted(sts)
            (skips if all(x.startswith("skipped") for x in st) else fails).append(f"{name}: {st[0][:800]}")
            continue
        per_rank = [{k.split("@", 1)[1]: v for k, v in res.items() if k.split("@", 1)[0] == name} for res in run["res"]]
        for r, got in enumerate(per_rank):
            err = check(spec, got, run["world"])
            if err:
                fails.append(f"rank {r} of {run['world']} ({run['mode']}): {err}")
        n += 1
    assert not fails, f"{len(fails)} failures, e.g.\n" + "\n".join(fails[:8])
    assert n or skips, f"no case in group {group}"
    if skips:
        pytest.skip(f"{len(skips)} cases not run: {skips[0]}")


def same_bits(gx, wx):
    """Bit for bit; any NaN matches any NaN."""
    b = util_bits(gx) == util_bits(wx)
    if gx.dtype.kind == "f":
        b |= np.isnan(gx) & np.isnan(wx)
    return b


def util_bits(x):
    x = np.ascontiguousarray(x)
    return x.view(f"u{x.dtype.itemsize}") if x.dtype != np.bool_ else x


def ag_model(spec, world):
    typ, n, b = spec["type"], spec["n"], spec["bounds"]
    x, p = np.zeros(n, DT[typ]), np.zeros(n, np.uint8)
    for r in range(world):
        xs, ps = slice_data(spec["name"], typ, b[r + 1] - b[r], spec["fills"][r], r)
        x[b[r]:b[r + 1]] = xs
        p[b[r]:b[r + 1]] = 1 if ps is None else ps
    return x, p


def vec_diff(gx, gp, wx, wp, label):
    if not np.array_equal(gp != 0, wp != 0):
        d = np.flatnonzero((gp != 0) != (wp != 0))
        return f"{label}: presence differs at {d[:6].tolist()} (got {gp[d[:6]].tolist()}, want {wp[d[:6]].tolist()})"
    on = wp != 0
    ok = same_bits(gx[on], wx[on])
    if not ok.all():
        i = np.flatnonzero(on)[~ok][:6]
        return f"{label}: values differ at {i.tolist()}: got {gx[i].tolist()}, want {wx[i].tolist()}"
    return None


def check_ag(spec, got, world):
    wx, wp = ag_model(spec, world)
    if "digest" in got:
        return None if str(got["digest"]) == digest(wx, wp) else f"{spec['name']}: digest of the result differs from the model's"
    return vec_diff(got["x"], got["p"], wx, wp, spec["name"])


def check_fresh(spec, got, world):
    typ, n, row0, m = spec["type"], spec["n"], spec["row0"], spec["len"]
    xs, ps = slice_data(spec["name"], typ, m, spec["fill"], 0)
    wx, wp = np.zeros(n, DT[typ]), np.zeros(n, np.uint8)
    wx[row0:row0 + m] = xs
    wp[row0:row0 + m] = 1 if ps is None else ps
    return vec_diff(got["x"], got["p"], wx, wp, spec["name"])


def ar_fold(typ, op, X, P, label, gx, gp):
    """Compare an all-reduce result with the rank-order fold of partials X[r] present where P[r]."""
    import kernel_check as kc
    world, n = P.shape
    keys, want, cand_k, cand_v = [], [], [], []
    for i in range(n):
        rs = [r for r in range(world) if P[r, i]]
        if not rs:
            continue
        keys.append(i)
        want.append(vm.reduce(op, typ, {r: X[r][i] for r in rs}, 0) if op != "ANY" else X[rs[0]][i])
        cand_k += [i] * len(rs)
        cand_v += [X[r][i] for r in rs]
    gI = np.flatnonzero(gp != 0)
    cands = kc._candidates(np.array(cand_k, np.int64), np.array(cand_v, DT[typ])) if op == "ANY" else None
    return kc.compare(gI, gx[gI], keys, np.array(want, DT[typ]), typ, op, label, cands)


def check_ar(spec, got, world):
    P = ar_presence(spec, world)
    X = [ar_values(spec, r) for r in range(world)]
    return ar_fold(spec["type"], spec["op"], X, P, spec["name"], got["x"], got["p"])


def check_seq(spec, got, world):
    state = {}
    j = 0
    for k in range(SEQ_STEPS):
        what, which = seq_step(k)
        typ, n = SEQ_A if which == "A" else SEQ_B
        if what == "barrier":
            continue
        gx, gp = got[f"{j}x"], got[f"{j}p"]
        label = f"seq step {k} ({what} on {which})"
        if what == "ag":
            b = equal_row_blocks(n, world)
            wx, wp = ag_model({"name": f"seq{k}", "type": typ, "n": n, "bounds": b,
                               "fills": ["pres" if which == "A" else "full"] * world}, world)
            err = vec_diff(gx, gp, wx, wp, label)
        elif what == "ar":
            sp_ = {"name": f"seq{k}", "n": n, "variant": "sparse", "type": typ}
            wx = None
            err = ar_fold(typ, SEQ_B_MONOIDS[(k // 6) % 4], [ar_values(sp_, r) for r in range(world)], ar_presence(sp_, world), label, gx, gp)
        else:
            px, pp = state[which]
            err = ar_fold(typ, "MIN", [px] * world, np.tile(pp != 0, (world, 1)), label, gx, gp)
        if err:
            return err
        state[which] = (gx, gp)          # the next step is checked against its actual input, so one error is reported once
        j += 1
    return None


def check_views(spec, got, world):
    b = equal_row_blocks(32, world)
    wx, wp = ag_model({"name": "views", "type": "INT32", "n": 32, "bounds": b, "fills": ["pres"] * world}, world)
    return (vec_diff(got["freshx"], got["freshp"], wx, np.zeros(32, np.uint8), "B200_Comm_result before any collective")
            or vec_diff(got["smallx"], got["smallp"], wx, wp, "all-gather")
            or vec_diff(got["bigx"], got["bigp"], np.tile(wx, world), np.tile(wp, world), "a view as the next slice")
            or ar_fold("INT32", "MAX", [wx] * world, np.tile(wp != 0, (world, 1)), "a view as the next partial", got["maxx"], got["maxp"]))


def check_recreate(spec, got, world):
    b = equal_row_blocks(48, world)
    for j, fill in enumerate(("full", "pres")):
        wx, wp = ag_model({"name": f"recreate{j}", "type": "INT64", "n": 48, "bounds": b, "fills": [fill] * world}, world)
        err = (vec_diff(got[f"fresh{j}x"], got[f"fresh{j}p"], wx, np.zeros(48, np.uint8), f"communicator {j} before any collective")
               or vec_diff(got[f"{j}x"], got[f"{j}p"], wx, wp, f"communicator {j}"))
        if err:
            return err
    return None


def single_process_mxv(sr, u_steps):
    """The same chain through the library in this process, on the whole matrix (the reference for MIN_PLUS)."""
    import pygraphblas_b200 as gb
    n, indptr, indices, vals, u0 = bench_graph()
    A = gb.Matrix.from_csr(indptr, indices, vals, n, n, gb.FP32)
    u, out = gb.Vector.from_numpy(u0), []
    for _ in range(u_steps):
        u = A.mxv(u, semiring=getattr(gb.FP32, sr))
        out.append(u.to_numpy())
    return out


def check_mxv(spec, got, world):
    import scipy.sparse as sp
    n, indptr, indices, vals, u0 = bench_graph()
    if spec["sr"] == "MIN_PLUS":
        for k, (wx, wp) in enumerate(single_process_mxv("MIN_PLUS", 4)):
            err = vec_diff(got[f"{k}x"], got[f"{k}p"], wx, wp, f"MIN_PLUS step {k}")
            if err:
                return err
        return None
    # PLUS_TIMES: each step against the fp64 product of the step's actual input, within the error bound of a
    # (deg + 1)-term fp32 dot product
    A = sp.csr_matrix((vals.astype(np.float64), indices, indptr), shape=(n, n))
    Pat = sp.csr_matrix((np.ones(len(indices)), indices, indptr), shape=(n, n))
    deg = np.diff(indptr)
    ux, up = u0.astype(np.float64), np.ones(n, bool)
    for k in range(4):
        gx, gp = got[f"{k}x"], got[f"{k}p"] != 0
        ref = A @ np.where(up, ux, 0.0)
        wp = (Pat @ up.astype(np.float64)) > 0
        if not np.array_equal(gp, wp):
            return f"PLUS_TIMES step {k}: presence differs at {np.flatnonzero(gp != wp)[:6].tolist()}"
        tol = (deg + 2) * 2.0 ** -24 * ref                  # all terms are positive: sum |a u| = ref
        bad = np.flatnonzero(gp & ~(np.abs(gx.astype(np.float64) - ref) <= tol))
        if len(bad):
            return f"PLUS_TIMES step {k}: beyond the fp32 error bound at {bad[:6].tolist()}: got {gx[bad[:6]].tolist()}, fp64 {ref[bad[:6]].tolist()}"
        ux, up = gx.astype(np.float64), gp
    return None


def check_bfs(spec, got, world):
    import scipy.sparse as sp
    from scipy.sparse import csgraph
    n, indptr, indices, vals, u0 = bench_graph()
    S = sp.csr_matrix((np.ones(len(indices)), indices, indptr), shape=(n, n))
    d = csgraph.shortest_path(S, directed=True, unweighted=True, indices=0)
    fin = np.isfinite(d)
    assert d[fin].max() < BFS_LEVELS, "the BFS needs more levels than the case runs"
    want = np.where(fin, d, -1).astype(np.int64)
    bad = np.flatnonzero(got["level"] != want)
    return f"BFS levels differ from scipy's at {bad[:6].tolist()}: got {got['level'][bad[:6]].tolist()}, want {want[bad[:6]].tolist()}" if len(bad) else None


def check_sssp(spec, got, world):
    import pygraphblas_b200 as gb
    from pygraphblas_b200 import descriptor
    n, indptr, indices, vals, u0 = bench_graph()
    A = gb.Matrix.from_csr(indptr, indices, vals, n, n, gb.FP32)
    dx, dp = np.zeros(n, np.float32), np.zeros(n, bool)
    dp[0] = True
    for _ in range(SSSP_ITERS):
        rx, rp = A.mxv(gb.Vector.from_numpy(dx, present=dp.astype(np.uint8)), semiring=gb.FP32.MIN_PLUS, desc=descriptor.T0).to_numpy()
        dx, dp = sssp_update(dx, dp, rx, rp)
    return vec_diff(got["x"], got["p"], dx, dp.astype(np.uint8), "SSSP distances")


# ------------------------------------------------------------------ the tests
def test_world1_accepts_every_form(runs):
    """Every argument form the ranks pass at world 2-4 is accepted at world 1: an empty slice at any row0 <= n included
    (equal_row_blocks starts empty trailing blocks at n, which need not be a multiple of 16)."""
    refused = runs("shared", 1)["status"][0]["refused"]
    assert not refused, f"{len(refused)} forms refused at world 1, e.g. {refused[:4]}"


@pytest.mark.parametrize("mode,world", RUNS, ids=[f"{m}-w{w}" for m, w in RUNS])
@pytest.mark.parametrize("typ", util.ALL_T)
def test_allgather(runs, mode, world, typ):
    """equal_row_blocks and hand-cut layouts, full slices, slices with presence and slices with no entries, at every n of
    ag_ns(typ), edge values: every rank's view holds exactly the slices."""
    check_group(runs(mode, world), f"ag-{typ}", check_ag)


def test_fresh_communicator_holds_only_the_slice(runs):
    """A slice of 1, 10, 16 or 17 entries into a fresh n = 64 communicator (both buffers zero): the result holds the slice's
    entries and nothing at any other position -- the push reads and writes exactly [row0, row0 + len)."""
    check_group(runs("shared", 1), "fresh", check_fresh)


@pytest.mark.parametrize("mode,world", RUNS, ids=[f"{m}-w{w}" for m, w in RUNS])
@pytest.mark.parametrize("typ", util.ALL_T)
def test_allreduce(runs, mode, world, typ):
    """Every builtin monoid of the type, dense, sparse and mixed partials, per-position presence patterns (none, only rank r,
    all, random), n = 17 and 1000: the rank-order fold of the present partials (LXNOR included)."""
    check_group(runs(mode, world), f"ar-{typ}", check_ar)


@pytest.mark.parametrize("mode,world", RUNS, ids=[f"{m}-w{w}" for m, w in RUNS])
def test_sequence_back_to_back(runs, mode, world):
    """200 all-gathers, all-reduces and barriers on two communicators of different types, enqueued without a host
    synchronisation, one rank held back before each step: every step's view, dup'd on the stream, is right."""
    check_group(runs(mode, world), "seq", check_seq)


@pytest.mark.parametrize("mode,world", RUNS, ids=[f"{m}-w{w}" for m, w in RUNS])
def test_views_and_recreate(runs, mode, world):
    """A view used as the next slice and as the next partial; B200_Comm_result before any collective; free and create
    again in the same processes."""
    run = runs(mode, world)
    check_group(run, "views", check_views)
    check_group(run, "recreate", check_recreate)


@pytest.mark.parametrize("mode,world", RUNS, ids=[f"{m}-w{w}" for m, w in RUNS])
def test_bench_forms(runs, mode, world):
    """What bench.py --gpus N runs, on an R-MAT scale-12 graph: row-block mxv + all-gather (PLUS_TIMES within the fp32
    bound, MIN_PLUS bit for bit against one process), BFS levels through a BOOL all-gather against scipy, SSSP through a
    T0 partial + MIN all-reduce bit for bit against one process."""
    run = runs(mode, world)
    check_group(run, "bench-mxv", check_mxv)
    check_group(run, "bench-bfs", check_bfs)
    check_group(run, "bench-sssp", check_sssp)


# ------------------------------------------------------------------ refusals, at world 1 in this process
def _comm(n, typ):
    from pygraphblas_b200.distributed import Comm
    return Comm(n, typ, 0, 1)


def _err():
    from pygraphblas_b200 import ffi, lib
    return ffi.string(lib.B200_last_error()).decode()


def test_refuses_a_slice_or_partial_of_another_type_of_the_same_size():
    import pygraphblas_b200 as gb
    lib = gb.lib
    c = _comm(64, gb.FP32)
    s = gb.Vector.from_numpy(np.arange(16, dtype=np.int32))
    assert lib.B200_Comm_allgather(c._comm[0], s._vector[0], 0) == lib.GrB_DOMAIN_MISMATCH, _err()
    p = gb.Vector.from_numpy(np.arange(64, dtype=np.int32))
    assert lib.B200_Comm_allreduce(c._comm[0], p._vector[0], gb.INT32.PLUS_MONOID.get_op()) == lib.GrB_DOMAIN_MISMATCH, _err()
    c2 = _comm(64, gb.UINT8)
    i8, b8, f32 = (gb.Vector.from_numpy(np.zeros(16, dt)) for dt in (np.int8, np.bool_, np.float32))
    assert lib.B200_Comm_allgather(c2._comm[0], i8._vector[0], 0) == lib.GrB_DOMAIN_MISMATCH, _err()
    assert lib.B200_Comm_allgather(c2._comm[0], b8._vector[0], 0) == lib.GrB_DOMAIN_MISMATCH, _err()
    # the same type is accepted
    assert lib.B200_Comm_allgather(c._comm[0], f32._vector[0], 0) == lib.GrB_SUCCESS, _err()
    c.close(); c2.close()


def test_refuses_a_user_defined_or_mismatched_monoid():
    import pygraphblas_b200 as gb
    from pygraphblas_b200 import ffi
    lib = gb.lib
    c = _comm(64, gb.FP32)
    p = gb.Vector.from_numpy(np.ones(64, np.float32))

    @ffi.callback("void(void*, const void*, const void*)")
    def fn(z, x, y):
        pass
    op = ffi.new("GrB_BinaryOp*")
    assert lib.GrB_BinaryOp_new(op, fn, lib.GrB_FP32, lib.GrB_FP32, lib.GrB_FP32) == 0
    mon = ffi.new("GrB_Monoid*")
    assert lib.GrB_Monoid_new_FP32(mon, op[0], 0.0) == 0
    assert lib.B200_Comm_allreduce(c._comm[0], p._vector[0], mon[0]) == lib.GrB_DOMAIN_MISMATCH, _err()
    for m in (gb.FP64.PLUS_MONOID, gb.INT32.MIN_MONOID, gb.BOOL.LOR_MONOID):
        assert lib.B200_Comm_allreduce(c._comm[0], p._vector[0], m.get_op()) == lib.GrB_DOMAIN_MISMATCH, (m, _err())
    assert lib.B200_Comm_allreduce(c._comm[0], p._vector[0], gb.FP32.PLUS_MONOID.get_op()) == lib.GrB_SUCCESS, _err()
    c.close()


def test_refuses_misplaced_slices_and_partials():
    import pygraphblas_b200 as gb
    lib = gb.lib
    c = _comm(64, gb.FP32)
    h = c._comm[0]
    v = lambda m: gb.Vector.from_numpy(np.ones(m, np.float32))
    keep_ = [v(1), v(17), v(16), v(63), v(65)]
    assert lib.B200_Comm_allgather(h, keep_[0]._vector[0], 8) == lib.GrB_INVALID_VALUE, _err()      # non-empty, row0 % 16 != 0
    assert lib.B200_Comm_allgather(h, keep_[1]._vector[0], 48) == lib.GrB_INVALID_VALUE, _err()     # runs past n
    assert lib.B200_Comm_allgather(h, keep_[2]._vector[0], 49) == lib.GrB_INVALID_VALUE, _err()
    # an empty slice writes nothing: accepted at any row0 <= n, refused past n
    e = gb.Vector.sparse(gb.FP32, 0)
    for row0 in (0, 7, 17, 63, 64):
        assert lib.B200_Comm_allgather(h, e._vector[0], row0) == lib.GrB_SUCCESS, (row0, _err())
    assert lib.B200_Comm_allgather(h, e._vector[0], 65) == lib.GrB_INVALID_VALUE, _err()
    for m in (63, 65):
        assert lib.B200_Comm_allreduce(h, keep_[3 if m == 63 else 4]._vector[0], gb.FP32.PLUS_MONOID.get_op()) == lib.GrB_DIMENSION_MISMATCH, _err()
    c.close()


def test_refuses_world_17_and_collectives_before_connect():
    import pygraphblas_b200 as gb
    from pygraphblas_b200 import ffi
    lib = gb.lib
    h = ffi.new("B200_Comm*")
    assert lib.B200_Comm_create(h, 0, 17, 64, lib.GrB_FP32) == lib.GrB_INVALID_VALUE, _err()
    assert lib.B200_Comm_create(h, 0, 2, 64, lib.GrB_FP32) == lib.GrB_SUCCESS, _err()
    s = gb.Vector.from_numpy(np.ones(16, np.float32))
    p = gb.Vector.from_numpy(np.ones(64, np.float32))
    assert lib.B200_Comm_allgather(h[0], s._vector[0], 0) == lib.GrB_INVALID_VALUE, _err()
    assert lib.B200_Comm_allreduce(h[0], p._vector[0], gb.FP32.PLUS_MONOID.get_op()) == lib.GrB_INVALID_VALUE, _err()
    assert lib.B200_Comm_barrier(h[0]) == lib.GrB_INVALID_VALUE, _err()
    assert lib.B200_Comm_free(h) == lib.GrB_SUCCESS
