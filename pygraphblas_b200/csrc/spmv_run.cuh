// The run kernels and their launcher, as templates; instantiated by spmv_run.cu (FP32 / FP64 semirings),
// spmv_run_int.cu (integer / BOOL semirings) and spmv_run_generic.cu (run-time operator codes).
#pragma once
#include "spmv_args.cuh"
#include <map>
#include <tuple>

// ==================================================================================================
// Dense-u kernel for the specialised semirings: warp-independent RUNS.
//
// The entries are cut into runs of 256 (one warp, 8 consecutive entries per lane).  A cached plan gives
// every lane what the tile kernel has to discover with shared-memory marks, a row pass and barriers:
//   run_headw   one bit per entry: "this entry starts a row"
//   run_base    number of row starts before the run;  run_lane: row starts inside the run before the lane
//   nzrow       ids of the non-empty rows (row start rank -> row id);  pres_tmpl: the output's presence
// so a warp needs no shared memory and no barrier: stream 8 entries, gather, fold between the row-start
// bits (rows inside a lane are final), one segmented suffix scan over the 32 lanes, and the two partial
// rows sticking out of the run go to per-run slots that spmv_run_fixup_kernel combines in a fixed order
// (deterministic).  ~3.5x fewer instructions per entry than the tile kernel.
// HOT: persistent CTAs, hot_n most referenced entries of the (relabelled) u in a shared-memory table.


// A lane's share of a run in flight: its 8 matrix values, the 8 values of u it gathered (presence bytes for a sparse u),
// its row-start bits and the rank of its first row start.
template <typename XT> struct RunLane { XT a[8]; XT uv[8]; uint8_t up[8]; uint32_t hb; uint32_t rank; int nvalid; };

// Part 1: everything that ISSUES loads -- the plan words of the lane and the gathers of u.
// `gather(c)` returns u's value for an (encoded) column id of a dense u; SPARSE kernels read p.uval / p.upres directly.
template <typename XT, int MUL_C, bool SPARSE, typename Gather>
__device__ __forceinline__ void spmv_run_gather(const RunArgs &p, const int64_t run, const int lane, const int nvalid,
                                                const uint32_t (&c)[8], RunLane<XT> &L, Gather &&gather) {
    constexpr bool NEED_U = MUL_C < 0 || mul_reads_y(MUL_C);
    const int64_t q = run * RUN + lane * 8;
    const XT *uval = static_cast<const XT *>(p.uval);
    const uint32_t hw = nvalid > 0 ? __ldg(p.headw + (q >> 5)) : 0u;
    L.hb = (hw >> ((lane & 3) * 8)) & 0xffu;                               // this lane's 8 row-start bits
    L.rank = __ldg(p.run_base + run) + __ldg(p.lane_rank + run * 32 + lane);   // row starts before this lane's first entry
    L.nvalid = nvalid;
    if (SPARSE) {
        // u has holes: a product exists only where u(col) does; the values are fetched only for those
#pragma unroll
        for (int j = 0; j < 8; ++j) L.up[j] = j < nvalid ? __ldg(p.upres + c[j]) : (uint8_t)0;
#pragma unroll
        for (int j = 0; j < 8; ++j) L.uv[j] = (NEED_U && L.up[j]) ? gload<XT>(uval + c[j]) : (XT)0;
    } else if (NEED_U) {
#pragma unroll
        for (int j = 0; j < 8; ++j) L.uv[j] = gather(c[j]);
    }
}

// Part 2: multiply, fold between the row-start bits, segmented scan over the lanes, stores.
template <typename XT, typename ZT, int ADD_C, int MUL_C, bool SPARSE>
__device__ __forceinline__ void spmv_run_fold(const RunArgs &p, const int64_t run, const int lane, const RunLane<XT> &L) {
    // ADD_C / MUL_C >= 0: compile-time semiring; -1: run-time operator codes (both operands are read)
    constexpr bool NEED_A = MUL_C < 0 || mul_reads_x(MUL_C);
    constexpr bool NEED_U = MUL_C < 0 || mul_reads_y(MUL_C);
    const int ADD = ADD_C >= 0 ? ADD_C : p.add_op;
    const int MUL = MUL_C >= 0 ? MUL_C : p.mul_op;
    ZT *tval = static_cast<ZT *>(p.tval);
    const int nvalid = L.nvalid;
    const uint32_t hb = L.hb; uint32_t rank = L.rank;
    const uint8_t (&up)[8] = L.up;
    ZT prod[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const XT av = NEED_A ? L.a[j] : (XT)1, uu = NEED_U ? L.uv[j] : (XT)1;
        prod[j] = (MUL_C < 0 && p.flip) ? MulApply<XT, ZT>::f(MUL, uu, av) : MulApply<XT, ZT>::f(MUL, av, uu);
    }

    // ---- fold between row starts
    Part<ZT> acc{(ZT)0, 0}, lead{(ZT)0, 0};
    bool seen = false; uint32_t cur = 0;
    if (nvalid == 8 && !SPARSE) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if ((hb >> j) & 1u) {
                if (!seen) lead = acc;
                else tval[__ldg(p.nzrow + cur)] = acc.v;                    // row began and ended inside this lane
                seen = true; cur = rank++; acc.v = prod[j]; acc.has = 1;
            } else if (j == 0) { acc.v = prod[0]; acc.has = 1; }
            else acc.v = MulApply<ZT, ZT>::f(ADD, acc.v, prod[j]);
        }
    } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (j < nvalid) {
                if ((hb >> j) & 1u) {
                    if (!seen) lead = acc;
                    else { const uint32_t row = __ldg(p.nzrow + cur); tval[row] = acc.v; if (SPARSE) p.tpres[row] = (uint8_t)acc.has; }
                    seen = true; cur = rank++; acc.has = 0;
                }
                const Part<ZT> it{prod[j], SPARSE ? (int)up[j] : 1};
                acc = part_join<ZT>(ADD, acc, it);
            }
        }
    }
    if (!seen) { lead = acc; acc.has = 0; }

    // ---- segmented suffix scan of the leads over the 32 lanes
    Part<ZT> x = lead; int stop = seen ? 1 : 0;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        Part<ZT> y; y.v = shfl_down_t<ZT>(x.v, d);
        const int yf = __shfl_down_sync(0xffffffffu, x.has | (stop << 1), d);
        y.has = yf & 1;
        if (lane + d < 32) { if (!stop) x = part_join<ZT>(ADD, x, y); stop |= yf >> 1; }
    }
    Part<ZT> nxt; nxt.v = shfl_down_t<ZT>(x.v, 1);
    const int nf = __shfl_down_sync(0xffffffffu, x.has | (stop << 1), 1);
    nxt.has = nf & 1; int nxt_stop = nf >> 1;
    if (lane == 31) { nxt.has = 0; nxt_stop = 0; }

    // the lane holding the last row start of the run owns the row that is still open at the run's end
    // (which row that is, and where it ends, is structural: run_tail_row / run_tail_last of the plan)
    if (seen) {
        const Part<ZT> total = part_join<ZT>(ADD, acc, nxt);
        if (nxt_stop) { const uint32_t row = __ldg(p.nzrow + cur); tval[row] = total.v; if (SPARSE) p.tpres[row] = (uint8_t)total.has; }
        else { static_cast<ZT *>(p.tail_val)[run] = total.v; if (SPARSE) p.tail_has[run] = (uint8_t)total.has; }
    }
    if (lane == 0 && !(hb & 1u) && nvalid > 0) {                                            // the run starts inside a row of an earlier run
        static_cast<ZT *>(p.head_val)[run] = x.v; if (SPARSE) p.head_has[run] = (uint8_t)x.has;
    }
}

// ---- plain run kernel: 8 warps per CTA, each warp streams its run straight from global memory into registers
template <typename XT, typename ZT, int MUL_C>
__device__ __forceinline__ int spmv_run_load_global(const RunArgs &p, const int64_t run, const int lane, uint32_t (&c)[8], XT (&a)[8]) {
    constexpr bool NEED_A = MUL_C < 0 || mul_reads_x(MUL_C);
    const int64_t q = run * RUN + lane * 8;
    const int nvalid = (int)min((int64_t)8, max((int64_t)0, p.nnz - q));
    if (nvalid == 8) {
        load4<uint32_t>(p.col + q, &c[0]); load4<uint32_t>(p.col + q + 4, &c[4]);
        if (NEED_A) { load4<XT>(static_cast<const XT *>(p.aval) + q, &a[0]); load4<XT>(static_cast<const XT *>(p.aval) + q + 4, &a[4]); }
    } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            c[j] = j < nvalid ? p.col[q + j] : 0u;
            if (NEED_A) a[j] = j < nvalid ? static_cast<const XT *>(p.aval)[q + j] : (XT)1;
        }
    }
    return nvalid;
}

template <typename XT, typename ZT, int ADD, int MUL, bool SPARSE>
__global__ void __launch_bounds__(256) spmv_run_kernel(const RunArgs p) {
    const int64_t run = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (run >= p.nruns) return;
    const int lane = threadIdx.x & 31;
    uint32_t c[8]; RunLane<XT> L;
    const int nvalid = spmv_run_load_global<XT, ZT, MUL>(p, run, lane, c, L.a);
    const XT *uval = static_cast<const XT *>(p.uval);
    spmv_run_gather<XT, MUL, SPARSE>(p, run, lane, nvalid, c, L, [uval](uint32_t col) { return gload<XT>(uval + col); });
    spmv_run_fold<XT, ZT, ADD, MUL, SPARSE>(p, run, lane, L);
}

// ==================================================================================================
// Hot-table run kernel (dense u, specialised semirings, large skewed matrices) -- the benchmarked kernel.
//
// One persistent 1024-thread CTA per SM.  Shared memory holds
//   * the HOT TABLE: u at the most referenced columns, in the tiers below (a scattered 4-byte gather costs one L1 wavefront
//     per lane; a shared-memory lookup a few bank-conflict cycles per warp), filled once per CTA by bulk TMA
//     copies (cp.async.bulk -> SASS UBLKCP) from the gathered copy u_hot that the prep kernel writes;
//   * one STAGE per warp: the column ids and values of the warp's NEXT run, brought in by two bulk TMA copies
//     issued by lane 0 and completed on the warp's own mbarrier, so the DRAM stream of run r+1 is in flight
//     while the warp gathers and folds run r (registers are the second buffer: a run is copied out of the
//     stage before the next copy is issued).  A warp is its own producer and consumer: no CTA barrier after
//     the table is in.
// Column ids are ENCODED by the cached plan: id < henc -> rank among the hottest columns; id >= henc -> original column
// + henc, gathered from u itself.  u needs no permutation.
// The kernel runs as thread-block clusters of C CTAs (C = 1: plain CTAs), and the hot ranks fall in tiers:
//   id < T0        the replicated tier, in every CTA's own table: LDS;
//   id < T0 + T1   the distributed tier: rank T0 + k sits in the table of the cluster's CTA k mod C (index k / C), read
//                  through distributed shared memory (mapa + ld.shared::cluster), so a cluster holds C times more of the
//                  hottest columns on chip than one SM can;
//   id < henc      u_hot, in L2;   otherwise u itself.
// Every CTA passes a cluster barrier after its table is in (no peer reads a table before it is complete) and another
// before it exits (no CTA leaves while a peer may still read its table) -- CTAs without runs included.

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile("{\n\t.reg .pred p;\n\tWAIT_%=:\n\t"
                 "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
                 "@p bra DONE_%=;\n\tbra WAIT_%=;\n\tDONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}

__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
// a value in the shared memory of CTA `cta` of the cluster, at the address `saddr` has in this CTA's shared memory
template <typename XT> __device__ __forceinline__ XT ld_dsmem(uint32_t saddr, uint32_t cta) {
    uint32_t a; asm("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(a) : "r"(saddr), "r"(cta));
    if constexpr (sizeof(XT) == 8) { unsigned long long v; asm("ld.shared::cluster.b64 %0, [%1];" : "=l"(v) : "r"(a)); return reinterpret_cast<const XT &>(v); }
    else if constexpr (sizeof(XT) == 4) { uint32_t v; asm("ld.shared::cluster.b32 %0, [%1];" : "=r"(v) : "r"(a)); return reinterpret_cast<const XT &>(v); }
    else { uint16_t v; asm("ld.shared::cluster.u8 %0, [%1];" : "=h"(v) : "r"(a)); return (XT)(uint8_t)v; }
}

template <typename XT> __host__ __device__ constexpr int hot2_stage_bytes(bool need_a) { return RUN * 4 + (need_a ? RUN * (int)sizeof(XT) : 0); }
constexpr int HOT2_WARPS = 32;

template <typename XT, typename ZT, int ADD, int MUL, bool PIPE>
__global__ void __launch_bounds__(HOT2_WARPS * 32, 1) spmv_run_hot2_kernel(const RunArgs p, const Hot2Args h) {
    constexpr bool NEED_A = mul_reads_x(MUL);
    constexpr int STAGE = hot2_stage_bytes<XT>(NEED_A);
    extern __shared__ __align__(128) unsigned char smem_raw[];
    // layout: [warp stages][mbarriers][hot table]
    unsigned char *s_stage = smem_raw;
    uint64_t *s_bar = reinterpret_cast<uint64_t *>(smem_raw + HOT2_WARPS * STAGE);        // [HOT2_WARPS] per warp + [1] table
    XT *s_hot = reinterpret_cast<XT *>(smem_raw + HOT2_WARPS * STAGE + (HOT2_WARPS + 1) * 8 + 8);   // 16-byte aligned
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint64_t *bar = s_bar + warp;
    unsigned char *stage = s_stage + warp * STAGE;
    const int64_t stride = (int64_t)gridDim.x * HOT2_WARPS;
    int64_t run = (int64_t)blockIdx.x * HOT2_WARPS + warp;

    auto issue = [&](int64_t r) {             // lane 0: the bulk copies of run r into this warp's stage
        const int64_t q = r * RUN;
        const int64_t left = p.nnz - q;
        const uint32_t cnt = (uint32_t)(left < RUN ? left : RUN);
        const uint32_t cb = (cnt * 4u + 15u) & ~15u;                                      // arrays are padded by >= 16 bytes
        const uint32_t ab = NEED_A ? ((cnt * (uint32_t)sizeof(XT) + 15u) & ~15u) : 0u;
        mbar_expect_tx(bar, cb + ab);
        tma_bulk_g2s(stage, p.col + q, cb, bar);
        if (NEED_A) tma_bulk_g2s(stage + RUN * 4, static_cast<const XT *>(p.aval) + q, ab, bar);
    };

    const uint32_t t0 = h.t0, t1 = h.t1, slice = h.slice, henc = h.henc;
    const int lc = __ffs(h.cluster) - 1;                                   // C is a power of two
    if (lane == 0) mbar_init(bar, 1);
    if (threadIdx.x == 0) mbar_init(s_bar + HOT2_WARPS, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncthreads();
    const uint32_t tab_n = t0 + slice;
    if (threadIdx.x == 0 && tab_n) {          // the table: the replicated tier and this CTA's slice, bulk copies of <= 16 KB
        const unsigned char *src = static_cast<const unsigned char *>(h.u_hot);
        unsigned char *dst = reinterpret_cast<unsigned char *>(s_hot);
        const uint32_t rb = t0 * (uint32_t)sizeof(XT), sb = slice * (uint32_t)sizeof(XT);
        mbar_expect_tx(s_bar + HOT2_WARPS, rb + sb);
        for (uint32_t off = 0; off < rb; off += 16384u) tma_bulk_g2s(dst + off, src + off, min(16384u, rb - off), s_bar + HOT2_WARPS);
        src += rb + (size_t)cluster_ctarank() * sb; dst += rb;
        for (uint32_t off = 0; off < sb; off += 16384u) tma_bulk_g2s(dst + off, src + off, min(16384u, sb - off), s_bar + HOT2_WARPS);
    }
    if (lane == 0 && run < p.nruns) issue(run);
    if (tab_n) mbar_wait(s_bar + HOT2_WARPS, 0);
    cluster_sync_all();                       // every table of the cluster is in

    const XT *uval = static_cast<const XT *>(p.uval);
    const XT *urest = static_cast<const XT *>(h.u_hot) + ((slice << lc) - t1);   // ranks past the tiers (spmv_args.cuh)
    const uint32_t s_slice = smem_u32(s_hot + t0);
    auto gather = [=](uint32_t col) -> XT {
        if (col < t0) return s_hot[col];
        const uint32_t k = col - t0;
        if (k < t1) return ld_dsmem<XT>(s_slice + (k >> lc) * (uint32_t)sizeof(XT), k & ((1u << lc) - 1u));
        if (col < henc) return gload<XT>(urest + col);
        return gload<XT>(uval + (col - henc));
    };
    // Software pipeline over the warp's runs: the words of run r+1 are copied out of the stage and its gathers of u
    // are ISSUED before run r is multiplied, folded and stored, so the gather latency sits under a run's worth of
    // arithmetic instead of in front of it (and the bulk copy of run r+2 is in flight under both).
    uint32_t parity = 0;
    RunLane<XT> cur, nxt;
    int64_t cur_run = -1;
    auto fetch = [&](int64_t r, RunLane<XT> &L) {
        mbar_wait(bar, parity); parity ^= 1u;
        const int64_t q = r * RUN + lane * 8;
        const int nvalid = (int)min((int64_t)8, max((int64_t)0, p.nnz - q));
        uint32_t c[8];
        if (NEED_A) {
            const XT *sa = reinterpret_cast<const XT *>(stage + RUN * 4) + lane * 8;
            if constexpr (sizeof(XT) == 4) {
                const uint4 a0 = reinterpret_cast<const uint4 *>(sa)[0], a1 = reinterpret_cast<const uint4 *>(sa)[1];
                const uint32_t w[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
#pragma unroll
                for (int j = 0; j < 8; ++j) L.a[j] = reinterpret_cast<const XT &>(w[j]);
            } else {
#pragma unroll
                for (int j = 0; j < 8; ++j) L.a[j] = sa[j];
            }
        }
        const uint4 *sc = reinterpret_cast<const uint4 *>(stage) + lane * 2;
        const uint4 c0 = sc[0], c1 = sc[1];
        c[0] = c0.x; c[1] = c0.y; c[2] = c0.z; c[3] = c0.w; c[4] = c1.x; c[5] = c1.y; c[6] = c1.z; c[7] = c1.w;
        // WAR guard of the stage.  The bulk copy of the next run writes this stage through the async proxy; nothing orders it
        // after generic-proxy loads that were only ISSUED (a __syncwarp does not wait for their data), and under load a
        // shared-memory load can sit in the LSU queue longer than an L2-hit bulk copy takes -- a lane then folds words of the
        // NEXT run into this run's rows (seen as one wrong hub-row sum in ~1 % of the launches of the overlapped e2e loop).  A vote
        // that READS the first and last loaded word of every lane cannot issue before the warp's loads have written their
        // registers; its predicate is never true (encoded ids stay below 2^32 - 1: spmv_hot_plan), so the copy is always issued.
        uint32_t guard = c[0] & c[7];
        if (NEED_A) {                                                       // the value loads take part too (first and last word of the lane)
            uint32_t w0, w7;
            if constexpr (sizeof(XT) >= 4) { memcpy(&w0, &L.a[0], 4); memcpy(&w7, &L.a[7], 4); }
            else { w0 = (uint32_t)L.a[0]; w7 = (uint32_t)L.a[7]; }             // 1-byte values (BOOL)
            guard &= (w0 | 0x80000000u) & (w7 | 0x80000000u);
        }
        const unsigned never = __ballot_sync(0xffffffffu, guard == 0xFFFFFFFFu);
        if (nvalid < 8) {                                                   // tail of the last run: what lies past nnz is not data
#pragma unroll
            for (int j = 0; j < 8; ++j) { if (j >= nvalid) { c[j] = henc; if (NEED_A) L.a[j] = (XT)1; } }
        }
        if (lane == 0 && never == 0u && r + stride < p.nruns) issue(r + stride);
        spmv_run_gather<XT, MUL, false>(p, r, lane, nvalid, c, L, gather);
    };
    if constexpr (sizeof(XT) > 4 || !PIPE) {
        // one run at a time (8-byte values: two runs in flight do not fit in 64 registers per thread)
        for (; run < p.nruns; run += stride) { fetch(run, cur); spmv_run_fold<XT, ZT, ADD, MUL, false>(p, run, lane, cur); }
        (void)nxt; (void)cur_run;
    } else {
        if (run < p.nruns) { fetch(run, cur); cur_run = run; run += stride; }
        while (cur_run >= 0) {
            const bool more = run < p.nruns;
            if (more) fetch(run, nxt);
            spmv_run_fold<XT, ZT, ADD, MUL, false>(p, cur_run, lane, cur);
            if (more) { cur = nxt; cur_run = run; run += stride; } else cur_run = -1;
        }
    }
    cluster_sync_all();                       // no peer reads this CTA's table any more
}

// rows that continue past their run: tail partial (+) head partials of the following runs, 8 lanes per open row.
// Every run after `run` up to tail_last starts inside that row, so its head partial exists.
template <typename ZT, int ADD_C, bool SPARSE>
__global__ void __launch_bounds__(256) spmv_run_fixup_kernel(const RunArgs p) {
    const int ADD = ADD_C >= 0 ? ADD_C : p.add_op;
    const int sub = threadIdx.x & 7;
    const int64_t run = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 3;
    const int32_t r = run < p.nruns ? __ldg(p.tail_row + run) : -1;
    Part<ZT> acc{(ZT)0, 0};
    if (r >= 0) {
        const int64_t last_run = __ldg(p.tail_last + run);
        if (sub == 0) { acc.v = static_cast<const ZT *>(p.tail_val)[run]; acc.has = SPARSE ? (int)p.tail_has[run] : 1; }
        for (int64_t t = run + 1 + sub; t <= last_run; t += 8) {
            const Part<ZT> y{static_cast<const ZT *>(p.head_val)[t], SPARSE ? (int)p.head_has[t] : 1};
            acc = part_join<ZT>(ADD, acc, y);
        }
    }
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) {
        Part<ZT> y; y.v = shfl_xor_t<ZT>(acc.v, o); y.has = __shfl_xor_sync(0xffffffffu, acc.has, o);
        acc = part_join<ZT>(ADD, acc, y);
    }
    if (r >= 0 && sub == 0) { static_cast<ZT *>(p.tval)[r] = acc.v; if (SPARSE) p.tpres[r] = (uint8_t)acc.has; }
}

// shared memory the hot-table kernel can use for its table, after the warp stages and barriers
template <typename XT> static inline uint32_t hot2_table_entries(bool need_a, uint32_t henc, size_t limit_bytes) {
    static int max_optin = 0;                   // one device per process: ask once
    if (!max_optin) cudaDeviceGetAttribute(&max_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, G.device);
    const size_t fixed = (size_t)HOT2_WARPS * hot2_stage_bytes<XT>(need_a) + (HOT2_WARPS + 1) * 8 + 8;
    size_t avail = (size_t)max_optin > fixed + 256 ? (size_t)max_optin - fixed - 256 : 0;
    avail = std::min(avail, limit_bytes);
    return (uint32_t)std::min<size_t>(henc, avail / sizeof(XT)) & ~15u;
}

// tiers of a cluster of C CTAs whose tables hold `cap` entries each (spmv_args.cuh).  Plain CTAs (cluster = 1, the whole
// table local) when C = 1, when one table already holds every hot rank (cap = henc rounded down to 16 entries), and when
// the replicated tier takes the whole table: a cluster would then only read peers' tables for ranks it could hold itself,
// and clusters of 4 or more leave SMs idle (DESIGN.md section 3.1).
static inline void hot2_tiers(Hot2Args &h, int C, uint32_t cap) {
    h.cluster = 1; h.t0 = cap; h.t1 = 0; h.slice = 0;
    if (C == 1 || h.henc - cap < 16) return;                                  // cap <= henc
    const uint32_t t0 = std::min(h.want_repl & ~15u, cap);
    const uint32_t need = h.henc - t0;
    const uint32_t slice = std::min(cap - t0, (uint32_t)((ceil_div((int64_t)need, C) + 15) & ~15ll));
    if (slice == 0) return;
    h.cluster = C; h.t0 = t0; h.slice = slice; h.t1 = std::min<uint32_t>(need, slice * (uint32_t)C);
}

// how many clusters of C CTAs of this kernel the device runs at once (asked once per kernel, C and shared-memory size)
template <typename Kernel> static int hot2_max_clusters(Kernel kernel, int C, size_t smem) {
    static std::map<std::tuple<Kernel, int, size_t>, int> known;
    auto it = known.find({kernel, C, smem});
    if (it != known.end()) return it->second;
    if (C > 8) cudaFuncSetAttribute(kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)(C * ((G.num_sms + C - 1) / C))); cfg.blockDim = dim3(HOT2_WARPS * 32); cfg.dynamicSmemBytes = smem;
    cudaLaunchAttribute at[1]; at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim = {(unsigned)C, 1, 1};
    cfg.attrs = at; cfg.numAttrs = 1;
    int n = 0;
    if (cudaOccupancyMaxActiveClusters(&n, kernel, &cfg) != cudaSuccess) { cudaGetLastError(); n = 0; }
    known[{kernel, C, smem}] = n;
    return n;
}

template <typename XT, typename ZT, int ADD, int MUL, bool PIPE>
static void hot2_launch(const RunArgs &a, Hot2Args &h, size_t table_limit) {
    constexpr bool NEED_A = mul_reads_x(MUL);
    auto kernel = spmv_run_hot2_kernel<XT, ZT, ADD, MUL, PIPE>;
    const uint32_t cap = hot2_table_entries<XT>(NEED_A, h.henc, table_limit);
    const size_t fixed = (size_t)HOT2_WARPS * hot2_stage_bytes<XT>(NEED_A) + (HOT2_WARPS + 1) * 8 + 8;
    const size_t smem_max = fixed + (size_t)cap * sizeof(XT);
    // the dynamic shared-memory limit of a kernel is raised once per size (a driver call per launch is host time the
    // multi-GPU step cannot hide: its kernels take tens of microseconds)
    static size_t set_for = 0;
    if (set_for != smem_max) { cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_max); set_for = smem_max; }
    const int64_t want_ctas = ceil_div(a.nruns, HOT2_WARPS);
    // the largest cluster size up to the requested one that the device co-schedules, and the tiers it holds
    int C = 1, clusters = G.num_sms;
    for (int c = h.want_cluster; c > 1; c >>= 1) {
        hot2_tiers(h, c, cap);
        if (h.cluster == 1) break;                                            // nothing to spread: plain CTAs
        const int m = hot2_max_clusters(kernel, c, fixed + (size_t)(h.t0 + h.slice) * sizeof(XT));
        if (m > 0) { C = c; clusters = m; break; }
    }
    if (C == 1) hot2_tiers(h, 1, cap);
    const size_t smem = fixed + (size_t)(h.t0 + h.slice) * sizeof(XT);
    const int64_t ctas = std::min<int64_t>((int64_t)clusters * C, ceil_div(want_ctas, C) * C);
    h.ctas = (int)ctas;
    spmv_hot2_prep(h);
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)ctas); cfg.blockDim = dim3(HOT2_WARPS * 32); cfg.dynamicSmemBytes = smem; cfg.stream = G.stream;
    cudaLaunchAttribute at[1]; at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim = {(unsigned)C, 1, 1};
    cfg.attrs = at; cfg.numAttrs = 1;
    cudaLaunchKernelEx(&cfg, kernel, a, (const Hot2Args)h); GB_LAUNCHED();
}

template <typename XT, typename ZT, int ADD, int MUL>
static void spmv_run_launch(const RunArgs &a, Hot2Args *hot, size_t table_limit) {
    if constexpr (ADD >= 0) {
        if (hot && !a.upres) {
            if (sizeof(XT) <= 4 && tunables().spmv_pipe) hot2_launch<XT, ZT, ADD, MUL, true>(a, *hot, table_limit);
            else hot2_launch<XT, ZT, ADD, MUL, false>(a, *hot, table_limit);
            spmv_run_fixup_kernel<ZT, ADD, false><<<(unsigned)ceil_div(a.nruns * 8, 256), 256, 0, G.stream>>>(a); GB_LAUNCHED();
            return;
        }
    }
    if (a.upres) {
        spmv_run_kernel<XT, ZT, ADD, MUL, true><<<(unsigned)ceil_div(a.nruns, 8), 256, 0, G.stream>>>(a); GB_LAUNCHED();
        spmv_run_fixup_kernel<ZT, ADD, true><<<(unsigned)ceil_div(a.nruns * 8, 256), 256, 0, G.stream>>>(a); GB_LAUNCHED();
        return;
    }
    spmv_run_kernel<XT, ZT, ADD, MUL, false><<<(unsigned)ceil_div(a.nruns, 8), 256, 0, G.stream>>>(a); GB_LAUNCHED();
    spmv_run_fixup_kernel<ZT, ADD, false><<<(unsigned)ceil_div(a.nruns * 8, 256), 256, 0, G.stream>>>(a); GB_LAUNCHED();
}
