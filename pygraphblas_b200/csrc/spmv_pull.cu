// Masked pull kernels for the saturating monoids (LOR, LAND, ANY): the BFS step.
#include "spmv_args.cuh"

template <typename ZT> __device__ __forceinline__ bool monoid_saturated(int add, ZT v) {
    switch (add) {
        case OP_LOR: return v != (ZT)0;
        case OP_LAND: return v == (ZT)0;
        case OP_ANY: return true;
        default: return false;
    }
}
// The three monoids of this kernel (LOR, LAND, ANY) need no running value: the fold of a row's products is
// decided by how many there are (0, 1, more), whether one of them saturates, and the first one --
//   0 products: no entry;  1: that product, as is;  more: ANY -> any of them, LOR -> "one was non-zero",
//   LAND -> "none was zero" (1 or 0 in the monoid's type).
// A row may stop early once its result can no longer change.
template <typename ZT> __device__ __forceinline__ ZT pull_result(int add, int n, bool sat, ZT first) {
    if (n <= 1 || add == OP_ANY) return first;
    return add == OP_LOR ? (ZT)(sat ? 1 : 0) : (ZT)(sat ? 0 : 1);
}
template <typename ZT> __device__ __forceinline__ bool pull_settled(int add, ZT v) {     // saturating AND already the final value
    switch (add) {
        case OP_LOR: return v == (ZT)1;
        case OP_LAND: return v == (ZT)0;
        case OP_ANY: return true;
        default: return false;
    }
}
template <typename XT, typename ZT>
__device__ __forceinline__ ZT pull_product(const PullArgs &p, const XT *aval, const XT *uval, uint32_t k, uint32_t c) {
    const XT a = gload<XT>(aval + k), u = gload<XT>(uval + c);
    return p.flip ? MulApply<XT, ZT>::f(p.mul_op, u, a) : MulApply<XT, ZT>::f(p.mul_op, a, u);
}

// Warp batches of 32 rows, their entries flattened: lane i owns row base+i (mask, accumulators, result) while
// the entries of all 32 rows are walked 32 at a time, so short rows cost one slot per entry instead of one
// warp iteration per row.  Rows advance in rounds of at most `cap` entries each; a row whose result is settled
// leaves the batch at the end of the round.
template <typename XT, typename ZT>
__global__ void __launch_bounds__(256) spmv_masked_pull_kernel(const PullArgs p) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const XT *aval = static_cast<const XT *>(p.aval), *uval = static_cast<const XT *>(p.uval);
    ZT *tval = static_cast<ZT *>(p.tval);
    const int add = p.add_op;
    for (int64_t base = warp * 32; base < p.nrows; base += nwarps * 32) {
        const int64_t mr = base + lane;
        bool m = false;
        if (mr < p.nrows) {
            m = p.mpres ? p.mpres[mr] != 0 : true;
            if (m && !p.mask_struct) m = sc_cast(sc_load(p.mtc, p.mval, (size_t)mr), p.mtc, TC_BOOL).u != 0;
            if (p.mask_comp) m = !m;
            if (!m) p.tpres[mr] = 0;
        }
        uint32_t pos = 0, rem = 0;
        if (m) {
            pos = p.rowptr[mr]; rem = p.rowptr[mr + 1] - pos;
            if (rem > PULL_LONG) { p.long_rows[atomicAdd(p.long_count, 1)] = (uint32_t)mr; rem = 0; m = false; }
        }
        int n_it = 0; bool sat = false; ZT first = (ZT)0;
        unsigned active;
        while ((active = __ballot_sync(0xffffffffu, rem > 0)) != 0) {
            const uint32_t cap = __popc(active) > 8 ? 32u : 128u;
            const uint32_t take = rem < cap ? rem : cap;
            uint32_t incl = take;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
            const uint32_t off = incl - take, total = __shfl_sync(0xffffffffu, incl, 31);
            const uint32_t delta = pos - off;                  // entry index = delta(owner) + flat position
            for (uint32_t f0 = 0; f0 < total; f0 += 32) {
                const uint32_t f = f0 + lane;
                int own = 0;                                   // first lane whose inclusive end exceeds f
#pragma unroll
                for (int step = 16; step > 0; step >>= 1) { const uint32_t t = __shfl_sync(0xffffffffu, incl, own + step - 1); if (t <= f) own += step; }
                const uint32_t k = __shfl_sync(0xffffffffu, delta, own) + f;
                bool has = false; ZT v = (ZT)0;
                if (f < total) {
                    const uint32_t c = __ldg(p.col + k);
                    if (!p.upres || __ldg(p.upres + c)) { v = pull_product<XT, ZT>(p, aval, uval, k, c); has = true; }
                }
                const unsigned hasmask = __ballot_sync(0xffffffffu, has);
                const unsigned satmask = __ballot_sync(0xffffffffu, has && monoid_saturated<ZT>(add, v));
                // the slots of this chunk that belong to this lane's row
                const uint32_t s0 = off > f0 ? off : f0, s1 = (off + take) < (f0 + 32) ? (off + take) : (f0 + 32);
                unsigned seg = 0;
                if (s1 > s0) { const uint32_t len = s1 - s0; seg = (len >= 32 ? 0xffffffffu : ((1u << len) - 1u)) << (s0 - f0); }
                const unsigned mine = hasmask & seg;
                const ZT fv = shfl_idx_t<ZT>(v, mine ? __ffs(mine) - 1 : lane);
                if (mine) {
                    if (n_it == 0) first = fv;
                    n_it = min(2, n_it + __popc(mine));
                    sat |= (satmask & seg) != 0;
                }
            }
            if (sat && (n_it >= 2 || pull_settled<ZT>(add, first))) rem = 0;
            else { rem -= take; pos += take; }
        }
        if (m) { tval[mr] = pull_result<ZT>(add, n_it, sat, first); p.tpres[mr] = (uint8_t)(n_it > 0); }
    }
}
// Long rows (hubs): one 1024-thread CTA per row, 1024 entries per iteration, early exit CTA-wide.
template <typename XT, typename ZT>
__global__ void __launch_bounds__(1024) spmv_pull_long_kernel(const PullArgs p) {
    __shared__ int s_n[32]; __shared__ int s_sat[32]; __shared__ ZT s_first[32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const XT *aval = static_cast<const XT *>(p.aval), *uval = static_cast<const XT *>(p.uval);
    ZT *tval = static_cast<ZT *>(p.tval);
    const int add = p.add_op;
    const int nlong = *p.long_count;
    for (int w = blockIdx.x; w < nlong; w += gridDim.x) {
        const uint32_t r = p.long_rows[w];
        const uint32_t rs = p.rowptr[r], re = p.rowptr[r + 1];
        int n_it = 0; bool sat = false; ZT first = (ZT)0;
        for (uint32_t b0 = rs; b0 < re; b0 += 1024) {
            const uint32_t k = b0 + threadIdx.x;
            int stop = 0;
            if (k < re) {
                const uint32_t c = __ldg(p.col + k);
                if (!p.upres || __ldg(p.upres + c)) {
                    const ZT v = pull_product<XT, ZT>(p, aval, uval, k, c);
                    if (n_it == 0) first = v;
                    n_it = min(2, n_it + 1);
                    if (monoid_saturated<ZT>(add, v)) { sat = true; stop = pull_settled<ZT>(add, v); }
                }
            }
            if (__syncthreads_or(stop)) break;
        }
        const unsigned hasmask = __ballot_sync(0xffffffffu, n_it > 0);
        const int wn = min(2, __reduce_add_sync(0xffffffffu, n_it));
        const int wsat = __any_sync(0xffffffffu, sat);
        const ZT wfirst = shfl_idx_t<ZT>(first, hasmask ? __ffs(hasmask) - 1 : 0);
        if (lane == 0) { s_n[wid] = wn; s_sat[wid] = wsat; s_first[wid] = wfirst; }
        __syncthreads();
        if (threadIdx.x == 0) {
            int N = 0, S = 0; ZT F = (ZT)0;
            for (int q = 0; q < 32; ++q) { if (s_n[q] && !N) F = s_first[q]; N = min(2, N + s_n[q]); S |= s_sat[q]; }
            tval[r] = pull_result<ZT>(add, N, S != 0, F); p.tpres[r] = (uint8_t)(N > 0);
        }
        __syncthreads();
    }
}
GrB_Info spmv_masked_pull_dispatch(int xt, int zt, const PullArgs &a, std::string *err) {
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(a.nrows, 256), (int64_t)G.num_sms * 8));
    const int lgrid = (int)std::max<int64_t>(1, std::min<int64_t>(a.long_cap, (int64_t)G.num_sms * 2));
#define GB_PULL(XT_, ZT_) do { spmv_masked_pull_kernel<XT_, ZT_><<<grid, 256, 0, G.stream>>>(a); GB_LAUNCHED(); \
        if (a.has_long) { spmv_pull_long_kernel<XT_, ZT_><<<lgrid, 1024, 0, G.stream>>>(a); GB_LAUNCHED(); } return GrB_SUCCESS; } while (0)
    if (xt == zt) {
        switch (xt) {
#define GB_GEN(TC, T) case TC: GB_PULL(T, T);
            GB_GEN(TC_BOOL, bool) GB_GEN(TC_INT8, int8_t) GB_GEN(TC_INT16, int16_t) GB_GEN(TC_INT32, int32_t) GB_GEN(TC_INT64, int64_t)
            GB_GEN(TC_UINT8, uint8_t) GB_GEN(TC_UINT16, uint16_t) GB_GEN(TC_UINT32, uint32_t) GB_GEN(TC_UINT64, uint64_t)
            GB_GEN(TC_FP32, float) GB_GEN(TC_FP64, double)
#undef GB_GEN
        }
    } else if (zt == TC_BOOL) {
        switch (xt) {
#define GB_GEN(TC, T) case TC: GB_PULL(T, bool);
            GB_GEN(TC_INT8, int8_t) GB_GEN(TC_INT16, int16_t) GB_GEN(TC_INT32, int32_t) GB_GEN(TC_INT64, int64_t)
            GB_GEN(TC_UINT8, uint8_t) GB_GEN(TC_UINT16, uint16_t) GB_GEN(TC_UINT32, uint32_t) GB_GEN(TC_UINT64, uint64_t)
            GB_GEN(TC_FP32, float) GB_GEN(TC_FP64, double)
#undef GB_GEN
        }
    }
#undef GB_PULL
    return gb_fail(GrB_DOMAIN_MISMATCH, err, "mxv: unsupported semiring domains (x=%d, z=%d)", xt, zt);
}


// ------------------------------------------------------------------ push
constexpr int PUSH_CHUNK = 1024;
// size of the frontier and of its out-edge set: one atomic pair per CTA
__global__ void __launch_bounds__(256) push_stats_kernel(const PushArgs a) {
    __shared__ unsigned long long s_c[8], s_d[8];
    unsigned long long cnt = 0, deg = 0;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < a.nin; k += (int64_t)gridDim.x * blockDim.x)
        if (!a.upres || a.upres[k] != 0) { ++cnt; deg += (unsigned long long)(a.rowptr[k + 1] - a.rowptr[k]); }
    for (int o = 16; o > 0; o >>= 1) { cnt += __shfl_xor_sync(0xffffffffu, cnt, o); deg += __shfl_xor_sync(0xffffffffu, deg, o); }
    if ((threadIdx.x & 31) == 0) { s_c[threadIdx.x >> 5] = cnt; s_d[threadIdx.x >> 5] = deg; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int q = 1; q < 8; ++q) { cnt += s_c[q]; deg += s_d[q]; }
        if (cnt) { atomicAdd(&a.counters[0], cnt); atomicAdd(&a.counters[1], deg); }
    }
}
// the frontier as a list (order irrelevant): warp-aggregated append
__global__ void __launch_bounds__(256) push_frontier_kernel(const PushArgs a) {
    const int lane = threadIdx.x & 31;
    for (int64_t base = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) - lane; base < a.nin; base += (int64_t)gridDim.x * blockDim.x) {
        const int64_t k = base + lane;
        const bool in = k < a.nin && (!a.upres || a.upres[k] != 0);
        const unsigned m = __ballot_sync(0xffffffffu, in);
        if (!m) continue;
        unsigned long long pos = 0;
        if (lane == 0) pos = atomicAdd(&a.counters[2], (unsigned long long)__popc(m));
        pos = __shfl_sync(0xffffffffu, pos, 0);
        if (in) a.list[pos + __popc(m & ((1u << lane) - 1u))] = (uint32_t)k;
    }
}
__global__ void push_chunks_kernel(const PushArgs a, int64_t count) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= count; i += (int64_t)gridDim.x * blockDim.x) {
        int64_t c = 0;
        if (i < count) { const uint32_t k = a.list[i]; c = ((int64_t)(a.rowptr[k + 1] - a.rowptr[k]) + PUSH_CHUNK - 1) / PUSH_CHUNK; }
        a.chunk_scan[i] = c;
    }
}
template <typename ZT> __global__ void push_init_kernel(ZT *tval, uint8_t *tpres, int64_t n, ZT init) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) { tval[i] = init; tpres[i] = 0; }
}
// one warp per chunk of <= PUSH_CHUNK entries of a frontier row
template <typename XT, typename ZT>
__global__ void __launch_bounds__(256) push_kernel(const PushArgs a, int64_t count) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int64_t nchunks = a.chunk_scan[count];
    const XT *aval = static_cast<const XT *>(a.aval), *uval = static_cast<const XT *>(a.uval);
    ZT *tval = static_cast<ZT *>(a.tval);
    for (int64_t c = warp; c < nchunks; c += nwarps) {
        int64_t lo = 0, hi = count;                              // owner: last i with chunk_scan[i] <= c
        while (hi - lo > 1) { const int64_t mid = (lo + hi) >> 1; if (a.chunk_scan[mid] <= c) lo = mid; else hi = mid; }
        const uint32_t k = a.list[lo];
        const uint32_t rs = a.rowptr[k] + (uint32_t)(c - a.chunk_scan[lo]) * PUSH_CHUNK;
        const uint32_t re = min(a.rowptr[k + 1], rs + (uint32_t)PUSH_CHUNK);
        const XT uk = gload<XT>(uval + k);
        for (uint32_t e = rs + lane; e < re; e += 32) {
            const uint32_t j = __ldg(a.col + e);
            bool m = a.mpres ? a.mpres[j] != 0 : true;
            if (m && !a.mask_struct) m = mask_value_true(a.mtc, a.mval, (int64_t)j);
            if (a.mask_comp) m = !m;
            if (!m) continue;
            const XT av = gload<XT>(aval + e);
            const ZT v = a.flip ? MulApply<XT, ZT>::f(a.mul_op, uk, av) : MulApply<XT, ZT>::f(a.mul_op, av, uk);
            a.tpres[j] = 1;
            if (a.add_op == OP_LOR) { if (v != (ZT)0) tval[j] = (ZT)1; }
            else if (a.add_op == OP_LAND) { if (v == (ZT)0) tval[j] = (ZT)0; }
            else tval[j] = v;
        }
    }
}
template <typename XT, typename ZT> static void push_launch(const PushArgs &a, int64_t count, int64_t chunk_bound) {
    const ZT init = a.add_op == OP_LAND ? (ZT)1 : (ZT)0;
    const int g0 = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(a.nout, 256), (int64_t)G.num_sms * 16));
    push_init_kernel<ZT><<<g0, 256, 0, G.stream>>>(static_cast<ZT *>(a.tval), a.tpres, a.nout, init); GB_LAUNCHED();
    if (count > 0) {
        const int g1 = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(chunk_bound * 32, 256), (int64_t)G.num_sms * 16));
        push_kernel<XT, ZT><<<g1, 256, 0, G.stream>>>(a, count); GB_LAUNCHED();
    }
}
GrB_Info spmv_masked_push_try(int xt, int zt, PushArgs &a, int64_t nnz_total, bool *done, std::string *err) {
    *done = false;
    // LOR / LAND results are normalised only when the monoid type is BOOL (every builtin); ANY stores the product as is
    if ((a.add_op == OP_LOR || a.add_op == OP_LAND) && zt != TC_BOOL) return GrB_SUCCESS;
    if (!(xt == zt || zt == TC_BOOL)) return GrB_SUCCESS;
    DevBuf<unsigned long long> counters; DevBuf<uint32_t> list; DevBuf<int64_t> chunk_scan;
    GB_TRY(counters.alloc(4, err));
    a.counters = counters;
    CU_TRY(cudaMemsetAsync(a.counters, 0, 32, G.stream), err);
    const int g = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(a.nin, 256 * 4), (int64_t)G.num_sms * 8));
    push_stats_kernel<<<g, 256, 0, G.stream>>>(a); GB_LAUNCHED();
    unsigned long long h[2] = {0, 0};
    CU_TRY(cudaMemcpyAsync(h, a.counters, 16, cudaMemcpyDeviceToHost, G.stream), err);
    CU_TRY(cudaStreamSynchronize(G.stream), err);
    const int64_t count = (int64_t)h[0], edges = (int64_t)h[1];
    // push pays per frontier vertex and per frontier edge, pull per unmasked row: push only small frontiers
    if ((edges * 16 > nnz_total || count * 32 > a.nin) && !tunables().force_push) return GrB_SUCCESS;
    GB_TRY(list.alloc((size_t)count + 1, err));
    a.list = list;
    if (count > 0) {
        const int gf = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(a.nin, 256), (int64_t)G.num_sms * 16));
        push_frontier_kernel<<<gf, 256, 0, G.stream>>>(a); GB_LAUNCHED();
    }
    GB_TRY(chunk_scan.alloc((size_t)count + 2, err));
    a.chunk_scan = chunk_scan;
    if (count > 0) {
        const int g2 = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(count + 1, 256), (int64_t)G.num_sms * 16));
        push_chunks_kernel<<<g2, 256, 0, G.stream>>>(a, count); GB_LAUNCHED();
        GB_TRY(dev_exclusive_scan(a.chunk_scan, count + 1, err));
    } else CU_TRY(cudaMemsetAsync(a.chunk_scan, 0, 16, G.stream), err);
    const int64_t chunk_bound = edges / PUSH_CHUNK + count + 1;
    bool ok = true;
#define GB_PUSH(XT_, ZT_) do { push_launch<XT_, ZT_>(a, count, chunk_bound); } while (0)
    if (xt == zt) {
        switch (xt) {
#define GB_GEN(TC, T) case TC: GB_PUSH(T, T); break;
            GB_GEN(TC_BOOL, bool) GB_GEN(TC_INT8, int8_t) GB_GEN(TC_INT16, int16_t) GB_GEN(TC_INT32, int32_t) GB_GEN(TC_INT64, int64_t)
            GB_GEN(TC_UINT8, uint8_t) GB_GEN(TC_UINT16, uint16_t) GB_GEN(TC_UINT32, uint32_t) GB_GEN(TC_UINT64, uint64_t)
            GB_GEN(TC_FP32, float) GB_GEN(TC_FP64, double)
#undef GB_GEN
            default: ok = false;
        }
    } else {
        switch (xt) {
#define GB_GEN(TC, T) case TC: GB_PUSH(T, bool); break;
            GB_GEN(TC_INT8, int8_t) GB_GEN(TC_INT16, int16_t) GB_GEN(TC_INT32, int32_t) GB_GEN(TC_INT64, int64_t)
            GB_GEN(TC_UINT8, uint8_t) GB_GEN(TC_UINT16, uint16_t) GB_GEN(TC_UINT32, uint32_t) GB_GEN(TC_UINT64, uint64_t)
            GB_GEN(TC_FP32, float) GB_GEN(TC_FP64, double)
#undef GB_GEN
            default: ok = false;
        }
    }
#undef GB_PUSH
    CU_TRY(cudaGetLastError(), err);
    *done = ok;
    return GrB_SUCCESS;
}
