// Run plan, hot-column plan, and the FP32 / FP64 instantiations of the run kernels.
#include "spmv_run.cuh"
#include <cub/device/device_radix_sort.cuh>

// ---- run plan (cached per CSR)
__global__ void plan_nonempty_kernel(const uint32_t *rowptr, int64_t nrows, int64_t *flag, uint8_t *pres) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += (int64_t)gridDim.x * blockDim.x) {
        const int ne = rowptr[r + 1] > rowptr[r];
        flag[r] = ne; pres[r] = (uint8_t)ne;
    }
}
__global__ void plan_rows_kernel(const uint32_t *rowptr, const int64_t *rank, int64_t nrows, uint32_t *nzrow, uint32_t *headw) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t rs = rowptr[r];
        if (rowptr[r + 1] > rs) { nzrow[rank[r]] = (uint32_t)r; atomicOr(&headw[rs >> 5], 1u << (rs & 31)); }
    }
}
__global__ void plan_runs_kernel(const uint32_t *headw, int64_t nruns, int64_t nwords, uint16_t *lane_rank, int64_t *run_cnt) {
    const int lane = threadIdx.x & 31;
    const int64_t run = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (run >= nruns) return;
    const int64_t w = run * 8 + (lane >> 2);
    const uint32_t hw = w < nwords ? headw[w] : 0u;
    const int pc = __popc((hw >> ((lane & 3) * 8)) & 0xffu);
    int inc = pc;
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
    lane_rank[run * 32 + lane] = (uint16_t)(inc - pc);
    if (lane == 31) run_cnt[run] = inc;
}
__global__ void plan_base_kernel(const int64_t *scan, int64_t nruns, uint32_t *run_base) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k <= nruns; k += (int64_t)gridDim.x * blockDim.x) run_base[k] = (uint32_t)scan[k];
}
// the row that starts last inside a run always holds the run's last entry: it is the run's "open" row
// (possibly ending exactly at the run's end), completed by the fix-up kernel
__global__ void plan_tails_kernel(const uint32_t *run_base, const uint32_t *nzrow, const uint32_t *rowptr, int64_t nruns,
                                  int32_t *tail_row, uint32_t *tail_last) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < nruns; k += (int64_t)gridDim.x * blockDim.x) {
        int32_t tr = -1; uint32_t tl = 0;
        if (run_base[k + 1] > run_base[k]) {
            const uint32_t r = nzrow[run_base[k + 1] - 1];
            const uint32_t re = rowptr[r + 1];
            tr = (int32_t)r; tl = (re - 1) / RUN;
        }
        tail_row[k] = tr; tail_last[k] = tl;
    }
}
static inline int rgrid(int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n, 256), (int64_t)G.num_sms * 16)); }

GrB_Info spmv_run_plan(Csr &c, std::string *err) {
    if (c.run.headw) return GrB_SUCCESS;
    if (!c.rowptr32) return gb_fail(GrB_INVALID_VALUE, err, "mxv: matrices with >= 2^32 entries are not supported");
    RunPlan p;                 // moved into c only once complete
    const int64_t nwords = ceil_div(c.nnz, 32);
    p.nruns = ceil_div(c.nnz, RUN);
    DevBuf<int64_t> flag, cnt;
    GB_TRY(flag.alloc((size_t)c.nrows + 1, err));
    GB_TRY(cnt.alloc((size_t)p.nruns + 1, err));
    GB_TRY(p.pres_tmpl.alloc((size_t)c.nrows, err));
    GB_TRY(p.headw.alloc((size_t)nwords + 8, err));
    GB_TRY(p.lane.alloc((size_t)p.nruns * 32, err));
    GB_TRY(p.base.alloc((size_t)p.nruns + 1, err));
    GB_TRY(p.tail_row.alloc((size_t)p.nruns, err));
    GB_TRY(p.tail_last.alloc((size_t)p.nruns, err));
    CU_TRY(cudaMemsetAsync(p.headw, 0, ((size_t)nwords + 8) * 4, G.stream), err);
    CU_TRY(cudaMemsetAsync(flag + c.nrows, 0, 8, G.stream), err);
    plan_nonempty_kernel<<<rgrid(c.nrows), 256, 0, G.stream>>>(c.rowptr32, c.nrows, flag, p.pres_tmpl); GB_LAUNCHED();
    GB_TRY(dev_exclusive_scan(flag, c.nrows + 1, err));
    int64_t nz = 0;
    CU_TRY(cudaMemcpyAsync(&nz, flag + c.nrows, 8, cudaMemcpyDeviceToHost, G.stream), err);
    CU_TRY(cudaStreamSynchronize(G.stream), err);
    p.nnzrows = nz;
    GB_TRY(p.nzrow.alloc((size_t)nz, err));
    plan_rows_kernel<<<rgrid(c.nrows), 256, 0, G.stream>>>(c.rowptr32, flag, c.nrows, p.nzrow, p.headw); GB_LAUNCHED();
    CU_TRY(cudaMemsetAsync(cnt + p.nruns, 0, 8, G.stream), err);
    plan_runs_kernel<<<(unsigned)ceil_div(p.nruns * 32, 256), 256, 0, G.stream>>>(p.headw, p.nruns, nwords, p.lane, cnt); GB_LAUNCHED();
    GB_TRY(dev_exclusive_scan(cnt, p.nruns + 1, err));
    plan_base_kernel<<<rgrid(p.nruns + 1), 256, 0, G.stream>>>(cnt, p.nruns, p.base); GB_LAUNCHED();
    plan_tails_kernel<<<rgrid(p.nruns), 256, 0, G.stream>>>(p.base, p.nzrow, c.rowptr32, p.nruns, p.tail_row, p.tail_last); GB_LAUNCHED();
    flag.reset(); cnt.reset();
    // per-call scratch lives with the plan: partials of the rows that straddle runs (8 bytes covers every type)
    GB_TRY(p.ws_head.alloc((size_t)p.nruns * 8 + 16, err));
    GB_TRY(p.ws_tail.alloc((size_t)p.nruns * 8 + 16, err));
    GB_TRY(p.ws_head_has.alloc((size_t)p.nruns, err));
    GB_TRY(p.ws_tail_has.alloc((size_t)p.nruns, err));
    CU_TRY(cudaGetLastError(), err);
    c.run = std::move(p);
    return GrB_SUCCESS;
}

// ---- hot-column plan (cached per CSR): the HOT_EXT most referenced columns are renamed to their rank, every other
//      column c to c + henc, so the kernel tells a table lookup from a gather of u by compares and u itself is
//      read in place (no permuted copy per call).  Whether the hot-table kernel is used at all is decided on the
//      HOT_ENC hottest columns (`cover`); the ranks past them feed the tiers a thread-block cluster holds.
constexpr uint32_t HOT_ENC = 40960;
constexpr uint32_t HOT_EXT = 1u << 17;        // covers the tiers of the default cluster (DESIGN.md section 3.1: 2^17 to 2^19 measure alike)
__global__ void hot_count_kernel(const uint32_t *col, int64_t nnz, uint32_t *deg) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < nnz; k += (int64_t)gridDim.x * blockDim.x) atomicAdd(&deg[col[k]], 1u);
}
__global__ void hot_iota_kernel(uint32_t *a, int64_t n) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) a[k] = (uint32_t)k;
}
// inv[col] = rank for the first k ranks whose degree is non-zero; stats: {how many there are among the first HOT_ENC,
// the sum of their degrees, how many there are among all k}
__global__ void hot_invert_kernel(const uint32_t *perm, const uint32_t *deg_sorted, int64_t k, uint32_t *inv, unsigned long long *stats) {
    unsigned long long c = 0, d = 0, e = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < k; i += (int64_t)gridDim.x * blockDim.x) {
        if (deg_sorted[i] != 0) {
            inv[perm[i]] = (uint32_t)i; e += 1;
            if (i < HOT_ENC) { c += 1; d += deg_sorted[i]; }
        }
    }
    for (int o = 16; o > 0; o >>= 1) {
        c += __shfl_xor_sync(0xffffffffu, c, o); d += __shfl_xor_sync(0xffffffffu, d, o); e += __shfl_xor_sync(0xffffffffu, e, o);
    }
    if ((threadIdx.x & 31) == 0 && e) { atomicAdd(stats, c); atomicAdd(stats + 1, d); atomicAdd(stats + 2, e); }
}
__global__ void hot_encode_kernel(const uint32_t *col, const uint32_t *inv, int64_t nnz, uint32_t henc, uint32_t *out) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < nnz; k += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t c = col[k], r = inv[c];
        out[k] = r < henc ? r : c + henc;
    }
}

GrB_Info spmv_hot_plan(Csr &c, std::string *err) {
    if (c.hot.planned) return GrB_SUCCESS;
    const int64_t n = c.ncols;
    if (n + (int64_t)HOT_EXT >= ((int64_t)1 << 32)) { c.hot.planned = true; return GrB_SUCCESS; }
    HotPlan p;                 // moved into c only once complete
    DevBuf<uint32_t> deg, deg_sorted, ids, inv, perm; DevBuf<unsigned long long> stats;
    GB_TRY(deg.alloc((size_t)n, err)); GB_TRY(deg_sorted.alloc((size_t)n, err)); GB_TRY(ids.alloc((size_t)n, err));
    GB_TRY(inv.alloc((size_t)n, err)); GB_TRY(perm.alloc((size_t)n, err)); GB_TRY(stats.alloc(3, err));
    CU_TRY(cudaMemsetAsync(deg, 0, (size_t)n * 4, G.stream), err);
    CU_TRY(cudaMemsetAsync(inv, 0xff, (size_t)n * 4, G.stream), err);
    CU_TRY(cudaMemsetAsync(stats, 0, 24, G.stream), err);
    hot_count_kernel<<<hgrid(c.nnz), 256, 0, G.stream>>>(c.col, c.nnz, deg); GB_LAUNCHED();
    hot_iota_kernel<<<hgrid(n), 256, 0, G.stream>>>(ids, n); GB_LAUNCHED();
    size_t tmp_bytes = 0;     // stable sort: equal degrees keep ascending column order (deterministic plan)
    CU_TRY(cub::DeviceRadixSort::SortPairsDescending(nullptr, tmp_bytes, deg.get(), deg_sorted.get(), ids.get(), perm.get(), n, 0, 32, G.stream), err);
    DevBuf<void> tmp; GB_TRY(tmp.alloc(tmp_bytes, err));
    CU_TRY(cub::DeviceRadixSort::SortPairsDescending(tmp.get(), tmp_bytes, deg.get(), deg_sorted.get(), ids.get(), perm.get(), n, 0, 32, G.stream), err);
    G.launches += 8;
    const int64_t topk = std::min<int64_t>(n, HOT_EXT);
    hot_invert_kernel<<<hgrid(topk), 256, 0, G.stream>>>(perm, deg_sorted, topk, inv, stats); GB_LAUNCHED();
    unsigned long long h[3] = {0, 0, 0};
    CU_TRY(cudaMemcpyAsync(h, stats, 24, cudaMemcpyDeviceToHost, G.stream), err);
    CU_TRY(cudaStreamSynchronize(G.stream), err);
    p.cover = c.nnz ? (double)h[1] / (double)c.nnz : 0.0;
    p.planned = true;
    if (h[0] >= 16) {
        p.henc = (uint32_t)h[2];
        GB_TRY(p.perm.alloc((size_t)p.henc, err));
        GB_TRY(p.col.alloc((size_t)c.nnz, err));
        GB_TRY(p.ws_uhot.alloc(((size_t)p.henc + 256) * 8 + 16, err));      // + the unused tail of the last slices (< 16 per CTA)
        CU_TRY(cudaMemcpyAsync(p.perm, perm, (size_t)p.henc * 4, cudaMemcpyDeviceToDevice, G.stream), err);
        hot_encode_kernel<<<hgrid(c.nnz), 256, 0, G.stream>>>(c.col, inv, c.nnz, p.henc, p.col); GB_LAUNCHED();
    }
    CU_TRY(cudaGetLastError(), err);
    c.hot = std::move(p);
    return GrB_SUCCESS;
}

// prep for the hot-table kernel, one launch: u at the henc hottest columns into u_hot in the tier layout of the launch
// (spmv_args.cuh), T's values cleared and its presence bytes set from the plan's template (rows are structurally present
// or not: u is dense)
__global__ void __launch_bounds__(256) spmv_hot2_prep_kernel(const uint32_t *hperm, const uint8_t *u, uint8_t *u_hot, int vsize, uint32_t henc,
                                                            uint32_t t0, uint32_t t1, uint32_t slice, int lc,
                                                            uint4 *tval16, int64_t tval_n16, const uint4 *tmpl16, uint4 *tpres16, int64_t pres_n16) {
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, nth = (int64_t)gridDim.x * blockDim.x;
    const uint32_t past = (slice << lc) - t1;             // slots of the slices that hold no rank
    for (int64_t i = tid; i < henc; i += nth) {
        const uint32_t col = hperm[i], k = (uint32_t)i - t0;
        const uint32_t pos = i < t0 ? (uint32_t)i : k < t1 ? t0 + (k & ((1u << lc) - 1u)) * slice + (k >> lc) : (uint32_t)i + past;
        switch (vsize) {
            case 1: u_hot[pos] = u[col]; break;
            case 4: ((uint32_t *)u_hot)[pos] = ((const uint32_t *)u)[col]; break;
            default: ((uint64_t *)u_hot)[pos] = ((const uint64_t *)u)[col]; break;
        }
    }
    const uint4 z = make_uint4(0, 0, 0, 0);
    for (int64_t i = tid; i < tval_n16; i += nth) tval16[i] = z;
    for (int64_t i = tid; i < pres_n16; i += nth) tpres16[i] = tmpl16[i];
}

void spmv_hot2_prep(const Hot2Args &h) {
    const int64_t tv16 = (int64_t)((h.tval_bytes + 15) / 16), pr16 = (h.nrows + 15) / 16;      // buffers are padded by >= 16 bytes
    spmv_hot2_prep_kernel<<<G.num_sms * 8, 256, 0, G.stream>>>(h.hperm, (const uint8_t *)h.u, (uint8_t *)h.u_hot, h.vsize, h.henc,
                                                               h.t0, h.t1, h.slice, __builtin_ctz((unsigned)h.cluster),
                                                               (uint4 *)h.tval, tv16, (const uint4 *)h.pres_tmpl, (uint4 *)h.tpres, pr16);
    GB_LAUNCHED();
}

template <typename T> static bool spmv_run_fast(int add, int mul, const RunArgs &a, Hot2Args *hot, size_t table_limit) {
#define GB_FAST(A, M) if (add == A && mul == M) { spmv_run_launch<T, T, A, M>(a, hot, table_limit); return true; }
    GB_FAST(OP_PLUS, OP_TIMES) GB_FAST(OP_MIN, OP_PLUS) GB_FAST(OP_PLUS, OP_SECOND) GB_FAST(OP_PLUS, OP_FIRST)
    GB_FAST(OP_PLUS, OP_PAIR) GB_FAST(OP_MIN, OP_FIRST) GB_FAST(OP_MIN, OP_SECOND)
#undef GB_FAST
    return false;
}
bool spmv_run_fast_int(int xt, int add, int mul, const RunArgs &a, Hot2Args *hot, size_t table_limit);
bool spmv_run_dispatch(int xt, int add, int mul, const RunArgs &a, Hot2Args *hot, size_t table_limit) {
    switch (xt) {
        case TC_FP32: return spmv_run_fast<float>(add, mul, a, hot, table_limit);
        case TC_FP64: return spmv_run_fast<double>(add, mul, a, hot, table_limit);
        case TC_INT32:
        case TC_INT64:
        case TC_UINT32:
        case TC_UINT64:
        case TC_BOOL: return spmv_run_fast_int(xt, add, mul, a, hot, table_limit);
        default: return false;
    }
}
