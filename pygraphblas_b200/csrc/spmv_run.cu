// Run plan, hot-column plan, and the FP32 / FP64 instantiations of the run kernels.
#include "spmv_run.cuh"
#include <cub/device/device_radix_sort.cuh>

// ---- run plan (cached per CSR).  OT: the type of the row offsets read (uint32_t: rowptr32; int64_t: rowptr, the wide route)
template <typename OT>
__global__ void plan_nonempty_kernel(const OT *rowptr, int64_t nrows, int64_t *flag, uint8_t *pres) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += (int64_t)gridDim.x * blockDim.x) {
        const int ne = rowptr[r + 1] > rowptr[r];
        flag[r] = ne; pres[r] = (uint8_t)ne;
    }
}
template <typename OT>
__global__ void plan_rows_kernel(const OT *rowptr, const int64_t *rank, int64_t nrows, uint32_t *nzrow, uint32_t *headw) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += (int64_t)gridDim.x * blockDim.x) {
        const OT rs = rowptr[r];
        if (rowptr[r + 1] > rs) { nzrow[rank[r]] = (uint32_t)r; atomicOr(&headw[rs >> 5], 1u << (rs & 31)); }
    }
}
// row starts per run (a lane's rank inside its run is counted by the run kernels themselves: spmv_run_gather)
__global__ void plan_runs_kernel(const uint32_t *headw, int64_t nruns, int64_t nwords, int64_t *run_cnt) {
    const int lane = threadIdx.x & 31;
    const int64_t run = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (run >= nruns) return;
    const int64_t w = run * 8 + (lane >> 2);
    const uint32_t hw = (w < nwords && (lane & 3) == 0) ? headw[w] : 0u;
    const int cnt = (int)__reduce_add_sync(0xffffffffu, (unsigned)__popc(hw));
    if (lane == 0) run_cnt[run] = cnt;
}
__global__ void plan_base_kernel(const int64_t *scan, int64_t nruns, uint32_t *run_base) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k <= nruns; k += (int64_t)gridDim.x * blockDim.x) run_base[k] = (uint32_t)scan[k];
}
// the row that starts last inside a run always holds the run's last entry: it is the run's "open" row
// (possibly ending exactly at the run's end), completed by the fix-up kernel.  is_long[k]: that row reaches more than
// FIX_LONG runs past k (the fix-up gives it a warp)
template <typename OT>
__global__ void plan_tails_kernel(const uint32_t *run_base, const uint32_t *nzrow, const OT *rowptr, int64_t nruns,
                                  int32_t *tail_row, uint32_t *tail_last, int64_t *is_long) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < nruns; k += (int64_t)gridDim.x * blockDim.x) {
        int32_t tr = -1; uint32_t tl = 0;
        if (run_base[k + 1] > run_base[k]) {
            const uint32_t r = nzrow[run_base[k + 1] - 1];
            const OT re = rowptr[r + 1];
            tr = (int32_t)r; tl = (uint32_t)((re - 1) / RUN);
        }
        tail_row[k] = tr; tail_last[k] = tl;
        is_long[k] = tr >= 0 && (int64_t)tl - k > FIX_LONG;
    }
}
// the long runs in ascending order, from the exclusive scan of is_long
__global__ void plan_long_kernel(const int64_t *scan, int64_t nruns, uint32_t *long_run) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < nruns; k += (int64_t)gridDim.x * blockDim.x)
        if (scan[k + 1] > scan[k]) long_run[scan[k]] = (uint32_t)k;
}

template <typename OT> static GrB_Info spmv_run_plan_t(Csr &c, const OT *rowptr, std::string *err) {
    RunPlan p;                 // moved into c only once complete
    p.wide = sizeof(OT) == 8;
    const int64_t nwords = ceil_div(c.nnz, 32);
    p.nruns = ceil_div(c.nnz, RUN);
    DevBuf<int64_t> flag, cnt;
    GB_TRY(flag.alloc((size_t)c.nrows + 1, err));
    GB_TRY(cnt.alloc((size_t)p.nruns + 1, err));
    GB_TRY(p.pres_tmpl.alloc((size_t)c.nrows, err));
    GB_TRY(p.headw.alloc((size_t)nwords + 8, err));
    GB_TRY(p.base.alloc((size_t)p.nruns + 1, err));
    GB_TRY(p.tail_row.alloc((size_t)p.nruns, err));
    GB_TRY(p.tail_last.alloc((size_t)p.nruns, err));
    CU_TRY(cudaMemsetAsync(p.headw, 0, ((size_t)nwords + 8) * 4, G.stream), err);
    CU_TRY(cudaMemsetAsync(flag + c.nrows, 0, 8, G.stream), err);
    plan_nonempty_kernel<OT><<<grid_for(c.nrows), 256, 0, G.stream>>>(rowptr, c.nrows, flag, p.pres_tmpl); GB_LAUNCHED();
    GB_TRY(dev_exclusive_scan(flag, c.nrows + 1, err));
    int64_t nz = 0;
    CU_TRY(cudaMemcpyAsync(&nz, flag + c.nrows, 8, cudaMemcpyDeviceToHost, G.stream), err);
    CU_TRY(cudaStreamSynchronize(G.stream), err);
    p.nnzrows = nz;
    GB_TRY(p.nzrow.alloc((size_t)nz, err));
    plan_rows_kernel<OT><<<grid_for(c.nrows), 256, 0, G.stream>>>(rowptr, flag, c.nrows, p.nzrow, p.headw); GB_LAUNCHED();
    CU_TRY(cudaMemsetAsync(cnt + p.nruns, 0, 8, G.stream), err);
    plan_runs_kernel<<<(unsigned)ceil_div(p.nruns * 32, 256), 256, 0, G.stream>>>(p.headw, p.nruns, nwords, cnt); GB_LAUNCHED();
    GB_TRY(dev_exclusive_scan(cnt, p.nruns + 1, err));
    plan_base_kernel<<<grid_for(p.nruns + 1), 256, 0, G.stream>>>(cnt, p.nruns, p.base); GB_LAUNCHED();
    plan_tails_kernel<OT><<<grid_for(p.nruns), 256, 0, G.stream>>>(p.base, p.nzrow, rowptr, p.nruns, p.tail_row, p.tail_last, cnt); GB_LAUNCHED();
    CU_TRY(cudaMemsetAsync(cnt + p.nruns, 0, 8, G.stream), err);
    GB_TRY(dev_exclusive_scan(cnt, p.nruns + 1, err));
    CU_TRY(cudaMemcpyAsync(&p.nlong, cnt + p.nruns, 8, cudaMemcpyDeviceToHost, G.stream), err);
    CU_TRY(cudaStreamSynchronize(G.stream), err);
    GB_TRY(p.long_run.alloc((size_t)p.nlong + 1, err));
    plan_long_kernel<<<grid_for(p.nruns), 256, 0, G.stream>>>(cnt, p.nruns, p.long_run); GB_LAUNCHED();
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
// the plan of the route csr_wide picks: a plan built by the other route is built again (they are equal; B200_debug_wide tests both)
GrB_Info spmv_run_plan(Csr &c, std::string *err) {
    const bool wide = csr_wide(c);
    if (c.run.headw && c.run.wide == wide) return GrB_SUCCESS;
    c.run = RunPlan();
    return wide ? spmv_run_plan_t<int64_t>(c, c.rowptr, err) : spmv_run_plan_t<uint32_t>(c, c.rowptr32, err);
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
// the same ids in 3 bytes, packed run by run (spmv_args.cuh, HOT_IDS3_RUN): the slots of the last run past nnz hold henc
__global__ void hot_encode3_kernel(const uint32_t *col, const uint32_t *inv, int64_t nnz, int64_t nslots, uint32_t henc, uint8_t *out) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < nslots; k += (int64_t)gridDim.x * blockDim.x) {
        uint32_t id = henc;
        if (k < nnz) { const uint32_t c = col[k], r = inv[c]; id = r < henc ? r : c + henc; }
        uint8_t *run = out + (k / RUN) * HOT_IDS3_RUN;
        const int j = (int)(k % RUN);
        reinterpret_cast<uint16_t *>(run)[j] = (uint16_t)id;
        run[RUN * 2 + j] = (uint8_t)(id >> 16);
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
    hot_count_kernel<<<grid_for(c.nnz, 256, 32), 256, 0, G.stream>>>(c.col, c.nnz, deg); GB_LAUNCHED();
    hot_iota_kernel<<<grid_for(n, 256, 32), 256, 0, G.stream>>>(ids, n); GB_LAUNCHED();
    size_t tmp_bytes = 0;     // stable sort: equal degrees keep ascending column order (deterministic plan)
    CU_TRY(cub::DeviceRadixSort::SortPairsDescending(nullptr, tmp_bytes, deg.get(), deg_sorted.get(), ids.get(), perm.get(), n, 0, 32, G.stream), err);
    DevBuf<void> tmp; GB_TRY(tmp.alloc(tmp_bytes, err));
    CU_TRY(cub::DeviceRadixSort::SortPairsDescending(tmp.get(), tmp_bytes, deg.get(), deg_sorted.get(), ids.get(), perm.get(), n, 0, 32, G.stream), err);
    G.launches += 8;
    const int64_t topk = std::min<int64_t>(n, HOT_EXT);
    hot_invert_kernel<<<grid_for(topk, 256, 32), 256, 0, G.stream>>>(perm, deg_sorted, topk, inv, stats); GB_LAUNCHED();
    unsigned long long h[3] = {0, 0, 0};
    CU_TRY(cudaMemcpyAsync(h, stats, 24, cudaMemcpyDeviceToHost, G.stream), err);
    CU_TRY(cudaStreamSynchronize(G.stream), err);
    p.cover = c.nnz ? (double)h[1] / (double)c.nnz : 0.0;
    p.planned = true;
    if (h[0] >= 16) {
        p.henc = (uint32_t)h[2];
        // 3-byte ids when the largest, ncols - 1 + henc, stays below 2^24 - 1: the kernel's stage guard relies on no id being
        // all ones (spmv_run_hot2_kernel)
        p.id_bytes = n + (int64_t)p.henc < ((int64_t)1 << 24) ? 3 : 4;
        const int64_t nruns = ceil_div(c.nnz, RUN);
        GB_TRY(p.perm.alloc((size_t)p.henc, err));
        GB_TRY(p.col.alloc(p.id_bytes == 3 ? (size_t)nruns * HOT_IDS3_RUN : (size_t)c.nnz * 4 + 16, err));
        GB_TRY(p.ws_uhot.alloc(((size_t)p.henc + 256) * 8 + 16, err));      // + the unused tail of the last slices (< 16 per CTA)
        CU_TRY(cudaMemcpyAsync(p.perm, perm, (size_t)p.henc * 4, cudaMemcpyDeviceToDevice, G.stream), err);
        if (p.id_bytes == 3)
            hot_encode3_kernel<<<grid_for(nruns * RUN, 256, 32), 256, 0, G.stream>>>(c.col, inv, c.nnz, nruns * RUN, p.henc, (uint8_t *)p.col);
        else
            hot_encode_kernel<<<grid_for(c.nnz, 256, 32), 256, 0, G.stream>>>(c.col, inv, c.nnz, p.henc, (uint32_t *)p.col);
        GB_LAUNCHED();
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
    pdl_launch_dependents();                              // the hot-table kernel waits for this grid before it reads u_hot or writes T
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
