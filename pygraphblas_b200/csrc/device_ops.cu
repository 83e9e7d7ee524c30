// device_ops.cu -- small sm_90a utility kernels shared by the hot path:
// 64-bit exclusive scan, rowptr narrowing, CSR transpose (cached per matrix),
// run-time-typed value casts, presence counting.
#include "common.cuh"
#include <cub/device/device_radix_sort.cuh>

// ------------------------------------------------------------------ exclusive scan (int64, in place)
// Three-phase block scan: per-block totals -> recursive scan of totals -> per-block scan + offset.
static constexpr int SCAN_THREADS = 256;
static constexpr int SCAN_ITEMS = 8;
static constexpr int SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

__device__ __forceinline__ int64_t block_reduce_sum(int64_t v, int64_t *s_warp) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (lane == 0) s_warp[w] = v;
    __syncthreads();
    int64_t t = 0;
    if (threadIdx.x < 32) {
        t = threadIdx.x < (blockDim.x >> 5) ? s_warp[threadIdx.x] : 0;
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    }
    return t;   // valid in warp 0
}

__global__ void __launch_bounds__(SCAN_THREADS) scan_block_totals(const int64_t *in, int64_t n, int64_t *totals) {
    __shared__ int64_t s_warp[32];
    const int64_t base = (int64_t)blockIdx.x * SCAN_TILE;
    int64_t v = 0;
    for (int k = 0; k < SCAN_ITEMS; ++k) {
        const int64_t i = base + threadIdx.x + (int64_t)k * SCAN_THREADS;
        if (i < n) v += in[i];
    }
    const int64_t t = block_reduce_sum(v, s_warp);
    if (threadIdx.x == 0) totals[blockIdx.x] = t;
}

__global__ void __launch_bounds__(SCAN_THREADS) scan_block_apply(int64_t *data, int64_t n, const int64_t *offsets) {
    __shared__ int64_t s_warp[32];
    const int64_t base = (int64_t)blockIdx.x * SCAN_TILE + (int64_t)threadIdx.x * SCAN_ITEMS;
    int64_t x[SCAN_ITEMS]; int64_t sum = 0;
    for (int k = 0; k < SCAN_ITEMS; ++k) { x[k] = (base + k < n) ? data[base + k] : 0; sum += x[k]; }
    // exclusive scan of per-thread sums across the block
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int64_t inc = sum;
    for (int o = 1; o < 32; o <<= 1) { int64_t y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
    if (lane == 31) s_warp[w] = inc;
    __syncthreads();
    if (w == 0) {
        int64_t t = lane < (SCAN_THREADS >> 5) ? s_warp[lane] : 0;
        int64_t ti = t;
        for (int o = 1; o < 32; o <<= 1) { int64_t y = __shfl_up_sync(0xffffffffu, ti, o); if (lane >= o) ti += y; }
        s_warp[lane] = ti - t;
    }
    __syncthreads();
    int64_t run = (offsets ? offsets[blockIdx.x] : 0) + s_warp[w] + (inc - sum);
    for (int k = 0; k < SCAN_ITEMS; ++k) { if (base + k < n) data[base + k] = run; run += x[k]; }
}

// in-place exclusive prefix sum of data[0..n); returns nothing (total = data[n-1]+last, callers keep a slot n)
GrB_Info dev_exclusive_scan(int64_t *data, int64_t n, std::string *err) {
    if (n <= 0) return GrB_SUCCESS;
    const int64_t nb = ceil_div(n, SCAN_TILE);
    if (nb == 1) {
        scan_block_apply<<<1, SCAN_THREADS, 0, G.stream>>>(data, n, nullptr); GB_LAUNCHED();
        return GrB_SUCCESS;
    }
    DevBuf<int64_t> totals;
    GB_TRY(totals.alloc((size_t)nb, err));
    scan_block_totals<<<(unsigned)nb, SCAN_THREADS, 0, G.stream>>>(data, n, totals); GB_LAUNCHED();
    GB_TRY(dev_exclusive_scan(totals, nb, err));
    scan_block_apply<<<(unsigned)nb, SCAN_THREADS, 0, G.stream>>>(data, n, totals); GB_LAUNCHED();
    CU_TRY(cudaGetLastError(), err);
    return GrB_SUCCESS;
}

// ------------------------------------------------------------------ rowptr narrowing
__global__ void narrow_rowptr_kernel(const int64_t *rp, uint32_t *rp32, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        rp32[i] = (uint32_t)rp[i];
}
GrB_Info dev_build_rowptr32(Csr &c, std::string *err) {
    c.rowptr32.reset();
    c.drop_plans();
    if (c.nnz >= ((int64_t)1 << 32)) return GrB_SUCCESS;
    DevBuf<uint32_t> rp32;
    GB_TRY(rp32.alloc((size_t)c.nrows + 1, err));
    const int64_t n = c.nrows + 1;
    const int blocks = (int)std::min<int64_t>(ceil_div(n, 256), (int64_t)G.num_sms * 8);
    narrow_rowptr_kernel<<<blocks, 256, 0, G.stream>>>(c.rowptr, rp32, n); GB_LAUNCHED();
    CU_TRY(cudaGetLastError(), err);
    c.rowptr32 = std::move(rp32);
    return GrB_SUCCESS;
}

// ------------------------------------------------------------------ transpose (CSR of A')
__global__ void expand_rows_kernel(const int64_t *rowptr, int64_t nrows, uint32_t *rowid) {
    // one warp per row
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < nrows; r += nwarps)
        for (int64_t k = rowptr[r] + lane; k < rowptr[r + 1]; k += 32) rowid[k] = (uint32_t)r;
}
__global__ void count_cols_kernel(const uint32_t *col, int64_t nnz, int64_t *count) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < nnz; k += (int64_t)gridDim.x * blockDim.x)
        atomicAdd((unsigned long long *)&count[col[k]], 1ull);
}
__global__ void iota_kernel(uint32_t *a, int64_t n) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) a[k] = (uint32_t)k;
}
__global__ void permute_kernel(const uint32_t *perm, const uint32_t *rowid, const uint8_t *val, int vsize,
                               int64_t nnz, uint32_t *tcol, uint8_t *tval) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < nnz; k += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t p = perm[k];
        tcol[k] = rowid[p];
        switch (vsize) {
            case 1: tval[k] = val[p]; break;
            case 2: ((uint16_t *)tval)[k] = ((const uint16_t *)val)[p]; break;
            case 4: ((uint32_t *)tval)[k] = ((const uint32_t *)val)[p]; break;
            default: ((uint64_t *)tval)[k] = ((const uint64_t *)val)[p]; break;
        }
    }
}

static inline int grid_for(int64_t n, int threads = 256) {
    return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n, threads), (int64_t)G.num_sms * 16));
}

// T = A' as CSR.  A stable LSD radix sort of the entries by column keeps, inside
// every column, the row-major order of A, i.e. ascending row ids: T's rows come out sorted.
// (cub::DeviceRadixSort is used here only: this is a cached set-up step, not the hot path.)
GrB_Info dev_transpose(const Csr &a, size_t vsize, Csr &t, std::string *err) {
    if (a.nnz >= ((int64_t)1 << 32)) return gb_fail(GrB_INVALID_VALUE, err, "transpose: nnz >= 2^32 not supported");
    t = Csr(); t.nrows = a.ncols; t.ncols = a.nrows; t.nnz = a.nnz;
    GB_TRY(t.rowptr.alloc((size_t)t.nrows + 1, err));
    GB_TRY(t.col.alloc((size_t)t.nnz, err));
    GB_TRY(t.val.alloc((size_t)t.nnz * vsize + 16, err));
    CU_TRY(cudaMemsetAsync(t.rowptr, 0, ((size_t)t.nrows + 1) * 8, G.stream), err);
    if (a.nnz > 0) {
        DevBuf<uint32_t> rowid, perm_in, perm_out, keys_out;
        GB_TRY(rowid.alloc((size_t)a.nnz, err)); GB_TRY(perm_in.alloc((size_t)a.nnz, err));
        GB_TRY(perm_out.alloc((size_t)a.nnz, err)); GB_TRY(keys_out.alloc((size_t)a.nnz, err));
        expand_rows_kernel<<<grid_for(a.nrows * 32), 256, 0, G.stream>>>(a.rowptr, a.nrows, rowid); GB_LAUNCHED();
        count_cols_kernel<<<grid_for(a.nnz), 256, 0, G.stream>>>(a.col, a.nnz, t.rowptr); GB_LAUNCHED();
        iota_kernel<<<grid_for(a.nnz), 256, 0, G.stream>>>(perm_in, a.nnz); GB_LAUNCHED();
        int end_bit = 1; while (end_bit < 32 && ((int64_t)1 << end_bit) < a.ncols) ++end_bit;
        size_t tmp_bytes = 0;
        CU_TRY(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, a.col.get(), keys_out.get(), perm_in.get(), perm_out.get(), (int64_t)a.nnz, 0, end_bit, G.stream), err);
        DevBuf<void> tmp; GB_TRY(tmp.alloc(tmp_bytes, err));
        CU_TRY(cub::DeviceRadixSort::SortPairs(tmp.get(), tmp_bytes, a.col.get(), keys_out.get(), perm_in.get(), perm_out.get(), (int64_t)a.nnz, 0, end_bit, G.stream), err);
        G.launches += 8;
        permute_kernel<<<grid_for(a.nnz), 256, 0, G.stream>>>(perm_out, rowid, (const uint8_t *)a.val, (int)vsize, a.nnz, t.col, (uint8_t *)t.val); GB_LAUNCHED();
    }
    GB_TRY(dev_exclusive_scan(t.rowptr, t.nrows + 1, err));
    GB_TRY(dev_build_rowptr32(t, err));
    CU_TRY(cudaGetLastError(), err);
    return GrB_SUCCESS;
}

// ------------------------------------------------------------------ run-time typed cast
__global__ void cast_kernel(void *out, int to, const void *in, int from, int64_t n) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x)
        sc_store(to, out, (size_t)k, sc_cast(sc_load(from, in, (size_t)k), from, to));
}
GrB_Info dev_cast_values(DevBuf<void> &out, int to_code, const void *in, int from_code, int64_t n, std::string *err) {
    GB_TRY(out.alloc((size_t)n * tc_size(to_code) + 16, err));
    if (n > 0) { cast_kernel<<<grid_for(n), 256, 0, G.stream>>>(out, to_code, in, from_code, n); GB_LAUNCHED(); }
    CU_TRY(cudaGetLastError(), err);
    return GrB_SUCCESS;
}

// ------------------------------------------------------------------ presence count
__global__ void count_present_kernel(const uint8_t *pres, int64_t n, unsigned long long *out) {
    unsigned long long c = 0;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) c += pres[k] != 0;
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, c);
}
GrB_Info dev_count_present(const uint8_t *pres, int64_t n, int64_t *count, std::string *err) {
    DevBuf<unsigned long long> d;
    GB_TRY(d.alloc(1, err));
    CU_TRY(cudaMemsetAsync(d, 0, 8, G.stream), err);
    count_present_kernel<<<grid_for(n), 256, 0, G.stream>>>(pres, n, d); GB_LAUNCHED();
    unsigned long long h = 0;
    CU_TRY(cudaMemcpyAsync(&h, d, 8, cudaMemcpyDeviceToHost, G.stream), err);
    CU_TRY(cudaStreamSynchronize(G.stream), err);
    *count = (int64_t)h;
    return GrB_SUCCESS;
}
