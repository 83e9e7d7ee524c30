// spmm.cu -- GrB_mxm with a dense right operand (DESIGN.md section 3.6), and the conversions between a matrix's dense form
// and its CSR.
//
//   T = op(A) (+).(x) X,   X a dense-form n x k matrix (row-major values, optional presence bytes), T formed dense (m x k)
//
// A group of W lanes (W = the power of two >= k, at most 32) folds one row of op(A) for W consecutive output columns: lane j
// walks the row's entries in column order and gathers X(col, j), so the k lanes of one entry read one contiguous row of X and
// the fold is the oracle's left-to-right fold.  Rows longer than SPMM_SEG entries are cut into segments of SPMM_SEG entries;
// each segment's partial goes to scratch and a second kernel folds the partials of a row pairwise in a fixed tree over the
// segment order (deterministic, no atomics).  The result is written back through the vector write-back over the flattened m*k positions, so C keeps the
// dense form; only a CSR mask sends T through the CSR write-back.
//
// A dense X on the left, C = X (+).(x) op(B), runs as C' = op(B)' (+).(x)' X' on the same kernels (spmm_left_mxm), with the
// multiply's operands swapped and dense_transpose_kernel turning X into X' and T' into T.
#include "common.cuh"
#include "spmv_common.cuh"

// ------------------------------------------------------------------ dense form <-> CSR
__device__ __forceinline__ void copy_value(uint8_t *dst, int64_t d, const uint8_t *src, int64_t s, int vsize) {
    switch (vsize) {
        case 1: dst[d] = src[s]; break;
        case 2: ((uint16_t *)dst)[d] = ((const uint16_t *)src)[s]; break;
        case 4: ((uint32_t *)dst)[d] = ((const uint32_t *)src)[s]; break;
        default: ((uint64_t *)dst)[d] = ((const uint64_t *)src)[s]; break;
    }
}
// warp per row: present entries of the row (pres NULL: all ncols)
__global__ void dense_row_count_kernel(const uint8_t *pres, int64_t nrows, int64_t ncols, int64_t *cnt) {
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int lane = threadIdx.x & 31;
    for (int64_t r = warp; r < nrows; r += nwarps) {
        int64_t c = 0;
        if (pres) for (int64_t j = lane; j < ncols; j += 32) c += pres[r * ncols + j] != 0;
        else c = lane == 0 ? ncols : 0;
        for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
        if (lane == 0) cnt[r] = c;
    }
}
// warp per row: the present entries, in column order, at the row's offset (a ballot ranks them inside each 32-column slice)
__global__ void dense_compact_kernel(const uint8_t *val, const uint8_t *pres, int64_t nrows, int64_t ncols, int vsize,
                                     const int64_t *rowptr, uint32_t *col, uint8_t *cval) {
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int lane = threadIdx.x & 31;
    for (int64_t r = warp; r < nrows; r += nwarps) {
        int64_t out = rowptr[r];
        for (int64_t base = 0; base < ncols; base += 32) {
            const int64_t j = base + lane;
            const bool p = j < ncols && (!pres || pres[r * ncols + j] != 0);
            const unsigned b = __ballot_sync(0xffffffffu, p);
            if (p) {
                const int64_t o = out + __popc(b & ((1u << lane) - 1));
                col[o] = (uint32_t)j;
                copy_value(cval, o, val, r * ncols + j, vsize);
            }
            out += __popc(b);
        }
    }
}
// warp per row: every entry of a CSR to its place in zero-filled dense arrays
__global__ void csr_scatter_dense_kernel(const int64_t *rowptr, const uint32_t *col, const uint8_t *cval, int64_t nrows, int64_t ncols,
                                         int vsize, uint8_t *val, uint8_t *pres) {
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int lane = threadIdx.x & 31;
    for (int64_t r = warp; r < nrows; r += nwarps)
        for (int64_t e = rowptr[r] + lane; e < rowptr[r + 1]; e += 32) {
            const int64_t d = r * ncols + col[e];
            copy_value(val, d, cval, e, vsize);
            pres[d] = 1;
        }
}

GrB_Info dense_to_csr(const void *val, const uint8_t *pres, int64_t nrows, int64_t ncols, size_t vsize, Csr &c, std::string *err) {
    Csr r;
    GB_TRY(csr_from_row_counts(nrows, ncols, vsize, r, err,
        [&](int64_t *rowptr) {
            CU_TRY(cudaMemsetAsync(rowptr, 0, ((size_t)nrows + 1) * 8, G.stream), err);
            if (nrows > 0) { dense_row_count_kernel<<<grid_for(nrows * 32), 256, 0, G.stream>>>(pres, nrows, ncols, rowptr); GB_LAUNCHED(); }
            return GrB_SUCCESS;
        },
        [&](Csr &t) {
            dense_compact_kernel<<<grid_for(nrows * 32), 256, 0, G.stream>>>((const uint8_t *)val, pres, nrows, ncols, (int)vsize, t.rowptr,
                                                                             t.col, (uint8_t *)t.val.get());
            GB_LAUNCHED();
            return GrB_SUCCESS;
        }));
    c = std::move(r);
    return GrB_SUCCESS;
}

// out (cols x rows) = in (rows x cols)', both row-major, presence bytes carried along (ipres NULL: no presence is written).
// A CTA of 32 x 8 threads moves one 32 x 32 tile at a time through shared memory (one column of padding), so both the loads
// and the stores run along rows; the CTAs stride over the tiles, so any rows * cols < 2^31 fits a capped grid.
template <typename V>
__global__ void __launch_bounds__(256) dense_transpose_kernel(const V *in, const uint8_t *ipres, int64_t rows, int64_t cols,
                                                              V *out, uint8_t *opres) {
    __shared__ V tv[32][33];
    __shared__ uint8_t tp[32][33];
    const int64_t tcols = ceil_div(cols, 32), ntiles = ceil_div(rows, 32) * tcols;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const int64_t r0 = t / tcols * 32, c0 = t % tcols * 32;
        for (int y = ty; y < 32; y += 8) {
            const int64_t r = r0 + y, c = c0 + tx;
            if (r < rows && c < cols) {
                tv[y][tx] = in[r * cols + c];
                if (ipres) tp[y][tx] = ipres[r * cols + c];
            }
        }
        __syncthreads();
        for (int y = ty; y < 32; y += 8) {
            const int64_t c = c0 + y, r = r0 + tx;     // out(c, r) = in(r, c)
            if (c < cols && r < rows) {
                out[c * rows + r] = tv[tx][y];
                if (ipres) opres[c * rows + r] = tp[tx][y];
            }
        }
        __syncthreads();
    }
}

GrB_Info dense_transpose(const void *val,const uint8_t *pres, int64_t rows, int64_t cols, size_t vsize, void *oval, uint8_t *opres,
                         std::string *err) {
    if (rows == 0 || cols == 0) return GrB_SUCCESS;
    const int grid = grid_for(ceil_div(rows, 32) * ceil_div(cols, 32), 1);
    switch (vsize) {
        case 1: dense_transpose_kernel<uint8_t><<<grid, 256, 0, G.stream>>>((const uint8_t *)val, pres, rows, cols, (uint8_t *)oval, opres); break;
        case 2: dense_transpose_kernel<uint16_t><<<grid, 256, 0, G.stream>>>((const uint16_t *)val, pres, rows, cols, (uint16_t *)oval, opres); break;
        case 4: dense_transpose_kernel<uint32_t><<<grid, 256, 0, G.stream>>>((const uint32_t *)val, pres, rows, cols, (uint32_t *)oval, opres); break;
        default: dense_transpose_kernel<uint64_t><<<grid, 256, 0, G.stream>>>((const uint64_t *)val, pres, rows, cols, (uint64_t *)oval, opres); break;
    }
    GB_LAUNCHED();
    CU_TRY(cudaGetLastError(), err);
    return GrB_SUCCESS;
}

GrB_Info csr_to_dense(const Csr &c, size_t vsize, DevBuf<void> &val, DevBuf<uint8_t> &pres, std::string *err) {
    const size_t n = (size_t)(c.nrows * c.ncols);
    DevBuf<void> v; DevBuf<uint8_t> p;
    GB_TRY(v.alloc(n * vsize + 16, err));
    GB_TRY(p.alloc(n, err));
    if (n) {
        CU_TRY(cudaMemsetAsync(v, 0, n * vsize, G.stream), err);
        CU_TRY(cudaMemsetAsync(p, 0, n, G.stream), err);
    }
    if (c.nnz > 0) {
        csr_scatter_dense_kernel<<<grid_for(c.nrows * 32), 256, 0, G.stream>>>(c.rowptr, c.col, (const uint8_t *)c.val.get(), c.nrows, c.ncols,
                                                                               (int)vsize, (uint8_t *)v.get(), p);
        GB_LAUNCHED();
    }
    CU_TRY(cudaGetLastError(), err);
    val = std::move(v); pres = std::move(p);
    return GrB_SUCCESS;
}

// ------------------------------------------------------------------ the SpMM kernels
// OT: the type of the row offsets (uint32_t: rowptr32; int64_t: rowptr, the wide route of matrices with >= 2^32 entries)
template <typename OT> struct SpmmArgsT {
    const OT *rowptr; const uint32_t *col; const void *aval;   // op(A): m rows, values of the multiply's x type
    const void *xval; const uint8_t *xpres;             // X: n x k row-major, values of the multiply's y type
    int64_t m, k;
    int add, mul;
    int gshift;                 // log2 of the lanes of a group (one row or segment, up to 32 columns)
    int64_t nitems;             // m rows, then the segments of the long rows
    const int64_t *segoff;      // [m+1] first segment of each row (only rows longer than SPMM_SEG have segments)
    const uint32_t *segrow;     // [nseg] row of each segment
    void *tval; uint8_t *tpres; // T: m x k
    void *pval; uint8_t *ppres; // partials: nseg x k
};

template <typename XT, typename ZT, int ADD, int MUL, typename OT>
__global__ void __launch_bounds__(256, 2) spmm_kernel(const SpmmArgsT<OT> p) {
    const int add = ADD >= 0 ? ADD : p.add, mul = MUL >= 0 ? MUL : p.mul;
    const int64_t item = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> p.gshift;
    if (item >= p.nitems) return;                       // lanes fold independently: no warp-wide operation follows
    const bool seg = item >= p.m;                       // a segment of a long row (its partial goes to scratch)
    const int64_t q = item - p.m;
    const uint32_t r = seg ? p.segrow[q] : (uint32_t)item;
    const int64_t rb = p.rowptr[r], re = p.rowptr[r + 1];
    if (!seg && re - rb > SPMM_SEG) return;             // folded by its segments
    const int64_t beg = seg ? rb + (q - p.segoff[r]) * SPMM_SEG : rb;
    const int64_t end = seg ? min(beg + SPMM_SEG, re) : re;
    ZT *out = (ZT *)(seg ? p.pval : p.tval);
    uint8_t *outp = seg ? p.ppres : p.tpres;
    const int64_t o = (seg ? q : item) * p.k;
    const XT *av = (const XT *)p.aval, *xv = (const XT *)p.xval;
    const uint8_t *xp = p.xpres;
    const bool rx = mul_reads_x(mul), ry = mul_reads_y(mul);
    // the group's column tiles (blockIdx.y strides them; one tile when k <= 32)
    for (int64_t j = ((int64_t)blockIdx.y << p.gshift) + (threadIdx.x & ((1 << p.gshift) - 1)); j < p.k; j += (int64_t)gridDim.y << p.gshift) {
        ZT acc = (ZT)0; bool has = false;
        int64_t e = beg;
        constexpr int U = 4;    // entries whose loads are in flight together; folded in order afterwards
        for (; e + U <= end; e += U) {
            XT a[U], x[U]; bool pr[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int64_t xi = (int64_t)__ldg(p.col + e + u) * p.k + j;
                a[u] = rx ? gload(av + e + u) : (XT)0;
                x[u] = ry ? gload(xv + xi) : (XT)0;
                pr[u] = xp ? gload(xp + xi) != 0 : true;
            }
#pragma unroll
            for (int u = 0; u < U; ++u)
                if (pr[u]) {
                    const ZT z = MulApply<XT, ZT>::f(mul, a[u], x[u]);
                    acc = has ? MulApply<ZT, ZT>::f(add, acc, z) : z; has = true;
                }
        }
        for (; e < end; ++e) {
            const int64_t xi = (int64_t)__ldg(p.col + e) * p.k + j;
            if (xp && gload(xp + xi) == 0) continue;
            const ZT z = MulApply<XT, ZT>::f(mul, rx ? gload(av + e) : (XT)0, ry ? gload(xv + xi) : (XT)0);
            acc = has ? MulApply<ZT, ZT>::f(add, acc, z) : z; has = true;
        }
        out[o + j] = has ? acc : (ZT)0;
        outp[o + j] = has;
    }
}

// thread per (long row, column): the partials of the row's segments folded pairwise, in place, in a fixed tree over the
// segment order (deterministic; the rounding error of a long FP row grows with the log of its segment count, not linearly)
template <typename ZT, typename OT>
__global__ void __launch_bounds__(256) spmm_combine_kernel(const SpmmArgsT<OT> p, int64_t nseg) {
    ZT *pv = (ZT *)p.pval;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < nseg * p.k; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t q = t / p.k, j = t - q * p.k;
        const uint32_t r = p.segrow[q];
        if (q != p.segoff[r]) continue;                 // not the row's first segment
        const int64_t ns = p.segoff[r + 1] - q;
        for (int64_t w = 1; w < ns; w <<= 1)
            for (int64_t s = 0; s + w < ns; s += 2 * w) {
                const int64_t a = (q + s) * p.k + j, b = (q + s + w) * p.k + j;
                if (!p.ppres[b]) continue;
                pv[a] = p.ppres[a] ? MulApply<ZT, ZT>::f(p.add, pv[a], pv[b]) : pv[b];
                p.ppres[a] = 1;
            }
        const bool has = p.ppres[q * p.k + j] != 0;
        ((ZT *)p.tval)[r * p.k + j] = has ? pv[q * p.k + j] : (ZT)0;
        p.tpres[r * p.k + j] = has;
    }
}

template <typename OT> __global__ void spmm_seg_count_kernel(const OT *rowptr, int64_t m, int64_t *cnt) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < m; r += (int64_t)gridDim.x * blockDim.x) {
        const int64_t len = (int64_t)rowptr[r + 1] - rowptr[r];
        cnt[r] = len > SPMM_SEG ? ceil_div(len, SPMM_SEG) : 0;
    }
}
__global__ void spmm_seg_fill_kernel(const int64_t *segoff, int64_t m, uint32_t *segrow) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < m; r += (int64_t)gridDim.x * blockDim.x)
        for (int64_t q = segoff[r]; q < segoff[r + 1]; ++q) segrow[q] = (uint32_t)r;
}

// the specialised semirings (the SpMV list, spmv_common.cuh) on x = z = T
template <typename T, typename OT> static bool spmm_launch_fast(int add, int mul, const SpmmArgsT<OT> &p, dim3 grid) {
#define GB_SPMM_FAST(A, M) if (add == A && mul == M) { spmm_kernel<T, T, A, M, OT><<<grid, 256, 0, G.stream>>>(p); return true; }
    GB_SPMV_FAST_PAIRS(T, GB_SPMM_FAST)
#undef GB_SPMM_FAST
    return false;
}
template <typename OT> static bool spmm_launch(int xt, int zt, const SpmmArgsT<OT> &p, dim3 grid, bool *fast) {
    *fast = false;
    if (xt == zt) switch (xt) {
        case TC_FP32: *fast = spmm_launch_fast<float, OT>(p.add, p.mul, p, grid); break;
        case TC_FP64: *fast = spmm_launch_fast<double, OT>(p.add, p.mul, p, grid); break;
        case TC_INT32: *fast = spmm_launch_fast<int32_t, OT>(p.add, p.mul, p, grid); break;
        case TC_INT64: *fast = spmm_launch_fast<int64_t, OT>(p.add, p.mul, p, grid); break;
        case TC_UINT32: *fast = spmm_launch_fast<uint32_t, OT>(p.add, p.mul, p, grid); break;
        case TC_UINT64: *fast = spmm_launch_fast<uint64_t, OT>(p.add, p.mul, p, grid); break;
        case TC_BOOL: *fast = spmm_launch_fast<bool, OT>(p.add, p.mul, p, grid); break;
        default: break;
    }
    if (*fast) return true;
    bool matched = false;
    GB_FOR_DOMAINS(xt, zt, matched, (spmm_kernel<XT_, ZT_, -1, -1, OT><<<grid, 256, 0, G.stream>>>(p)));
    return matched;
}
template <typename OT> static bool spmm_combine(int zt, const SpmmArgsT<OT> &p, int64_t nseg) {
    const int grid = grid_for(nseg * p.k);
    bool matched = false;
    GB_FOR_DOMAINS(zt, zt, matched, (spmm_combine_kernel<ZT_, OT><<<grid, 256, 0, G.stream>>>(p, nseg)));
    return matched;
}

// T (m x k, type zt, presence per entry) = a (+).(x) X, reading a's row offsets through rowptr (of type OT)
template <typename OT>
static GrB_Info spmm_product_t(const Csr &a, const OT *rowptr, const void *aval, const void *xval, const uint8_t *xpres, int64_t k, int xt,
                               int zt, int add, int mul, void *tval, uint8_t *tpres, std::string *err) {
    const int64_t m = a.nrows;
    SpmmArgsT<OT> p{};
    p.rowptr = rowptr; p.col = a.col; p.aval = aval; p.xval = xval; p.xpres = xpres;
    p.m = m; p.k = k; p.add = add; p.mul = mul;
    while ((1 << p.gshift) < k && p.gshift < 5) ++p.gshift;
    p.tval = tval; p.tpres = tpres;
    // segments of the long rows
    DevBuf<int64_t> segoff; DevBuf<uint32_t> segrow; DevBuf<void> pval; DevBuf<uint8_t> ppres;
    GB_TRY(segoff.alloc((size_t)m + 1, err));
    CU_TRY(cudaMemsetAsync(segoff.get() + m, 0, 8, G.stream), err);
    spmm_seg_count_kernel<<<grid_for(m), 256, 0, G.stream>>>(rowptr, m, segoff); GB_LAUNCHED();
    GB_TRY(dev_exclusive_scan(segoff, m + 1, err));
    int64_t nseg = 0; GB_TRY(read_i64(segoff.get() + m, &nseg, err));
    if (nseg > 0) {
        GB_TRY(segrow.alloc((size_t)nseg, err));
        GB_TRY(pval.alloc((size_t)(nseg * k) * tc_size(zt) + 16, err));
        GB_TRY(ppres.alloc((size_t)(nseg * k), err));
        spmm_seg_fill_kernel<<<grid_for(m), 256, 0, G.stream>>>(segoff, m, segrow); GB_LAUNCHED();
    }
    p.segoff = segoff; p.segrow = segrow; p.pval = pval; p.ppres = ppres;
    p.nitems = m + nseg;
    const int64_t ntile = ceil_div(k, (int64_t)1 << p.gshift);
    const dim3 grid((unsigned)ceil_div(p.nitems << p.gshift, 256), (unsigned)std::min<int64_t>(ntile, 65535));
    bool fast = false;
    if (!spmm_launch(xt, zt, p, grid, &fast))
        return gb_fail(GrB_DOMAIN_MISMATCH, err, "GrB_mxm: unsupported semiring domains (x=%d, z=%d)", xt, zt);
    GB_LAUNCHED();
    gb_kernel_used(fast ? "spmm-fast" : "spmm-generic");
    if (sizeof(OT) == 8) gb_kernel_used("offsets=64");
    if (nseg > 0) {
        spmm_combine(zt, p, nseg); GB_LAUNCHED();
        gb_kernel_used("spmm-split");
    }
    CU_TRY(cudaGetLastError(), err);
    return GrB_SUCCESS;
}
// the wide route (csr_wide: nnz >= 2^32, or B200_debug_wide) reads the 64-bit row offsets; the kernels are otherwise the same
static GrB_Info spmm_product(const Csr &a, const void *aval, const void *xval, const uint8_t *xpres, int64_t k, int xt, int zt, int add, int mul,
                             void *tval, uint8_t *tpres, std::string *err) {
    return csr_wide(a) ? spmm_product_t<int64_t>(a, a.rowptr.get(), aval, xval, xpres, k, xt, zt, add, mul, tval, tpres, err)
                       : spmm_product_t<uint32_t>(a, a.rowptr32.get(), aval, xval, xpres, k, xt, zt, add, mul, tval, tpres, err);
}

// C<Mask> = accum(C, T) for a dense T (m x k).  With no mask or a dense-form mask, C is viewed as a vector of m*k positions and
// the vector write-back runs on it, so C keeps (or takes) the dense form.  A CSR mask sends T through the CSR write-back.
GrB_Info spmm_writeback(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const DescFlags &f,
                        DevBuf<void> &&tval, DevBuf<uint8_t> &&tpres, int zt, std::string *err) {
    const int64_t m = (int64_t)C->nrows, k = (int64_t)C->ncols;
    if (Mask && !Mask->dn.valid) {
        Csr T;
        GB_TRY(dense_to_csr(tval, tpres, m, k, tc_size(zt), T, err));
        tval.reset(); tpres.reset();
        gb_kernel_used("write=csr");
        return matrix_writeback(C, Mask, accum, f, std::move(T), zt, false, err);
    }
    gb_kernel_used("write=dense");
    // C's entries are read only under a mask or an accumulator: its dense form is borrowed, or a CSR C lends its dense image
    GB_Vector_opaque w{};
    w.magic = GB_MAGIC; w.type = C->type; w.n = (uint64_t)(m * k); w.host_valid = true;
    DevBuf<void> cval; DevBuf<uint8_t> cpres;
    if ((Mask || accum) && !matrix_known_empty(C)) {
        if (!C->dn.valid) {
            GB_TRY(matrix_ensure_device(C));
            GB_TRY(csr_to_dense(C->dev, C->type->size, cval, cpres, err));
        }
        w.host_valid = false;
        w.dv = C->dn.valid ? DenseForm::borrow(C->dn.val, C->dn.pres) : DenseForm::borrow(cval, cpres);
    }
    GB_Vector_opaque mv{};
    if (Mask) {
        mv.magic = GB_MAGIC; mv.type = Mask->type; mv.n = (uint64_t)(m * k); mv.host_valid = false;
        mv.dv = DenseForm::borrow(Mask->dn.val, Mask->dn.pres);
    }
    const GrB_Info r = vector_write(&w, Mask ? &mv : nullptr, accum, f, DenseForm{std::move(tval), std::move(tpres)}, zt, false, nullptr);
    if (w.dv.valid && !w.dv.val.borrowed()) matrix_adopt_dense(C, std::move(w.dv));    // the write-back's result: C's dense form
    if (r != GrB_SUCCESS && !w.err.empty()) *err = w.err;
    return r;
}

GrB_Info spmm_mxm(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const GrB_Semiring s, const GrB_Matrix A,
                  const GrB_Matrix B, const DescFlags &f, GbBurble &burble) {
    std::string *err = &C->err;
    const GrB_BinaryOp mulop = s->mul, addop = s->add->op;
    const int xt = mulop->xtype->code, zt = addop->ztype->code, add = addop->opcode, mul = mulop->opcode;
    gb_kernel_used("spmm");
    Csr *pa; GB_TRY(source_csr(A, f.tran0, &pa));
    const Csr &a = *pa;
    const int64_t m = a.nrows, n = a.ncols, k = (int64_t)B->ncols;
    // operands cast to the multiply's input types, as in the CSR path
    DevBuf<void> a_cast, x_cast;
    const void *aval = nullptr, *xval = nullptr;
    GB_TRY(mxm_values(a_cast, &aval, mul_reads_x(mul), xt, a.val, A->type->code, a.nnz, err));
    GB_TRY(mxm_values(x_cast, &xval, mul_reads_y(mul), xt, B->dn.val, B->type->code, n * k, err));
    // T in fresh buffers: C may alias A or X
    DevBuf<void> tval; DevBuf<uint8_t> tpres;
    GB_TRY(tval.alloc((size_t)(m * k) * tc_size(zt) + 16, err));
    GB_TRY(tpres.alloc((size_t)(m * k), err));
    if (m > 0 && k > 0) GB_TRY(spmm_product(a, aval, xval, B->dn.pres, k, xt, zt, add, mul, tval, tpres, err));
    a_cast.reset(); x_cast.reset();
    // algorithmic bytes: A (ids, values, row pointers), X once, T (values and presence)
    const bool wide = csr_wide(a);
    const double bytes = (double)a.nnz * (4 + tc_size(A->type->code)) + (double)(m + 1) * (wide ? 8 : 4) +
                         (double)(n * k) * (tc_size(B->type->code) + (B->dn.pres ? 1 : 0)) + (double)(m * k) * (tc_size(zt) + 1);
    burble.note(wide ? "spmm, 64-bit offsets" : "spmm", bytes);
    return spmm_writeback(C, Mask, accum, f, std::move(tval), std::move(tpres), zt, err);
}

int op_mirror(int op) {
    switch (op) {
        case OP_FIRST: return OP_SECOND;   case OP_SECOND: return OP_FIRST;
        case OP_ANY: return OP_FIRST;      // the device's ANY returns y, op(B)'s value: FIRST of the swapped operands
        case OP_MINUS: return OP_RMINUS;   case OP_RMINUS: return OP_MINUS;
        case OP_DIV: return OP_RDIV;       case OP_RDIV: return OP_DIV;
        case OP_ISGT: return OP_ISLT;      case OP_ISLT: return OP_ISGT;
        case OP_ISGE: return OP_ISLE;      case OP_ISLE: return OP_ISGE;
        case OP_GT: return OP_LT;          case OP_LT: return OP_GT;
        case OP_GE: return OP_LE;          case OP_LE: return OP_GE;
        case OP_TIMES: case OP_PLUS: case OP_PAIR: case OP_MIN: case OP_MAX: case OP_ISEQ: case OP_ISNE: case OP_EQ: case OP_NE:
        case OP_LOR: case OP_LAND: case OP_LXOR: case OP_BOR: case OP_BAND: case OP_BXOR: case OP_BXNOR: return op;
        default: return -1;                // POW, positional, user-defined
    }
}

// C<Mask> = accum(C, X (+).(x) op(B)) for a dense-form X = op(A) (k x n), as C' = op(B)' (+).(x)' X' on the kernel above, where
// (x)' is the multiply with its operands swapped.  op(B)' is B's cached transpose, or B's own CSR under INP1 = TRAN; X' (n x k) is
// A's dense form itself under INP0 = TRAN (or when k = 1), else its dense transpose, built per call.  T' (m x k) is transposed into
// T (k x m) in fresh buffers (C may alias A or B), unless m = 1, and T goes through the right route's write-back.
GrB_Info spmm_left_mxm(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const GrB_Semiring s, const GrB_Matrix A,
                       const GrB_Matrix B, const DescFlags &f, GbBurble &burble) {
    std::string *err = &C->err;
    const GrB_BinaryOp mulop = s->mul, addop = s->add->op;
    const int xt = mulop->xtype->code, zt = addop->ztype->code, add = addop->opcode, mul = op_mirror(mulop->opcode);
    gb_kernel_used("spmm");
    gb_kernel_used("spmm-left");
    if (f.tran1) GB_TRY(matrix_ensure_device(B)); else GB_TRY(matrix_ensure_transpose(B));
    const Csr &b = f.tran1 ? B->dev : B->devT;
    const int64_t m = b.nrows, n = b.ncols, k = (int64_t)(f.tran0 ? A->ncols : A->nrows);
    // operands cast to the multiply's input types, as in the CSR path: op(B)' takes the swapped multiply's x, X its y
    DevBuf<void> b_cast, x_cast;
    const void *bval = nullptr, *xval = nullptr;
    const uint8_t *xpres = A->dn.pres;
    GB_TRY(mxm_values(b_cast, &bval, mul_reads_x(mul), xt, b.val, B->type->code, b.nnz, err));
    GB_TRY(mxm_values(x_cast, &xval, mul_reads_y(mul), xt, A->dn.val, A->type->code, n * k, err));
    // X' (n x k): the row-major k x n form transposed, unless A already is n x k (INP0 = TRAN) or k = 1
    const bool xtr = !f.tran0 && k > 1;
    const size_t bx = mul_reads_y(mul) ? tc_size(xt) : tc_size(A->type->code);
    DevBuf<void> xtval; DevBuf<uint8_t> xtpres;
    if (xtr) {
        GB_TRY(xtval.alloc((size_t)(n * k) * bx + 16, err));
        if (xpres) GB_TRY(xtpres.alloc((size_t)(n * k), err));
        GB_TRY(dense_transpose(xval, xpres, k, n, bx, xtval, xtpres, err));
        x_cast.reset();
        xval = xtval; xpres = xtpres;
        gb_kernel_used("x-transpose");
    }
    // T' (m x k), then T (k x m); both in fresh buffers
    DevBuf<void> tval; DevBuf<uint8_t> tpres;
    GB_TRY(tval.alloc((size_t)(m * k) * tc_size(zt) + 16, err));
    GB_TRY(tpres.alloc((size_t)(m * k), err));
    if (m > 0 && k > 0) GB_TRY(spmm_product(b, bval, xval, xpres, k, xt, zt, add, mul, tval, tpres, err));
    b_cast.reset(); x_cast.reset(); xtval.reset(); xtpres.reset();
    if (m > 1) {
        DevBuf<void> uval; DevBuf<uint8_t> upres;
        GB_TRY(uval.alloc((size_t)(m * k) * tc_size(zt) + 16, err));
        GB_TRY(upres.alloc((size_t)(m * k), err));
        GB_TRY(dense_transpose(tval, tpres, m, k, tc_size(zt), uval, upres, err));
        tval = std::move(uval); tpres = std::move(upres);
        gb_kernel_used("t-transpose");
    }
    // algorithmic bytes: the right route's (op(B)', X once, T), plus the transposes (each reads and writes its array)
    const double xb = (double)(n * k) * (tc_size(A->type->code) + (A->dn.pres ? 1 : 0)), tb = (double)(m * k) * (tc_size(zt) + 1);
    const bool wide = csr_wide(b);
    const double bytes = (double)b.nnz * (4 + tc_size(B->type->code)) + (double)(m + 1) * (wide ? 8 : 4) + xb + tb + (xtr ? 2 * xb : 0.0) +
                         (m > 1 ? 2 * tb : 0.0);
    burble.note(wide ? "spmm-left, 64-bit offsets" : "spmm-left", bytes);
    return spmm_writeback(C, Mask, accum, f, std::move(tval), std::move(tpres), zt, err);
}
