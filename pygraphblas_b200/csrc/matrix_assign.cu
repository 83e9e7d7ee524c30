// matrix_assign.cu -- sub-matrix assignment and extraction on the device (SURVEY.md section 8(b) / 8(f)3):
//
//   GrB_Matrix_assign_<T>   C<Mask>(I,J) = accum(C(I,J), x)     reference: pygraphblas/matrix.py:3106-3238 (assign_scalar;
//                                                               Matrix.dense :183 -> :179, used by tests/test_matrix.py:858-864 test_pow)
//   GrB_Matrix_extract      C<Mask> = accum(C, A(I,J))          matrix.py:2807-2860 (extract_matrix, M[0:1, :] slices)
//   GrB_Matrix_assign       C<Mask>(I,J) = accum(C(I,J), A)     matrix.py:3057-3104 (assign_matrix)
//   GrB_Col_extract / GrB_Row_assign / GrB_Col_assign           matrix.py:2862-2897, 3005-3031
//   GxB_Matrix_diag / GxB_Vector_diag                           matrix.py:2202-2236 / vector.py diag
//   GrB_Matrix_kronecker_BinaryOp                               matrix.py:2739-2805
//
// Every operation forms T (a CSR in HBM) with one or two streaming kernels and hands it to the common write-back
// C<Mask> = accum(C, T) of spgemm.cu.  GrB_assign semantics (C API 1.3 section 4.3.7): the result Z is C with the
// region I x J replaced by T (no accumulator: entries of C inside the region that T lacks are deleted) or merged with
// it (accumulator), and only then the mask -- which spans all of C -- and GrB_REPLACE apply.
// Index lists (GrB_ALL, explicit, GxB_RANGE / STRIDE / BACKWARDS as reference: pygraphblas/base.py:216-252 builds
// them) are expanded on the host: they are call arguments, not data.  Nothing here computes values on the host.
#include "common.cuh"
#include <algorithm>
#include <vector>
#include "../../include/b200grb_compat.h"

static inline int agrid(int64_t n, int threads = 256) { return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n, threads), (int64_t)G.num_sms * 16)); }

GrB_Info index_list(const GrB_Index *I, GrB_Index ni, uint64_t dim, bool *all, std::vector<uint64_t> &out, std::string *err, const char *fn);   // vector_ops.cu
extern "C" GrB_Info GrB_Matrix_dup(GrB_Matrix *C, const GrB_Matrix A);
extern "C" GrB_Info GrB_Matrix_free(GrB_Matrix *A);
extern "C" GrB_Info GrB_Matrix_new(GrB_Matrix *A, GrB_Type type, GrB_Index nrows, GrB_Index ncols);

static GrB_BinaryOp second_op(int tc) {
    switch (tc) {
        case TC_BOOL: return GrB_SECOND_BOOL;     case TC_INT8: return GrB_SECOND_INT8;     case TC_INT16: return GrB_SECOND_INT16;
        case TC_INT32: return GrB_SECOND_INT32;   case TC_INT64: return GrB_SECOND_INT64;   case TC_UINT8: return GrB_SECOND_UINT8;
        case TC_UINT16: return GrB_SECOND_UINT16; case TC_UINT32: return GrB_SECOND_UINT32; case TC_UINT64: return GrB_SECOND_UINT64;
        case TC_FP32: return GrB_SECOND_FP32;     default: return GrB_SECOND_FP64;
    }
}

template <typename T> static GrB_Info upload(const std::vector<T> &h, DevBuf<T> &d, std::string *err) {
    GB_TRY(d.alloc(h.size(), err));
    if (!h.empty()) CU_TRY(cudaMemcpyAsync(d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice, G.stream), err);
    CU_TRY(cudaStreamSynchronize(G.stream), err);          // h is a caller-owned temporary
    return GrB_SUCCESS;
}
static GrB_Info read_i64(const int64_t *d, int64_t *h, std::string *err) {
    CU_TRY(cudaMemcpyAsync(h, d, 8, cudaMemcpyDeviceToHost, G.stream), err);
    CU_TRY(cudaStreamSynchronize(G.stream), err);
    return GrB_SUCCESS;
}

// ------------------------------------------------------------------ the region I x J of a matrix
struct Region {
    bool all_rows = true, all_cols = true;
    std::vector<uint64_t> I, J;          // as given (after expansion), empty when all
    DevBuf<uint8_t> rowflag;             // [nrows] 1 where the row is in I   (NULL: every row)
    DevBuf<uint8_t> colflag;             // [ncols] 1 where the column is in J (NULL: every column)
    DevBuf<uint32_t> jsorted;            // sorted distinct columns of J        (NULL: 0..ncols-1)
    int64_t nj_distinct = 0, ni_distinct = 0;
};
__global__ void flag_kernel(const uint64_t *idx, int64_t k, uint8_t *flag) {
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < k; q += (int64_t)gridDim.x * blockDim.x) flag[idx[q]] = 1;
}
static GrB_Info region_build(Region &R, const GrB_Index *I, GrB_Index ni, const GrB_Index *J, GrB_Index nj, uint64_t nrows, uint64_t ncols,
                             std::string *err, const char *fn) {
    GB_TRY(index_list(I, ni, nrows, &R.all_rows, R.I, err, fn));
    GB_TRY(index_list(J, nj, ncols, &R.all_cols, R.J, err, fn));
    R.ni_distinct = (int64_t)nrows; R.nj_distinct = (int64_t)ncols;
    if (!R.all_rows) {
        std::vector<uint64_t> s(R.I); std::sort(s.begin(), s.end()); s.erase(std::unique(s.begin(), s.end()), s.end());
        R.ni_distinct = (int64_t)s.size();
        DevBuf<uint64_t> d; GB_TRY(upload(s, d, err));
        GB_TRY(R.rowflag.alloc((size_t)nrows, err));
        CU_TRY(cudaMemsetAsync(R.rowflag, 0, (size_t)nrows, G.stream), err);
        if (!s.empty()) { flag_kernel<<<agrid((int64_t)s.size()), 256, 0, G.stream>>>(d, (int64_t)s.size(), R.rowflag); GB_LAUNCHED(); }
    }
    if (!R.all_cols) {
        std::vector<uint64_t> s(R.J); std::sort(s.begin(), s.end()); s.erase(std::unique(s.begin(), s.end()), s.end());
        R.nj_distinct = (int64_t)s.size();
        std::vector<uint32_t> s32(s.begin(), s.end());
        GB_TRY(upload(s32, R.jsorted, err));
        DevBuf<uint64_t> d; GB_TRY(upload(s, d, err));
        GB_TRY(R.colflag.alloc((size_t)ncols, err));
        CU_TRY(cudaMemsetAsync(R.colflag, 0, (size_t)ncols, G.stream), err);
        if (!s.empty()) { flag_kernel<<<agrid((int64_t)s.size()), 256, 0, G.stream>>>(d, (int64_t)s.size(), R.colflag); GB_LAUNCHED(); }
    }
    return GrB_SUCCESS;
}

// ------------------------------------------------------------------ T = the region filled with one value
__global__ void fill_count_kernel(const uint8_t *rowflag, int64_t nrows, int64_t per_row, int64_t *rowptr) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r <= nrows; r += (int64_t)gridDim.x * blockDim.x)
        rowptr[r] = (r < nrows && (!rowflag || rowflag[r])) ? per_row : 0;
}
__global__ void fill_entries_kernel(const int64_t *rowptr, int64_t nrows, const uint32_t *jsorted, uint32_t *col, void *val, int tc, Sc x) {
    // one warp per row
    const int lane = threadIdx.x & 31;
    for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < nrows; r += ((int64_t)gridDim.x * blockDim.x) >> 5) {
        const int64_t b = rowptr[r], e = rowptr[r + 1];
        for (int64_t k = b + lane; k < e; k += 32) { col[k] = jsorted ? jsorted[k - b] : (uint32_t)(k - b); sc_store(tc, val, (size_t)k, x); }
    }
}
static GrB_Info region_filled(const Region &R, int64_t nrows, int64_t ncols, int tc, Sc x, Csr &T, std::string *err) {
    T = Csr(); T.nrows = nrows; T.ncols = ncols;
    GB_TRY(T.rowptr.alloc((size_t)nrows + 1, err));
    fill_count_kernel<<<agrid(nrows + 1), 256, 0, G.stream>>>(R.rowflag, nrows, R.nj_distinct, T.rowptr); GB_LAUNCHED();
    GB_TRY(dev_exclusive_scan(T.rowptr, nrows + 1, err));
    T.nnz = R.ni_distinct * R.nj_distinct;
    GB_TRY(T.col.alloc((size_t)T.nnz, err));
    GB_TRY(T.val.alloc((size_t)T.nnz * tc_size(tc) + 16, err));
    if (T.nnz > 0) { fill_entries_kernel<<<agrid(nrows * 32), 256, 0, G.stream>>>(T.rowptr, nrows, R.jsorted, T.col, T.val, tc, x); GB_LAUNCHED(); }
    GB_TRY(dev_build_rowptr32(T, err));
    CU_TRY(cudaGetLastError(), err);
    return GrB_SUCCESS;
}

// ------------------------------------------------------------------ C minus the region (entries of C outside I x J)
__global__ void outside_count_kernel(const int64_t *ptr, const uint32_t *col, int64_t nrows, const uint8_t *rowflag, const uint8_t *colflag, int64_t *cnt) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r <= nrows; r += (int64_t)gridDim.x * blockDim.x) {
        int64_t c = 0;
        if (r < nrows) {
            const bool rin = !rowflag || rowflag[r];
            for (int64_t k = ptr[r]; k < ptr[r + 1]; ++k) c += !(rin && (!colflag || colflag[col[k]]));
        }
        cnt[r] = c;
    }
}
__global__ void outside_fill_kernel(const int64_t *ptr, const uint32_t *col, const uint8_t *val, int vsize, int64_t nrows, const uint8_t *rowflag,
                                    const uint8_t *colflag, const int64_t *optr, uint32_t *ocol, uint8_t *oval) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += (int64_t)gridDim.x * blockDim.x) {
        const bool rin = !rowflag || rowflag[r];
        int64_t o = optr[r];
        for (int64_t k = ptr[r]; k < ptr[r + 1]; ++k) if (!(rin && (!colflag || colflag[col[k]]))) {
            ocol[o] = col[k];
            for (int b = 0; b < vsize; ++b) oval[o * vsize + b] = val[k * vsize + b];
            ++o;
        }
    }
}
static GrB_Info csr_outside_region(const Csr &c, size_t vsize, const Region &R, Csr &out, std::string *err) {
    out = Csr(); out.nrows = c.nrows; out.ncols = c.ncols;
    GB_TRY(out.rowptr.alloc((size_t)c.nrows + 1, err));
    outside_count_kernel<<<agrid(c.nrows + 1), 256, 0, G.stream>>>(c.rowptr, c.col, c.nrows, R.rowflag, R.colflag, out.rowptr); GB_LAUNCHED();
    GB_TRY(dev_exclusive_scan(out.rowptr, c.nrows + 1, err));
    GB_TRY(read_i64(out.rowptr + c.nrows, &out.nnz, err));
    GB_TRY(out.col.alloc((size_t)out.nnz, err));
    GB_TRY(out.val.alloc((size_t)out.nnz * vsize + 16, err));
    if (out.nnz > 0) {
        outside_fill_kernel<<<agrid(c.nrows), 256, 0, G.stream>>>(c.rowptr, c.col, (const uint8_t *)c.val, (int)vsize, c.nrows, R.rowflag, R.colflag,
                                                                  out.rowptr, out.col, (uint8_t *)out.val); GB_LAUNCHED();
    }
    GB_TRY(dev_build_rowptr32(out, err));
    CU_TRY(cudaGetLastError(), err);
    return GrB_SUCCESS;
}

// ------------------------------------------------------------------ GrB_assign write-back:  C<Mask>(region) = accum(C(region), T)
// T is a CSR of C's dimensions holding the new content of the region (type ttc); consumed.
// t_covers_region: T has an entry at every position of the region (scalar fill), so nothing needs deleting first.
static GrB_Info assign_writeback(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const DescFlags &f, const Region &R,
                                 Csr &&T, int ttc, bool t_covers_region, std::string *err) {
    const int ctc = C->type->code;
    if (!Mask && f.mask_comp) return matrix_writeback(C, nullptr, accum, f, std::move(T), ttc, false, err);     // nothing is let through
    DescFlags plain{}; plain.replace = false; plain.mask_comp = false; plain.mask_struct = false; plain.tran0 = plain.tran1 = false; plain.axb = f.axb;
    const GrB_BinaryOp merge = accum ? accum : second_op(ctc);
    const bool whole = R.all_rows && R.all_cols;
    // Z = C with the region replaced by / merged with T, built in a scratch matrix unless it can go straight into C
    GrB_Matrix Zm = C;
    if (Mask) GB_TRY(GrB_Matrix_dup(&Zm, C));
    GrB_Info r = GrB_SUCCESS;
    if (!accum && !t_covers_region && !whole) {
        // entries of C inside the region that T lacks are deleted: drop the region from C first
        r = matrix_ensure_device(Zm);
        if (r == GrB_SUCCESS && Zm->dev.nnz > 0) {
            Csr keep;
            r = csr_outside_region(Zm->dev, Zm->type->size, R, keep, err);
            if (r == GrB_SUCCESS) matrix_adopt_device(Zm, std::move(keep));
        }
    }
    if (r == GrB_SUCCESS) {
        if (!accum && whole) r = matrix_writeback(Zm, nullptr, nullptr, plain, std::move(T), ttc, false, err);        // Z = T
        else r = matrix_writeback(Zm, nullptr, merge, plain, std::move(T), ttc, false, err);                          // Z = C (+) T
    }
    if (!Mask || r != GrB_SUCCESS) { if (Zm != C) GrB_Matrix_free(&Zm); return r; }
    // C<Mask> = Z  (mask and GrB_REPLACE span all of C)
    r = matrix_ensure_device(Zm);
    if (r == GrB_SUCCESS) {
        Csr z = std::move(Zm->dev); Zm->host_valid = true;      // steal Z's CSR (values already of C's type)
        r = matrix_writeback(C, Mask, nullptr, f, std::move(z), ctc, false, err);
    }
    GrB_Matrix_free(&Zm);
    return r;
}

static GrB_Info matrix_assign_scalar(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, Sc x, int xtc, const GrB_Index *I, GrB_Index ni,
                                     const GrB_Index *J, GrB_Index nj, const GrB_Descriptor desc, const char *fn) {
    GB_LOCK; GB_CHECK_INIT;
    if (!C) return gb_fail(GrB_NULL_POINTER, nullptr, "%s: NULL argument", fn);
    if (!gb_valid_matrix(C) || (Mask && !gb_valid_matrix(Mask))) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "%s: invalid object", fn);
    std::string *err = &C->err;
    if (accum && accum->opcode == OP_USER) return gb_fail(GrB_INVALID_VALUE, err, "%s: user-defined accumulators are host function pointers and cannot run on the GPU", fn);
    if (Mask && (Mask->nrows != C->nrows || Mask->ncols != C->ncols)) return gb_fail(GrB_DIMENSION_MISMATCH, err, "%s: the mask must have C's dimensions", fn);
    if (!G.have_device) return gb_fail(GrB_PANIC, err, "%s: no CUDA device: libb200grb computes only on the GPU (no CPU fallback)", fn);
    if (C->nrows >= ((uint64_t)1 << 31) || C->ncols >= ((uint64_t)1 << 31)) return gb_fail(GrB_INVALID_VALUE, err, "%s: dimensions beyond 2^31 cannot be filled", fn);
    GbBurble burble(fn);
    const DescFlags f = desc_flags(desc);
    Region R;
    GB_TRY(region_build(R, I, ni, J, nj, C->nrows, C->ncols, err, fn));
    if ((double)R.ni_distinct * (double)R.nj_distinct >= 4.0e9) return gb_fail(GrB_OUT_OF_MEMORY, err, "%s: the filled region would hold >= 4e9 entries", fn);
    Csr T;
    GB_TRY(region_filled(R, (int64_t)C->nrows, (int64_t)C->ncols, xtc, x, T, err));
    burble.note("region fill + write-back", (double)T.nnz * (4 + tc_size(xtc)));
    return assign_writeback(C, Mask, accum, f, R, std::move(T), xtc, /*t_covers_region=*/true, err);
}

#define GB_MASSIGN(TN, CT, TC, FIELD) \
    extern "C" GrB_Info GrB_Matrix_assign_##TN(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, CT x, const GrB_Index *I, GrB_Index ni, \
                                               const GrB_Index *J, GrB_Index nj, const GrB_Descriptor desc) { \
        Sc s; s.u = 0; s.FIELD = x; return matrix_assign_scalar(C, Mask, accum, s, TC, I, ni, J, nj, desc, "GrB_Matrix_assign_" #TN); }
GB_MASSIGN(BOOL, bool, TC_BOOL, u) GB_MASSIGN(INT8, int8_t, TC_INT8, i) GB_MASSIGN(INT16, int16_t, TC_INT16, i) GB_MASSIGN(INT32, int32_t, TC_INT32, i)
GB_MASSIGN(INT64, int64_t, TC_INT64, i) GB_MASSIGN(UINT8, uint8_t, TC_UINT8, u) GB_MASSIGN(UINT16, uint16_t, TC_UINT16, u) GB_MASSIGN(UINT32, uint32_t, TC_UINT32, u)
GB_MASSIGN(UINT64, uint64_t, TC_UINT64, u) GB_MASSIGN(FP32, float, TC_FP32, d) GB_MASSIGN(FP64, double, TC_FP64, d)
#undef GB_MASSIGN

// ================================================================== GrB_Matrix_extract:  C<Mask> = accum(C, op(A)(I,J))
// T(p, q) = A'(I[p], J[q]).  Rows are gathered by I; columns are mapped through J sorted by value (a column that J names
// several times appears several times); when J is not ascending the rows of T are sorted by column afterwards.
__global__ void extract_count_kernel(const uint32_t *rows, int64_t ni, const int64_t *a_ptr, const uint32_t *a_col,
                                     const uint32_t *jsv, int64_t njs, int64_t *cnt) {
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p <= ni; p += (int64_t)gridDim.x * blockDim.x) {
        int64_t c = 0;
        if (p < ni) {
            const int64_t r = rows ? rows[p] : p;
            if (!jsv) c = a_ptr[r + 1] - a_ptr[r];
            else for (int64_t k = a_ptr[r]; k < a_ptr[r + 1]; ++k) {
                const uint32_t col = a_col[k];
                int64_t lo = 0, hi = njs;
                while (lo < hi) { const int64_t mid = (lo + hi) >> 1; if (jsv[mid] < col) lo = mid + 1; else hi = mid; }
                while (lo < njs && jsv[lo] == col) { ++c; ++lo; }
            }
        }
        cnt[p] = c;
    }
}
__global__ void extract_fill_kernel(const uint32_t *rows, int64_t ni, const int64_t *a_ptr, const uint32_t *a_col, const uint8_t *a_val, int vsize,
                                    const uint32_t *jsv, const uint32_t *jsq, int64_t njs, const int64_t *t_ptr, uint32_t *t_col, uint8_t *t_val) {
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < ni; p += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = rows ? rows[p] : p;
        int64_t o = t_ptr[p];
        for (int64_t k = a_ptr[r]; k < a_ptr[r + 1]; ++k) {
            const uint32_t col = a_col[k];
            if (!jsv) { t_col[o] = col; for (int b = 0; b < vsize; ++b) t_val[o * vsize + b] = a_val[k * vsize + b]; ++o; continue; }
            int64_t lo = 0, hi = njs;
            while (lo < hi) { const int64_t mid = (lo + hi) >> 1; if (jsv[mid] < col) lo = mid + 1; else hi = mid; }
            while (lo < njs && jsv[lo] == col) {
                t_col[o] = jsq[lo]; for (int b = 0; b < vsize; ++b) t_val[o * vsize + b] = a_val[k * vsize + b];
                ++o; ++lo;
            }
        }
    }
}
// sort each row's (column, value) pairs by column: the rows here are short lists produced by an unsorted J
__global__ void rows_insertion_sort_kernel(const int64_t *t_ptr, int64_t nrows, uint32_t *t_col, uint8_t *t_val, int vsize) {
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < nrows; p += (int64_t)gridDim.x * blockDim.x) {
        const int64_t b = t_ptr[p], e = t_ptr[p + 1];
        for (int64_t x = b + 1; x < e; ++x) {
            const uint32_t c = t_col[x]; uint8_t v[8];
            for (int q = 0; q < vsize; ++q) v[q] = t_val[x * vsize + q];
            int64_t y = x - 1;
            while (y >= b && t_col[y] > c) { t_col[y + 1] = t_col[y]; for (int q = 0; q < vsize; ++q) t_val[(y + 1) * vsize + q] = t_val[y * vsize + q]; --y; }
            t_col[y + 1] = c; for (int q = 0; q < vsize; ++q) t_val[(y + 1) * vsize + q] = v[q];
        }
    }
}

extern "C" GrB_Info GrB_Matrix_extract(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const GrB_Matrix A, const GrB_Index *I, GrB_Index ni,
                                       const GrB_Index *J, GrB_Index nj, const GrB_Descriptor desc) {
    GB_LOCK; GB_CHECK_INIT;
    const char *fn = "GrB_Matrix_extract";
    if (!C || !A) return gb_fail(GrB_NULL_POINTER, nullptr, "%s: NULL argument", fn);
    if (!gb_valid_matrix(C) || !gb_valid_matrix(A) || (Mask && !gb_valid_matrix(Mask))) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "%s: invalid object", fn);
    std::string *err = &C->err;
    if (accum && accum->opcode == OP_USER) return gb_fail(GrB_INVALID_VALUE, err, "%s: user-defined accumulators cannot run on the GPU", fn);
    const DescFlags f = desc_flags(desc);
    const uint64_t an = f.tran0 ? A->ncols : A->nrows, am = f.tran0 ? A->nrows : A->ncols;
    bool all_i, all_j; std::vector<uint64_t> Iv, Jv;
    GB_TRY(index_list(I, ni, an, &all_i, Iv, err, fn));
    GB_TRY(index_list(J, nj, am, &all_j, Jv, err, fn));
    const uint64_t tn = all_i ? an : Iv.size(), tm = all_j ? am : Jv.size();
    if (C->nrows != tn || C->ncols != tm || (Mask && (Mask->nrows != tn || Mask->ncols != tm)))
        return gb_fail(GrB_DIMENSION_MISMATCH, err, "%s: C is %llux%llu, the index lists select %llux%llu", fn, (unsigned long long)C->nrows,
                       (unsigned long long)C->ncols, (unsigned long long)tn, (unsigned long long)tm);
    if (!G.have_device) return gb_fail(GrB_PANIC, err, "%s: no CUDA device: libb200grb computes only on the GPU (no CPU fallback)", fn);
    GbBurble burble(fn);
    if (f.tran0) GB_TRY(matrix_ensure_transpose(A)); else GB_TRY(matrix_ensure_device(A));
    const Csr &a = f.tran0 ? A->devT : A->dev;
    const size_t vsize = A->type->size;
    DevBuf<uint32_t> d_rows, d_jsv, d_jsq;
    bool need_sort = false;
    if (!all_i) { std::vector<uint32_t> r32(Iv.begin(), Iv.end()); GB_TRY(upload(r32, d_rows, err)); }
    if (!all_j) {
        std::vector<uint32_t> ord(Jv.size());
        for (size_t q = 0; q < ord.size(); ++q) ord[q] = (uint32_t)q;
        std::stable_sort(ord.begin(), ord.end(), [&](uint32_t x, uint32_t y) { return Jv[x] < Jv[y]; });
        std::vector<uint32_t> jsv(ord.size());
        for (size_t q = 0; q < ord.size(); ++q) { jsv[q] = (uint32_t)Jv[ord[q]]; if (ord[q] != q) need_sort = true; }
        GB_TRY(upload(jsv, d_jsv, err)); GB_TRY(upload(ord, d_jsq, err));
    }
    Csr T; T.nrows = (int64_t)tn; T.ncols = (int64_t)tm;
    GB_TRY(T.rowptr.alloc((size_t)tn + 1, err));
    extract_count_kernel<<<agrid((int64_t)tn + 1), 256, 0, G.stream>>>(d_rows, (int64_t)tn, a.rowptr, a.col, d_jsv, (int64_t)Jv.size(), T.rowptr); GB_LAUNCHED();
    GB_TRY(dev_exclusive_scan(T.rowptr, (int64_t)tn + 1, err));
    GB_TRY(read_i64(T.rowptr + tn, &T.nnz, err));
    GB_TRY(T.col.alloc((size_t)T.nnz, err));
    GB_TRY(T.val.alloc((size_t)T.nnz * vsize + 16, err));
    if (T.nnz > 0) {
        extract_fill_kernel<<<agrid((int64_t)tn), 256, 0, G.stream>>>(d_rows, (int64_t)tn, a.rowptr, a.col, (const uint8_t *)a.val, (int)vsize, d_jsv, d_jsq,
                                                                    (int64_t)Jv.size(), T.rowptr, T.col, (uint8_t *)T.val); GB_LAUNCHED();
        if (need_sort) { rows_insertion_sort_kernel<<<agrid((int64_t)tn), 256, 0, G.stream>>>(T.rowptr, (int64_t)tn, T.col, (uint8_t *)T.val, (int)vsize); GB_LAUNCHED(); }
    }
    GB_TRY(dev_build_rowptr32(T, err));
    d_rows.reset(); d_jsv.reset(); d_jsq.reset();
    burble.note("row gather + column map", (double)T.nnz * (4 + vsize) * 2);
    return matrix_writeback(C, Mask, accum, f, std::move(T), A->type->code, false, err);
}

// ================================================================== GxB_Matrix_diag / GxB_Vector_diag
__global__ void diag_build_kernel(const uint8_t *pres, int64_t n, int64_t k, int64_t dim, int64_t *rowptr_cnt) {
    // row of entry i of v: i (k >= 0) or i - k (k < 0)
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r <= dim; r += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = k >= 0 ? r : r + k;
        rowptr_cnt[r] = (r < dim && i >= 0 && i < n && (!pres || pres[i])) ? 1 : 0;
    }
}
__global__ void diag_fill_kernel(const uint8_t *vval, int vsize, int64_t n, int64_t k, int64_t dim, const int64_t *rowptr, uint32_t *col, uint8_t *val) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < dim; r += (int64_t)gridDim.x * blockDim.x) {
        if (rowptr[r + 1] > rowptr[r]) {
            const int64_t i = k >= 0 ? r : r + k, o = rowptr[r];
            col[o] = (uint32_t)(k >= 0 ? i + k : i);
            for (int b = 0; b < vsize; ++b) val[o * vsize + b] = vval[i * vsize + b];
        }
    }
}
extern "C" GrB_Info GxB_Matrix_diag(GrB_Matrix C, const GrB_Vector v, int64_t k, const GrB_Descriptor desc) {
    (void)desc; GB_LOCK; GB_CHECK_INIT;
    const char *fn = "GxB_Matrix_diag";
    if (!C || !v) return gb_fail(GrB_NULL_POINTER, nullptr, "%s: NULL argument", fn);
    if (!gb_valid_matrix(C) || !gb_valid_vector(v)) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "%s: invalid object", fn);
    std::string *err = &C->err;
    const uint64_t dim = v->n + (uint64_t)(k >= 0 ? k : -k);
    if (C->nrows != dim || C->ncols != dim) return gb_fail(GrB_DIMENSION_MISMATCH, err, "%s: C must be %llux%llu", fn, (unsigned long long)dim, (unsigned long long)dim);
    if (!G.have_device) return gb_fail(GrB_PANIC, err, "%s: no CUDA device: libb200grb computes only on the GPU (no CPU fallback)", fn);
    if (dim >= ((uint64_t)1 << 31)) return gb_fail(GrB_INVALID_VALUE, err, "%s: dimensions beyond 2^31 are not supported in HBM", fn);
    GB_TRY(vector_ensure_device(v));
    const size_t vsize = v->type->size;
    Csr T; T.nrows = T.ncols = (int64_t)dim;
    GB_TRY(T.rowptr.alloc((size_t)dim + 1, err));
    diag_build_kernel<<<agrid((int64_t)dim + 1), 256, 0, G.stream>>>(v->dpres, (int64_t)v->n, k, (int64_t)dim, T.rowptr); GB_LAUNCHED();
    GB_TRY(dev_exclusive_scan(T.rowptr, (int64_t)dim + 1, err));
    GB_TRY(read_i64(T.rowptr + dim, &T.nnz, err));
    GB_TRY(T.col.alloc((size_t)T.nnz, err));
    GB_TRY(T.val.alloc((size_t)T.nnz * vsize + 16, err));
    if (T.nnz > 0) { diag_fill_kernel<<<agrid((int64_t)dim), 256, 0, G.stream>>>((const uint8_t *)v->dval, (int)vsize, (int64_t)v->n, k, (int64_t)dim, T.rowptr, T.col, (uint8_t *)T.val); GB_LAUNCHED(); }
    GB_TRY(dev_build_rowptr32(T, err));
    DescFlags plain{};
    return matrix_writeback(C, nullptr, nullptr, plain, std::move(T), v->type->code, false, err);
}
__global__ void diag_extract_kernel(const int64_t *a_ptr, const uint32_t *a_col, const uint8_t *a_val, int vsize, int64_t nrows, int64_t ncols, int64_t k, int64_t n,
                                    uint8_t *oval, uint8_t *opres) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = k >= 0 ? i : i - k, c = k >= 0 ? i + k : i;
        uint8_t has = 0;
        if (r < nrows && c < ncols) {
            int64_t lo = a_ptr[r], hi = a_ptr[r + 1];
            while (lo < hi) { const int64_t mid = (lo + hi) >> 1; if (a_col[mid] < (uint32_t)c) lo = mid + 1; else hi = mid; }
            if (lo < a_ptr[r + 1] && a_col[lo] == (uint32_t)c) { has = 1; for (int b = 0; b < vsize; ++b) oval[i * vsize + b] = a_val[lo * vsize + b]; }
        }
        opres[i] = has;
    }
}
extern "C" GrB_Info GxB_Vector_diag(GrB_Vector v, const GrB_Matrix A, int64_t k, const GrB_Descriptor desc) {
    (void)desc; GB_LOCK; GB_CHECK_INIT;
    const char *fn = "GxB_Vector_diag";
    if (!v || !A) return gb_fail(GrB_NULL_POINTER, nullptr, "%s: NULL argument", fn);
    if (!gb_valid_matrix(A) || !gb_valid_vector(v)) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "%s: invalid object", fn);
    std::string *err = &v->err;
    // length of diagonal k of an nrows x ncols matrix
    const int64_t nr = (int64_t)A->nrows, nc = (int64_t)A->ncols;
    const int64_t len = k >= 0 ? std::max<int64_t>(0, std::min(nr, nc - k)) : std::max<int64_t>(0, std::min(nr + k, nc));
    if ((int64_t)v->n != len) return gb_fail(GrB_DIMENSION_MISMATCH, err, "%s: v must have %lld positions", fn, (long long)len);
    if (!G.have_device) return gb_fail(GrB_PANIC, err, "%s: no CUDA device: libb200grb computes only on the GPU (no CPU fallback)", fn);
    GB_TRY(matrix_ensure_device(A));
    const size_t vsize = A->type->size;
    DevBuf<void> oval; DevBuf<uint8_t> opres;
    GB_TRY(oval.alloc((size_t)len * vsize + 16, err));
    GB_TRY(opres.alloc((size_t)len, err));
    CU_TRY(cudaMemsetAsync(oval, 0, (size_t)len * vsize, G.stream), err);
    if (len > 0) { diag_extract_kernel<<<agrid(len), 256, 0, G.stream>>>(A->dev.rowptr, A->dev.col, (const uint8_t *)A->dev.val, (int)vsize, nr, nc, k, len, (uint8_t *)oval, opres); GB_LAUNCHED(); }
    DescFlags plain{};
    return vector_write(v, nullptr, nullptr, plain, oval, opres, A->type->code, false, nullptr, std::move(oval), std::move(opres));
}

// ================================================================== GrB_Matrix_kronecker_BinaryOp:  C<Mask> = accum(C, kron(op(A), op(B)))
__global__ void kron_count_kernel(const int64_t *a_ptr, const int64_t *b_ptr, int64_t am, int64_t bm, int64_t *cnt) {
    const int64_t n = am * bm;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r <= n; r += (int64_t)gridDim.x * blockDim.x)
        cnt[r] = r < n ? (a_ptr[r / bm + 1] - a_ptr[r / bm]) * (b_ptr[r % bm + 1] - b_ptr[r % bm]) : 0;
}
__global__ void kron_fill_kernel(const int64_t *a_ptr, const uint32_t *a_col, const void *a_val, int atc, const int64_t *b_ptr, const uint32_t *b_col, const void *b_val, int btc,
                                 int64_t am, int64_t bm, int64_t bn, int op, int xtc, int ytc, int ztc, const int64_t *t_ptr, uint32_t *t_col, void *t_val) {
    const int64_t n = am * bm;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        const int64_t ia = r / bm, ib = r % bm;
        int64_t o = t_ptr[r];
        for (int64_t ka = a_ptr[ia]; ka < a_ptr[ia + 1]; ++ka) {
            const Sc x = sc_cast(sc_load(atc, a_val, (size_t)ka), atc, xtc);
            for (int64_t kb = b_ptr[ib]; kb < b_ptr[ib + 1]; ++kb) {
                // the operator's two inputs share one type for every builtin operator
                const Sc y = sc_cast(sc_load(btc, b_val, (size_t)kb), btc, ytc);
                t_col[o] = (uint32_t)((int64_t)a_col[ka] * bn + b_col[kb]);
                sc_store(ztc, t_val, (size_t)o, sc_binop(op, xtc, x, y));
                ++o;
            }
        }
    }
}
extern "C" GrB_Info GrB_Matrix_kronecker_BinaryOp(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const GrB_BinaryOp op, const GrB_Matrix A,
                                                  const GrB_Matrix B, const GrB_Descriptor desc) {
    GB_LOCK; GB_CHECK_INIT;
    const char *fn = "GrB_Matrix_kronecker_BinaryOp";
    if (!C || !op || !A || !B) return gb_fail(GrB_NULL_POINTER, nullptr, "%s: NULL argument", fn);
    if (!gb_valid_matrix(C) || !gb_valid_matrix(A) || !gb_valid_matrix(B) || (Mask && !gb_valid_matrix(Mask)) || op->magic != GB_MAGIC)
        return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "%s: invalid object", fn);
    std::string *err = &C->err;
    if (op->opcode == OP_USER || (accum && accum->opcode == OP_USER)) return gb_fail(GrB_INVALID_VALUE, err, "%s: user-defined operators cannot run on the GPU", fn);
    const DescFlags f = desc_flags(desc);
    const uint64_t am = f.tran0 ? A->ncols : A->nrows, an = f.tran0 ? A->nrows : A->ncols;
    const uint64_t bm = f.tran1 ? B->ncols : B->nrows, bn = f.tran1 ? B->nrows : B->ncols;
    if (C->nrows != am * bm || C->ncols != an * bn || (Mask && (Mask->nrows != C->nrows || Mask->ncols != C->ncols)))
        return gb_fail(GrB_DIMENSION_MISMATCH, err, "%s: C must be %llux%llu", fn, (unsigned long long)(am * bm), (unsigned long long)(an * bn));
    if (!G.have_device) return gb_fail(GrB_PANIC, err, "%s: no CUDA device: libb200grb computes only on the GPU (no CPU fallback)", fn);
    if (am * bm >= ((uint64_t)1 << 31) || an * bn >= ((uint64_t)1 << 31)) return gb_fail(GrB_INVALID_VALUE, err, "%s: result dimensions beyond 2^31 are not supported in HBM", fn);
    GbBurble burble(fn);
    if (f.tran0) GB_TRY(matrix_ensure_transpose(A)); else GB_TRY(matrix_ensure_device(A));
    if (f.tran1) GB_TRY(matrix_ensure_transpose(B)); else GB_TRY(matrix_ensure_device(B));
    const Csr &a = f.tran0 ? A->devT : A->dev; const Csr &b = f.tran1 ? B->devT : B->dev;
    const int ztc = op->ztype->code;
    Csr T; T.nrows = (int64_t)(am * bm); T.ncols = (int64_t)(an * bn);
    GB_TRY(T.rowptr.alloc((size_t)T.nrows + 1, err));
    kron_count_kernel<<<agrid(T.nrows + 1), 256, 0, G.stream>>>(a.rowptr, b.rowptr, (int64_t)am, (int64_t)bm, T.rowptr); GB_LAUNCHED();
    GB_TRY(dev_exclusive_scan(T.rowptr, T.nrows + 1, err));
    GB_TRY(read_i64(T.rowptr + T.nrows, &T.nnz, err));
    GB_TRY(T.col.alloc((size_t)T.nnz, err));
    GB_TRY(T.val.alloc((size_t)T.nnz * tc_size(ztc) + 16, err));
    if (T.nnz > 0) {
        kron_fill_kernel<<<agrid(T.nrows), 256, 0, G.stream>>>(a.rowptr, a.col, a.val, A->type->code, b.rowptr, b.col, b.val, B->type->code, (int64_t)am, (int64_t)bm,
                                                              (int64_t)bn, op->opcode, op->xtype->code, op->ytype->code, ztc, T.rowptr, T.col, T.val); GB_LAUNCHED();
    }
    GB_TRY(dev_build_rowptr32(T, err));
    burble.note("row-pair expansion", (double)T.nnz * (4 + tc_size(ztc)));
    return matrix_writeback(C, Mask, accum, f, std::move(T), ztc, false, err);
}

// ================================================================== rows / columns of a matrix as vectors, and back
extern "C" GrB_Info GrB_Vector_new(GrB_Vector *v, GrB_Type type, GrB_Index n);
extern "C" GrB_Info GrB_Vector_free(GrB_Vector *v);
extern "C" GrB_Info GrB_Vector_assign(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_Vector u, const GrB_Index *I, GrB_Index ni, const GrB_Descriptor desc);
extern "C" GrB_Info GrB_Vector_extract(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_Vector u, const GrB_Index *I, GrB_Index ni, const GrB_Descriptor desc);

__global__ void row_to_dense_kernel(const int64_t *ptr, const uint32_t *col, const uint8_t *val, int vsize, int64_t row, uint8_t *oval, uint8_t *opres) {
    for (int64_t k = ptr[row] + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < ptr[row + 1]; k += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t c = col[k];
        for (int b = 0; b < vsize; ++b) oval[(size_t)c * vsize + b] = val[k * vsize + b];
        opres[c] = 1;
    }
}
__global__ void col_to_dense_kernel(const int64_t *ptr, const uint32_t *col, const uint8_t *val, int vsize, int64_t nrows, uint32_t j, uint8_t *oval, uint8_t *opres) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += (int64_t)gridDim.x * blockDim.x) {
        int64_t lo = ptr[r], hi = ptr[r + 1];
        while (lo < hi) { const int64_t mid = (lo + hi) >> 1; if (col[mid] < j) lo = mid + 1; else hi = mid; }
        if (lo < ptr[r + 1] && col[lo] == j) { for (int b = 0; b < vsize; ++b) oval[(size_t)r * vsize + b] = val[lo * vsize + b]; opres[r] = 1; }
    }
}
// a temporary vector holding row i (along = 0) or column j (along = 1) of the CSR
static GrB_Info slice_vector(const Csr &a, GrB_Type type, int along, uint64_t index, GrB_Vector *out, std::string *err) {
    const int64_t n = along == 0 ? a.ncols : a.nrows;
    const size_t vsize = type->size;
    DevBuf<void> val; DevBuf<uint8_t> pres;
    GB_TRY(val.alloc((size_t)n * vsize + 16, err));
    GB_TRY(pres.alloc((size_t)n, err));
    CU_TRY(cudaMemsetAsync(val, 0, (size_t)n * vsize, G.stream), err);
    CU_TRY(cudaMemsetAsync(pres, 0, (size_t)n, G.stream), err);
    if (a.nnz > 0) {
        if (along == 0) row_to_dense_kernel<<<agrid(4096), 256, 0, G.stream>>>(a.rowptr, a.col, (const uint8_t *)a.val, (int)vsize, (int64_t)index, (uint8_t *)val, pres);
        else col_to_dense_kernel<<<agrid(a.nrows), 256, 0, G.stream>>>(a.rowptr, a.col, (const uint8_t *)a.val, (int)vsize, a.nrows, (uint32_t)index, (uint8_t *)val, pres);
        GB_LAUNCHED();
    }
    GB_TRY(GrB_Vector_new(out, type, (GrB_Index)n));
    vector_adopt_device(*out, val.release(), pres.release());
    return GrB_SUCCESS;
}
__global__ void vec_flags_kernel(const uint8_t *pres, int64_t n, int64_t *flag) {
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q <= n; q += (int64_t)gridDim.x * blockDim.x) flag[q] = (q < n && (!pres || pres[q])) ? 1 : 0;
}
__global__ void vec_to_row_kernel(const uint8_t *vval, const uint8_t *pres, int vsize, int64_t n, const int64_t *pos, int64_t base, uint32_t *col, uint8_t *val) {
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (int64_t)gridDim.x * blockDim.x) if (!pres || pres[q]) {
        const int64_t o = base + pos[q];
        col[o] = (uint32_t)q;
        for (int b = 0; b < vsize; ++b) val[o * vsize + b] = vval[(size_t)q * vsize + b];
    }
}
__global__ void row_only_ptr_kernel(int64_t nrows, int64_t row, int64_t cnt, int64_t *rowptr) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r <= nrows; r += (int64_t)gridDim.x * blockDim.x) rowptr[r] = r <= row ? 0 : cnt;
}
__global__ void vec_to_col_kernel(const uint8_t *vval, const uint8_t *pres, int vsize, int64_t n, const int64_t *rowptr, uint32_t j, uint32_t *col, uint8_t *val) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) if (!pres || pres[r]) {
        const int64_t o = rowptr[r];
        col[o] = j;
        for (int b = 0; b < vsize; ++b) val[o * vsize + b] = vval[(size_t)r * vsize + b];
    }
}
// T (nrows x ncols): row `index` (along = 0) or column `index` (along = 1) holds the vector, everything else is empty
static GrB_Info vector_as_slice_csr(GrB_Vector v, int along, uint64_t index, int64_t nrows, int64_t ncols, Csr &T, std::string *err) {
    GB_TRY(vector_ensure_device(v));
    const int64_t n = (int64_t)v->n; const size_t vsize = v->type->size;
    T = Csr(); T.nrows = nrows; T.ncols = ncols;
    DevBuf<int64_t> pos;
    GB_TRY(pos.alloc((size_t)n + 1, err));
    vec_flags_kernel<<<agrid(n + 1), 256, 0, G.stream>>>(v->dpres, n, pos); GB_LAUNCHED();
    GB_TRY(dev_exclusive_scan(pos, n + 1, err));
    GB_TRY(read_i64(pos + n, &T.nnz, err));
    GB_TRY(T.col.alloc((size_t)T.nnz, err));
    GB_TRY(T.val.alloc((size_t)T.nnz * vsize + 16, err));
    if (along == 0) {
        GB_TRY(T.rowptr.alloc((size_t)nrows + 1, err));
        row_only_ptr_kernel<<<agrid(nrows + 1), 256, 0, G.stream>>>(nrows, (int64_t)index, T.nnz, T.rowptr); GB_LAUNCHED();
        if (T.nnz > 0) { vec_to_row_kernel<<<agrid(n), 256, 0, G.stream>>>((const uint8_t *)v->dval, v->dpres, (int)vsize, n, pos, 0, T.col, (uint8_t *)T.val); GB_LAUNCHED(); }
        pos.reset();
    } else {
        T.rowptr = std::move(pos);       // one entry per present position: the scan IS the row pointer
        if (T.nnz > 0) { vec_to_col_kernel<<<agrid(n), 256, 0, G.stream>>>((const uint8_t *)v->dval, v->dpres, (int)vsize, n, T.rowptr, (uint32_t)index, T.col, (uint8_t *)T.val); GB_LAUNCHED(); }
    }
    GB_TRY(dev_build_rowptr32(T, err));
    CU_TRY(cudaGetLastError(), err);
    return GrB_SUCCESS;
}

// C<mask'>(i, J) = accum(C(i,J), u')   /   C<mask>(I, j) = accum(C(I,j), u)
static GrB_Info slice_assign(GrB_Matrix C, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_Vector u, int along, GrB_Index index,
                             const GrB_Index *K, GrB_Index nk, const GrB_Descriptor desc, const char *fn) {
    GB_LOCK; GB_CHECK_INIT;
    if (!C || !u) return gb_fail(GrB_NULL_POINTER, nullptr, "%s: NULL argument", fn);
    if (!gb_valid_matrix(C) || !gb_valid_vector(u) || (mask && !gb_valid_vector(mask))) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "%s: invalid object", fn);
    std::string *err = &C->err;
    if (index >= (along == 0 ? C->nrows : C->ncols)) return gb_fail(GrB_INVALID_INDEX, err, "%s: index %llu out of bounds", fn, (unsigned long long)index);
    if (!G.have_device) return gb_fail(GrB_PANIC, err, "%s: no CUDA device: libb200grb computes only on the GPU (no CPU fallback)", fn);
    if (C->nrows >= ((uint64_t)1 << 31) || C->ncols >= ((uint64_t)1 << 31)) return gb_fail(GrB_INVALID_VALUE, err, "%s: dimensions beyond 2^31 are not supported in HBM", fn);
    GbBurble burble(fn);
    GB_TRY(matrix_ensure_device(C));
    // 1. the row / column as a vector;  2. the vector assignment (mask, accumulator, GrB_REPLACE act inside the slice);  3. put it back
    GrB_Vector sv = nullptr;
    GB_TRY(slice_vector(C->dev, C->type, along, index, &sv, err));
    GrB_Info r = GrB_Vector_assign(sv, mask, accum, u, K, nk, desc);
    if (r != GrB_SUCCESS) { *err = sv->err; GrB_Vector_free(&sv); return r; }
    Csr T;
    r = vector_as_slice_csr(sv, along, index, (int64_t)C->nrows, (int64_t)C->ncols, T, err);
    GrB_Vector_free(&sv);
    if (r != GrB_SUCCESS) return r;
    Region R;
    std::vector<uint64_t> one(1, index);
    if (along == 0) { R.all_rows = false; R.I = one; R.ni_distinct = 1; R.nj_distinct = (int64_t)C->ncols; }
    else { R.all_cols = false; R.J = one; R.nj_distinct = 1; R.ni_distinct = (int64_t)C->nrows; }
    DevBuf<uint64_t> d;
    GB_TRY(upload(one, d, err));
    DevBuf<uint8_t> &flag = along == 0 ? R.rowflag : R.colflag;
    const size_t fn_ = (size_t)(along == 0 ? C->nrows : C->ncols);
    GB_TRY(flag.alloc(fn_, err));
    cudaMemsetAsync(flag, 0, fn_, G.stream);
    flag_kernel<<<1, 32, 0, G.stream>>>(d, 1, flag); GB_LAUNCHED();
    DescFlags plain{};
    return assign_writeback(C, nullptr, nullptr, plain, R, std::move(T), C->type->code, /*t_covers_region=*/false, err);     // the slice vector has C's type
}

extern "C" GrB_Info GrB_Row_assign(GrB_Matrix C, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_Vector u, GrB_Index i, const GrB_Index *J, GrB_Index nj,
                                   const GrB_Descriptor desc) {
    return slice_assign(C, mask, accum, u, 0, i, J, nj, desc, "GrB_Row_assign");
}
extern "C" GrB_Info GrB_Col_assign(GrB_Matrix C, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_Vector u, const GrB_Index *I, GrB_Index ni, GrB_Index j,
                                   const GrB_Descriptor desc) {
    return slice_assign(C, mask, accum, u, 1, j, I, ni, desc, "GrB_Col_assign");
}

// w<mask> = accum(w, op(A)(I, j))
extern "C" GrB_Info GrB_Col_extract(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_Matrix A, const GrB_Index *I, GrB_Index ni, GrB_Index j,
                                    const GrB_Descriptor desc) {
    GB_LOCK; GB_CHECK_INIT;
    const char *fn = "GrB_Col_extract";
    if (!w || !A) return gb_fail(GrB_NULL_POINTER, nullptr, "%s: NULL argument", fn);
    if (!gb_valid_vector(w) || !gb_valid_matrix(A) || (mask && !gb_valid_vector(mask))) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "%s: invalid object", fn);
    std::string *err = &w->err;
    const DescFlags f = desc_flags(desc);
    if (j >= (f.tran0 ? A->nrows : A->ncols)) return gb_fail(GrB_INVALID_INDEX, err, "%s: column %llu out of bounds", fn, (unsigned long long)j);
    if (!G.have_device) return gb_fail(GrB_PANIC, err, "%s: no CUDA device: libb200grb computes only on the GPU (no CPU fallback)", fn);
    GbBurble burble(fn);
    GB_TRY(matrix_ensure_device(A));
    GrB_Vector cv = nullptr;                 // column j of op(A): row j of A when INP0 = TRAN
    GB_TRY(slice_vector(A->dev, A->type, f.tran0 ? 0 : 1, j, &cv, err));
    const GrB_Info r = GrB_Vector_extract(w, mask, accum, cv, I, ni, desc);
    GrB_Vector_free(&cv);
    return r;
}

// ================================================================== GrB_Matrix_assign:  C<Mask>(I,J) = accum(C(I,J), op(A))
__global__ void massign_count_kernel(const int32_t *rowsrc, int64_t nrows, const int64_t *a_ptr, int64_t *cnt) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r <= nrows; r += (int64_t)gridDim.x * blockDim.x) {
        const int32_t p = r < nrows ? (rowsrc ? rowsrc[r] : (int32_t)r) : -1;
        cnt[r] = p >= 0 ? a_ptr[p + 1] - a_ptr[p] : 0;
    }
}
__global__ void massign_fill_kernel(const int32_t *rowsrc, int64_t nrows, const int64_t *a_ptr, const uint32_t *a_col, const uint8_t *a_val, int vsize,
                                    const uint32_t *jmap, const int64_t *t_ptr, uint32_t *t_col, uint8_t *t_val) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += (int64_t)gridDim.x * blockDim.x) {
        const int32_t p = rowsrc ? rowsrc[r] : (int32_t)r;
        if (p < 0) continue;
        int64_t o = t_ptr[r];
        for (int64_t k = a_ptr[p]; k < a_ptr[p + 1]; ++k, ++o) {
            t_col[o] = jmap ? jmap[a_col[k]] : a_col[k];
            for (int b = 0; b < vsize; ++b) t_val[o * vsize + b] = a_val[k * vsize + b];
        }
    }
}
extern "C" GrB_Info GrB_Matrix_assign(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const GrB_Matrix A, const GrB_Index *I, GrB_Index ni,
                                      const GrB_Index *J, GrB_Index nj, const GrB_Descriptor desc) {
    GB_LOCK; GB_CHECK_INIT;
    const char *fn = "GrB_Matrix_assign";
    if (!C || !A) return gb_fail(GrB_NULL_POINTER, nullptr, "%s: NULL argument", fn);
    if (!gb_valid_matrix(C) || !gb_valid_matrix(A) || (Mask && !gb_valid_matrix(Mask))) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "%s: invalid object", fn);
    std::string *err = &C->err;
    if (accum && accum->opcode == OP_USER) return gb_fail(GrB_INVALID_VALUE, err, "%s: user-defined accumulators cannot run on the GPU", fn);
    if (Mask && (Mask->nrows != C->nrows || Mask->ncols != C->ncols)) return gb_fail(GrB_DIMENSION_MISMATCH, err, "%s: the mask must have C's dimensions", fn);
    const DescFlags f = desc_flags(desc);
    Region R;
    if (G.have_device && C->nrows < ((uint64_t)1 << 31) && C->ncols < ((uint64_t)1 << 31)) GB_TRY(region_build(R, I, ni, J, nj, C->nrows, C->ncols, err, fn));
    else return G.have_device ? gb_fail(GrB_INVALID_VALUE, err, "%s: dimensions beyond 2^31 are not supported in HBM", fn)
                              : gb_fail(GrB_PANIC, err, "%s: no CUDA device: libb200grb computes only on the GPU (no CPU fallback)", fn);
    const uint64_t an = f.tran0 ? A->ncols : A->nrows, am = f.tran0 ? A->nrows : A->ncols;
    const uint64_t tn = R.all_rows ? C->nrows : R.I.size(), tm = R.all_cols ? C->ncols : R.J.size();
    if (an != tn || am != tm) return gb_fail(GrB_DIMENSION_MISMATCH, err, "%s: A is %llux%llu, the index lists select %llux%llu", fn,
                                             (unsigned long long)an, (unsigned long long)am, (unsigned long long)tn, (unsigned long long)tm);
    GbBurble burble(fn);
    GB_TRY(f.tran0 ? matrix_ensure_transpose(A) : matrix_ensure_device(A));
    const Csr &a = f.tran0 ? A->devT : A->dev;
    const size_t vsize = A->type->size;
    DevBuf<int32_t> d_rowsrc; DevBuf<uint32_t> d_jmap; bool need_sort = false;
    if (!R.all_rows) {
        std::vector<int32_t> rowsrc((size_t)C->nrows, -1);
        for (size_t p = 0; p < R.I.size(); ++p) rowsrc[R.I[p]] = (int32_t)p;       // a row named twice takes the later source row
        GB_TRY(upload(rowsrc, d_rowsrc, err));
    }
    if (!R.all_cols) {
        std::vector<uint32_t> jmap(R.J.begin(), R.J.end());
        for (size_t q = 1; q < jmap.size(); ++q) if (jmap[q] <= jmap[q - 1]) need_sort = true;
        GB_TRY(upload(jmap, d_jmap, err));
    }
    Csr T; T.nrows = (int64_t)C->nrows; T.ncols = (int64_t)C->ncols;
    GB_TRY(T.rowptr.alloc((size_t)T.nrows + 1, err));
    massign_count_kernel<<<agrid(T.nrows + 1), 256, 0, G.stream>>>(d_rowsrc, T.nrows, a.rowptr, T.rowptr); GB_LAUNCHED();
    GB_TRY(dev_exclusive_scan(T.rowptr, T.nrows + 1, err));
    GB_TRY(read_i64(T.rowptr + T.nrows, &T.nnz, err));
    GB_TRY(T.col.alloc((size_t)T.nnz, err));
    GB_TRY(T.val.alloc((size_t)T.nnz * vsize + 16, err));
    if (T.nnz > 0) {
        massign_fill_kernel<<<agrid(T.nrows), 256, 0, G.stream>>>(d_rowsrc, T.nrows, a.rowptr, a.col, (const uint8_t *)a.val, (int)vsize, d_jmap, T.rowptr, T.col, (uint8_t *)T.val); GB_LAUNCHED();
        if (need_sort) { rows_insertion_sort_kernel<<<agrid(T.nrows), 256, 0, G.stream>>>(T.rowptr, T.nrows, T.col, (uint8_t *)T.val, (int)vsize); GB_LAUNCHED(); }
    }
    GB_TRY(dev_build_rowptr32(T, err));
    d_rowsrc.reset(); d_jmap.reset();
    return assign_writeback(C, Mask, accum, f, R, std::move(T), A->type->code, /*t_covers_region=*/false, err);
}
