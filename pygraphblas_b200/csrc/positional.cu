// positional.cu -- the positional operators of SuiteSparse v4: FIRSTI ... SECONDJ1 (binary), POSITIONI ... POSITIONJ1 (unary).
//
// A positional operator never reads a value: it returns where its operands sit, as INT32 / INT64.  So no kernel of the
// library ever sees a positional opcode.  The callers (spmv.cu, spgemm.cu, matrix_ops.cu, vector_ops.cu) rewrite the call
// into one the existing kernels run, with the positions supplied as VALUES by the kernels below (DESIGN.md section 3.5):
//
//   inner form   the product is the inner index k (FIRSTJ, SECONDI): the operand that sits at k gets k as its value
//                (an iota over u, or the column / row index of each entry of op(A) / op(B)), then FIRST or SECOND
//   count form   the product is an output coordinate or 0 (FIRSTI, SECONDJ): every product at output position p has the
//                same value v(p), so T(p) = v(p) folded cnt(p) times; cnt comes from PLUS.PAIR (ANY.PAIR when the
//                monoid is idempotent) and the fold is closed-form: MIN / MAX / ANY -> v, PLUS -> v * cnt, TIMES -> v^cnt
//
// All arithmetic is modulo 2^64, then truncated for INT32 (a C cast), which is what the INT32 monoids compute.
#include "common.cuh"

// the index a position stands for: its original id (hypersparse operands) or the position itself, plus the offset
__device__ __forceinline__ uint64_t pos_index(int64_t p, const uint64_t *ids, int64_t off) {
    return (ids ? ids[p] : (uint64_t)p) + (uint64_t)off;
}
// v folded cnt times with the monoid add (cnt >= 1), modulo 2^64
__device__ __forceinline__ uint64_t pos_fold(int add, uint64_t v, int64_t cnt) {
    if (add == OP_PLUS) return v * (uint64_t)cnt;
    if (add == OP_TIMES) {
        uint64_t r = 1, b = v;
        for (uint64_t e = (uint64_t)cnt; e; e >>= 1) { if (e & 1) r *= b; b *= b; }
        return r;
    }
    return v;                              // MIN, MAX, ANY: every product is v
}

template <typename T>
__global__ void pos_vector_kernel(T *out, const int64_t *cnt, int add, int64_t n, int zero, const uint64_t *ids, int64_t off) {
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x) {
        const uint64_t v = zero ? (uint64_t)off : pos_index(p, ids, off);
        out[p] = (T)(cnt ? pos_fold(add, v, cnt[p]) : v);
    }
}

// one thread per entry; the row of entry e is found by binary search in rowptr (balanced whatever the row lengths)
template <typename T>
__global__ void pos_csr_kernel(T *out, const int64_t *cnt, int add, const int64_t *rowptr, const uint32_t *col, int64_t nrows, int64_t nnz,
                               int by_col, const uint64_t *ids, int64_t off) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += (int64_t)gridDim.x * blockDim.x) {
        int64_t idx;
        if (by_col) idx = (int64_t)col[e];
        else {
            int64_t lo = 0, hi = nrows - 1;                // last row r with rowptr[r] <= e
            while (lo < hi) { const int64_t mid = (lo + hi + 1) >> 1; if (rowptr[mid] <= e) lo = mid; else hi = mid - 1; }
            idx = lo;
        }
        const uint64_t v = pos_index(idx, ids, off);
        out[e] = (T)(cnt ? pos_fold(add, v, cnt[e]) : v);
    }
}

GrB_Info pos_vector_values(void *out, int tc, const int64_t *cnt, int add, int64_t n, bool zero, const uint64_t *ids, int64_t off,
                           std::string *err) {
    if (n <= 0) return GrB_SUCCESS;
    if (tc == TC_INT32) pos_vector_kernel<int32_t><<<grid_for(n), 256, 0, G.stream>>>((int32_t *)out, cnt, add, n, zero, ids, off);
    else if (tc == TC_INT64) pos_vector_kernel<int64_t><<<grid_for(n), 256, 0, G.stream>>>((int64_t *)out, cnt, add, n, zero, ids, off);
    else return gb_fail(GrB_DOMAIN_MISMATCH, err, "positional operators compute INT32 or INT64 values");
    GB_LAUNCHED();
    CU_TRY(cudaGetLastError(), err);
    return GrB_SUCCESS;
}

GrB_Info pos_csr_values(void *out, int tc, const int64_t *cnt, int add, const Csr &c, bool by_col, const uint64_t *ids, int64_t off,
                        std::string *err) {
    if (c.nnz <= 0) return GrB_SUCCESS;
    if (tc == TC_INT32)
        pos_csr_kernel<int32_t><<<grid_for(c.nnz), 256, 0, G.stream>>>((int32_t *)out, cnt, add, c.rowptr, c.col, c.nrows, c.nnz, by_col, ids, off);
    else if (tc == TC_INT64)
        pos_csr_kernel<int64_t><<<grid_for(c.nnz), 256, 0, G.stream>>>((int64_t *)out, cnt, add, c.rowptr, c.col, c.nrows, c.nnz, by_col, ids, off);
    else return gb_fail(GrB_DOMAIN_MISMATCH, err, "positional operators compute INT32 or INT64 values");
    GB_LAUNCHED();
    CU_TRY(cudaGetLastError(), err);
    return GrB_SUCCESS;
}

GrB_Info gb_refuse_positional_accum(const GrB_BinaryOp accum, const char *fn) {
    if (accum && accum->magic == GB_MAGIC && op_is_positional(accum->opcode))
        return gb_fail(GrB_DOMAIN_MISMATCH, nullptr, "%s: a positional operator (%s) cannot be an accumulator", fn, accum->name);
    return GrB_SUCCESS;
}
GrB_Info gb_refuse_user_with_positional(const GrB_Semiring s, const GrB_BinaryOp accum, const char *fn) {
    if (!s || s->magic != GB_MAGIC || !op_is_positional(s->mul->opcode)) return GrB_SUCCESS;
    if (s->add->op->opcode == OP_USER || (accum && accum->opcode == OP_USER))
        return gb_fail(GrB_INVALID_VALUE, nullptr, "%s: user-defined operators are host function pointers and cannot run on the GPU (no CPU fallback)", fn);
    return GrB_SUCCESS;
}
GrB_Info gb_refuse_positional(const GrB_BinaryOp op, const char *fn) {
    if (op && op->magic == GB_MAGIC && op_is_positional(op->opcode))
        return gb_fail(GrB_INVALID_VALUE, nullptr, "positional operators are not supported by %s", fn);
    return GrB_SUCCESS;
}
GrB_Info gb_refuse_positional(const GrB_Semiring s, const char *fn) {
    return s && s->magic == GB_MAGIC ? gb_refuse_positional(s->mul, fn) : GrB_SUCCESS;
}
