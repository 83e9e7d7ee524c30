// Matrix-side consumers of the hot path, on the device (SURVEY.md section 8(f)3): what the reference's
// algorithms wrap around a masked SpGEMM or a sweep of SpMVs so that they run end to end in HBM --
//
//   GxB_Matrix_select / GxB_Vector_select   tril / triu / diag / offdiag / nonzero / comparisons with zero or a thunk
//                                           reference: pygraphblas/matrix.py:2042-2140 (select, tril, triu, ...),
//                                           demo/Triangle-Counting.ipynb:581 (L = A.tril(-1))
//   GrB_Matrix_apply (+ BinaryOp1st / 2nd)  matrix.py:1870-1990
//   GrB_Matrix_reduce_<T>                   matrix.py:1782-1840 (reduce_bool / reduce_int / reduce_float): triangle count = C.reduce_int()
//   GrB_Matrix_reduce_Monoid / _BinaryOp    matrix.py:1842-1868 (reduce_vector): out-degrees for PageRank
//   GrB_Matrix_eWiseAdd_* / eWiseMult_*     matrix.py:1494-1700 (eadd / emult and the operators built on them)
//
// All of them read CSR panels (rows sorted, columns sorted inside a row), form a CSR or vector T with one warp per
// row, and finish with the common write-back (matrix_writeback / vector_write).  Values travel on the 64-bit
// carrier, so one code path serves the 11 builtin types and their typecasts; these kernels stream each operand
// once and are HBM-bound.
#include "common.cuh"
#include <algorithm>
#include <vector>
#include "../../include/b200grb_compat.h"

#define GB_MAT_OK(A, fn) do { if (!(A)) return gb_fail(GrB_NULL_POINTER, nullptr, "%s: NULL matrix", fn); \
    if (!gb_valid_matrix(A)) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "%s: invalid matrix handle", fn); } while (0)
#define GB_VEC_OK(v, fn) do { if (!(v)) return gb_fail(GrB_NULL_POINTER, nullptr, "%s: NULL vector", fn); \
    if (!gb_valid_vector(v)) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "%s: invalid vector handle", fn); } while (0)
#define GB_NEED_DEVICE(errp, fn) do { if (!G.have_device) return gb_fail(GrB_PANIC, errp, "%s: no CUDA device: libb200grb computes only on the GPU (no CPU fallback)", fn); } while (0)

// ------------------------------------------------------------------ select
struct SelectArgs {
    const int64_t *rowptr; const uint32_t *col; const void *val; int tc; int64_t nrows;
    int code; int64_t k; Sc thunk;              // k: diagonal of TRIL / TRIU / DIAG / OFFDIAG; thunk: already of type tc
    int64_t *o_ptr; uint32_t *o_col; void *o_val;
};
__device__ __forceinline__ bool select_keep(const SelectArgs &a, int64_t i, int64_t j, Sc x) {
    switch (a.code) {
        case SEL_TRIL: return j - i <= a.k;
        case SEL_TRIU: return j - i >= a.k;
        case SEL_DIAG: return j - i == a.k;
        case SEL_OFFDIAG: return j - i != a.k;
        default: break;
    }
    Sc zero; zero.u = 0;
    const Sc y = a.code >= SEL_NE_THUNK ? a.thunk : zero;
    int cmp;
    switch (a.code) {
        case SEL_NONZERO: case SEL_NE_THUNK: cmp = OP_NE; break;
        case SEL_EQ_ZERO: case SEL_EQ_THUNK: cmp = OP_EQ; break;
        case SEL_GT_ZERO: case SEL_GT_THUNK: cmp = OP_GT; break;
        case SEL_GE_ZERO: case SEL_GE_THUNK: cmp = OP_GE; break;
        case SEL_LT_ZERO: case SEL_LT_THUNK: cmp = OP_LT; break;
        default: cmp = OP_LE; break;
    }
    return sc_binop(cmp, a.tc, x, y).u != 0;
}
// one warp per row; FILL = false counts the survivors of each row into o_ptr[row], FILL = true writes them
template <bool FILL>
__global__ void __launch_bounds__(256) select_kernel(const SelectArgs a) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int vs = tc_size(a.tc);
    for (int64_t r = warp; r < a.nrows; r += nwarps) {
        const int64_t rs = a.rowptr[r], re = a.rowptr[r + 1];
        int64_t out = FILL ? a.o_ptr[r] : 0;
        for (int64_t b = rs; b < re; b += 32) {
            const int64_t e = b + lane;
            bool keep = false; uint32_t c = 0;
            if (e < re) { c = a.col[e]; keep = select_keep(a, r, (int64_t)c, sc_load(a.tc, a.val, (size_t)e)); }
            const unsigned m = __ballot_sync(0xffffffffu, keep);
            if (FILL && keep) {
                const int64_t o = out + __popc(m & ((1u << lane) - 1u));
                a.o_col[o] = c;
                if (a.o_val) {                          // no value array: the pattern only (mask_true_pattern)
                    const uint8_t *src = (const uint8_t *)a.val + (size_t)e * vs; uint8_t *dst = (uint8_t *)a.o_val + (size_t)o * vs;
                    for (int q = 0; q < vs; ++q) dst[q] = src[q];
                }
            }
            out += __popc(m);
        }
        if (!FILL && lane == 0) a.o_ptr[r] = out;
    }
}
static GrB_Info select_args(const GxB_SelectOp op, const GxB_Scalar thunk, int tc, SelectArgs &a, const char *fn) {
    if (!op) return gb_fail(GrB_NULL_POINTER, nullptr, "%s: NULL select operator", fn);
    if (op->magic != GB_MAGIC) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "%s: invalid select operator (user-defined select functions cannot run on the GPU)", fn);
    a.code = op->code; a.k = 0; a.thunk.u = 0;
    const bool has_thunk = thunk && thunk->magic == GB_MAGIC && thunk->has;
    if (a.code <= SEL_OFFDIAG) { if (has_thunk) a.k = sc_cast(thunk->v, thunk->type->code, TC_INT64).i; }
    else if (a.code >= SEL_NE_THUNK) {
        if (!has_thunk) return gb_fail(GrB_INVALID_VALUE, nullptr, "%s: %s needs a thunk", fn, op->name);
        a.thunk = sc_cast(thunk->v, thunk->type->code, tc);
    }
    return GrB_SUCCESS;
}
// T = the entries of src that a (code, k, thunk, tc set) keeps, with their values when vsize > 0, only their pattern when 0
static GrB_Info select_csr(const Csr &src, SelectArgs a, size_t vsize, Csr &T, std::string *err) {
    a.rowptr = src.rowptr; a.col = src.col; a.val = src.val; a.nrows = src.nrows;
    const int grid = grid_for(src.nrows * 32);
    return csr_from_row_counts(src.nrows, src.ncols, vsize, T, err,
        [&](int64_t *rowptr) {
            CU_TRY(cudaMemsetAsync(rowptr, 0, ((size_t)src.nrows + 1) * 8, G.stream), err);
            a.o_ptr = rowptr;       // without entries there is nothing to count: the memset has zeroed every slot
            if (src.nnz > 0) { select_kernel<false><<<grid, 256, 0, G.stream>>>(a); GB_LAUNCHED(); }
            return GrB_SUCCESS;
        },
        [&](Csr &t) {
            a.o_col = t.col; a.o_val = vsize ? t.val.get() : nullptr;
            select_kernel<true><<<grid, 256, 0, G.stream>>>(a); GB_LAUNCHED();
            return GrB_SUCCESS;
        });
}
extern "C" GrB_Info GxB_Matrix_select(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const GxB_SelectOp op, const GrB_Matrix A,
                                      const GxB_Scalar thunk, const GrB_Descriptor desc) {
    GB_LOCK; GB_CHECK_INIT;
    const char *fn = "GxB_Matrix_select";
    GB_MAT_OK(C, fn); GB_MAT_OK(A, fn);
    if (Mask) GB_MAT_OK(Mask, fn);
    GB_TRY(gb_refuse_positional_accum(accum, fn));
    if (accum && accum->opcode == OP_USER) return gb_fail(GrB_INVALID_VALUE, nullptr, "%s: user-defined accumulators cannot run on the GPU", fn);
    std::string *err = &C->err;
    const DescFlags f = desc_flags(desc);
    const uint64_t an = f.tran0 ? A->ncols : A->nrows, am = f.tran0 ? A->nrows : A->ncols;
    if (C->nrows != an || C->ncols != am || (Mask && (Mask->nrows != an || Mask->ncols != am))) return gb_fail(GrB_DIMENSION_MISMATCH, err, "%s: dimensions do not match", fn);
    SelectArgs a{};
    GB_TRY(select_args(op, thunk, A->type->code, a, fn));
    GB_NEED_DEVICE(err, fn);
    Csr *src; GB_TRY(source_csr(A, f.tran0, &src));
    a.tc = A->type->code;
    Csr T; GB_TRY(select_csr(*src, a, A->type->size, T, err));
    return matrix_writeback(C, Mask, accum, f, std::move(T), A->type->code, false, err);
}
GrB_Info mask_true_pattern(const Csr &M, int mtc, Csr &out, std::string *err) {
    SelectArgs a{};
    a.code = SEL_NONZERO; a.tc = mtc;
    return select_csr(M, a, 0, out, err);       // the filter reads the pattern only
}
__global__ void vec_select_kernel(const SelectArgs a, const uint8_t *upres, uint8_t *tpres) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.nrows; i += (int64_t)gridDim.x * blockDim.x) {
        const bool up = upres ? upres[i] != 0 : true;
        tpres[i] = up && select_keep(a, i, 0, sc_load(a.tc, a.val, (size_t)i));
    }
}
extern "C" GrB_Info GxB_Vector_select(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GxB_SelectOp op, const GrB_Vector u,
                                      const GxB_Scalar thunk, const GrB_Descriptor desc) {
    GB_LOCK; GB_CHECK_INIT;
    const char *fn = "GxB_Vector_select";
    GB_VEC_OK(w, fn); GB_VEC_OK(u, fn);
    if (mask) GB_VEC_OK(mask, fn);
    GB_TRY(gb_refuse_positional_accum(accum, fn));
    if (accum && accum->opcode == OP_USER) return gb_fail(GrB_INVALID_VALUE, nullptr, "%s: user-defined accumulators cannot run on the GPU", fn);
    if (w->n != u->n || (mask && mask->n != w->n)) return gb_fail(GrB_DIMENSION_MISMATCH, &w->err, "%s: dimensions do not match", fn);
    SelectArgs a{};
    GB_TRY(select_args(op, thunk, u->type->code, a, fn));
    GB_NEED_DEVICE(&w->err, fn);
    GB_TRY(vector_ensure_device(u));
    a.val = u->dv.val; a.tc = u->type->code; a.nrows = (int64_t)u->n;
    // T keeps u's values and narrows its presence: a vector is a column, i = position, j = 0
    const size_t bytes = (size_t)u->n * u->type->size;
    DevBuf<void> tval; DevBuf<uint8_t> tpres;
    GB_TRY(tval.alloc(bytes + 16, &w->err));
    GB_TRY(tpres.alloc((size_t)u->n, &w->err));
    CU_TRY(cudaMemcpyAsync(tval, u->dv.val, bytes, cudaMemcpyDeviceToDevice, G.stream), &w->err);
    vec_select_kernel<<<grid_for(a.nrows), 256, 0, G.stream>>>(a, u->dv.pres, tpres); GB_LAUNCHED();
    return vector_write(w, mask, accum, desc_flags(desc), DenseForm{std::move(tval), std::move(tpres)}, u->type->code, false, nullptr);
}

// ------------------------------------------------------------------ apply:  T has A's pattern, z = f(a) / op(x, a) / op(a, y)
enum { AP_UNARY = 0, AP_BIND1 = 1, AP_BIND2 = 2 };
struct ApplyArgs { int64_t nnz; const void *aval; int atc; int mode; int op; int xtc, ztc; Sc scalar; void *tval; };
__global__ void mat_apply_kernel(const ApplyArgs a) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < a.nnz; e += (int64_t)gridDim.x * blockDim.x) {
        const Sc x = sc_cast(sc_load(a.atc, a.aval, (size_t)e), a.atc, a.xtc);
        const Sc z = a.mode == AP_UNARY ? sc_unop(a.op, a.xtc, x) : (a.mode == AP_BIND1 ? sc_binop(a.op, a.xtc, a.scalar, x) : sc_binop(a.op, a.xtc, x, a.scalar));
        sc_store(a.ztc, a.tval, (size_t)e, z);
    }
}
static GrB_Info mat_apply(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, int mode, int opcode, int xtc, int ztc, Sc scalar,
                          const GrB_Matrix A, const GrB_Descriptor desc, const char *fn) {
    GB_MAT_OK(C, fn); GB_MAT_OK(A, fn);
    if (Mask) GB_MAT_OK(Mask, fn);
    GB_TRY(gb_refuse_positional_accum(accum, fn));
    if (accum && accum->opcode == OP_USER) return gb_fail(GrB_INVALID_VALUE, nullptr, "%s: user-defined accumulators cannot run on the GPU", fn);
    std::string *err = &C->err;
    const DescFlags f = desc_flags(desc);
    const uint64_t an = f.tran0 ? A->ncols : A->nrows, am = f.tran0 ? A->nrows : A->ncols;
    if (C->nrows != an || C->ncols != am || (Mask && (Mask->nrows != an || Mask->ncols != am))) return gb_fail(GrB_DIMENSION_MISMATCH, err, "%s: dimensions do not match", fn);
    GB_NEED_DEVICE(err, fn);
    Csr *src; GB_TRY(source_csr(A, f.tran0, &src));
    Csr T; GB_TRY(csr_copy(*src, (size_t)tc_size(ztc), false, T, err));
    ApplyArgs a{};
    a.nnz = src->nnz; a.aval = src->val; a.atc = A->type->code; a.mode = mode; a.op = opcode; a.xtc = xtc; a.ztc = ztc; a.scalar = scalar; a.tval = T.val;
    if (mode == AP_UNARY ? uop_is_positional(opcode) : op_is_positional(opcode)) {
        // POSITIONI / J, and FIRSTI ... SECONDJ1 bound to a scalar (the scalar is ignored): the row or column of each entry of op(A)
        const PosOp p = mode == AP_UNARY ? pos_unop(opcode) : pos_binop(opcode);
        GB_TRY(pos_csr_values(T.val, ztc, nullptr, OP_ANY, *src, p.col, nullptr, p.off, err));
    } else if (a.nnz > 0) { mat_apply_kernel<<<grid_for(a.nnz), 256, 0, G.stream>>>(a); GB_LAUNCHED(); }
    GB_TRY(dev_build_rowptr32(T, err));
    return matrix_writeback(C, Mask, accum, f, std::move(T), ztc, false, err);
}
extern "C" GrB_Info GrB_Matrix_apply(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const GrB_UnaryOp op, const GrB_Matrix A, const GrB_Descriptor desc) {
    GB_LOCK; GB_CHECK_INIT;
    if (!op) return gb_fail(GrB_NULL_POINTER, nullptr, "GrB_Matrix_apply: NULL operator");
    if (op->magic != GB_MAGIC) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "GrB_Matrix_apply: invalid operator");
    Sc none; none.u = 0;
    return mat_apply(C, Mask, accum, AP_UNARY, op->opcode, op->xtype->code, op->ztype->code, none, A, desc, "GrB_Matrix_apply");
}
static GrB_Info mat_bind(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const GrB_BinaryOp op, int first, const void *x, int xtc_in,
                         const GrB_Matrix A, const GrB_Descriptor desc, const char *fn) {
    if (!op) return gb_fail(GrB_NULL_POINTER, nullptr, "%s: NULL operator", fn);
    if (op->magic != GB_MAGIC) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "%s: invalid operator", fn);
    if (op->opcode == OP_USER) return gb_fail(GrB_INVALID_VALUE, nullptr, "%s: user-defined operators cannot run on the GPU", fn);
    const int xtc = op->xtype->code;
    const Sc s = xtc_in >= 0 ? sc_cast(sc_load(xtc_in, x, 0), xtc_in, xtc) : sc_cast(*(const Sc *)x, -1 - xtc_in, xtc);
    return mat_apply(C, Mask, accum, first ? AP_BIND1 : AP_BIND2, op->opcode, xtc, op->ztype->code, s, A, desc, fn);
}
extern "C" GrB_Info GxB_Matrix_apply_BinaryOp1st(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const GrB_BinaryOp op, const GxB_Scalar x,
                                                  const GrB_Matrix A, const GrB_Descriptor desc) {
    GB_LOCK; GB_CHECK_INIT;
    if (!x || x->magic != GB_MAGIC || !x->has) return gb_fail(GrB_INVALID_VALUE, nullptr, "GxB_Matrix_apply_BinaryOp1st: empty or invalid scalar");
    return mat_bind(C, Mask, accum, op, 1, &x->v, -1 - x->type->code, A, desc, "GxB_Matrix_apply_BinaryOp1st");
}
extern "C" GrB_Info GxB_Matrix_apply_BinaryOp2nd(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const GrB_BinaryOp op, const GrB_Matrix A,
                                                  const GxB_Scalar y, const GrB_Descriptor desc) {
    GB_LOCK; GB_CHECK_INIT;
    if (!y || y->magic != GB_MAGIC || !y->has) return gb_fail(GrB_INVALID_VALUE, nullptr, "GxB_Matrix_apply_BinaryOp2nd: empty or invalid scalar");
    return mat_bind(C, Mask, accum, op, 0, &y->v, -1 - y->type->code, A, desc, "GxB_Matrix_apply_BinaryOp2nd");
}

// ------------------------------------------------------------------ reduce to a scalar / to a vector
static GrB_Info mat_reduce_scalar(void *c, int ctc, const GrB_BinaryOp accum, const GrB_Monoid monoid, const GrB_Matrix A, const char *fn) {
    if (!G.have_device) return gb_fail(GrB_PANIC, nullptr, "%s: no CUDA device: libb200grb computes only on the GPU (no CPU fallback)", fn);
    if (!c || !monoid) return gb_fail(GrB_NULL_POINTER, nullptr, "%s: NULL argument", fn);
    GB_MAT_OK(A, fn);
    if (monoid->magic != GB_MAGIC) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "%s: invalid monoid", fn);
    const GrB_BinaryOp op = monoid->op;
    GB_TRY(gb_refuse_positional_accum(accum, fn));
    if (op->opcode == OP_USER || (accum && accum->opcode == OP_USER)) return gb_fail(GrB_INVALID_VALUE, nullptr, "%s: user-defined operators cannot run on the GPU", fn);
    GB_TRY(matrix_ensure_device(A));
    const int mtc = op->ztype->code;
    Sc r; bool rh = false;
    GB_TRY(dev_reduce_values(A->dev.val, nullptr, A->type->code, A->dev.nnz, op->opcode, mtc, &r, &rh, &A->err));
    const Sc acc = rh ? r : sc_monoid_identity(op->opcode, mtc);
    Sc out = sc_cast(acc, mtc, ctc);
    if (accum) {
        const int atc = accum->xtype->code;
        const Sc old = sc_cast(sc_load(ctc, c, 0), ctc, atc);
        out = sc_cast(sc_binop(accum->opcode, atc, old, sc_cast(acc, mtc, atc)), accum->ztype->code, ctc);
    }
    sc_store(ctc, c, 0, out);
    return GrB_SUCCESS;
}
struct RowReduceArgs { const int64_t *rowptr; const void *val; int atc; int64_t nrows; int op; int mtc; void *tval; uint8_t *tpres; };
__global__ void __launch_bounds__(256) row_reduce_kernel(const RowReduceArgs a) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < a.nrows; r += nwarps) {
        const int64_t rs = a.rowptr[r], re = a.rowptr[r + 1];
        Sc acc; acc.u = 0; int has = 0;
        for (int64_t e = rs + lane; e < re; e += 32) {
            const Sc x = sc_cast(sc_load(a.atc, a.val, (size_t)e), a.atc, a.mtc);
            acc = has ? sc_binop(a.op, a.mtc, acc, x) : x; has = 1;
        }
        for (int o = 16; o > 0; o >>= 1) {
            Sc y; y.u = __shfl_xor_sync(0xffffffffu, (unsigned long long)acc.u, o);
            const int yh = __shfl_xor_sync(0xffffffffu, has, o);
            if (yh) { acc = has ? sc_binop(a.op, a.mtc, acc, y) : y; has = 1; }
        }
        if (lane == 0) { if (has) sc_store(a.mtc, a.tval, (size_t)r, acc); a.tpres[r] = (uint8_t)has; }
    }
}
static GrB_Info mat_reduce_vector(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_BinaryOp op, const GrB_Matrix A,
                                  const GrB_Descriptor desc, const char *fn) {
    GB_VEC_OK(w, fn); GB_MAT_OK(A, fn);
    if (mask) GB_VEC_OK(mask, fn);
    if (!op) return gb_fail(GrB_NULL_POINTER, nullptr, "%s: NULL operator", fn);
    if (op->magic != GB_MAGIC) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "%s: invalid operator", fn);
    GB_TRY(gb_refuse_positional_accum(accum, fn));
    if (op->opcode == OP_USER || (accum && accum->opcode == OP_USER)) return gb_fail(GrB_INVALID_VALUE, nullptr, "%s: user-defined operators cannot run on the GPU", fn);
    GB_TRY(gb_refuse_positional(op, fn));
    const DescFlags f = desc_flags(desc);
    const uint64_t rows = f.tran0 ? A->ncols : A->nrows;
    if (w->n != rows || (mask && mask->n != rows)) return gb_fail(GrB_DIMENSION_MISMATCH, &w->err, "%s: dimensions do not match", fn);
    GB_NEED_DEVICE(&w->err, fn);
    Csr *src; GB_TRY(source_csr(A, f.tran0, &src));
    RowReduceArgs a{};
    a.rowptr = src->rowptr; a.val = src->val; a.atc = A->type->code; a.nrows = src->nrows; a.op = op->opcode; a.mtc = op->ztype->code;
    DevBuf<void> tval; DevBuf<uint8_t> tpres;
    GB_TRY(tval.alloc((size_t)rows * tc_size(a.mtc) + 16, &w->err));
    GB_TRY(tpres.alloc((size_t)rows, &w->err));
    a.tval = tval; a.tpres = tpres;
    row_reduce_kernel<<<grid_for(a.nrows * 32), 256, 0, G.stream>>>(a); GB_LAUNCHED();
    return vector_write(w, mask, accum, f, DenseForm{std::move(tval), std::move(tpres)}, a.mtc, false, nullptr);
}
extern "C" GrB_Info GrB_Matrix_reduce_Monoid(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_Monoid monoid, const GrB_Matrix A, const GrB_Descriptor desc) {
    GB_LOCK; GB_CHECK_INIT;
    if (!monoid) return gb_fail(GrB_NULL_POINTER, nullptr, "GrB_Matrix_reduce_Monoid: NULL monoid");
    return mat_reduce_vector(w, mask, accum, monoid->op, A, desc, "GrB_Matrix_reduce_Monoid");
}
extern "C" GrB_Info GrB_Matrix_reduce_BinaryOp(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_BinaryOp op, const GrB_Matrix A, const GrB_Descriptor desc) {
    GB_LOCK; GB_CHECK_INIT;
    return mat_reduce_vector(w, mask, accum, op, A, desc, "GrB_Matrix_reduce_BinaryOp");
}

// ------------------------------------------------------------------ eWiseAdd / eWiseMult: merge of two sorted rows
struct MergeArgs {
    const int64_t *a_ptr; const uint32_t *a_col; const void *a_val; int atc;
    const int64_t *b_ptr; const uint32_t *b_col; const void *b_val; int btc;
    int64_t nrows; int mult; int op; int xtc, ztc;
    int64_t *o_ptr; uint32_t *o_col; void *o_val;
};
// one thread per row (two-pointer merge).  FILL = false: sizes only.
template <bool FILL>
__global__ void merge_rows_kernel(const MergeArgs a) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < a.nrows; r += (int64_t)gridDim.x * blockDim.x) {
        int64_t i = a.a_ptr[r], j = a.b_ptr[r];
        const int64_t ie = a.a_ptr[r + 1], je = a.b_ptr[r + 1];
        int64_t o = FILL ? a.o_ptr[r] : 0;
        while (i < ie || j < je) {
            const uint32_t ca = i < ie ? a.a_col[i] : 0xffffffffu, cb = j < je ? a.b_col[j] : 0xffffffffu;
            if (ca == cb) {
                if (FILL) {
                    a.o_col[o] = ca;
                    sc_store(a.ztc, a.o_val, (size_t)o, sc_binop(a.op, a.xtc, sc_cast(sc_load(a.atc, a.a_val, (size_t)i), a.atc, a.xtc),
                                                                  sc_cast(sc_load(a.btc, a.b_val, (size_t)j), a.btc, a.xtc)));
                }
                ++o; ++i; ++j;
            } else if (ca < cb) {
                if (!a.mult) { if (FILL) { a.o_col[o] = ca; sc_store(a.ztc, a.o_val, (size_t)o, sc_cast(sc_load(a.atc, a.a_val, (size_t)i), a.atc, a.ztc)); } ++o; }
                ++i;
            } else {
                if (!a.mult) { if (FILL) { a.o_col[o] = cb; sc_store(a.ztc, a.o_val, (size_t)o, sc_cast(sc_load(a.btc, a.b_val, (size_t)j), a.btc, a.ztc)); } ++o; }
                ++j;
            }
        }
        if (!FILL) a.o_ptr[r] = o;
    }
}
static GrB_Info mat_ewise(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const GrB_BinaryOp op, const GrB_Matrix A, const GrB_Matrix B,
                          const GrB_Descriptor desc, int mult, const char *fn) {
    GB_MAT_OK(C, fn); GB_MAT_OK(A, fn); GB_MAT_OK(B, fn);
    if (Mask) GB_MAT_OK(Mask, fn);
    if (!op) return gb_fail(GrB_NULL_POINTER, nullptr, "%s: NULL operator", fn);
    if (op->magic != GB_MAGIC || (accum && accum->magic != GB_MAGIC)) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "%s: invalid operator", fn);
    GB_TRY(gb_refuse_positional_accum(accum, fn));
    if (op->opcode == OP_USER || (accum && accum->opcode == OP_USER)) return gb_fail(GrB_INVALID_VALUE, nullptr, "%s: user-defined operators cannot run on the GPU", fn);
    GB_TRY(gb_refuse_positional(op, fn));
    std::string *err = &C->err;
    const DescFlags f = desc_flags(desc);
    const uint64_t an = f.tran0 ? A->ncols : A->nrows, am = f.tran0 ? A->nrows : A->ncols;
    const uint64_t bn = f.tran1 ? B->ncols : B->nrows, bm = f.tran1 ? B->nrows : B->ncols;
    if (an != bn || am != bm || C->nrows != an || C->ncols != am || (Mask && (Mask->nrows != an || Mask->ncols != am)))
        return gb_fail(GrB_DIMENSION_MISMATCH, err, "%s: dimensions do not match", fn);
    GB_NEED_DEVICE(err, fn);
    Csr *sa, *sb; GB_TRY(source_csr(A, f.tran0, &sa)); GB_TRY(source_csr(B, f.tran1, &sb));
    MergeArgs a{};
    a.a_ptr = sa->rowptr; a.a_col = sa->col; a.a_val = sa->val; a.atc = A->type->code;
    a.b_ptr = sb->rowptr; a.b_col = sb->col; a.b_val = sb->val; a.btc = B->type->code;
    a.nrows = sa->nrows; a.mult = mult; a.op = op->opcode; a.xtc = op->xtype->code; a.ztc = op->ztype->code;
    Csr T;
    GB_TRY(csr_from_row_counts(sa->nrows, sa->ncols, tc_size(a.ztc), T, err,
        [&](int64_t *rowptr) {
            CU_TRY(cudaMemsetAsync(rowptr, 0, ((size_t)a.nrows + 1) * 8, G.stream), err);
            a.o_ptr = rowptr;
            merge_rows_kernel<false><<<grid_for(a.nrows), 256, 0, G.stream>>>(a); GB_LAUNCHED();
            return GrB_SUCCESS;
        },
        [&](Csr &t) {
            a.o_col = t.col; a.o_val = t.val;
            merge_rows_kernel<true><<<grid_for(a.nrows), 256, 0, G.stream>>>(a); GB_LAUNCHED();
            return GrB_SUCCESS;
        }));
    return matrix_writeback(C, Mask, accum, f, std::move(T), a.ztc, false, err);
}
#define GB_MAT_EWISE(NAME, KIND, OPEXPR, MULT) \
    extern "C" GrB_Info NAME(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const KIND op, const GrB_Matrix A, const GrB_Matrix B, const GrB_Descriptor desc) { \
        GB_LOCK; GB_CHECK_INIT; if (!op) return gb_fail(GrB_NULL_POINTER, nullptr, #NAME ": NULL operator"); \
        GB_TRY(gb_refuse_positional(op, #NAME)); \
        return mat_ewise(C, Mask, accum, OPEXPR, A, B, desc, MULT, #NAME); }
GB_MAT_EWISE(GrB_Matrix_eWiseAdd_BinaryOp, GrB_BinaryOp, op, 0)
GB_MAT_EWISE(GrB_Matrix_eWiseAdd_Monoid, GrB_Monoid, op->op, 0)
GB_MAT_EWISE(GrB_Matrix_eWiseAdd_Semiring, GrB_Semiring, op->add->op, 0)
GB_MAT_EWISE(GrB_Matrix_eWiseMult_Monoid, GrB_Monoid, op->op, 1)
GB_MAT_EWISE(GrB_Matrix_eWiseMult_Semiring, GrB_Semiring, op->mul, 1)
extern "C" GrB_Info GrB_Matrix_eWiseMult_BinaryOp(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const GrB_BinaryOp op, const GrB_Matrix A,
                                                   const GrB_Matrix B, const GrB_Descriptor desc) {
    GB_LOCK; GB_CHECK_INIT;
    return mat_ewise(C, Mask, accum, op, A, B, desc, 1, "GrB_Matrix_eWiseMult_BinaryOp");
}

#define GB_MAT_TYPED(TN, CT, TC) \
    extern "C" GrB_Info GrB_Matrix_reduce_##TN(CT *c, const GrB_BinaryOp accum, const GrB_Monoid m, const GrB_Matrix A, const GrB_Descriptor d) { \
        (void)d; GB_LOCK; GB_CHECK_INIT; return mat_reduce_scalar(c, TC, accum, m, A, "GrB_Matrix_reduce_" #TN); } \
    extern "C" GrB_Info GrB_Matrix_apply_BinaryOp1st_##TN(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const GrB_BinaryOp op, CT x, const GrB_Matrix A, const GrB_Descriptor desc) { \
        GB_LOCK; GB_CHECK_INIT; return mat_bind(C, Mask, accum, op, 1, &x, TC, A, desc, "GrB_Matrix_apply_BinaryOp1st_" #TN); } \
    extern "C" GrB_Info GrB_Matrix_apply_BinaryOp2nd_##TN(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const GrB_BinaryOp op, const GrB_Matrix A, CT y, const GrB_Descriptor desc) { \
        GB_LOCK; GB_CHECK_INIT; return mat_bind(C, Mask, accum, op, 0, &y, TC, A, desc, "GrB_Matrix_apply_BinaryOp2nd_" #TN); }
GB_MAT_TYPED(BOOL, bool, TC_BOOL) GB_MAT_TYPED(INT8, int8_t, TC_INT8) GB_MAT_TYPED(INT16, int16_t, TC_INT16) GB_MAT_TYPED(INT32, int32_t, TC_INT32)
GB_MAT_TYPED(INT64, int64_t, TC_INT64) GB_MAT_TYPED(UINT8, uint8_t, TC_UINT8) GB_MAT_TYPED(UINT16, uint16_t, TC_UINT16)
GB_MAT_TYPED(UINT32, uint32_t, TC_UINT32) GB_MAT_TYPED(UINT64, uint64_t, TC_UINT64) GB_MAT_TYPED(FP32, float, TC_FP32) GB_MAT_TYPED(FP64, double, TC_FP64)
