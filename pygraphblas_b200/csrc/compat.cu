// compat.cu -- the part of the GraphBLAS C API that is NOT the mxm/mxv/vxm hot path but that the
// unmodified reference package touches at import time or around its hot-path tests (SURVEY.md
// section 8b): GxB_Scalar, options, select-operator handles, complex type handles, resize and
// memoryUsage.  Handle plumbing only: nothing here computes (every arithmetic entry point lives in
// spmv*.cu / spgemm.cu / vector_ops.cu / matrix_ops.cu and needs the GPU).  What the library does not
// implement is a generated stub that refuses (compat_stubs.inc).
#include "common.cuh"
#include <stdarg.h>
#include <string.h>
#include <algorithm>
#include "../../include/b200grb_compat.h"


static GB_Type_opaque type_FC32 = {GB_MAGIC, TC_COUNT, 8, "FC32"};
static GB_Type_opaque type_FC64 = {GB_MAGIC, TC_COUNT + 1, 16, "FC64"};
static const GrB_Index gb_all_sentinel = 0;
extern "C" {
GrB_Type GxB_FC32 = &type_FC32, GxB_FC64 = &type_FC64;
const GrB_Index *GrB_ALL = &gb_all_sentinel;
const double GxB_ALWAYS_HYPER = 1.0, GxB_NEVER_HYPER = -1.0, GxB_HYPER_DEFAULT = 0.0625;
#define GB_SELOP(N) static GB_SelectOp_opaque selop_##N = {GB_MAGIC, "GxB_" #N, SEL_##N}; GxB_SelectOp GxB_##N = &selop_##N;
GB_SELOP(TRIL) GB_SELOP(TRIU) GB_SELOP(DIAG) GB_SELOP(OFFDIAG) GB_SELOP(NONZERO) GB_SELOP(EQ_ZERO) GB_SELOP(GT_ZERO) GB_SELOP(GE_ZERO)
GB_SELOP(LT_ZERO) GB_SELOP(LE_ZERO) GB_SELOP(NE_THUNK) GB_SELOP(EQ_THUNK) GB_SELOP(GT_THUNK) GB_SELOP(GE_THUNK) GB_SELOP(LT_THUNK) GB_SELOP(LE_THUNK)
}

#include "compat_stubs.inc"

// ------------------------------------------------------------------ GxB_Scalar
static bool valid_scalar(const GxB_Scalar s) { return s && s->magic == GB_MAGIC; }
extern "C" GrB_Info GxB_Scalar_new(GxB_Scalar *s, GrB_Type type) {
    if (!s) return gb_fail(GrB_NULL_POINTER, nullptr, "GxB_Scalar_new: NULL");
    if (!type || type->magic != GB_MAGIC || type->code >= TC_COUNT) return gb_fail(GrB_DOMAIN_MISMATCH, nullptr, "GxB_Scalar_new: unsupported type");
    *s = new GB_Scalar_opaque{GB_MAGIC, type, false, Sc{}};
    return GrB_SUCCESS;
}
extern "C" GrB_Info GxB_Scalar_dup(GxB_Scalar *s, const GxB_Scalar t) {
    if (!s) return gb_fail(GrB_NULL_POINTER, nullptr, "GxB_Scalar_dup: NULL");
    if (!valid_scalar(t)) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "GxB_Scalar_dup: invalid scalar");
    *s = new GB_Scalar_opaque(*t); return GrB_SUCCESS;
}
extern "C" GrB_Info GxB_Scalar_free(GxB_Scalar *s) {
    if (!s || !*s) return GrB_SUCCESS;
    if ((*s)->magic == GB_MAGIC) { (*s)->magic = GB_FREED; delete *s; }
    *s = nullptr; return GrB_SUCCESS;
}
extern "C" GrB_Info GxB_Scalar_clear(GxB_Scalar s) {
    if (!valid_scalar(s)) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "GxB_Scalar_clear: invalid scalar");
    s->has = false; return GrB_SUCCESS;
}
extern "C" GrB_Info GxB_Scalar_nvals(GrB_Index *nvals, const GxB_Scalar s) {
    if (!nvals) return gb_fail(GrB_NULL_POINTER, nullptr, "GxB_Scalar_nvals: NULL");
    if (!valid_scalar(s)) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "GxB_Scalar_nvals: invalid scalar");
    *nvals = s->has ? 1 : 0; return GrB_SUCCESS;
}
extern "C" GrB_Info GxB_Scalar_wait(GxB_Scalar *s) { (void)s; return GrB_SUCCESS; }
extern "C" GrB_Info GxB_Scalar_type(GrB_Type *type, const GxB_Scalar s) {
    if (!type) return gb_fail(GrB_NULL_POINTER, nullptr, "GxB_Scalar_type: NULL");
    if (!valid_scalar(s)) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "GxB_Scalar_type: invalid scalar");
    *type = s->type; return GrB_SUCCESS;
}
static GrB_Info scalar_set(GxB_Scalar s, int tc, const void *x) {
    if (!valid_scalar(s)) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "GxB_Scalar_setElement: invalid scalar");
    s->v = sc_cast(sc_load(tc, x, 0), tc, s->type->code); s->has = true; return GrB_SUCCESS;
}
static GrB_Info scalar_get(void *x, int tc, const GxB_Scalar s) {
    if (!x) return gb_fail(GrB_NULL_POINTER, nullptr, "GxB_Scalar_extractElement: NULL");
    if (!valid_scalar(s)) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "GxB_Scalar_extractElement: invalid scalar");
    if (!s->has) return GrB_NO_VALUE;
    sc_store(tc, x, 0, sc_cast(s->v, s->type->code, tc)); return GrB_SUCCESS;
}
extern "C" GrB_Info GxB_Scalar_fprint(GxB_Scalar s, const char *name, int pr, FILE *f) {
    if (!valid_scalar(s)) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "GxB_Scalar_fprint: invalid scalar");
    if (pr > 0) fprintf(f ? f : stdout, "\n  B200 GraphBLAS %s scalar %s: %d entries\n", s->type->name, name ? name : "", s->has ? 1 : 0);
    return GrB_SUCCESS;
}
extern "C" GrB_Info GxB_SelectOp_fprint(GxB_SelectOp op, const char *name, int pr, FILE *f) {
    if (!op) return gb_fail(GrB_NULL_POINTER, nullptr, "GxB_SelectOp_fprint: NULL");
    if (pr > 0) fprintf(f ? f : stdout, "\n    B200 GraphBLAS SelectOp: %s %s (handle only)\n", name ? name : "", op->name);
    return GrB_SUCCESS;
}
extern "C" GrB_Info GxB_UnaryOp_fprint(GrB_UnaryOp op, const char *name, int pr, FILE *f) {
    (void)op; if (pr > 0) fprintf(f ? f : stdout, "\n    B200 GraphBLAS UnaryOp: %s (handle only)\n", name ? name : "");
    return GrB_SUCCESS;
}

#define GB_COMPAT_TYPED(TN, CT, TC) \
    extern "C" GrB_Info GxB_Scalar_setElement_##TN(GxB_Scalar s, CT x) { return scalar_set(s, TC, &x); } \
    extern "C" GrB_Info GxB_Scalar_extractElement_##TN(CT *x, const GxB_Scalar s) { return scalar_get(x, TC, s); }
GB_COMPAT_TYPED(BOOL, bool, TC_BOOL) GB_COMPAT_TYPED(INT8, int8_t, TC_INT8) GB_COMPAT_TYPED(INT16, int16_t, TC_INT16) GB_COMPAT_TYPED(INT32, int32_t, TC_INT32)
GB_COMPAT_TYPED(INT64, int64_t, TC_INT64) GB_COMPAT_TYPED(UINT8, uint8_t, TC_UINT8) GB_COMPAT_TYPED(UINT16, uint16_t, TC_UINT16)
GB_COMPAT_TYPED(UINT32, uint32_t, TC_UINT32) GB_COMPAT_TYPED(UINT64, uint64_t, TC_UINT64) GB_COMPAT_TYPED(FP32, float, TC_FP32) GB_COMPAT_TYPED(FP64, double, TC_FP64)

// ------------------------------------------------------------------ resize / memory usage
extern "C" GrB_Info GrB_Matrix_resize(GrB_Matrix A, GrB_Index nrows, GrB_Index ncols) {
    GB_LOCK;
    if (!gb_valid_matrix(A)) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "GrB_Matrix_resize: invalid matrix");
    if (nrows == 0 || ncols == 0) return gb_fail(GrB_INVALID_VALUE, &A->err, "GrB_Matrix_resize: dimensions must be positive");
    GB_TRY(matrix_ensure_host(A));
    matrix_invalidate_device(A);
    const size_t sz = A->type->size; size_t o = 0;
    for (size_t k = 0; k < A->hi.size(); ++k) if (A->hi[k] < nrows && A->hj[k] < ncols) {
        A->hi[o] = A->hi[k]; A->hj[o] = A->hj[k]; memmove(&A->hx[o * sz], &A->hx[k * sz], sz); ++o;
    }
    A->hi.resize(o); A->hj.resize(o); A->hx.resize(o * sz);
    A->nrows = nrows; A->ncols = ncols;
    return GrB_SUCCESS;
}
extern "C" GrB_Info GrB_Vector_resize(GrB_Vector v, GrB_Index n) {
    GB_LOCK;
    if (!gb_valid_vector(v)) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "GrB_Vector_resize: invalid vector");
    if (n == 0) return gb_fail(GrB_INVALID_VALUE, &v->err, "GrB_Vector_resize: size must be positive");
    GB_TRY(vector_ensure_host(v));
    vector_invalidate_device(v);
    const size_t sz = v->type->size; size_t o = 0;
    for (size_t k = 0; k < v->hi.size(); ++k) if (v->hi[k] < n) { v->hi[o] = v->hi[k]; memmove(&v->hx[o * sz], &v->hx[k * sz], sz); ++o; }
    v->hi.resize(o); v->hx.resize(o * sz); v->n = n;
    return GrB_SUCCESS;
}
extern "C" GrB_Info GxB_Matrix_memoryUsage(size_t *size, const GrB_Matrix A) {
    if (!size) return gb_fail(GrB_NULL_POINTER, nullptr, "GxB_Matrix_memoryUsage: NULL");
    if (!gb_valid_matrix(A)) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "GxB_Matrix_memoryUsage: invalid matrix");
    *size = sizeof(*A) + A->hi.size() * (16 + A->type->size) + (A->dev.valid ? (size_t)A->dev.nnz * (4 + A->type->size) + ((size_t)A->dev.nrows + 1) * 12 : 0)
          + (A->dn.valid ? (size_t)(A->nrows * A->ncols) * (A->type->size + (A->dn.pres ? 1 : 0)) : 0);
    return GrB_SUCCESS;
}
extern "C" GrB_Info GxB_Vector_memoryUsage(size_t *size, const GrB_Vector v) {
    if (!size) return gb_fail(GrB_NULL_POINTER, nullptr, "GxB_Vector_memoryUsage: NULL");
    if (!gb_valid_vector(v)) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "GxB_Vector_memoryUsage: invalid vector");
    *size = sizeof(*v) + v->hi.size() * (8 + v->type->size) + (v->dv.valid ? (size_t)v->n * (1 + v->type->size) : 0);
    return GrB_SUCCESS;
}

// ------------------------------------------------------------------ options (variadic, as reference: pygraphblas/base.py:49-130 passes them)
static struct { int nthreads = 1; double chunk = 65536; int burble = 0; double hyper = 0.0625; int format = GxB_BY_ROW; double bitmap[8] = {0.04, 0.05, 0.06, 0.08, 0.10, 0.20, 0.30, 0.40}; } g_opt;
extern "C" GrB_Info GxB_Global_Option_set(GxB_Option_Field field, ...) {
    va_list ap; va_start(ap, field); GrB_Info r = GrB_SUCCESS;
    switch (field) {
        case GxB_GLOBAL_NTHREADS: g_opt.nthreads = va_arg(ap, int); break;
        case GxB_GLOBAL_CHUNK: g_opt.chunk = va_arg(ap, double); break;
        case GxB_BURBLE: g_opt.burble = va_arg(ap, int); G.burble = g_opt.burble; break;
        case GxB_HYPER_SWITCH: g_opt.hyper = va_arg(ap, double); break;
        case GxB_BITMAP_SWITCH: { const double *p = va_arg(ap, const double *); if (p) memcpy(g_opt.bitmap, p, sizeof g_opt.bitmap); } break;
        case GxB_FORMAT: { const int f = va_arg(ap, int);                // default storage hint of new matrices: recorded, no effect on the HBM layout
            if (f == GxB_BY_ROW || f == GxB_BY_COL) g_opt.format = f; else r = gb_fail(GrB_INVALID_VALUE, nullptr, "GxB_FORMAT: GxB_BY_ROW or GxB_BY_COL"); } break;
        default: r = gb_fail(GrB_INVALID_VALUE, nullptr, "GxB_Global_Option_set: unknown option %d", (int)field);
    }
    va_end(ap); return r;
}
extern "C" GrB_Info GxB_Global_Option_get(GxB_Option_Field field, ...) {
    va_list ap; va_start(ap, field); GrB_Info r = GrB_SUCCESS;
    void *out = va_arg(ap, void *);
    if (!out) r = gb_fail(GrB_NULL_POINTER, nullptr, "GxB_Global_Option_get: NULL");
    else switch (field) {
        case GxB_GLOBAL_NTHREADS: *(int *)out = g_opt.nthreads; break;
        case GxB_GLOBAL_CHUNK: *(double *)out = g_opt.chunk; break;
        case GxB_BURBLE: *(int *)out = G.burble; break;
        case GxB_HYPER_SWITCH: *(double *)out = g_opt.hyper; break;
        case GxB_BITMAP_SWITCH: memcpy(out, g_opt.bitmap, sizeof g_opt.bitmap); break;
        case GxB_FORMAT: *(int *)out = g_opt.format; break;
        case GxB_MODE: *(int *)out = GrB_NONBLOCKING; break;
        default: r = gb_fail(GrB_INVALID_VALUE, nullptr, "GxB_Global_Option_get: unknown option %d", (int)field);
    }
    va_end(ap); return r;
}
static GrB_Info object_option_set(GBObjOpts &o, GxB_Option_Field field, va_list ap) {
    switch (field) {
        case GxB_HYPER_SWITCH: o.hyper = va_arg(ap, double); return GrB_SUCCESS;
        case GxB_BITMAP_SWITCH: (void)va_arg(ap, double); return GrB_SUCCESS;
        case GxB_SPARSITY_CONTROL: o.sparsity = va_arg(ap, int); return GrB_SUCCESS;      // HBM layout is fixed (CSR / dense+presence)
        case GxB_FORMAT: { const int f = va_arg(ap, int);                                   // a storage hint: recorded, no effect
            if (f != GxB_BY_ROW && f != GxB_BY_COL) return gb_fail(GrB_INVALID_VALUE, nullptr, "GxB_FORMAT: GxB_BY_ROW or GxB_BY_COL");
            o.format = f; return GrB_SUCCESS; }
        default: return gb_fail(GrB_INVALID_VALUE, nullptr, "Option_set: unknown option %d", (int)field);
    }
}
static GrB_Info object_option_get(const GBObjOpts &o, GxB_Option_Field field, bool huge, va_list ap) {
    void *out = va_arg(ap, void *);
    if (!out) return gb_fail(GrB_NULL_POINTER, nullptr, "Option_get: NULL");
    switch (field) {
        case GxB_HYPER_SWITCH: *(double *)out = o.hyper; return GrB_SUCCESS;
        case GxB_BITMAP_SWITCH: *(double *)out = 0.04; return GrB_SUCCESS;
        case GxB_FORMAT: *(int *)out = o.format; return GrB_SUCCESS;
        case GxB_SPARSITY_CONTROL: *(int *)out = o.sparsity; return GrB_SUCCESS;
        case GxB_SPARSITY_STATUS: *(int *)out = huge ? GxB_HYPERSPARSE : GxB_SPARSE; return GrB_SUCCESS;
        default: return gb_fail(GrB_INVALID_VALUE, nullptr, "Option_get: unknown option %d", (int)field);
    }
}
extern "C" GrB_Info GxB_Matrix_Option_set(GrB_Matrix A, GxB_Option_Field field, ...) {
    if (!gb_valid_matrix(A)) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "GxB_Matrix_Option_set: invalid matrix");
    va_list ap; va_start(ap, field); const GrB_Info r = object_option_set(A->opts, field, ap); va_end(ap); return r;
}
extern "C" GrB_Info GxB_Matrix_Option_get(GrB_Matrix A, GxB_Option_Field field, ...) {
    if (!gb_valid_matrix(A)) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "GxB_Matrix_Option_get: invalid matrix");
    // host-only tuple form (no HBM CSR yet, or dimensions beyond 2^31) reports HYPERSPARSE, tests/test_matrix.py:555,570;
    // a dense form reports FULL (no presence bytes) or BITMAP
    va_list ap; va_start(ap, field);
    GrB_Info r;
    if (field == GxB_SPARSITY_STATUS && A->dn.valid) {
        int *out = va_arg(ap, int *);
        if (out) { *out = A->dn.pres ? GxB_BITMAP : GxB_FULL; r = GrB_SUCCESS; }
        else r = gb_fail(GrB_NULL_POINTER, nullptr, "Option_get: NULL");
    } else r = object_option_get(A->opts, field, !A->dev.valid, ap);
    va_end(ap); return r;
}
extern "C" GrB_Info GxB_Vector_Option_set(GrB_Vector v, GxB_Option_Field field, ...) {
    if (!gb_valid_vector(v)) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "GxB_Vector_Option_set: invalid vector");
    va_list ap; va_start(ap, field); const GrB_Info r = object_option_set(v->opts, field, ap); va_end(ap); return r;
}
extern "C" GrB_Info GxB_Vector_Option_get(GrB_Vector v, GxB_Option_Field field, ...) {
    if (!gb_valid_vector(v)) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "GxB_Vector_Option_get: invalid vector");
    va_list ap; va_start(ap, field); const GrB_Info r = object_option_get(v->opts, field, !v->dv.valid, ap); va_end(ap); return r;
}
