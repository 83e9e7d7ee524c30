/* b200grb.h -- C ABI of libb200grb.so, the H100-native GraphBLAS hot-path core.
 *
 * This is the drop-in boundary of the project: a subset of the GraphBLAS C API
 * (spec 1.3 / SuiteSparse:GraphBLAS 5.x naming, numbering and calling
 * conventions) that the reference, Graphegon/pygraphblas, binds through CFFI
 * as `suitesparse_graphblas.lib` (reference: pygraphblas/__init__.py:248,
 * reference: pygraphblas/base.py:7).  The three hot entry points are
 *
 *     GrB_mxm   <- reference: pygraphblas/matrix.py:2574   (Matrix.mxm, @, @=, **)
 *     GrB_mxv   <- reference: pygraphblas/matrix.py:2716   (Matrix.mxv, @)
 *     GrB_vxm   <- reference: pygraphblas/vector.py:961    (Vector.vxm, @)
 *
 * everything else in this file is the handle plumbing those calls need
 * (create / fill / read / sync / destroy; SURVEY.md section 8b).
 *
 * Conventions (same as the reference's binding expects):
 *   - every function returns GrB_Info; 0 = success, 1 = GrB_NO_VALUE, 2..13 errors
 *     numbered as reference: pygraphblas/base.py:189-203 maps them;
 *   - objects are opaque pointers, allocated by *_new/_dup, released by *_free(&h)
 *     (which also accepts NULL handles and builtin objects,
 *     reference: pygraphblas/descriptor.py:76-78);
 *   - plain C types only: no CUDA, torch or C++ types appear in any signature;
 *   - arithmetic runs ONLY on the GPU (sm_90a kernels).  Without a CUDA device
 *     the library loads and all host-side plumbing works, but GrB_mxm/mxv/vxm
 *     return GrB_PANIC with an explanatory GrB_*_error string: there is no CPU
 *     fallback.
 *
 * The file is written so that cffi can parse it after dropping preprocessor
 * lines (see pygraphblas_b200/_ffi.py).
 */
#ifndef B200GRB_H
#define B200GRB_H

#include <stdint.h>
#include <stddef.h>
#include <stdbool.h>
#include <stdio.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef uint64_t GrB_Index;

typedef struct GB_Type_opaque       *GrB_Type;
typedef struct GB_UnaryOp_opaque    *GrB_UnaryOp;
typedef struct GB_BinaryOp_opaque   *GrB_BinaryOp;
typedef struct GB_Monoid_opaque     *GrB_Monoid;
typedef struct GB_Semiring_opaque   *GrB_Semiring;
typedef struct GB_Descriptor_opaque *GrB_Descriptor;
typedef struct GB_Vector_opaque     *GrB_Vector;
typedef struct GB_Matrix_opaque     *GrB_Matrix;

typedef void (*GxB_binary_function)(void *, const void *, const void *);

/* reference: pygraphblas/base.py:189-203 */
typedef enum {
    GrB_SUCCESS = 0,
    GrB_NO_VALUE = 1,
    GrB_UNINITIALIZED_OBJECT = 2,
    GrB_INVALID_OBJECT = 3,
    GrB_NULL_POINTER = 4,
    GrB_INVALID_VALUE = 5,
    GrB_INVALID_INDEX = 6,
    GrB_DOMAIN_MISMATCH = 7,
    GrB_DIMENSION_MISMATCH = 8,
    GrB_OUTPUT_NOT_EMPTY = 9,
    GrB_OUT_OF_MEMORY = 10,
    GrB_INSUFFICIENT_SPACE = 11,
    GrB_INDEX_OUT_OF_BOUNDS = 12,
    GrB_PANIC = 13
} GrB_Info;

typedef enum { GrB_NONBLOCKING = 0, GrB_BLOCKING = 1 } GrB_Mode;

/* descriptor fields / values: reference: pygraphblas/descriptor.py:10-145 */
typedef enum {
    GrB_OUTP = 0,
    GrB_MASK = 1,
    GrB_INP0 = 2,
    GrB_INP1 = 3,
    GxB_DESCRIPTOR_NTHREADS = 5,
    GxB_DESCRIPTOR_CHUNK = 7,
    GxB_SORT = 35,
    GxB_AxB_METHOD = 1000
} GrB_Desc_Field;

typedef enum {
    GxB_DEFAULT = 0,
    GrB_REPLACE = 1,
    GrB_COMP = 2,
    GrB_TRAN = 3,
    GrB_STRUCTURE = 4,
    GxB_AxB_GUSTAVSON = 1001,
    GxB_AxB_DOT = 1003,
    GxB_AxB_HASH = 1004,
    GxB_AxB_SAXPY = 1005
} GrB_Desc_Value;

/* ------------------------------------------------------------------ lifecycle */
GrB_Info GrB_init(GrB_Mode mode);
GrB_Info GrB_finalize(void);
/* last error text of the calling thread (library-owned string) */
const char *B200_last_error(void);

/* ------------------------------------------------------------------ types */
extern GrB_Type GrB_BOOL, GrB_INT8, GrB_INT16, GrB_INT32, GrB_INT64,
                GrB_UINT8, GrB_UINT16, GrB_UINT32, GrB_UINT64, GrB_FP32, GrB_FP64;
GrB_Info GxB_Type_size(size_t *size, GrB_Type type);
/* B200 extension: the name ("FP32", ...) and the small integer code of a type */
GrB_Info B200_Type_info(const char **name, int *code, GrB_Type type);

/* ------------------------------------------------------------------ operators */
#include "b200grb_ops.h"

GrB_Info GrB_BinaryOp_new(GrB_BinaryOp *op, GxB_binary_function fn, GrB_Type ztype, GrB_Type xtype, GrB_Type ytype);
GrB_Info GrB_BinaryOp_free(GrB_BinaryOp *op);
GrB_Info GxB_BinaryOp_ztype(GrB_Type *ztype, GrB_BinaryOp op);
GrB_Info GxB_BinaryOp_xtype(GrB_Type *xtype, GrB_BinaryOp op);
GrB_Info GxB_BinaryOp_ytype(GrB_Type *ytype, GrB_BinaryOp op);
GrB_Info GrB_Monoid_free(GrB_Monoid *monoid);
GrB_Info GxB_Monoid_operator(GrB_BinaryOp *op, GrB_Monoid monoid);
GrB_Info GrB_Semiring_new(GrB_Semiring *semiring, GrB_Monoid add, GrB_BinaryOp multiply);
GrB_Info GrB_Semiring_free(GrB_Semiring *semiring);
GrB_Info GxB_Semiring_add(GrB_Monoid *add, GrB_Semiring semiring);
GrB_Info GxB_Semiring_multiply(GrB_BinaryOp *multiply, GrB_Semiring semiring);
GrB_Info GxB_BinaryOp_fprint(GrB_BinaryOp op, const char *name, int pr, FILE *f);
GrB_Info GxB_Monoid_fprint(GrB_Monoid monoid, const char *name, int pr, FILE *f);
GrB_Info GxB_Semiring_fprint(GrB_Semiring semiring, const char *name, int pr, FILE *f);
/* B200 extension: look a builtin operator up by its C name; kind 0 = BinaryOp,
 * 1 = Monoid, 2 = Semiring.  *obj receives the same pointer the global holds. */
GrB_Info B200_lookup(void **obj, int kind, const char *name);
GrB_Info B200_object_name(const char **name, int kind, const void *obj);

/* ------------------------------------------------------------------ descriptors */
extern GrB_Descriptor
    GrB_DESC_T1, GrB_DESC_T0, GrB_DESC_T0T1,
    GrB_DESC_C, GrB_DESC_CT1, GrB_DESC_CT0, GrB_DESC_CT0T1,
    GrB_DESC_S, GrB_DESC_ST1, GrB_DESC_ST0, GrB_DESC_ST0T1,
    GrB_DESC_SC, GrB_DESC_SCT1, GrB_DESC_SCT0, GrB_DESC_SCT0T1,
    GrB_DESC_R, GrB_DESC_RT1, GrB_DESC_RT0, GrB_DESC_RT0T1,
    GrB_DESC_RC, GrB_DESC_RCT1, GrB_DESC_RCT0, GrB_DESC_RCT0T1,
    GrB_DESC_RS, GrB_DESC_RST1, GrB_DESC_RST0, GrB_DESC_RST0T1,
    GrB_DESC_RSC, GrB_DESC_RSCT1, GrB_DESC_RSCT0, GrB_DESC_RSCT0T1;
GrB_Info GrB_Descriptor_new(GrB_Descriptor *descriptor);
GrB_Info GrB_Descriptor_free(GrB_Descriptor *descriptor);
GrB_Info GrB_Descriptor_set(GrB_Descriptor desc, GrB_Desc_Field field, GrB_Desc_Value value);
GrB_Info GxB_Desc_set(GrB_Descriptor desc, GrB_Desc_Field field, ...);
GrB_Info GxB_Desc_get(GrB_Descriptor desc, GrB_Desc_Field field, ...);

/* ------------------------------------------------------------------ matrices */
GrB_Info GrB_Matrix_new(GrB_Matrix *A, GrB_Type type, GrB_Index nrows, GrB_Index ncols);
GrB_Info GrB_Matrix_dup(GrB_Matrix *C, const GrB_Matrix A);
GrB_Info GrB_Matrix_free(GrB_Matrix *A);
GrB_Info GrB_Matrix_clear(GrB_Matrix A);
GrB_Info GrB_Matrix_nrows(GrB_Index *nrows, const GrB_Matrix A);
GrB_Info GrB_Matrix_ncols(GrB_Index *ncols, const GrB_Matrix A);
GrB_Info GrB_Matrix_nvals(GrB_Index *nvals, const GrB_Matrix A);
GrB_Info GxB_Matrix_type(GrB_Type *type, const GrB_Matrix A);
GrB_Info GrB_Matrix_wait(GrB_Matrix *A);                       /* 1-arg v1.3 form: matrix.py:3353 */
GrB_Info GrB_Matrix_error(const char **error, const GrB_Matrix A);
GrB_Info GrB_Matrix_removeElement(GrB_Matrix C, GrB_Index i, GrB_Index j);
GrB_Info GrB_transpose(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const GrB_Matrix A, const GrB_Descriptor desc);
GrB_Info GxB_Matrix_fprint(GrB_Matrix A, const char *name, int pr, FILE *f);

/* ------------------------------------------------------------------ vectors */
GrB_Info GrB_Vector_new(GrB_Vector *v, GrB_Type type, GrB_Index n);
GrB_Info GrB_Vector_dup(GrB_Vector *w, const GrB_Vector u);
GrB_Info GrB_Vector_free(GrB_Vector *v);
GrB_Info GrB_Vector_clear(GrB_Vector v);
GrB_Info GrB_Vector_size(GrB_Index *n, const GrB_Vector v);
GrB_Info GrB_Vector_nvals(GrB_Index *nvals, const GrB_Vector v);
GrB_Info GxB_Vector_type(GrB_Type *type, const GrB_Vector v);
GrB_Info GrB_Vector_wait(GrB_Vector *v);
GrB_Info GrB_Vector_error(const char **error, const GrB_Vector v);
GrB_Info GrB_Vector_removeElement(GrB_Vector v, GrB_Index i);
GrB_Info GxB_Vector_fprint(GrB_Vector v, const char *name, int pr, FILE *f);

/* per-type element access / build (setElement, extractElement, extractTuples, build, Monoid_new) */
#include "b200grb_typed.h"

/* ------------------------------------------------------------------ THE HOT PATH
 * C<Mask> = accum(C, op(A) (+).(x) op(B))      reference: pygraphblas/matrix.py:2574
 * w<mask> = accum(w, op(A) (+).(x) u)          reference: pygraphblas/matrix.py:2716
 * w'<mask'> = accum(w', u' (+).(x) op(A))      reference: pygraphblas/vector.py:961
 * Mask, accum and desc may be NULL; the output may alias an input.            */
GrB_Info GrB_mxm(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const GrB_Semiring semiring,
                 const GrB_Matrix A, const GrB_Matrix B, const GrB_Descriptor desc);
GrB_Info GrB_mxv(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_Semiring semiring,
                 const GrB_Matrix A, const GrB_Vector u, const GrB_Descriptor desc);
GrB_Info GrB_vxm(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_Semiring semiring,
                 const GrB_Vector u, const GrB_Matrix A, const GrB_Descriptor desc);

/* ------------------------------------------------------------------ B200 extensions
 * Bulk ingest / egress (the reference has none: Matrix.from_lists loops
 * setElement, reference: pygraphblas/matrix.py:325-330) and device interop.
 * `where`: 0 = the pointers are host memory, 1 = CUDA device memory of the
 * current device (e.g. a torch tensor's data_ptr()), 2 (vector set / export only) = PINNED host
 * memory copied on the library's copy streams, overlapping kernels already enqueued: GraphBLAS
 * non-blocking mode -- an export's data is in host memory after GrB_Vector_wait / B200_device_synchronize. */
GrB_Info B200_Matrix_import_CSR(GrB_Matrix *A, GrB_Type type, GrB_Index nrows, GrB_Index ncols,
                                const int64_t *Ap, const uint32_t *Aj, const void *Ax,
                                GrB_Index nvals, int where);
/* Ap must hold nrows+1, Aj/Ax nvals entries; any pointer may be NULL to skip it.
 * Rows are sorted by column. */
GrB_Info B200_Matrix_export_CSR(const GrB_Matrix A, int64_t *Ap, uint32_t *Aj, void *Ax, int where);
/* dense matrix import: x[nrows*ncols] row-major values of `type`; present[nrows*ncols] bytes, entry (i,j) present where
 * present[i*ncols+j] != 0, or NULL when every entry is present.  where = 0 or 1.  The matrix holds the dense form in HBM
 * (GxB_SPARSITY_STATUS reports GxB_FULL without presence bytes, GxB_BITMAP with them); GrB_mxm with it as the
 * untransposed B runs the dense-operand kernel, and every other operation sees its CSR, built on first use.
 * nrows*ncols must be at most 2^31-1 (GrB_INVALID_VALUE otherwise). */
GrB_Info B200_Matrix_import_dense(GrB_Matrix *A, GrB_Type type, GrB_Index nrows, GrB_Index ncols,
                                  const void *x, const uint8_t *present, int where);
/* dense matrix export of any matrix: x[nrows*ncols] row-major values (0 where absent), present[nrows*ncols] bytes (1 / 0);
 * either pointer may be NULL to skip it.  where = 0 or 1; returns once the data is in place. */
GrB_Info B200_Matrix_export_dense(const GrB_Matrix A, void *x, uint8_t *present, int where);
/* dense import: every position present (present == NULL) or present[i] != 0 */
GrB_Info B200_Vector_import_dense(GrB_Vector *v, GrB_Type type, GrB_Index n,
                                  const void *x, const uint8_t *present, int where);
GrB_Info B200_Vector_export_dense(const GrB_Vector v, void *x, uint8_t *present, int where);
/* refill an existing vector's device buffers from (x, present) without reallocating */
GrB_Info B200_Vector_set_dense(GrB_Vector v, const void *x, const uint8_t *present, int where);
/* raw device buffers of a vector (valid until the vector is next modified or freed):
 * values[n] of the vector's type and present[n] bytes (NULL when all present). */
GrB_Info B200_Vector_device_ptrs(GrB_Vector v, void **values, uint8_t **present);
/* the CUDA stream (cudaStream_t) all kernels of this library are launched on */
GrB_Info B200_get_stream(void **stream);
GrB_Info B200_device_synchronize(void);
/* 1 when a CUDA device is usable, 0 otherwise (host plumbing only) */
int B200_have_device(void);
/* statistics of the last hot-path call: kernel launch count (cumulative) */
uint64_t B200_kernel_launches(void);
/* allocation test seam: the k-th device allocation from now fails with GrB_OUT_OF_MEMORY before it reaches
 * the device (k = 0 switches it off); and the number of device blocks allocated and not yet freed */
void B200_debug_fail_alloc(int64_t k);
int64_t B200_debug_live_allocs(void);
/* wide-route test seam: chunk > 0 puts every GrB_mxv / GrB_vxm, every transpose and the SpMM, dense-left and SDDMM routes of
 * GrB_mxm on the code that serves matrices with 2^32 or more entries (64-bit entry offsets; transposes and SDDMM masks cut into
 * chunks of `chunk` entries), whatever the matrix's size; 0 switches it off.  The 32-bit row offsets stay built for the other
 * operations.  The unmasked and complemented-mask CSR x CSR products of GrB_mxm stay on their 32-bit kernels under it */
void B200_debug_wide(int64_t chunk);
/* wide-route test seam of the unmasked and complemented-mask CSR x CSR products of GrB_mxm: chunk > 0 puts every such product on
 * the code that serves operands with 2^32 or more entries (row panels of A and of the mask's blocking entries with 32-bit
 * offsets, B's 64-bit offsets), whatever the operands' size, with panels of at most `chunk` entries of A and of the mask.
 * result_limit > 0 stands for 2^32 in that route's size rule (a product whose result would have that many entries or more
 * is refused with GrB_INVALID_VALUE), and spa_budget > 0 for the 2^32 bytes the dense accumulators of one panel may take
 * (0: the defaults).  chunk = 0 switches all three off */
void B200_debug_wide_gemm(int64_t chunk, int64_t result_limit, int64_t spa_budget);
/* kernel-path test seam: the paths the last GrB_mxv / GrB_vxm / GrB_mxm took, separated by ';' ("run",
 * "run (sparse u)", "run+hot-table (TMA-staged)", "pull", "push", "esc-small", "esc-medium", "spa", "spa-split", "masked-warp", "stream-L",
 * "dot", ...); recorded whether the burble is on or not, valid until the next such call.  Host-decided variants follow
 * their entry as "key=value" tokens: "filter=exact" or "filter=bloom" after each "stream-S" / "stream-M" / "stream-L"
 * (the mask-row membership filter is an exact bitmap or a one-hash Bloom filter), and "mxv=in-place" after an mxv / vxm
 * entry when the product was formed straight in w's buffers.  "offsets=64" follows the first entry of a call that ran on the
 * wide route (64-bit offsets).  An unmasked or complemented-mask product lists "esc-small", "esc-medium", "spa" and "spa-split"
 * once each, in that order, however many row panels ran them, with "offsets=64" after the first on the wide route; a
 * complemented-mask product whose rows took the pull route lists "pull" after them, followed by "pull=dot" (GxB_AxB_DOT on
 * the descriptor) or "pull=auto" (the B200GRB_MXM_PULL rule) */
const char *B200_debug_last_kernel(void);
/* per-matrix SpGEMM/SpMV work figures of the most recent GrB_mxm (flops = number of
 * multiplies, nnz_out = nvals of the product T as the kernels formed it, before the accumulator and the write-back:
 * unmasked calls report the whole product, masked ones (complemented or not) only the entries the mask lets through) */
GrB_Info B200_last_mxm_stats(uint64_t *flops, uint64_t *nnz_out);
/* ------------------------------------------------------------------ multi-GPU exchange (csrc/dist.cu)
 * One process per GPU; A is 1-D row-block partitioned (SURVEY.md section 8e).  The library moves the output
 * slices itself, with its own kernels over CUDA-IPC-mapped peer HBM (NVLink / NVSwitch): the host only carries
 * the 64-byte IPC handles between the processes.  Replaces nothing in the reference (which is single-process,
 * reference: pygraphblas/matrix.py:2586-2726); it is the exchange step north_star asks for after GrB_mxv.  */
typedef struct B200_Comm_opaque *B200_Comm;
/* a communicator for replicated vectors of n values of `type` among `world` ranks (this process is `rank`) */
GrB_Info B200_Comm_create(B200_Comm *comm, int rank, int world, GrB_Index n, GrB_Type type);
/* this rank's 64-byte IPC handle; gather all ranks' handles (rank order) and pass them to connect */
GrB_Info B200_Comm_handle(B200_Comm comm, void *handle64);
GrB_Info B200_Comm_connect(B200_Comm comm, const void *all_handles);
GrB_Info B200_Comm_free(B200_Comm *comm);
/* all-gather: positions [row0, row0 + size(slice)) of the replicated vector := slice, on EVERY rank, for all ranks'
 * slices (row0 a multiple of 16); enqueued on the library stream, complete (stream order) when it returns */
GrB_Info B200_Comm_allgather(B200_Comm comm, const GrB_Vector slice, GrB_Index row0);
/* all-reduce: every rank passes a full-length partial; the replicated vector := the monoid fold of the partials
 * present at each position, taken in rank order (deterministic) */
GrB_Info B200_Comm_allreduce(B200_Comm comm, const GrB_Vector partial, GrB_Monoid monoid);
/* the replicated vector produced by the last collective, as a GrB_Vector that borrows the communicator's buffer
 * (valid until the next collective on this communicator; usable as the input of GrB_mxv / GrB_vxm) */
GrB_Info B200_Comm_result(B200_Comm comm, GrB_Vector *view);
/* flags-only round: every rank has enqueued everything before this point */
GrB_Info B200_Comm_barrier(B200_Comm comm);

/* kernel-choice switches (B200GRB_* environment variables) are read once at GrB_init; re-read them now */
GrB_Info B200_reload_tunables(void);
/* same switch as GxB_Global_Option_set(GxB_BURBLE, on) (reference: pygraphblas/base.py:84-86): every compute
 * call prints the kernel it chose, its algorithmic bytes and its device time */
void B200_set_burble(int on);
int B200_get_burble(void);

/* ------------------------------------------------------------------ import compatibility
 * Names the unmodified reference package resolves at import time or calls around its hot-path tests
 * (GxB_Scalar, options, iseq helpers, per-type families, select-operator and complex-type handles).
 * Most are stubs that refuse: they are not on the mxm/mxv/vxm hot path. */
#include "b200grb_compat.h"

#ifdef __cplusplus
}
#endif
#endif /* B200GRB_H */
