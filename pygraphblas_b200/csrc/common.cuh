// common.cuh -- internal declarations of libb200grb (not part of the C ABI).
//
// Object model behind the opaque GraphBLAS handles of include/b200grb.h, the
// scalar "carrier" used wherever a value's type is only known at run time
// (typecasts, accumulators, dup operators), and the typed operator templates
// that the sm_90a kernels instantiate.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>
#include <math.h>
#include <float.h>
#include <limits.h>
#include <algorithm>
#include <string>
#include <vector>
#include <mutex>
#include <type_traits>
#include <utility>
#include "../../include/b200grb.h"

#define GB_MAGIC 0x42323030  /* "B200" */
#define GB_FREED 0x0DEAD000

// ---------------------------------------------------------------- type codes
enum TypeCode : int {
    TC_BOOL = 0, TC_INT8, TC_INT16, TC_INT32, TC_INT64,
    TC_UINT8, TC_UINT16, TC_UINT32, TC_UINT64, TC_FP32, TC_FP64, TC_COUNT
};

// ---------------------------------------------------------------- operator codes
enum OpCode : int {
    OP_FIRST = 0, OP_SECOND, OP_PAIR, OP_ANY, OP_MIN, OP_MAX, OP_PLUS, OP_MINUS, OP_RMINUS,
    OP_TIMES, OP_DIV, OP_RDIV, OP_POW, OP_ISEQ, OP_ISNE, OP_ISGT, OP_ISLT, OP_ISGE, OP_ISLE,
    OP_LOR, OP_LAND, OP_LXOR, OP_BOR, OP_BAND, OP_BXOR, OP_BXNOR,
    OP_EQ, OP_NE, OP_GT, OP_LT, OP_GE, OP_LE,   // z = BOOL
    // positional (z = INT32 / INT64, an index of x or y; never handed to a kernel: positional.cu rewrites the call)
    OP_FIRSTI, OP_FIRSTI1, OP_FIRSTJ, OP_FIRSTJ1, OP_SECONDI, OP_SECONDI1, OP_SECONDJ, OP_SECONDJ1,
    OP_USER, OP_COUNT
};
static inline bool op_is_cmp(int op) { return op >= OP_EQ && op <= OP_LE; }
static inline bool op_is_positional(int op) { return op >= OP_FIRSTI && op <= OP_SECONDJ1; }

// ---------------------------------------------------------------- opaque objects
struct GB_Type_opaque { int magic; int code; size_t size; const char *name; };
struct GB_BinaryOp_opaque {
    int magic; int opcode; GrB_Type xtype, ytype, ztype; const char *name; void *user_fn;
};
struct GB_Monoid_opaque { int magic; GrB_BinaryOp op; const char *name; bool builtin; };
struct GB_Semiring_opaque { int magic; GrB_Monoid add; GrB_BinaryOp mul; const char *name; bool builtin; };
struct GB_Descriptor_opaque {
    int magic; int outp, mask, inp0, inp1; int axb; int nthreads; double chunk; int sort;
    bool builtin; const char *name;
};
struct GB_UnaryOp_opaque { int magic; int opcode; GrB_Type xtype, ztype; const char *name; };
enum UnaryCode : int {
    UOP_IDENTITY = 0, UOP_AINV, UOP_MINV, UOP_LNOT, UOP_ONE, UOP_ABS, UOP_BNOT,
    // floating point only
    UOP_SQRT, UOP_LOG, UOP_EXP, UOP_LOG2, UOP_SIN, UOP_COS, UOP_TAN, UOP_ACOS, UOP_ASIN, UOP_ATAN, UOP_SINH, UOP_COSH,
    UOP_TANH, UOP_ACOSH, UOP_ASINH, UOP_ATANH, UOP_SIGNUM, UOP_CEIL, UOP_FLOOR, UOP_ROUND, UOP_TRUNC, UOP_EXP2,
    UOP_EXPM1, UOP_LOG10, UOP_LOG1P, UOP_LGAMMA, UOP_TGAMMA, UOP_ERF, UOP_ERFC,
    UOP_ISINF, UOP_ISNAN, UOP_ISFINITE,      // z = BOOL
    UOP_POSITIONI, UOP_POSITIONI1, UOP_POSITIONJ, UOP_POSITIONJ1,      // z = INT32 / INT64, the row or column of the entry
    UOP_COUNT
};
static inline bool uop_is_positional(int op) { return op >= UOP_POSITIONI && op <= UOP_POSITIONJ1; }

// device memory (stream-ordered pool on G.stream)
GrB_Info dmalloc(void **p, size_t bytes, std::string *err);
void dfree(void *p);
template <typename T> static inline GrB_Info dalloc(T **p, size_t count, std::string *err) {
    return dmalloc((void **)p, count * sizeof(T) + 16, err);   // +16: bulk copies may over-read a tail
}

// Owner of one dmalloc block, released at scope exit (stream-ordered after the kernels already enqueued).  It converts
// to the raw pointer, so it can stand wherever a device pointer is read.  DevBuf<void> takes an exact byte count.
// A borrowed block (borrow) belongs to someone else -- another container, a communicator's cudaMalloc region -- and is
// never freed here.
template <typename T> class DevBuf {
    T *p_ = nullptr;
    bool borrowed_ = false;
public:
    DevBuf() = default;                 // move-only: declaring the moves deletes the copies
    DevBuf(DevBuf &&o) noexcept : p_(o.p_), borrowed_(o.borrowed_) { o.p_ = nullptr; o.borrowed_ = false; }
    DevBuf &operator=(DevBuf &&o) noexcept {
        if (this != &o) { reset(); p_ = o.p_; borrowed_ = o.borrowed_; o.p_ = nullptr; o.borrowed_ = false; }
        return *this;
    }
    ~DevBuf() { reset(); }
    GrB_Info alloc(size_t count, std::string *err) {
        reset();
        if constexpr (std::is_void<T>::value) return dmalloc(&p_, count, err);
        else return dalloc(&p_, count, err);
    }
    void borrow(T *p) { reset(); p_ = p; borrowed_ = true; }
    bool borrowed() const { return borrowed_; }
    T *get() const { return p_; }
    operator T *() const { return p_; }
    template <typename U> explicit operator U *() const { return (U *)p_; }
    void reset() { if (!borrowed_) dfree(p_); p_ = nullptr; borrowed_ = false; }
};

// run plan (spmv_run.cu, warp-independent kernels): entries cut into warp-sized runs of 256
struct RunPlan {
    DevBuf<uint32_t> headw;          // [ceil(nnz/32)] bit q = entry q starts a row
    DevBuf<uint32_t> base;           // [nruns+1] row starts before the run (= rank of its first row start)
    DevBuf<int32_t> tail_row;        // [nruns] row still open at the end of the run (its last row start), or -1
    DevBuf<uint32_t> tail_last;      // [nruns] last run that row reaches
    DevBuf<uint32_t> long_run;       // [nlong] ascending: the runs whose open row reaches more than FIX_LONG runs further
    int64_t nlong = 0;
    DevBuf<uint32_t> nzrow;          // [nnzrows] ids of the non-empty rows, ascending
    DevBuf<uint8_t> pres_tmpl;       // [nrows] 1 where the row is non-empty
    int64_t nruns = 0, nnzrows = 0;
    bool wide = false;               // built from the 64-bit row offsets (the wide route)
    // per-call scratch of the run kernels, kept with the plan (no allocation on the call path)
    DevBuf<void> ws_head, ws_tail;   // [nruns] x 8 bytes: partials of the rows a run starts / ends inside
    DevBuf<uint8_t> ws_head_has, ws_tail_has;
};
// hot-column plan (spmv_run.cu): the henc most referenced columns get their rank as id, the others col + henc
struct HotPlan {
    DevBuf<uint32_t> perm;           // [henc] hot rank -> original column
    DevBuf<void> col;                // encoded column ids: 3-byte ids packed run by run ([nruns] x 768 bytes), or [nnz] x 4 bytes
    int id_bytes = 4;                // 3 when every encoded id is below 2^24 - 1 (ncols + henc < 2^24), else 4
    DevBuf<void> ws_uhot;            // [henc + 256] x 8 bytes: u at the hot columns, in the tier layout of the launch (spmv_args.cuh)
    uint32_t henc = 0;               // ids below this are hot ranks
    bool planned = false;            // the plan was attempted (col stays NULL when the gathers are not concentrated)
    double cover = 0.0;              // share of the entries whose column is among the HOT_ENC most referenced
};

// Device CSR panel: rows sorted, columns sorted inside each row.  Owns its arrays and cached plans.
struct CsrFields {
    int64_t nrows = 0, ncols = 0, nnz = 0;
    DevBuf<int64_t> rowptr;          // [nrows+1] 64-bit offsets (canonical)
    DevBuf<uint32_t> rowptr32;       // [nrows+1] 32-bit shadow, built when nnz < 2^32
    DevBuf<uint32_t> col;            // [nnz]
    DevBuf<void> val;                // [nnz] of the matrix type
    // cached SpMV plans, each either complete or absent
    RunPlan run;
    HotPlan hot;
    bool valid = false;
};
// A move is the member-wise move of every field, then a reset of the source: a moved-from Csr is empty, not
// "valid with null arrays", whatever fields are added later.
struct Csr : CsrFields {
    Csr() = default;
    Csr(Csr &&o) noexcept : CsrFields(std::move(o)) { o.clear(); }
    Csr &operator=(Csr &&o) noexcept { if (this != &o) { CsrFields::operator=(std::move(o)); o.clear(); } return *this; }
    void clear() { static_cast<CsrFields &>(*this) = CsrFields(); }
    // the cached SpMV plans and scratch (dropped whenever the structure changes)
    void drop_plans() { run = RunPlan(); hot = HotPlan(); }
};

// per-object storage hints of SuiteSparse's GxB_*_Option_set/get: recorded and reported back, without effect on the HBM
// layout (always CSR by row / dense + presence) -- the API is format-agnostic, results do not depend on them
struct GBObjOpts { double hyper = 0.0625; int format = 0 /* GxB_BY_ROW */; int sparsity = 15 /* GxB_AUTO_SPARSITY */; };

// Dense device form: values of the container's type, one per position, and one presence byte per position (pres NULL: every
// position present).  It is the device form of every vector, and of a dense matrix (DESIGN.md section 3.6): nrows x ncols
// positions, row-major, created only by B200_Matrix_import_dense and the SpMM result of GrB_mxm.  A matrix's dense form is
// authoritative while it is held: the CSR and the host tuples beside it are caches built from it on demand, and any
// modification drops it (matrix_invalidate_device).  nrows * ncols <= 2^31-1, so the flattened form is a legal vector.
// A view (a communicator's result, a stack-built operand) borrows its buffers: dropping the form frees nothing.
struct DenseForm {
    DevBuf<void> val;
    DevBuf<uint8_t> pres;
    bool valid = false;
    static DenseForm borrow(void *val, uint8_t *pres) {
        DenseForm d; d.val.borrow(val); d.pres.borrow(pres); d.valid = true; return d;
    }
};

struct GB_Matrix_opaque {
    int magic; GrB_Type type; uint64_t nrows, ncols;
    GBObjOpts opts;
    // host form: row-major sorted unique COO
    std::vector<uint64_t> hi, hj; std::vector<uint8_t> hx; bool host_valid;
    // pending setElement tuples (in call order; later wins)
    std::vector<uint64_t> pi, pj; std::vector<uint8_t> px;
    // device form (+ cached transpose)
    Csr dev, devT;
    DenseForm dn;
    std::string err;
};

struct GB_Vector_opaque {
    int magic; GrB_Type type; uint64_t n;
    GBObjOpts opts;
    // host form: sorted unique (index, value)
    std::vector<uint64_t> hi; std::vector<uint8_t> hx; bool host_valid;
    std::vector<uint64_t> pi; std::vector<uint8_t> px;
    // device form, and its entry count when known (-1: count the presence bytes)
    DenseForm dv; int64_t dev_nvals = -1;
    // overlapped host copies (B200_Vector_set_dense / export_dense with where = 2): the copy streams' hand-shakes with the compute stream
    cudaEvent_t ev_h2d = nullptr, ev_d2h = nullptr, ev_use = nullptr;
    bool h2d_pending = false, d2h_pending = false, use_recorded = false;
    std::string err;
};

// ---------------------------------------------------------------- globals (objects.cu)
struct GBGlobal {
    bool initialized = false;
    bool have_device = false;
    int device = 0;
    int num_sms = 0;
    cudaStream_t stream = nullptr;
    cudaStream_t h2d = nullptr, d2h = nullptr;     // copy streams of the overlapped import / export (where = 2)
    uint64_t launches = 0;
    uint64_t last_flops = 0, last_nnz_out = 0;
    int burble = 0;
    cudaEvent_t burble_e0 = nullptr, burble_e1 = nullptr;
    std::string last_kernel;      // kernel paths of the last GrB_mxv / GrB_vxm / GrB_mxm, separated by ';' (B200_debug_last_kernel)
    int64_t debug_wide = 0;       // B200_debug_wide: > 0 puts every mxv / vxm / transpose, the SpMM, dense-left and SDDMM routes
                                  // of mxm and its masked CSR x CSR methods (not complemented) on the wide route; transposes and
                                  // SDDMM masks go in chunks of this many entries, masked products in row panels of at most this
                                  // many entries of A and of M (a longer row makes a panel of its own)
    // B200_debug_wide_gemm: chunk > 0 puts every unmasked and complemented-mask CSR x CSR mxm on the wide route, in row panels of
    // at most this many entries of A and of M'; limit > 0 stands for 2^32 in that route's size rule, spa_budget > 0 for
    // WIDE_SPA_BUDGET (spgemm.cu)
    int64_t debug_wide_gemm = 0, debug_gemm_limit = 0, debug_spa_budget = 0;
    std::recursive_mutex mu;
};
extern GBGlobal G;
static inline void gb_kernel_used(const char *k) { if (!G.last_kernel.empty()) G.last_kernel += ';'; G.last_kernel += k; }
// the wide route of mxv / vxm, of the dense-operand mxm and of the masked CSR x CSR mxm (DESIGN.md sections 3.1, 3.2 and 3.6):
// 64-bit entry offsets, for a CSR
// without rowptr32 (nnz >= 2^32), and for every CSR while B200_debug_wide is on
static inline bool csr_wide(const Csr &c) { return !c.rowptr32 || G.debug_wide > 0; }
// entries per chunk of the wide route's chunked passes (the transpose, the mask of SDDMM): 2^27, or B200_debug_wide's chunk,
// at most 2^31 (the transpose's permutations are 32-bit)
static constexpr int64_t TRANSPOSE_CHUNK = (int64_t)1 << 27;
static inline int64_t wide_chunk() { return G.debug_wide > 0 ? std::min(G.debug_wide, (int64_t)1 << 31) : TRANSPOSE_CHUNK; }
extern thread_local std::string tl_error;

GrB_Info gb_fail(GrB_Info code, std::string *where, const char *fmt, ...);

// every entry point: take the library lock and make the library's device current for the calling host thread
// (the reference drives `lib` from a ThreadPool, reference: demo/dnn/challenge.py:48-51; a new thread starts on device 0)
static inline void gb_thread_enter() {
    // the embedding application (torch, another library) may have switched this thread to another GPU since the last call:
    // ask, do not cache
    if (G.have_device) { int cur = -1; if (cudaGetDevice(&cur) != cudaSuccess || cur != G.device) cudaSetDevice(G.device); }
    tl_error.clear();                      // GrB_*_error / B200_last_error report the failure of the LAST call of this thread
}
#define GB_LOCK std::lock_guard<std::recursive_mutex> _lk(G.mu); gb_thread_enter()
#define GB_CHECK_INIT  do { if (!G.initialized) return gb_fail(GrB_PANIC, nullptr, "GrB_init not called"); } while (0)
#define GB_TRY(expr) do { GrB_Info _i = (expr); if (_i != GrB_SUCCESS) return _i; } while (0)
#define CU_TRY(expr, errstr) do { cudaError_t _e = (expr); if (_e != cudaSuccess) \
    return gb_fail(_e == cudaErrorMemoryAllocation ? GrB_OUT_OF_MEMORY : GrB_PANIC, errstr, \
                   "CUDA error %s at %s:%d", cudaGetErrorString(_e), __FILE__, __LINE__); } while (0)

// kernel-choice switches read from the environment ONCE (GrB_init) and again only on B200_reload_tunables()
// (tests flip them between calls); nothing on a call path touches getenv
struct Tunables {
    int spmv_hot_kb = -1;      // B200GRB_SPMV_HOT     -1 default (on when the gathers are concentrated), 0 off, >0 table cap in KB
    bool no_pull = false, no_push = false, force_push = false;
    int spmv_cluster = 2;      // B200GRB_SPMV_CLUSTER thread-block cluster size of the hot-table kernel (1 / 2 / 4 / 8 / 16)
    int spmv_hot_repl_kb = 32; // B200GRB_SPMV_HOT_REPL KB of the hot table replicated in every CTA of a cluster (the rest is spread)
    bool spgemm_trace = false; // B200GRB_SPGEMM_TRACE phase times of GrB_mxm (masked) on stderr
    int stream_blk_log2 = 7;   // B200GRB_STREAM_BLK   log2 of the block of a long B row one warp takes (masked SpGEMM)
    int mxv_inplace = 1;       // B200GRB_MXV_INPLACE  0: mxv / vxm never form T in w's own buffers; 1: when w has no copy in flight;
                               //                      2: always, the compute stream first joins w's last overlapped copies
    double mxm_pull = 0.0;     // B200GRB_MXM_PULL     alpha of the per-row pull rule of a complemented-mask mxm (LOR / LAND / ANY);
                               //                      0: off (only GxB_AxB_DOT pulls).  DESIGN.md section 3.2
    int64_t mxm_pull_budget = (int64_t)1 << 28;   // B200GRB_MXM_PULL_BUDGET  bytes of bitmaps of one group of pull rows
};
const Tunables &tunables();

// GxB_BURBLE (reference: pygraphblas/base.py:84-86): when on, every compute entry point prints which kernel it
// chose, the algorithmic bytes of the call and its device time; every entry point is also an NVTX range
struct GbBurble {
    bool on; const char *fn; const char *kernel = ""; double bytes = 0.0;
    explicit GbBurble(const char *fn);
    void note(const char *k, double b) { kernel = k; bytes = b; }
    ~GbBurble();
};

// Persistent scratch of the compute calls: slot k keeps its buffer between calls and only grows (calls are serialised on one
// stream, so a slot is never in use twice).  Large transient cudaMallocAsync / cudaFreeAsync pairs were measured to cost
// 10-70 ms per call when the pool has to map fresh memory (masked GrB_mxm: 620 MB of column maps) -- these buffers never leave.
enum WsSlot : int { WS_WORDS = 0, WS_FOUND, WS_FLOPS, WS_TOTAL, WS_CS, WS_CM, WS_CL, WS_C1, WS_SROW, WS_SIDX, WS_SCNT, WS_MROW, WS_MIDX, WS_MCNT,
                    WS_LROW, WS_LIDX, WS_LCNT, WS_WROWS, WS_QUEUES, WS_SPA_SLOT, WS_MASK_ROW,
                    WS_SPLIT_BUF, WS_SPLIT_ROWS, WS_SPLIT_CHUNKS, WS_SPLIT_RANGES, WS_PANEL_A, WS_PANEL_M, WS_GEMM_TREE,
                    WS_PULL_ROWS, WS_PULL_BUF, WS_COUNT };
GrB_Info ws_get(int slot, void **p, size_t bytes, std::string *err, bool *fresh = nullptr);
template <typename T> static inline GrB_Info ws_array(int slot, T **p, size_t count, std::string *err, bool *fresh = nullptr) {
    return ws_get(slot, (void **)p, count * sizeof(T) + 16, err, fresh);
}

// host <-> device sync of containers (objects.cu)
GrB_Info matrix_flush_pending(GrB_Matrix A);
GrB_Info matrix_ensure_host(GrB_Matrix A);
GrB_Info matrix_ensure_device(GrB_Matrix A);
GrB_Info matrix_ensure_transpose(GrB_Matrix A);     // builds A->devT on the device
void matrix_invalidate_device(GrB_Matrix A);
void matrix_adopt_device(GrB_Matrix A, Csr &&c);    // A takes ownership of c, host form dropped
void matrix_adopt_dense(GrB_Matrix A, DenseForm &&d);   // A takes a dense form, every other form dropped
bool matrix_known_empty(const GrB_Matrix A);        // A has no entries, as far as can be told without reading the device
GrB_Info vector_ensure_host(GrB_Vector v);
GrB_Info vector_ensure_device(GrB_Vector v);
void vector_invalidate_device(GrB_Vector v);
void vector_adopt_device(GrB_Vector v, DenseForm &&d);   // v takes d as its device form, host form dropped
void vector_mark_used(GrB_Vector v);               // after the kernels reading v were enqueued (lets the next overlapped import of v start early)
bool gb_valid_matrix(const GrB_Matrix A);
bool gb_valid_vector(const GrB_Vector v);

struct DescFlags { bool replace, mask_comp, mask_struct, tran0, tran1; int axb; };
// hypersparse operands (dimension beyond 2^31-1): computed on in their compact index space (hyper.cu)
bool gb_hyper_matrix(const GrB_Matrix A);
bool gb_hyper_vector(const GrB_Vector v);
GrB_Info hyper_mxv(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_Semiring s, const GrB_Matrix A, const GrB_Vector u,
                   const GrB_Descriptor desc, bool vxm);
GrB_Info hyper_mxm(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const GrB_Semiring s, const GrB_Matrix A, const GrB_Matrix B,
                   const GrB_Descriptor desc);
DescFlags desc_flags(const GrB_Descriptor d);

struct Sc;
// C<Mask> = accum(C, T) for a CSR T of type ttc (spgemm.cu); consumes T
GrB_Info matrix_writeback(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const DescFlags &f,
                          Csr &&T, int ttc, bool t_already_masked, std::string *err);
// fold of n values (presence bytes optional) with a builtin monoid operator on the device (vector_ops.cu)
GrB_Info dev_reduce_values(const void *val, const uint8_t *pres, int vtc, int64_t n, int op, int mtc, Sc *out, bool *has, std::string *err);
// w<mask> = accum(w, T) on the device (vector_ops.cu).  T (val, pres) is of type ttc over w->n positions
// (pres NULL: every position present; t_scalar: val is ONE value standing for all positions).  region
// (NULL = everything) limits the write to the positions it flags, GrB_assign style.  w may adopt the buffers of a T
// that owns them; a borrowed T (another vector's form) is only read.  T is consumed.
GrB_Info vector_write(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const DescFlags &f,
                      DenseForm &&T, int ttc, bool t_scalar, const uint8_t *region);

// positional operators (positional.cu).  What a positional operator returns, decoded: the index of the first or the second
// operand (`second`), its row or its column (`col`), plus `off` (0, or 1 for the ...1 forms)
struct PosOp { bool second, col; int64_t off; };
static inline PosOp pos_binop(int op) { const int d = op - OP_FIRSTI; return PosOp{(d >> 2) != 0, ((d >> 1) & 1) != 0, (int64_t)(d & 1)}; }
static inline PosOp pos_unop(int op) { const int d = op - UOP_POSITIONI; return PosOp{false, (d >> 1) != 0, (int64_t)(d & 1)}; }
// A positional operator as accumulator, or in an operation that has no positional form: refused before anything is read
GrB_Info gb_refuse_positional_accum(const GrB_BinaryOp accum, const char *fn);
// A positional semiring with a user-defined monoid or accumulator: GrB_INVALID_VALUE, like every other call with a user-defined
// operator, and before the hypersparse dispatch and the device check (the rewrite would hand them to the write-back)
GrB_Info gb_refuse_user_with_positional(const GrB_Semiring s, const GrB_BinaryOp accum, const char *fn);
GrB_Info gb_refuse_positional(const GrB_BinaryOp op, const char *fn);
GrB_Info gb_refuse_positional(const GrB_Semiring s, const char *fn);
static inline GrB_Info gb_refuse_positional(const GrB_Monoid, const char *) { return GrB_SUCCESS; }   // no monoid is positional
// out[p] (type tc = INT32 / INT64, n positions) = v(p) folded cnt[p] times with the monoid `add`: v(p) = (zero ? 0 : ids[p] or p)
// + off, truncated like a C cast.  cnt NULL: v(p) itself (one product per position).  ids NULL: the position is the index.
GrB_Info pos_vector_values(void *out, int tc, const int64_t *cnt, int add, int64_t n, bool zero, const uint64_t *ids, int64_t off,
                           std::string *err);
// the same over the entries of a CSR: v(e) = the column (by_col) or the row of entry e, through ids when given
GrB_Info pos_csr_values(void *out, int tc, const int64_t *cnt, int add, const Csr &c, bool by_col, const uint64_t *ids, int64_t off,
                        std::string *err);
// GrB_mxv / GrB_vxm / GrB_mxm with a positional multiply (spmv.cu / spgemm.cu).  ids_*: the original index of every position of
// a compact (hypersparse) operand, in device memory; NULL when the positions are the indices
GrB_Info positional_mxv(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_Semiring s, const GrB_Matrix A,
                        const GrB_Vector u, const DescFlags &f, bool vxm, const uint64_t *ids_in, const uint64_t *ids_out);
GrB_Info positional_mxm(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const GrB_Semiring s, const GrB_Matrix A,
                        const GrB_Matrix B, const DescFlags &f, const uint64_t *ids_m, const uint64_t *ids_k, const uint64_t *ids_n);

// kernels (device_ops.cu / spmv.cu / spgemm.cu)
GrB_Info dev_build_rowptr32(Csr &c, std::string *err);
GrB_Info dev_exclusive_scan(int64_t *data, int64_t n, std::string *err);
GrB_Info dev_transpose(const Csr &a, size_t vsize, Csr &t, std::string *err);
GrB_Info dev_cast_values(DevBuf<void> &out, int to_code, const void *in, int from_code, int64_t n, std::string *err);
// *out = the n values `in` (of type from_code) of an mxm operand as the multiply reads them: cast into `cast` to its x type xt
// when it reads them (reads) and the types differ, else `in` itself.  The cast buffer belongs to the caller.
static inline GrB_Info mxm_values(DevBuf<void> &cast, const void **out, bool reads, int xt, const void *in, int from_code, int64_t n,
                                  std::string *err) {
    *out = in;
    if (reads && from_code != xt) { GB_TRY(dev_cast_values(cast, xt, in, from_code, n, err)); *out = cast; }
    return GrB_SUCCESS;
}
GrB_Info dev_count_present(const uint8_t *pres, int64_t n, int64_t *count, std::string *err);
GrB_Info upload_indices(const std::vector<uint64_t> &idx, DevBuf<uint64_t> &d, std::string *err);     // host list -> device (vector_ops.cu)
// dense form <-> CSR (spmm.cu).  dense_to_csr compacts the present entries (pres NULL: all) into c, rowptr32 included;
// csr_to_dense scatters c into fresh zero-filled values and presence bytes
GrB_Info dense_to_csr(const void *val, const uint8_t *pres, int64_t nrows, int64_t ncols, size_t vsize, Csr &c, std::string *err);
GrB_Info csr_to_dense(const Csr &c, size_t vsize, DevBuf<void> &val, DevBuf<uint8_t> &pres, std::string *err);
// C<Mask> = accum(C, op(A) (+).(x) B) for a dense-form B, not transposed, and a builtin non-positional semiring (spmm.cu)
GrB_Info spmm_mxm(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const GrB_Semiring s, const GrB_Matrix A,
                  const GrB_Matrix B, const DescFlags &f, GbBurble &burble);
// the multiply with its operands swapped, mirror(y, x) = op(x, y), by opcode; -1 when the library has none (POW)
int op_mirror(int op);
// C<Mask> = accum(C, op(A) (+).(x) op(B)) for a dense-form A, a B without one, a multiply with a mirror and a k x m C of at most
// 2^31-1 entries (spmm.cu)
GrB_Info spmm_left_mxm(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const GrB_Semiring s, const GrB_Matrix A,
                       const GrB_Matrix B, const DescFlags &f, GbBurble &burble);
// values one lane folds in order before a dot product is split (bounds the FP32 rounding error of a sequential fold; the
// partials are folded pairwise): entries of a row of op(A) in the SpMM kernel, positions k in the masked dense-dense kernel
static constexpr int SPMM_SEG = 64;
// out (cols x rows) = in (rows x cols)', both row-major, presence bytes carried along when pres is given (spmm.cu)
GrB_Info dense_transpose(const void *val, const uint8_t *pres, int64_t rows, int64_t cols, size_t vsize, void *oval, uint8_t *opres,
                         std::string *err);
// (pattern of M, one found flag and one value of vsize bytes per entry of M) -> the CSR T of the found entries, rowptr32
// included, of M's dimensions (spgemm.cu)
GrB_Info masked_compact(const Csr &M, const uint8_t *found, const void *tval, size_t vsize, Csr &T, std::string *err);
// the entries of a valued mask M (type mtc) that are true, x != 0 as in mask_value_true (NaN true, +-0 false), as a CSR pattern with
// 32-bit row pointers: the columns a complemented mask blocks (select_kernel with SEL_NONZERO, matrix_ops.cu)
GrB_Info mask_true_pattern(const Csr &M, int mtc, Csr &out, std::string *err);
// C<Mask> = accum(C, op(A) (+).(x) op(B)) for dense-form A and B, a builtin non-positional semiring and a CSR mask of fewer than
// 2^32 entries, already on the device and not complemented: one dot product per entry of the mask (sddmm.cu)
GrB_Info sddmm_mxm(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const GrB_Semiring s, const GrB_Matrix A,
                   const GrB_Matrix B, const DescFlags &f, GbBurble &burble);
// C<Mask> = accum(C, T) for a dense m x n T, presence bytes optional (tpres NULL: every position present): the vector write-back
// over the m*n positions with no mask or a dense-form mask, so C keeps or takes a dense form; the CSR write-back under a CSR
// mask (spmm.cu).  Consumes T.
GrB_Info spmm_writeback(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const DescFlags &f, DevBuf<void> &&tval,
                        DevBuf<uint8_t> &&tpres, int zt, std::string *err);
// C<Mask> = accum(C, op(A) (+).(x) op(B)) for dense-form A and B without presence bytes, a builtin non-positional semiring, an
// m x n result of at most 2^31-1 positions, and no sparse non-complemented mask: the tiled semiring GEMM (gemm.cu)
GrB_Info gemm_mxm(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const GrB_Semiring s, const GrB_Matrix A,
                  const GrB_Matrix B, const DescFlags &f, GbBurble &burble);

// ---------------------------------------------------------------- scalar carrier
// A value of any builtin type held in 64 bits: BOOL/UINT* in .u, INT* in .i, FP* in .d
// (a float is held as the exactly-equal double).
struct Sc { union { int64_t i; uint64_t u; double d; }; };
struct GB_Scalar_opaque { int magic; GrB_Type type; bool has; Sc v; };     // GxB_Scalar (compat.cu)
enum SelectCode : int { SEL_TRIL = 0, SEL_TRIU, SEL_DIAG, SEL_OFFDIAG, SEL_NONZERO, SEL_EQ_ZERO, SEL_GT_ZERO, SEL_GE_ZERO, SEL_LT_ZERO, SEL_LE_ZERO,
                        SEL_NE_THUNK, SEL_EQ_THUNK, SEL_GT_THUNK, SEL_GE_THUNK, SEL_LT_THUNK, SEL_LE_THUNK };
struct GB_SelectOp_opaque { int magic; const char *name; int code; };

__host__ __device__ static inline int tc_size(int tc) {
    switch (tc) {
        case TC_BOOL: case TC_INT8: case TC_UINT8: return 1;
        case TC_INT16: case TC_UINT16: return 2;
        case TC_INT32: case TC_UINT32: case TC_FP32: return 4;
        default: return 8;
    }
}
__host__ __device__ static inline bool tc_is_float(int tc) { return tc == TC_FP32 || tc == TC_FP64; }
__host__ __device__ static inline bool tc_is_signed(int tc) { return tc >= TC_INT8 && tc <= TC_INT64; }

__host__ __device__ static inline Sc sc_load(int tc, const void *p, size_t k) {
    Sc s; s.u = 0;
    switch (tc) {
        case TC_BOOL:   s.u = ((const uint8_t *)p)[k] != 0; break;
        case TC_INT8:   s.i = ((const int8_t *)p)[k]; break;
        case TC_INT16:  s.i = ((const int16_t *)p)[k]; break;
        case TC_INT32:  s.i = ((const int32_t *)p)[k]; break;
        case TC_INT64:  s.i = ((const int64_t *)p)[k]; break;
        case TC_UINT8:  s.u = ((const uint8_t *)p)[k]; break;
        case TC_UINT16: s.u = ((const uint16_t *)p)[k]; break;
        case TC_UINT32: s.u = ((const uint32_t *)p)[k]; break;
        case TC_UINT64: s.u = ((const uint64_t *)p)[k]; break;
        case TC_FP32:   s.d = (double)((const float *)p)[k]; break;
        case TC_FP64:   s.d = ((const double *)p)[k]; break;
    }
    return s;
}
__host__ __device__ static inline void sc_store(int tc, void *p, size_t k, Sc s) {
    switch (tc) {
        case TC_BOOL:   ((uint8_t *)p)[k] = (uint8_t)(s.u != 0); break;
        case TC_INT8:   ((int8_t *)p)[k] = (int8_t)s.i; break;
        case TC_INT16:  ((int16_t *)p)[k] = (int16_t)s.i; break;
        case TC_INT32:  ((int32_t *)p)[k] = (int32_t)s.i; break;
        case TC_INT64:  ((int64_t *)p)[k] = s.i; break;
        case TC_UINT8:  ((uint8_t *)p)[k] = (uint8_t)s.u; break;
        case TC_UINT16: ((uint16_t *)p)[k] = (uint16_t)s.u; break;
        case TC_UINT32: ((uint32_t *)p)[k] = (uint32_t)s.u; break;
        case TC_UINT64: ((uint64_t *)p)[k] = s.u; break;
        case TC_FP32:   ((float *)p)[k] = (float)s.d; break;
        case TC_FP64:   ((double *)p)[k] = s.d; break;
    }
}

// float -> integer conversion as GraphBLAS defines it (NaN -> 0, saturate, truncate).
__host__ __device__ static inline int64_t sat_i64(double d, int64_t lo, int64_t hi) {
    if (d != d) return 0;
    if (d <= (double)lo) return lo;
    if (d >= (double)hi) return hi;
    return (int64_t)d;
}
__host__ __device__ static inline uint64_t sat_u64(double d, uint64_t hi) {
    if (d != d) return 0;
    if (d <= 0.0) return 0;
    if (d >= (double)hi) return hi;
    return (uint64_t)d;
}

// C-style typecast between builtin types, on the carrier.
__host__ __device__ static inline Sc sc_cast(Sc x, int from, int to) {
    if (from == to) return x;
    Sc r; r.u = 0;
    const bool ff = tc_is_float(from), fs = tc_is_signed(from);
    if (to == TC_BOOL) { r.u = ff ? (x.d != 0.0) : (x.u != 0); return r; }
    if (to == TC_FP64) { r.d = ff ? x.d : (fs ? (double)x.i : (double)x.u); return r; }
    if (to == TC_FP32) { r.d = ff ? (double)(float)x.d : (fs ? (double)(float)x.i : (double)(float)x.u); return r; }
    if (ff) {
        switch (to) {
            case TC_INT8:   r.i = sat_i64(x.d, INT8_MIN, INT8_MAX); break;
            case TC_INT16:  r.i = sat_i64(x.d, INT16_MIN, INT16_MAX); break;
            case TC_INT32:  r.i = sat_i64(x.d, INT32_MIN, INT32_MAX); break;
            case TC_INT64:  r.i = sat_i64(x.d, INT64_MIN, INT64_MAX); break;
            case TC_UINT8:  r.u = sat_u64(x.d, UINT8_MAX); break;
            case TC_UINT16: r.u = sat_u64(x.d, UINT16_MAX); break;
            case TC_UINT32: r.u = sat_u64(x.d, UINT32_MAX); break;
            case TC_UINT64: r.u = sat_u64(x.d, UINT64_MAX); break;
        }
        return r;
    }
    // integer/bool -> integer: modular truncation, then sign- or zero-extension
    switch (to) {
        case TC_INT8:   r.i = (int8_t)x.u; break;
        case TC_INT16:  r.i = (int16_t)x.u; break;
        case TC_INT32:  r.i = (int32_t)x.u; break;
        case TC_INT64:  r.i = (int64_t)x.u; break;
        case TC_UINT8:  r.u = (uint8_t)x.u; break;
        case TC_UINT16: r.u = (uint16_t)x.u; break;
        case TC_UINT32: r.u = (uint32_t)x.u; break;
        case TC_UINT64: r.u = x.u; break;
    }
    return r;
}

// ---------------------------------------------------------------- typed operators
template <typename T> struct TypeOf;
template <> struct TypeOf<bool>     { static constexpr int code = TC_BOOL; };
template <> struct TypeOf<int8_t>   { static constexpr int code = TC_INT8; };
template <> struct TypeOf<int16_t>  { static constexpr int code = TC_INT16; };
template <> struct TypeOf<int32_t>  { static constexpr int code = TC_INT32; };
template <> struct TypeOf<int64_t>  { static constexpr int code = TC_INT64; };
template <> struct TypeOf<uint8_t>  { static constexpr int code = TC_UINT8; };
template <> struct TypeOf<uint16_t> { static constexpr int code = TC_UINT16; };
template <> struct TypeOf<uint32_t> { static constexpr int code = TC_UINT32; };
template <> struct TypeOf<uint64_t> { static constexpr int code = TC_UINT64; };
template <> struct TypeOf<float>    { static constexpr int code = TC_FP32; };
template <> struct TypeOf<double>   { static constexpr int code = TC_FP64; };

template <typename T> struct NumTraits {
    static constexpr bool is_float = false;
    static constexpr bool is_signed = ((T)-1) < (T)0;
    __host__ __device__ static inline T maxv() {
        return is_signed ? (T)((((uint64_t)1) << (sizeof(T) * 8 - 1)) - 1) : (T)~(T)0;
    }
    __host__ __device__ static inline T minv() {
        return is_signed ? (T)(((uint64_t)1) << (sizeof(T) * 8 - 1)) : (T)0;
    }
};
template <> struct NumTraits<float> {
    static constexpr bool is_float = true; static constexpr bool is_signed = true;
    __host__ __device__ static inline float maxv() { return INFINITY; }
    __host__ __device__ static inline float minv() { return -INFINITY; }
};
template <> struct NumTraits<double> {
    static constexpr bool is_float = true; static constexpr bool is_signed = true;
    __host__ __device__ static inline double maxv() { return (double)INFINITY; }
    __host__ __device__ static inline double minv() { return -(double)INFINITY; }
};

template <typename T> struct UnsignedOf { typedef T type; };
template <> struct UnsignedOf<int8_t>  { typedef uint8_t type; };
template <> struct UnsignedOf<int16_t> { typedef uint16_t type; };
template <> struct UnsignedOf<int32_t> { typedef uint32_t type; };
template <> struct UnsignedOf<int64_t> { typedef uint64_t type; };

template <typename T> __host__ __device__ static inline T t_from_double(double d) {
    if (NumTraits<T>::is_float) return (T)d;
    if (NumTraits<T>::is_signed) return (T)sat_i64(d, (int64_t)NumTraits<T>::minv(), (int64_t)NumTraits<T>::maxv());
    return (T)sat_u64(d, (uint64_t)NumTraits<T>::maxv());
}

// pow of two integers in double, before the saturating cast.  The device's pow may miss an exact integer result by an
// ulp (just below 3), which the truncating cast would turn into 2: a result within 2^-40 of an
// integer is that integer.  Integer operands have no other result so close to an integer (1 / x^k, |x| >= 2, is at most
// 1/2 away from the nearest one, or rounds to 0 either way), so this only undoes the rounding error.
__host__ __device__ static inline double int_pow_double(double x, double y) {
    double p = pow(x, y);
    const double r = rint(p);
    if (fabs(p) < 9007199254740992.0 && fabs(p - r) <= 0x1p-40 * fmax(1.0, fabs(r))) p = r;
    return p;
}

// integer division with GraphBLAS' defined results for x/0 and INT_MIN/-1
template <typename T> __host__ __device__ static inline T int_div(T x, T y) {
    if constexpr (NumTraits<T>::is_signed) {
        if (y == (T)-1) return (T)(0 - (typename UnsignedOf<T>::type)x);
        if (y == 0) return x == 0 ? (T)0 : (x < 0 ? NumTraits<T>::minv() : NumTraits<T>::maxv());
        return (T)(x / y);
    } else {
        if (y == 0) return x == 0 ? (T)0 : NumTraits<T>::maxv();
        return (T)(x / y);
    }
}

// z = op(x, y) with z of the operand type T (arithmetic, logical and IS* operators).
template <typename T> __host__ __device__ __forceinline__ T op_apply(int op, T x, T y) {
    typedef typename UnsignedOf<T>::type U;
    constexpr bool F = NumTraits<T>::is_float;
    switch (op) {
        case OP_FIRST:  return x;
        case OP_SECOND: return y;
        case OP_ANY:    return y;
        case OP_PAIR:   return (T)1;
        case OP_MIN:    if (F) return (T)fmin((double)x, (double)y); return x < y ? x : y;
        case OP_MAX:    if (F) return (T)fmax((double)x, (double)y); return x > y ? x : y;
        case OP_PLUS:   if (F) return x + y; return (T)((U)x + (U)y);
        case OP_MINUS:  if (F) return x - y; return (T)((U)x - (U)y);
        case OP_RMINUS: if (F) return y - x; return (T)((U)y - (U)x);
        case OP_TIMES:  if (F) return x * y; return (T)((U)x * (U)y);
        case OP_DIV:    if constexpr (F) return x / y; else return int_div<T>(x, y);
        case OP_RDIV:   if constexpr (F) return y / x; else return int_div<T>(y, x);
        case OP_POW:    if constexpr (F) return (T)pow((double)x, (double)y); else return t_from_double<T>(int_pow_double((double)x, (double)y));
        case OP_ISEQ:   return (T)(x == y);
        case OP_ISNE:   return (T)(x != y);
        case OP_ISGT:   return (T)(x > y);
        case OP_ISLT:   return (T)(x < y);
        case OP_ISGE:   return (T)(x >= y);
        case OP_ISLE:   return (T)(x <= y);
        case OP_LOR:    return (T)((x != 0) || (y != 0));
        case OP_LAND:   return (T)((x != 0) && (y != 0));
        case OP_LXOR:   return (T)((x != 0) != (y != 0));
        case OP_BOR:    if constexpr (F) return x; else return (T)((U)x | (U)y);
        case OP_BAND:   if constexpr (F) return x; else return (T)((U)x & (U)y);
        case OP_BXOR:   if constexpr (F) return x; else return (T)((U)x ^ (U)y);
        case OP_BXNOR:  if constexpr (F) return x; else return (T)~((U)x ^ (U)y);
        default:        return x;
    }
}
template <> __host__ __device__ __forceinline__ float op_apply<float>(int op, float x, float y) {
    switch (op) {
        case OP_FIRST: return x;
        case OP_SECOND: case OP_ANY: return y;
        case OP_PAIR:   return 1.0f;
        case OP_MIN:    return fminf(x, y);
        case OP_MAX:    return fmaxf(x, y);
        case OP_PLUS:   return x + y;
        case OP_MINUS:  return x - y;
        case OP_RMINUS: return y - x;
        case OP_TIMES:  return x * y;
        case OP_DIV:    return x / y;
        case OP_RDIV:   return y / x;
        case OP_POW:    return powf(x, y);
        case OP_ISEQ:   return (float)(x == y);
        case OP_ISNE:   return (float)(x != y);
        case OP_ISGT:   return (float)(x > y);
        case OP_ISLT:   return (float)(x < y);
        case OP_ISGE:   return (float)(x >= y);
        case OP_ISLE:   return (float)(x <= y);
        case OP_LOR:    return (float)((x != 0) || (y != 0));
        case OP_LAND:   return (float)((x != 0) && (y != 0));
        case OP_LXOR:   return (float)((x != 0) != (y != 0));
        default:        return x;
    }
}
// BOOL: arithmetic names alias logical ones (PLUS=LOR, TIMES=LAND, MIN=LAND, MAX=LOR, MINUS=LXOR, DIV=FIRST ...)
template <> __host__ __device__ __forceinline__ bool op_apply<bool>(int op, bool x, bool y) {
    switch (op) {
        case OP_FIRST: case OP_DIV: return x;
        case OP_SECOND: case OP_RDIV: case OP_ANY: return y;
        case OP_PAIR:   return true;
        case OP_MIN: case OP_TIMES: case OP_LAND: return x && y;
        case OP_MAX: case OP_PLUS: case OP_LOR: return x || y;
        case OP_MINUS: case OP_RMINUS: case OP_LXOR: case OP_ISNE: return x != y;
        case OP_POW:    return x || !y;
        case OP_ISEQ:   return x == y;
        case OP_ISGT:   return x && !y;
        case OP_ISLT:   return !x && y;
        case OP_ISGE:   return x || !y;
        case OP_ISLE:   return !x || y;
        default:        return x;
    }
}
// z = cmp(x, y), z BOOL
template <typename T> __host__ __device__ __forceinline__ bool cmp_apply(int op, T x, T y) {
    switch (op) {
        case OP_EQ: return x == y;
        case OP_NE: return x != y;
        case OP_GT: return x > y;
        case OP_LT: return x < y;
        case OP_GE: return x >= y;
        case OP_LE: return x <= y;
        default:    return false;
    }
}
// multiply of a semiring: ZT == XT for arithmetic operators, ZT == bool for comparisons
template <typename XT, typename ZT> struct MulApply {
    __host__ __device__ static __forceinline__ ZT f(int op, XT a, XT b) { return (ZT)cmp_apply<XT>(op, a, b); }
};
template <typename T> struct MulApply<T, T> {
    __host__ __device__ static __forceinline__ T f(int op, T a, T b) {
        if (op >= OP_EQ && op <= OP_LE) return (T)cmp_apply<T>(op, a, b);
        return op_apply<T>(op, a, b);
    }
};

// identity / terminal value of a monoid operator on type T
template <typename T> __host__ __device__ static inline T monoid_identity(int op) {
    switch (op) {
        case OP_MIN:   return NumTraits<T>::maxv();
        case OP_MAX:   return NumTraits<T>::minv();
        case OP_TIMES: return (T)1;
        case OP_LAND:  return (T)1;
        case OP_EQ:    return (T)1;
        case OP_BAND: case OP_BXNOR: return (T)~(uint64_t)0;
        default:       return (T)0;   // PLUS, LOR, LXOR, ANY, BOR, BXOR
    }
}
template <> __host__ __device__ inline bool monoid_identity<bool>(int op) {
    switch (op) {
        case OP_MIN: case OP_TIMES: case OP_LAND: case OP_EQ: return true;
        default: return false;
    }
}
template <> __host__ __device__ inline float monoid_identity<float>(int op) {
    switch (op) { case OP_MIN: return INFINITY; case OP_MAX: return -INFINITY;
                  case OP_TIMES: case OP_LAND: case OP_EQ: return 1.0f; default: return 0.0f; }
}
template <> __host__ __device__ inline double monoid_identity<double>(int op) {
    switch (op) { case OP_MIN: return (double)INFINITY; case OP_MAX: return -(double)INFINITY;
                  case OP_TIMES: case OP_LAND: case OP_EQ: return 1.0; default: return 0.0; }
}

// carrier-level operator: x, y, z all of the operator's type `tc` (z BOOL for comparisons)
__host__ __device__ static inline Sc sc_binop(int op, int tc, Sc x, Sc y) {
    Sc r; r.u = 0;
#define GB_CASE(TC, T, FIELD) case TC: { T a = (T)x.FIELD, b = (T)y.FIELD; \
        if (op >= OP_EQ && op <= OP_LE) r.u = cmp_apply<T>(op, a, b); \
        else { T z = op_apply<T>(op, a, b); Sc t; t.u = 0; t.FIELD = z; r = t; } } break;
    switch (tc) {
        case TC_BOOL: { bool a = x.u != 0, b = y.u != 0;
            if (op >= OP_EQ && op <= OP_LE) r.u = cmp_apply<bool>(op, a, b); else r.u = op_apply<bool>(op, a, b); } break;
        GB_CASE(TC_INT8, int8_t, i) GB_CASE(TC_INT16, int16_t, i) GB_CASE(TC_INT32, int32_t, i) GB_CASE(TC_INT64, int64_t, i)
        GB_CASE(TC_UINT8, uint8_t, u) GB_CASE(TC_UINT16, uint16_t, u) GB_CASE(TC_UINT32, uint32_t, u) GB_CASE(TC_UINT64, uint64_t, u)
        case TC_FP32: { float a = (float)x.d, b = (float)y.d;
            if (op >= OP_EQ && op <= OP_LE) r.u = cmp_apply<float>(op, a, b); else r.d = (double)op_apply<float>(op, a, b); } break;
        case TC_FP64: { double a = x.d, b = y.d;
            if (op >= OP_EQ && op <= OP_LE) r.u = cmp_apply<double>(op, a, b); else r.d = op_apply<double>(op, a, b); } break;
    }
#undef GB_CASE
    return r;
}

// carrier-level unary operator: x of type `tc`; z of type `tc` (BOOL for ISINF / ISNAN / ISFINITE)
template <typename T> __host__ __device__ static inline T uop_apply(int op, T x) {
    typedef typename UnsignedOf<T>::type U;
    constexpr bool F = NumTraits<T>::is_float;
    switch (op) {
        case UOP_IDENTITY: return x;
        case UOP_AINV: if (F) return -x; return (T)((U)0 - (U)x);
        case UOP_MINV: if constexpr (F) return (T)1 / x; else return int_div<T>((T)1, x);
        case UOP_LNOT: return (T)!(x != (T)0);
        case UOP_ONE:  return (T)1;
        case UOP_ABS:  if constexpr (F) return (T)fabs((double)x); else if constexpr (NumTraits<T>::is_signed) return x < 0 ? (T)((U)0 - (U)x) : x; else return x;
        case UOP_BNOT: if constexpr (F) return x; else return (T)~(U)x;
        default: break;
    }
    if constexpr (F) {
        const double d = (double)x;
        switch (op) {
            case UOP_SQRT: return (T)sqrt(d);   case UOP_LOG: return (T)log(d);     case UOP_EXP: return (T)exp(d);
            case UOP_LOG2: return (T)log2(d);   case UOP_SIN: return (T)sin(d);     case UOP_COS: return (T)cos(d);
            case UOP_TAN: return (T)tan(d);     case UOP_ACOS: return (T)acos(d);   case UOP_ASIN: return (T)asin(d);
            case UOP_ATAN: return (T)atan(d);   case UOP_SINH: return (T)sinh(d);   case UOP_COSH: return (T)cosh(d);
            case UOP_TANH: return (T)tanh(d);   case UOP_ACOSH: return (T)acosh(d); case UOP_ASINH: return (T)asinh(d);
            case UOP_ATANH: return (T)atanh(d); case UOP_SIGNUM: return (T)(d != d ? d : (d > 0) - (d < 0));
            case UOP_CEIL: return (T)ceil(d);   case UOP_FLOOR: return (T)floor(d); case UOP_ROUND: return (T)round(d);
            case UOP_TRUNC: return (T)trunc(d); case UOP_EXP2: return (T)exp2(d);   case UOP_EXPM1: return (T)expm1(d);
            case UOP_LOG10: return (T)log10(d); case UOP_LOG1P: return (T)log1p(d); case UOP_LGAMMA: return (T)lgamma(d);
            case UOP_TGAMMA: return (T)tgamma(d); case UOP_ERF: return (T)erf(d);   case UOP_ERFC: return (T)erfc(d);
            default: break;
        }
    }
    return x;
}
__host__ __device__ static inline Sc sc_unop(int op, int tc, Sc x) {
    Sc r; r.u = 0;
    if (op >= UOP_ISINF && op <= UOP_ISFINITE) {
        const double d = tc == TC_FP32 ? (double)(float)x.d : x.d;
        const bool inf = d == (double)INFINITY || d == -(double)INFINITY, nan = d != d;
        r.u = op == UOP_ISINF ? inf : (op == UOP_ISNAN ? nan : (!inf && !nan));
        return r;
    }
#define GB_CASE(TC, T, FIELD) case TC: { Sc t; t.u = 0; t.FIELD = uop_apply<T>(op, (T)x.FIELD); r = t; } break;
    switch (tc) {
        case TC_BOOL: r.u = uop_apply<bool>(op, x.u != 0); break;
        GB_CASE(TC_INT8, int8_t, i) GB_CASE(TC_INT16, int16_t, i) GB_CASE(TC_INT32, int32_t, i) GB_CASE(TC_INT64, int64_t, i)
        GB_CASE(TC_UINT8, uint8_t, u) GB_CASE(TC_UINT16, uint16_t, u) GB_CASE(TC_UINT32, uint32_t, u) GB_CASE(TC_UINT64, uint64_t, u)
        case TC_FP32: r.d = (double)uop_apply<float>(op, (float)x.d); break;
        case TC_FP64: r.d = uop_apply<double>(op, x.d); break;
    }
#undef GB_CASE
    return r;
}
// identity of a builtin monoid operator, on the carrier (same table the kernels use)
__host__ __device__ static inline Sc sc_monoid_identity(int op, int tc) {
    Sc acc; acc.u = 0;
    switch (tc) {
#define GB_ID(TC, T, F) case TC: { Sc t; t.u = 0; t.F = monoid_identity<T>(op); acc = t; } break;
        case TC_BOOL: acc.u = monoid_identity<bool>(op); break;
        GB_ID(TC_INT8, int8_t, i) GB_ID(TC_INT16, int16_t, i) GB_ID(TC_INT32, int32_t, i) GB_ID(TC_INT64, int64_t, i)
        GB_ID(TC_UINT8, uint8_t, u) GB_ID(TC_UINT16, uint16_t, u) GB_ID(TC_UINT32, uint32_t, u) GB_ID(TC_UINT64, uint64_t, u)
        case TC_FP32: acc.d = (double)monoid_identity<float>(op); break;
        case TC_FP64: acc.d = monoid_identity<double>(op); break;
#undef GB_ID
    }
    return acc;
}

// value of a mask entry as a truth value (any builtin type), without the carrier
__host__ __device__ static inline bool mask_value_true(int mtc, const void *mval, int64_t i) {
    switch (mtc) {
        case TC_FP32: return ((const float *)mval)[i] != 0.0f;
        case TC_FP64: return ((const double *)mval)[i] != 0.0;
        default: break;
    }
    switch (tc_size(mtc)) {
        case 1: return ((const uint8_t *)mval)[i] != 0;
        case 2: return ((const uint16_t *)mval)[i] != 0;
        case 4: return ((const uint32_t *)mval)[i] != 0;
        default: return ((const uint64_t *)mval)[i] != 0;
    }
}

// which operands a multiply reads (compile-time for the specialised semirings)
__host__ __device__ constexpr bool mul_reads_x(int op) { return !(op == OP_SECOND || op == OP_PAIR); }
__host__ __device__ constexpr bool mul_reads_y(int op) { return !(op == OP_FIRST || op == OP_PAIR || op == OP_ANY); }

// gather of one value through the read-only path (1-byte types as unsigned char: there is no __ldg of bool)
template <typename T> __device__ __forceinline__ T gload(const T *p) {
    if constexpr (sizeof(T) == 1) { const unsigned char v = __ldg(reinterpret_cast<const unsigned char *>(p)); return reinterpret_cast<const T &>(v); }
    else return __ldg(p);
}

// The (x, z) domains of the kernels with run-time operator codes: z = x on the 11 types, z = BOOL (comparisons) on the 10
// others.  Runs the statement BODY with XT_ / ZT_ naming the C++ types of (xt, zt), and sets `matched` to whether the pair
// is one of them.
#define GB_DOMAIN_CASE_(TC, X, Z, ...) case TC: { typedef X XT_; typedef Z ZT_; __VA_ARGS__; } break;
#define GB_FOR_DOMAINS(xt, zt, matched, ...)                                                                                \
    do {                                                                                                                   \
        matched = true;                                                                                                    \
        if ((xt) == (zt)) switch (xt) {                                                                                    \
            GB_DOMAIN_CASE_(TC_BOOL, bool, bool, __VA_ARGS__)          GB_DOMAIN_CASE_(TC_INT8, int8_t, int8_t, __VA_ARGS__)         \
            GB_DOMAIN_CASE_(TC_INT16, int16_t, int16_t, __VA_ARGS__)   GB_DOMAIN_CASE_(TC_INT32, int32_t, int32_t, __VA_ARGS__)      \
            GB_DOMAIN_CASE_(TC_INT64, int64_t, int64_t, __VA_ARGS__)   GB_DOMAIN_CASE_(TC_UINT8, uint8_t, uint8_t, __VA_ARGS__)      \
            GB_DOMAIN_CASE_(TC_UINT16, uint16_t, uint16_t, __VA_ARGS__) GB_DOMAIN_CASE_(TC_UINT32, uint32_t, uint32_t, __VA_ARGS__)  \
            GB_DOMAIN_CASE_(TC_UINT64, uint64_t, uint64_t, __VA_ARGS__) GB_DOMAIN_CASE_(TC_FP32, float, float, __VA_ARGS__)          \
            GB_DOMAIN_CASE_(TC_FP64, double, double, __VA_ARGS__)      default: matched = false;                                    \
        } else if ((zt) == TC_BOOL) switch (xt) {                                                                          \
            GB_DOMAIN_CASE_(TC_INT8, int8_t, bool, __VA_ARGS__)        GB_DOMAIN_CASE_(TC_INT16, int16_t, bool, __VA_ARGS__)         \
            GB_DOMAIN_CASE_(TC_INT32, int32_t, bool, __VA_ARGS__)      GB_DOMAIN_CASE_(TC_INT64, int64_t, bool, __VA_ARGS__)         \
            GB_DOMAIN_CASE_(TC_UINT8, uint8_t, bool, __VA_ARGS__)      GB_DOMAIN_CASE_(TC_UINT16, uint16_t, bool, __VA_ARGS__)       \
            GB_DOMAIN_CASE_(TC_UINT32, uint32_t, bool, __VA_ARGS__)    GB_DOMAIN_CASE_(TC_UINT64, uint64_t, bool, __VA_ARGS__)       \
            GB_DOMAIN_CASE_(TC_FP32, float, bool, __VA_ARGS__)         GB_DOMAIN_CASE_(TC_FP64, double, bool, __VA_ARGS__)           \
            default: matched = false;                                                                                      \
        } else matched = false;                                                                                            \
    } while (0)

// ---------------------------------------------------------------- launch helpers
__host__ __device__ static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }
#define GB_LAUNCHED() (G.launches++)
// grid of a grid-stride kernel: one CTA per `threads` items, at most `per_sm` CTAs per SM, at least one
static inline int grid_for(int64_t n, int threads = 256, int per_sm = 16) {
    const int64_t g = std::min<int64_t>(ceil_div(n, threads), (int64_t)G.num_sms * per_sm);
    return (int)std::max<int64_t>(1, g);
}
// one 8-byte count from the device (synchronises the compute stream)
GrB_Info read_i64(const int64_t *d, int64_t *h, std::string *err);

// ---------------------------------------------------------------- CSR results
// op(A): the CSR of A, or of its cached transpose when tran
static inline GrB_Info source_csr(GrB_Matrix A, bool tran, Csr **out) {
    if (tran) { GB_TRY(matrix_ensure_transpose(A)); *out = &A->devT; }
    else { GB_TRY(matrix_ensure_device(A)); *out = &A->dev; }
    return GrB_SUCCESS;
}
// T = a fresh nrows x ncols CSR formed row by row.  count(rowptr) enqueues the work that leaves all nrows + 1 slots defined:
// the entry count of row r in slot r, 0 in slot nrows.  The slots are scanned into row offsets, T.nnz is read back, and T gets
// col and, when vsize > 0, val (vsize bytes per entry, plus the 16-byte tail of every value array).  fill(T) writes them and
// runs only when T has entries.  Both return GrB_Info.  rowptr32 is built last.  check(nnz), when given, sees T's entry count
// before col and val are allocated, and its failure is the call's.
template <typename Count, typename Fill, typename Check>
static GrB_Info csr_from_row_counts(int64_t nrows, int64_t ncols, size_t vsize, Csr &T, std::string *err, Count &&count, Fill &&fill,
                                    Check &&check) {
    T = Csr(); T.nrows = nrows; T.ncols = ncols;
    GB_TRY(T.rowptr.alloc((size_t)nrows + 1, err));
    GB_TRY(count(T.rowptr.get()));
    GB_TRY(dev_exclusive_scan(T.rowptr, nrows + 1, err));
    GB_TRY(read_i64(T.rowptr + nrows, &T.nnz, err));
    GB_TRY(check(T.nnz));
    GB_TRY(T.col.alloc((size_t)T.nnz, err));
    if (vsize) GB_TRY(T.val.alloc((size_t)T.nnz * vsize + 16, err));
    if (T.nnz > 0) GB_TRY(fill(T));
    return dev_build_rowptr32(T, err);
}
template <typename Count, typename Fill>
static GrB_Info csr_from_row_counts(int64_t nrows, int64_t ncols, size_t vsize, Csr &T, std::string *err, Count &&count, Fill &&fill) {
    return csr_from_row_counts(nrows, ncols, vsize, T, err, count, fill, [](int64_t) { return GrB_SUCCESS; });
}
// T = src's pattern in fresh arrays, with a value array of vsize bytes per entry holding src's values when with_values
// (device_ops.cu).  rowptr32 is left to the caller, to be built once the values are in place.
GrB_Info csr_copy(const Csr &src, size_t vsize, bool with_values, Csr &T, std::string *err);
