// Argument blocks of the run and pull kernels (host side fills them in spmv.cu).
#pragma once
#include "spmv_common.cuh"

static constexpr int RUN = 256;
struct RunArgs {
    const uint32_t *col; const void *aval; const void *uval;
    const uint32_t *headw; const uint16_t *lane_rank; const uint32_t *run_base; const uint32_t *nzrow; const uint32_t *rowptr;
    const int32_t *tail_row; const uint32_t *tail_last;       // structural: which row is open at a run's end, how far it reaches
    int64_t nruns; int64_t nnz;
    void *tval;
    void *head_val; void *tail_val;                            // per run: partial of the row it starts inside / of the row open at its end
    int add_op, mul_op, flip;                                  // run-time operator codes (kernels instantiated with ADD = MUL = -1)
    const uint8_t *upres;                                      // SPARSE kernels: presence bytes of u ...
    uint8_t *tpres; uint8_t *head_has; uint8_t *tail_has;      // ... and of everything they produce
};

// hot-table run kernel (spmv_run.cuh).  The host fills u_hot .. tpres and the two requests; spmv_run_launch lays out the
// table tiers, runs the prep kernel and the hot-table kernel, and fills in the layout and the cluster size it used.
// u_hot layout: [T0 ranks, replicated in every CTA | slice 0 | ... | slice C-1 (S entries each) | ranks T0+T1 .. henc-1]
// hot rank T0 + k (k < T1) lives in slice k mod C at index k / C, in the shared memory of the cluster's CTA k mod C.
struct Hot2Args {
    void *u_hot;              // the plan's u_hot buffer (written by the prep kernel)
    const uint32_t *hperm;    // [henc] column of each hot rank
    const void *u; int vsize; // u and its value size (prep kernel)
    void *tval; size_t tval_bytes; const uint8_t *pres_tmpl; uint8_t *tpres; int64_t nrows;   // T cleared, T's presence (prep kernel)
    uint32_t henc;            // ids below this are hot ranks
    int want_cluster;         // requested cluster size C (1, 2, 4, 8, 16)
    uint32_t want_repl;       // requested replicated tier T0 (entries), used when C > 1
    // filled in by spmv_run_launch
    int cluster;              // cluster size launched
    int ctas;                 // grid of the launch: (clusters the device co-schedules) x C, or fewer when the runs run out
    uint32_t t0, t1, slice;   // replicated tier, distributed tier (C * slice >= t1), slice entries per CTA
};

// ------------------------------------------------------------------ masked pull with early exit (BFS-shaped calls)
// w<mask> = A (+).(x) u for monoids with a terminal value (LOR, LAND, ANY): one warp per row, rows the mask
// rules out are skipped entirely (their entries are never read), and a row stops as soon as its monoid
// saturates -- the BFS step `A.mxv(q, mask=visited, desc=RC, semiring=LOR_LAND)` of
// reference: tests/test_descriptor.py:13-30 touches only the unvisited rows and, for each, only the
// entries up to the first frontier hit.  Output: T restricted to the rows the mask lets through.
struct PullArgs {
    const uint32_t *rowptr; const uint32_t *col; const void *aval; int64_t nrows;
    const void *uval; const uint8_t *upres;
    const void *mval; const uint8_t *mpres; int mtc; int mask_comp, mask_struct;
    void *tval; uint8_t *tpres;
    int add_op, mul_op, flip;
    int has_long; int64_t long_cap;
    uint32_t *long_rows; int *long_count;                      // work list of the rows left to the CTA-per-row kernel
};
constexpr uint32_t PULL_LONG = 4096;          // rows longer than this go to the CTA-per-row kernel

// ------------------------------------------------------------------ masked push for small frontiers (same three monoids)
// The transpose of the pull: for every present u(k), walk row k of the OTHER orientation's CSR and store into
// T(j) for the columns j the mask lets through.  LOR / LAND / ANY need no atomics: T(j) starts at the monoid's
// identity-like value and every store is idempotent (LOR: "a product was true", LAND: "a product was false",
// ANY: any product).  Work is proportional to the frontier's out-edges; used when those are < nnz / 16.
struct PushArgs {
    const uint32_t *rowptr; const uint32_t *col; const void *aval; int64_t nin;    // CSR whose rows are the input positions k
    const void *uval; const uint8_t *upres;
    const void *mval; const uint8_t *mpres; int mtc; int mask_comp, mask_struct;
    void *tval; uint8_t *tpres; int64_t nout;
    int add_op, mul_op, flip;
    uint32_t *list; int64_t *chunk_scan; unsigned long long *counters;           // frontier list, chunk offsets, {count, edges}
};
GrB_Info spmv_masked_push_try(int xt, int zt, PushArgs &a, int64_t nnz_total, bool *done, std::string *err);
