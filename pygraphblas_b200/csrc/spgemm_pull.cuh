// The pull route of a complemented-mask mxm with a saturating monoid (spgemm_pull.cu, DESIGN.md section 3.2):
// T(i,j) for the open columns j of a row i is the fold of op(A)(i,p) (x) op(B)(p,j) over column j of op(B) -- row j of
// op(B)' -- in ascending p, stopped once the value is settled.
#pragma once
#include "common.cuh"

// The operands of one narrow-route call: op(A) rows, M' rows (the mask entries that block; m_ptr null when none do) and
// op(B)' rows, all with 32-bit offsets.  a_val and bt_val are of the multiply's x type (null when the multiply does not read them).
struct PullOperands {
    const uint32_t *a_ptr, *a_col; const void *a_val;
    const uint32_t *m_ptr, *m_col;
    const uint32_t *bt_ptr, *bt_col; const void *bt_val;
    int64_t nrows, ncols;                  // of T
    int64_t inner;                         // nrows(op(B)) = ncols(op(A))
    int xt, zt, add, mul; bool need_a, need_b;
};

// The pull rows of one call, processed in groups whose bitmaps fit tunables().mxm_pull_budget
struct PullPlan {
    int64_t n = 0, group = 0, words = 0, iwords = 0;
    int32_t *rows = nullptr;               // the pull rows (any order)
    uint32_t *abit = nullptr, *mbit = nullptr, *hit = nullptr;   // per group row: op(A)(i,:), M'(i,:) and the columns with a product
    int64_t *wcnt = nullptr;               // per group row and 32-column word: the entries of T there, then their exclusive scan
};

// The rule: row i pulls when flops[i] > 0 and (dot, or alpha > 0 and alpha * flops[i] * ncols >= open_i * bnnz, open_i = ncols - |M'(i,:)|).
// The pull rows get flops[i] = 0, so that no push bin takes them; pp gets the rows and its scratch (its bitmaps cleared).
GrB_Info pull_plan(const PullOperands &o, int64_t *flops, bool dot, double alpha, int64_t bnnz, PullPlan &pp, std::string *err);
// cnt[i] += the entries of T(i,:) of every pull row i
GrB_Info pull_count(const PullOperands &o, const PullPlan &pp, int64_t *cnt, std::string *err);
// the columns (ascending) and values of the pull rows of T, at the row offsets c_ptr
GrB_Info pull_fill(const PullOperands &o, const PullPlan &pp, const int64_t *c_ptr, uint32_t *c_col, void *c_val, std::string *err);
