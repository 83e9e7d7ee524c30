// The fold of the pull kernels for the saturating monoids (LOR, LAND, ANY): the masked mxv pull (spmv_pull.cu) and the
// complemented-mask mxm pull (spgemm_pull.cu) state it once, here.
#pragma once
#include "common.cuh"

template <typename ZT> __device__ __forceinline__ bool monoid_saturated(int add, ZT v) {
    switch (add) {
        case OP_LOR: return v != (ZT)0;
        case OP_LAND: return v == (ZT)0;
        case OP_ANY: return true;
        default: return false;
    }
}
// The three monoids of this kernel (LOR, LAND, ANY) need no running value: the fold of a row's products is
// decided by how many there are (0, 1, more), whether one of them saturates, and the first one --
//   0 products: no entry;  1: that product, as is;  more: ANY -> any of them, LOR -> "one was non-zero",
//   LAND -> "none was zero" (1 or 0 in the monoid's type).
// A row may stop early once its result can no longer change.
template <typename ZT> __device__ __forceinline__ ZT pull_result(int add, int n, bool sat, ZT first) {
    if (n <= 1 || add == OP_ANY) return first;
    return add == OP_LOR ? (ZT)(sat ? 1 : 0) : (ZT)(sat ? 0 : 1);
}
template <typename ZT> __device__ __forceinline__ bool pull_settled(int add, ZT v) {     // saturating AND already the final value
    switch (add) {
        case OP_LOR: return v == (ZT)1;
        case OP_LAND: return v == (ZT)0;
        case OP_ANY: return true;
        default: return false;
    }
}
