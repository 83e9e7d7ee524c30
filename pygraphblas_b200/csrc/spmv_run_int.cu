// Integer and BOOL instantiations of the run kernels.
#include "spmv_run.cuh"

template <typename T> static bool spmv_run_fast(int add, int mul, const RunArgs &a, Hot2Args *hot, size_t table_limit) {
#define GB_FAST(A, M) if (add == A && mul == M) { spmv_run_launch<T, T, A, M>(a, hot, table_limit); return true; }
    GB_FAST(OP_PLUS, OP_TIMES) GB_FAST(OP_MIN, OP_PLUS) GB_FAST(OP_PLUS, OP_SECOND) GB_FAST(OP_PLUS, OP_FIRST)
    GB_FAST(OP_PLUS, OP_PAIR) GB_FAST(OP_MIN, OP_FIRST) GB_FAST(OP_MIN, OP_SECOND)
#undef GB_FAST
    return false;
}
static bool spmv_run_fast_bool(int add, int mul, const RunArgs &a, Hot2Args *hot, size_t table_limit) {
#define GB_FAST(A, M) if (add == A && mul == M) { spmv_run_launch<bool, bool, A, M>(a, hot, table_limit); return true; }
    GB_FAST(OP_LOR, OP_LAND) GB_FAST(OP_ANY, OP_PAIR) GB_FAST(OP_LOR, OP_PAIR) GB_FAST(OP_LOR, OP_SECOND) GB_FAST(OP_LOR, OP_FIRST)
#undef GB_FAST
    return false;
}
bool spmv_run_fast_int(int xt, int add, int mul, const RunArgs &a, Hot2Args *hot, size_t table_limit) {
    switch (xt) {
        case TC_INT32: return spmv_run_fast<int32_t>(add, mul, a, hot, table_limit);
        case TC_INT64: return spmv_run_fast<int64_t>(add, mul, a, hot, table_limit);
        case TC_UINT32: return spmv_run_fast<uint32_t>(add, mul, a, hot, table_limit);
        case TC_UINT64: return spmv_run_fast<uint64_t>(add, mul, a, hot, table_limit);
        case TC_BOOL: return spmv_run_fast_bool(add, mul, a, hot, table_limit);
        default: return false;
    }
}
