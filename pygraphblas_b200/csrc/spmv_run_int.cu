// Integer and BOOL instantiations of the run kernels.
#include "spmv_run.cuh"

bool spmv_run_fast_int(int xt, int add, int mul, const RunArgs &a, Hot2Args *hot, size_t table_limit) {
    switch (xt) {
        case TC_INT32: return spmv_run_fast<int32_t>(add, mul, a, hot, table_limit);
        case TC_INT64: return spmv_run_fast<int64_t>(add, mul, a, hot, table_limit);
        case TC_UINT32: return spmv_run_fast<uint32_t>(add, mul, a, hot, table_limit);
        case TC_UINT64: return spmv_run_fast<uint64_t>(add, mul, a, hot, table_limit);
        case TC_BOOL: return spmv_run_fast<bool>(add, mul, a, hot, table_limit);
        default: return false;
    }
}
