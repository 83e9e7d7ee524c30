// Run kernels with run-time operator codes (every builtin semiring that has no compile-time specialisation).
#include "spmv_run.cuh"

bool spmv_run_generic(int xt, int zt, const RunArgs &a) {
    bool ok;
    GB_FOR_DOMAINS(xt, zt, ok, spmv_run_launch<XT_, ZT_, -1, -1>(a, nullptr, 0));
    return ok;
}
