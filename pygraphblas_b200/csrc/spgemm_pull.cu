// The pull route of a complemented-mask mxm with a saturating monoid (LOR, LAND, ANY): the direction-optimising step of
// multi-source BFS (DESIGN.md section 3.2).  For a pull row i, every column j that M'(i,:) leaves open walks column j of
// op(B) (row j of op(B)') in ascending p and tests op(A)(i,p) in a bitmap of the row, stopping once the value is settled.
//
// A group of pull rows holds, per row, a bitmap of op(A)(i,:) (nrows(op(B)) bits), one of M'(i,:) and one of the columns that
// have a product (ncols bits each), and a count per 32-column word.  A warp takes one (row, word): a lane per open column walks
// its op(B)' row serially, and columns longer than MXM_PULL_LONG are walked by the whole warp, 32 probes per step.
// The count pass only asks whether a column has a product (it stops at the first); the fill pass recounts the group, scans the
// word counts into positions and folds the products of the columns that have one.
#include "spgemm_pull.cuh"
#include "pull_fold.cuh"
#include "spmv_common.cuh"

static constexpr uint32_t MXM_PULL_LONG = 128;      // op(B)' rows longer than this are walked by a warp, not a lane

__global__ void pull_pick_kernel(const PullOperands o, int64_t *flops, bool dot, double alpha, int64_t bnnz, int32_t *rows,
                                 unsigned int *count) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < o.nrows; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t f = flops[i];
        if (f == 0) continue;
        const int64_t open = o.ncols - (o.m_ptr ? (int64_t)(o.m_ptr[i + 1] - o.m_ptr[i]) : 0);
        if (dot || (alpha > 0 && alpha * (double)f * (double)o.ncols >= (double)open * (double)bnnz)) {
            rows[atomicAdd(count, 1u)] = (int32_t)i;
            flops[i] = 0;
        }
    }
}

// SET: the bits of op(A)(i,:) and M'(i,:) of every row of the group; else the words that hold them are cleared again
template <bool SET>
__global__ void __launch_bounds__(256) pull_bits_kernel(const PullOperands o, const PullPlan pp, int64_t ng) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t g = warp; g < ng; g += nwarps) {
        const int32_t i = pp.rows[g];
        uint32_t *ab = pp.abit + g * pp.iwords;
        for (uint32_t e = o.a_ptr[i] + lane; e < o.a_ptr[i + 1]; e += 32) {
            const uint32_t p = __ldg(o.a_col + e);
            if (SET) atomicOr(ab + (p >> 5), 1u << (p & 31)); else ab[p >> 5] = 0;
        }
        if (!o.m_ptr) continue;
        uint32_t *mb = pp.mbit + g * pp.words;
        for (uint32_t e = o.m_ptr[i] + lane; e < o.m_ptr[i + 1]; e += 32) {
            const uint32_t j = __ldg(o.m_col + e);
            if (SET) atomicOr(mb + (j >> 5), 1u << (j & 31)); else mb[j >> 5] = 0;
        }
    }
}

__device__ __forceinline__ bool pull_bit(const uint32_t *b, uint32_t p) { return (__ldg(b + (p >> 5)) >> (p & 31)) & 1u; }

// Per (row, word) of the group: which open columns have at least one product -> pp.hit, pp.wcnt, and cnt[i] when given
__global__ void __launch_bounds__(256) pull_count_kernel(const PullOperands o, const PullPlan pp, int64_t ng, int64_t *cnt) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t w = warp; w < ng * pp.words; w += nwarps) {
        const int64_t g = w / pp.words, wd = w - g * pp.words;
        const uint32_t *ab = pp.abit + g * pp.iwords;
        const uint32_t j = (uint32_t)(wd * 32 + lane);
        const bool open = j < o.ncols && !((pp.mbit[g * pp.words + wd] >> lane) & 1u);
        uint32_t s = 0, e = 0;
        if (open) { s = o.bt_ptr[j]; e = o.bt_ptr[j + 1]; }
        const bool lng = e - s > MXM_PULL_LONG;
        bool hit = false;
        if (!lng)
            for (uint32_t k = s; k < e; ++k)
                if (pull_bit(ab, __ldg(o.bt_col + k))) { hit = true; break; }
        for (unsigned lm = __ballot_sync(0xffffffffu, lng); lm; lm &= lm - 1) {
            const int c = __ffs(lm) - 1;
            const uint32_t cs = __shfl_sync(0xffffffffu, s, c), ce = __shfl_sync(0xffffffffu, e, c);
            bool found = false;
            for (uint32_t k0 = cs; k0 < ce && !found; k0 += 32) {
                const uint32_t k = k0 + lane;
                found = __any_sync(0xffffffffu, k < ce && pull_bit(ab, __ldg(o.bt_col + k)));
            }
            if (lane == c) hit = found;
        }
        const unsigned hits = __ballot_sync(0xffffffffu, hit);
        if (lane == 0) {
            pp.hit[w] = hits; pp.wcnt[w] = __popc(hits);
            if (cnt && hits) atomicAdd(reinterpret_cast<unsigned long long *>(cnt + pp.rows[g]), (unsigned long long)__popc(hits));
        }
    }
}

// T(i,j) sits at c_ptr[i] + the entries of the row's earlier words (pp.wcnt, scanned over the group) + its rank in the word
__device__ __forceinline__ int64_t pull_pos(const PullPlan &pp, const int64_t *c_ptr, int32_t i, int64_t g, int64_t w, unsigned hits, int lane) {
    return c_ptr[i] + (pp.wcnt[w] - pp.wcnt[g * pp.words]) + __popc(hits & ((1u << lane) - 1u));
}

// op(A)(i,p) (x) op(B)(p,j), where k is the position of op(B)(p,j) in op(B)'; op(A)(i,p) by a search of op(A)'s sorted row i
template <typename XT, typename ZT>
__device__ __forceinline__ ZT pull_mxm_product(const PullOperands &o, int32_t i, uint32_t p, uint32_t k) {
    XT av = (XT)1, bv = (XT)1;
    if (o.need_a) {
        uint32_t lo = o.a_ptr[i], hi = o.a_ptr[i + 1];
        while (lo < hi) {
            const uint32_t mid = (lo + hi) >> 1;
            if (__ldg(o.a_col + mid) < p) lo = mid + 1; else hi = mid;
        }
        av = gload<XT>(static_cast<const XT *>(o.a_val) + lo);
    }
    if (o.need_b) bv = gload<XT>(static_cast<const XT *>(o.bt_val) + k);
    return MulApply<XT, ZT>::f(o.mul, av, bv);
}

template <typename XT, typename ZT>
__global__ void __launch_bounds__(256) pull_fill_kernel(const PullOperands o, const PullPlan pp, int64_t ng, const int64_t *c_ptr,
                                                        uint32_t *c_col, ZT *c_val) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int add = o.add;
    for (int64_t w = warp; w < ng * pp.words; w += nwarps) {
        const unsigned hits = pp.hit[w];
        if (!hits) continue;
        const int64_t g = w / pp.words, wd = w - g * pp.words;
        const int32_t i = pp.rows[g];
        const uint32_t *ab = pp.abit + g * pp.iwords;
        const uint32_t j = (uint32_t)(wd * 32 + lane);
        const bool mine = (hits >> lane) & 1u;
        uint32_t s = 0, e = 0;
        if (mine) { s = o.bt_ptr[j]; e = o.bt_ptr[j + 1]; }
        const bool lng = e - s > MXM_PULL_LONG;
        int n = 0; bool sat = false; ZT first = (ZT)0;
        if (mine && !lng)
            for (uint32_t k = s; k < e; ++k) {
                const uint32_t p = __ldg(o.bt_col + k);
                if (!pull_bit(ab, p)) continue;
                const ZT v = pull_mxm_product<XT, ZT>(o, i, p, k);
                if (n == 0) first = v;
                n = min(2, n + 1);
                sat |= monoid_saturated<ZT>(add, v);
                if (sat && (n >= 2 || pull_settled<ZT>(add, first))) break;
            }
        for (unsigned lm = __ballot_sync(0xffffffffu, lng); lm; lm &= lm - 1) {
            const int c = __ffs(lm) - 1;
            const uint32_t cs = __shfl_sync(0xffffffffu, s, c), ce = __shfl_sync(0xffffffffu, e, c);
            int cn = 0; bool csat = false; ZT cfirst = (ZT)0;
            for (uint32_t k0 = cs; k0 < ce; k0 += 32) {
                const uint32_t k = k0 + lane;
                bool has = false; ZT v = (ZT)0;
                if (k < ce) {
                    const uint32_t p = __ldg(o.bt_col + k);
                    if (pull_bit(ab, p)) { v = pull_mxm_product<XT, ZT>(o, i, p, k); has = true; }
                }
                const unsigned hm = __ballot_sync(0xffffffffu, has), sm = __ballot_sync(0xffffffffu, has && monoid_saturated<ZT>(add, v));
                if (hm) {
                    const ZT fv = shfl_idx_t<ZT>(v, __ffs(hm) - 1);      // the lowest lane: the smallest p of the step
                    if (cn == 0) cfirst = fv;
                    cn = min(2, cn + __popc(hm));
                    csat |= sm != 0;
                }
                if (csat && (cn >= 2 || pull_settled<ZT>(add, cfirst))) break;
            }
            if (lane == c) { n = cn; sat = csat; first = cfirst; }
        }
        if (mine) {
            const int64_t pos = pull_pos(pp, c_ptr, i, g, w, hits, lane);
            c_col[pos] = j;
            c_val[pos] = pull_result<ZT>(add, n, sat, first);
        }
    }
}

// PAIR multiplies: every product is 1, and so is the fold of any number of them under LOR, LAND and ANY -- no walk, no values
__global__ void __launch_bounds__(256) pull_fill_pair_kernel(const PullOperands o, const PullPlan pp, int64_t ng, const int64_t *c_ptr,
                                                             uint32_t *c_col, uint8_t *c_val, uint64_t one, int zsz) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t w = warp; w < ng * pp.words; w += nwarps) {
        const unsigned hits = pp.hit[w];
        if (!((hits >> lane) & 1u)) continue;
        const int64_t g = w / pp.words, wd = w - g * pp.words;
        const int64_t pos = pull_pos(pp, c_ptr, pp.rows[g], g, w, hits, lane);
        c_col[pos] = (uint32_t)(wd * 32 + lane);
        for (int b = 0; b < zsz; ++b) c_val[pos * zsz + b] = (uint8_t)(one >> (8 * b));
    }
}

// ------------------------------------------------------------------ host side
GrB_Info pull_plan(const PullOperands &o, int64_t *flops, bool dot, double alpha, int64_t bnnz, PullPlan &pp, std::string *err) {
    pp = PullPlan();
    DevBuf<unsigned int> count;
    GB_TRY(count.alloc(1, err));
    CU_TRY(cudaMemsetAsync(count, 0, 4, G.stream), err);
    int32_t *rows = nullptr;
    GB_TRY(ws_array(WS_PULL_ROWS, &rows, (size_t)o.nrows, err));
    pull_pick_kernel<<<grid_for(o.nrows), 256, 0, G.stream>>>(o, flops, dot, alpha, bnnz, rows, count); GB_LAUNCHED();
    unsigned int n = 0;
    CU_TRY(cudaMemcpyAsync(&n, count, 4, cudaMemcpyDeviceToHost, G.stream), err);
    CU_TRY(cudaStreamSynchronize(G.stream), err);
    if (!n) return GrB_SUCCESS;
    pp.rows = rows; pp.words = ceil_div(o.ncols, 32); pp.iwords = ceil_div(o.inner, 32);
    const int64_t per_row = (pp.iwords + 2 * pp.words) * 4 + pp.words * 8;
    pp.group = std::max<int64_t>(1, std::min<int64_t>(n, tunables().mxm_pull_budget / per_row));
    void *buf = nullptr;
    GB_TRY(ws_get(WS_PULL_BUF, &buf, (size_t)(pp.group * per_row) + 8 + 16, err));
    pp.wcnt = static_cast<int64_t *>(buf);                        // group * words + 1: the scan's total in the last slot
    pp.abit = reinterpret_cast<uint32_t *>(pp.wcnt + pp.group * pp.words + 1);
    pp.mbit = pp.abit + pp.group * pp.iwords;
    pp.hit = pp.mbit + pp.group * pp.words;
    CU_TRY(cudaMemsetAsync(pp.abit, 0, (size_t)pp.group * (pp.iwords + pp.words) * 4, G.stream), err);   // both bitmaps
    pp.n = n;
    return GrB_SUCCESS;
}

// the rows [g0, g0 + ng) of the plan
static PullPlan pull_group(const PullPlan &pp, int64_t g0, int64_t *ng) {
    PullPlan q = pp;
    q.rows = pp.rows + g0;
    *ng = std::min(pp.group, pp.n - g0);
    return q;
}

GrB_Info pull_count(const PullOperands &o, const PullPlan &pp, int64_t *cnt, std::string *err) {
    for (int64_t g0 = 0; g0 < pp.n; g0 += pp.group) {
        int64_t ng = 0;
        const PullPlan q = pull_group(pp, g0, &ng);
        pull_bits_kernel<true><<<grid_for(ng * 32), 256, 0, G.stream>>>(o, q, ng);
        pull_count_kernel<<<grid_for(ng * q.words * 32), 256, 0, G.stream>>>(o, q, ng, cnt);
        pull_bits_kernel<false><<<grid_for(ng * 32), 256, 0, G.stream>>>(o, q, ng);
        G.launches += 3;
    }
    CU_TRY(cudaGetLastError(), err);
    return GrB_SUCCESS;
}

static uint64_t one_bits(int tc) {
    if (tc == TC_FP32) { const float f = 1.0f; uint32_t u; memcpy(&u, &f, 4); return u; }
    if (tc == TC_FP64) { const double d = 1.0; uint64_t u; memcpy(&u, &d, 8); return u; }
    return 1;
}

GrB_Info pull_fill(const PullOperands &o, const PullPlan &pp, const int64_t *c_ptr, uint32_t *c_col, void *c_val, std::string *err) {
    for (int64_t g0 = 0; g0 < pp.n; g0 += pp.group) {
        int64_t ng = 0;
        const PullPlan q = pull_group(pp, g0, &ng);
        const int grid = grid_for(ng * q.words * 32);
        pull_bits_kernel<true><<<grid_for(ng * 32), 256, 0, G.stream>>>(o, q, ng);
        pull_count_kernel<<<grid, 256, 0, G.stream>>>(o, q, ng, nullptr);
        G.launches += 2;
        CU_TRY(cudaMemsetAsync(q.wcnt + ng * q.words, 0, 8, G.stream), err);
        GB_TRY(dev_exclusive_scan(q.wcnt, ng * q.words + 1, err));
        if (o.mul == OP_PAIR) {
            pull_fill_pair_kernel<<<grid, 256, 0, G.stream>>>(o, q, ng, c_ptr, c_col, static_cast<uint8_t *>(c_val), one_bits(o.zt),
                                                              (int)tc_size(o.zt));
            GB_LAUNCHED();
        } else {
            bool ok;
            GB_FOR_DOMAINS(o.xt, o.zt, ok, pull_fill_kernel<XT_, ZT_><<<grid, 256, 0, G.stream>>>(o, q, ng, c_ptr, c_col, static_cast<ZT_ *>(c_val));
                           GB_LAUNCHED());
            if (!ok) return gb_fail(GrB_DOMAIN_MISMATCH, err, "mxm: unsupported semiring domains (x=%d, z=%d)", o.xt, o.zt);
        }
        pull_bits_kernel<false><<<grid_for(ng * 32), 256, 0, G.stream>>>(o, q, ng); GB_LAUNCHED();
    }
    CU_TRY(cudaGetLastError(), err);
    return GrB_SUCCESS;
}
