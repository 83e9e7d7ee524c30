// spgemm.cu -- GrB_mxm on sm_90a:  C<M> = accum(C, op(A) (+).(x) op(B))
//
// Replaces the SuiteSparse call behind reference: pygraphblas/matrix.py:2574
// (Matrix.mxm, `@`, `@=`, `**`).  Gustavson row-wise formulation, three methods:
//
//   unmasked    per-row flop count -> rows binned by flops -> symbolic pass (distinct
//               columns per row) -> scan -> numeric pass.  Small / medium rows count their
//               columns in a shared-memory hash table (atomicCAS probing) and form their
//               values by expand-sort-compress in shared memory; rows beyond the shared-memory
//               budget use a dense accumulator in HBM owned by a persistent CTA.  Rows come out
//               sorted (in-smem bitonic sort / ordered bitmap sweep).  A complemented mask runs the same pipeline
//               with the mask's blocking entries filtered inside each kernel (COMP instantiations).
//   masked      C<M> = A*B with a non-complemented mask: the mask row M(i,:) is loaded into
//               the table first, products are accumulated only where they hit it, so both
//               the work kept and the output are bounded by nnz(M) (triangle counting,
//               reference: demo/Triangle-Counting.ipynb:581-582).
//   masked dot  C<M> = A*B' (INP1 = TRAN) with a mask: sorted-row intersection per mask
//               entry, no transpose materialised (reference: demo/TriangleCentrality.ipynb:596).
//
// The general write-back  C<M> = accum(C, T)  (mask value/structure/complement, replace,
// accumulator, typecasts) is a row-wise three-way merge (matrix_finalize).
#include "common.cuh"
#include "spgemm_pull.cuh"
#include <algorithm>
#include <functional>
#include <limits>
#include <type_traits>

static constexpr uint32_t EMPTY_KEY = 0xFFFFFFFFu;

// ------------------------------------------------------------------ device helpers
// storage word of an accumulator slot: 32-bit for types up to 4 bytes, 64-bit otherwise
template <typename ZT> struct SlotWord { typedef typename std::conditional<sizeof(ZT) == 8, unsigned long long, unsigned int>::type W; };
template <typename ZT> __host__ __device__ __forceinline__ typename SlotWord<ZT>::W pack_slot(ZT v) {
    typename SlotWord<ZT>::W w = 0;
    memcpy(&w, &v, sizeof(ZT));
    return w;
}
template <typename ZT> __host__ __device__ __forceinline__ ZT unpack_slot(typename SlotWord<ZT>::W w) {
    ZT v; memcpy(&v, &w, sizeof(ZT)); return v;
}

// Starting value of an accumulator slot that the products of one entry are folded into (its presence is kept apart: keys,
// bitmaps or found flags).  Integer and BOOL monoids start from their identity.  FP monoids start from the identity of the IEEE
// operation, which fmin / fmax / + leave every x unchanged with: fmin(NaN, x) = fmax(NaN, x) = x and -0.0 + x = x.  The monoid
// identities are not that: fmin(+Inf, NaN) = +Inf and +0.0 + -0.0 = +0.0, so an entry whose only product is NaN (or -0.0)
// would come out +Inf (or +0.0) where the fold from the first product gives NaN (-0.0).
template <typename ZT> __host__ __device__ __forceinline__ ZT accum_init(int add) {
    if constexpr (std::is_floating_point<ZT>::value) {
        if (add == OP_MIN || add == OP_MAX) return std::numeric_limits<ZT>::quiet_NaN();
        if (add == OP_PLUS) return (ZT)-0.0;
    }
    return monoid_identity<ZT>(add);
}

// *addr = add(*addr, v) atomically; works on shared and global addresses.
//
// FP32 PLUS: atomicAdd(float *) on a global address is RED.ADD.F32.FTZ on sm_90, which flushes subnormal operands and results to
// zero.  For |v| >= 2^-100 (or v = +-Inf) the flush cannot change the sum, so the reduction is used there: (i) a subnormal *addr
// is below half an ulp of v, so the exact sum rounds to v, which is what the flushed operand gives; (ii) for a normal *addr the
// sum is 0 or at least 2^-124 in magnitude (either |*addr| < |v| / 2, or both are multiples of 2^-124), never subnormal.
// Smaller v, zeros and NaN take the compare-and-swap loop, whose plain add keeps subnormals.
template <typename ZT> __device__ __forceinline__ void atomic_combine(typename SlotWord<ZT>::W *addr, ZT v, int add) {
    typedef typename SlotWord<ZT>::W W;
    if (add == OP_ANY) { *addr = pack_slot<ZT>(v); return; }
    if constexpr (std::is_same<ZT, float>::value) {
        if (add == OP_PLUS && fabsf(v) >= 0x1p-100f) { atomicAdd(reinterpret_cast<float *>(addr), v); return; }
    }
    if constexpr (std::is_same<ZT, double>::value) { if (add == OP_PLUS) { atomicAdd(reinterpret_cast<double *>(addr), v); return; } }
    if constexpr (std::is_same<ZT, int32_t>::value || std::is_same<ZT, uint32_t>::value) {
        if (add == OP_PLUS) { atomicAdd(reinterpret_cast<unsigned int *>(addr), (unsigned int)v); return; }
    }
    if constexpr (std::is_same<ZT, int64_t>::value || std::is_same<ZT, uint64_t>::value) {
        if (add == OP_PLUS) { atomicAdd(reinterpret_cast<unsigned long long *>(addr), (unsigned long long)v); return; }
    }
    if constexpr (std::is_same<ZT, int32_t>::value) {
        if (add == OP_MIN) { atomicMin(reinterpret_cast<int *>(addr), v); return; }
        if (add == OP_MAX) { atomicMax(reinterpret_cast<int *>(addr), v); return; }
    }
    if constexpr (std::is_same<ZT, uint32_t>::value) {
        if (add == OP_MIN) { atomicMin(reinterpret_cast<unsigned int *>(addr), v); return; }
        if (add == OP_MAX) { atomicMax(reinterpret_cast<unsigned int *>(addr), v); return; }
    }
    if constexpr (std::is_same<ZT, int64_t>::value) {
        if (add == OP_MIN) { atomicMin(reinterpret_cast<long long *>(addr), (long long)v); return; }
        if (add == OP_MAX) { atomicMax(reinterpret_cast<long long *>(addr), (long long)v); return; }
    }
    if constexpr (std::is_same<ZT, uint64_t>::value) {
        if (add == OP_MIN) { atomicMin(reinterpret_cast<unsigned long long *>(addr), (unsigned long long)v); return; }
        if (add == OP_MAX) { atomicMax(reinterpret_cast<unsigned long long *>(addr), (unsigned long long)v); return; }
    }
    W old = *addr;
    while (true) {
        const ZT n = MulApply<ZT, ZT>::f(add, unpack_slot<ZT>(old), v);
        const W seen = atomicCAS(addr, old, pack_slot<ZT>(n));
        if (seen == old) break;
        old = seen;
    }
}

// multiplicative (Fibonacci) hashing: the HIGH bits of c * 2^32/phi index a table of 2^k slots (shift = 32 - k);
// the low bits would only permute the low bits of c and cluster structured column ids
__device__ __forceinline__ uint32_t hash_col(uint32_t c, int shift) { return (c * 2654435761u) >> shift; }

// BT: the type of B's row offsets (uint32_t: rowptr32; int64_t: rowptr, the wide route of the masked methods).  A's and M's
// offsets stay 32-bit: the wide route hands the kernels row panels of A and M with offsets rebased to the panel.
template <typename BT> struct GemmArgsT {
    const uint32_t *a_ptr, *a_col; const void *a_val;
    const BT *b_ptr; const uint32_t *b_col; const void *b_val;
    const uint32_t *m_ptr, *m_col; const void *m_val; int m_tc; int m_struct;   // mask (masked kernels)
    int64_t nrows, ncols;
    const int32_t *rows; int64_t nbin;          // rows of this bin
    int64_t *c_cnt;                              // symbolic: c_cnt[row] = nnz(C(row,:))
    const int64_t *c_ptr; uint32_t *c_col; void *c_val;   // numeric outputs
    uint8_t *t_found;                            // masked: per mask entry "has a value"
    int add_op, mul_op, need_a, need_b;
    int table;                                   // hash table size (power of two)
    int group;                                   // threads per row: 32 (warp) or blockDim (CTA)
    // dense accumulator workspace (one slice per CTA)
    uint32_t *spa_bits; void *spa_val; int64_t spa_words; unsigned int *queue;
};
typedef GemmArgsT<uint32_t> GemmArgs;

// ------------------------------------------------------------------ flop count + binning
template <typename BT>
__global__ void flops_kernel(const uint32_t *a_ptr, const uint32_t *a_col, const BT *b_ptr, int64_t nrows,
                             int64_t *flops, unsigned long long *total) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    unsigned long long mine = 0;
    for (int64_t r = warp; r < nrows; r += nwarps) {
        int64_t f = 0;
        for (uint32_t p = a_ptr[r] + lane; p < a_ptr[r + 1]; p += 32) { const uint32_t k = a_col[p]; f += b_ptr[k + 1] - b_ptr[k]; }
        for (int o = 16; o > 0; o >>= 1) f += __shfl_xor_sync(0xffffffffu, f, o);
        if (lane == 0) { flops[r] = f; mine += (unsigned long long)f; }
    }
    if (lane == 0 && mine) atomicAdd(total, mine);
}

// bins: 0 = nothing to do, 1 = warp per row (shared memory), 2 = CTA per row (shared memory), 3 = dense accumulator
struct BinLimits { int64_t small_max, medium_max; };
__global__ void bin_count_kernel(const int64_t *work, int64_t nrows, BinLimits lim, unsigned int *counts) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += (int64_t)gridDim.x * blockDim.x) {
        const int64_t f = work[r];
        const int b = f == 0 ? 0 : (f <= lim.small_max ? 1 : (f <= lim.medium_max ? 2 : 3));
        atomicAdd(&counts[b], 1u);
    }
}
__global__ void bin_fill_kernel(const int64_t *work, int64_t nrows, BinLimits lim, const unsigned int *offsets,
                                unsigned int *cursor, int32_t *rows) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += (int64_t)gridDim.x * blockDim.x) {
        const int64_t f = work[r];
        const int b = f == 0 ? 0 : (f <= lim.small_max ? 1 : (f <= lim.medium_max ? 2 : 3));
        rows[offsets[b] + atomicAdd(&cursor[b], 1u)] = (int32_t)r;
    }
}

// ------------------------------------------------------------------ bitonic sort of 64-bit words in shared memory
template <bool WARP> __device__ __forceinline__ void group_sync() { if (WARP) __syncwarp(); else __syncthreads(); }

template <bool WARP> __device__ void bitonic_sort_u64(unsigned long long *a, int n, int tid, int nthreads) {
    for (int k = 2; k <= n; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = tid; i < n; i += nthreads) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const unsigned long long x = a[i], y = a[ixj];
                    const bool up = (i & k) == 0;
                    if ((x > y) == up) { a[i] = y; a[ixj] = x; }
                }
            }
            group_sync<WARP>();
        }
    }
}

// ------------------------------------------------------------------ complemented mask: the columns that block a position
// COMP instantiations of the unmasked kernels compute T = (A (+).(x) B)<!M'> where M' (m_ptr / m_col, sorted rows) holds the
// mask entries that block: a column j of row i survives when it is not in M'(i, [ms, me)).  A binary search of the mask row
// keeps the test at log2(ncols) loads however long the row is (the path counts of betweenness centrality are full rows).
__device__ __forceinline__ bool mask_blocks(const uint32_t *m_col, uint32_t ms, uint32_t me, uint32_t j) {
    uint32_t lo = ms, hi = me;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (__ldg(m_col + mid) < j) lo = mid + 1; else hi = mid;
    }
    return lo < me && __ldg(m_col + lo) == j;
}

// ------------------------------------------------------------------ unmasked, symbolic pass: shared-memory hash
// One row per group (a warp, or the whole CTA): count its distinct columns (COMP: those not blocked by M', tested once per
// distinct column, when it first enters the table).
template <bool WARP, bool COMP, typename BT>
__global__ void __launch_bounds__(256) hash_symbolic_kernel(const GemmArgsT<BT> p) {
    extern __shared__ unsigned char smem_raw[];
    const int gsize = WARP ? 32 : blockDim.x;
    const int gid = WARP ? (threadIdx.x >> 5) : 0;
    const int tid = WARP ? (threadIdx.x & 31) : threadIdx.x;
    const int groups = WARP ? (blockDim.x >> 5) : 1;
    uint32_t *keys = reinterpret_cast<uint32_t *>(smem_raw) + (size_t)gid * p.table;
    __shared__ int s_count[8];
    const int64_t idx = (int64_t)blockIdx.x * groups + gid;
    const bool active = idx < p.nbin;
    const uint32_t tmask = (uint32_t)p.table - 1;
    const int hshift = __clz(p.table) + 1;                            // 32 - log2(table)
    for (int s = tid; s < p.table; s += gsize) keys[s] = EMPTY_KEY;
    if (tid == 0) s_count[gid] = 0;
    group_sync<WARP>();
    int mine = 0;
    if (active) {
        const int64_t row = p.rows[idx];
        const uint32_t as = p.a_ptr[row], ae = p.a_ptr[row + 1];
        uint32_t ms = 0, me = 0;
        if (COMP) { ms = p.m_ptr[row]; me = p.m_ptr[row + 1]; }
        if (WARP) {       // lane per A entry, each lane walks its B row
            for (uint32_t pa = as + tid; pa < ae; pa += 32) {
                const uint32_t k = p.a_col[pa];
                for (BT pb = p.b_ptr[k]; pb < p.b_ptr[k + 1]; ++pb) {
                    const uint32_t j = __ldg(p.b_col + pb);
                    uint32_t s = hash_col(j, hshift);
                    while (true) {
                        const uint32_t seen = atomicCAS(&keys[s], EMPTY_KEY, j);
                        if (seen == EMPTY_KEY) { if (!COMP || !mask_blocks(p.m_col, ms, me, j)) ++mine; break; }
                        if (seen == j) break;
                        s = (s + 1) & tmask;
                    }
                }
            }
        } else {          // warp per A entry, lanes stride the B row
            const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
            for (uint32_t pa = as + warp; pa < ae; pa += nwarps) {
                const uint32_t k = p.a_col[pa];
                for (BT pb = p.b_ptr[k] + lane; pb < p.b_ptr[k + 1]; pb += 32) {
                    const uint32_t j = __ldg(p.b_col + pb);
                    uint32_t s = hash_col(j, hshift);
                    while (true) {
                        const uint32_t seen = atomicCAS(&keys[s], EMPTY_KEY, j);
                        if (seen == EMPTY_KEY) { if (!COMP || !mask_blocks(p.m_col, ms, me, j)) ++mine; break; }
                        if (seen == j) break;
                        s = (s + 1) & tmask;
                    }
                }
            }
        }
    }
    for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
    if ((threadIdx.x & 31) == 0 && mine) atomicAdd(&s_count[gid], mine);
    group_sync<WARP>();
    if (active && tid == 0) p.c_cnt[p.rows[idx]] = s_count[gid];
}

// ------------------------------------------------------------------ unmasked: dense accumulator in HBM
// Persistent CTAs pull rows from a queue; each owns a bitmap (+ value array) over all columns.
// The ordered sweep of the bitmap yields the row already sorted.
__device__ __forceinline__ int block_exclusive_scan(int v, int *s_warp, int *total) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    int inc = v;
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
    if (lane == 31) s_warp[w] = inc;
    __syncthreads();
    if (w == 0) {
        int t = lane < nw ? s_warp[lane] : 0, ti = t;
        for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, ti, o); if (lane >= o) ti += y; }
        s_warp[lane] = ti - t;
        if (lane == 31) s_warp[32] = ti;
    }
    __syncthreads();
    const int r = s_warp[w] + inc - v;
    *total = s_warp[32];
    __syncthreads();
    return r;
}

// ------------------------------------------------------------------ unmasked, numeric pass: expand - sort - compress (ESC)
// The numeric pass of the two shared-memory bins.  The products of a row are EXPANDED into shared memory in their Gustavson order
// (key = column << 32 | position, the value stays at its position), the keys are SORTED by a bitonic network over the next
// power of two of the row's own product count, and equal columns are COMPRESSED by folding their values in position order.  No
// atomics and no table to clear; a floating-point PLUS monoid gives the same bit pattern on every run.  One warp per row of the
// small bin (<= 128 products), one CTA per row of the medium bin (<= 2048).  The row's output count comes from the symbolic
// pass (c_ptr).  COMP: a column blocked by M' is dropped at the compress step, one test per distinct column, and output positions
// are ranks among the survivors (the symbolic pass counted the same survivors).
static constexpr int ESC_SMALL = 128, ESC_MEDIUM = 2048;
static constexpr size_t ESC_SMEM_SMALL = (size_t)8 * ESC_SMALL * 16;                       // 8 warps x (keys 8 B + value words 8 B)
static constexpr size_t ESC_SMEM_MEDIUM = (size_t)ESC_MEDIUM * 16 + 3 * 256 * 4 + 256 * 8;   // + offsets, starts, lengths, A values of a chunk
// the medium bin with B's 64-bit offsets: the B row starts of a chunk take 8 bytes each
template <typename BT> static constexpr size_t esc_smem_medium() { return ESC_SMEM_MEDIUM + 256 * (sizeof(BT) - 4); }

template <typename XT, typename ZT, int ADD, int MUL, bool WARP, bool COMP, typename BT>
__global__ void __launch_bounds__(256) esc_numeric_kernel(const GemmArgsT<BT> p) {
    typedef typename SlotWord<ZT>::W W;
    constexpr int CAP = WARP ? ESC_SMALL : ESC_MEDIUM;
    extern __shared__ unsigned char smem_raw[];
    __shared__ int s_warp[33];
    const int add = ADD >= 0 ? ADD : p.add_op;
    const int mul = MUL >= 0 ? MUL : p.mul_op;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const int groups = WARP ? nwarps : 1, gid = WARP ? warp : 0;
    const int tid = WARP ? lane : (int)threadIdx.x, gsize = WARP ? 32 : (int)blockDim.x;
    unsigned long long *keys = reinterpret_cast<unsigned long long *>(smem_raw) + (size_t)gid * CAP;
    W *vals = reinterpret_cast<W *>(smem_raw + (size_t)groups * CAP * 8) + (size_t)gid * CAP;
    const int64_t idx = (int64_t)blockIdx.x * groups + gid;
    if (idx >= p.nbin) return;                  // a whole warp (WARP) or never (one CTA per row): no CTA barrier is skipped
    const int64_t row = p.rows[idx];
    const uint32_t as = p.a_ptr[row], ae = p.a_ptr[row + 1];
    const XT *aval = static_cast<const XT *>(p.a_val), *bval = static_cast<const XT *>(p.b_val);
    int F = 0;                                  // products expanded so far (uniform over the group)

    // ---- expand
    if constexpr (WARP) {
        for (uint32_t pa0 = as; pa0 < ae; pa0 += 32) {          // a lane per A entry, each lane walks its B row
            const uint32_t pa = pa0 + lane;
            BT bs = 0; uint32_t len = 0; XT av = (XT)1;
            if (pa < ae) {
                const uint32_t k = p.a_col[pa];
                bs = p.b_ptr[k]; len = (uint32_t)(p.b_ptr[k + 1] - bs);
                if (p.need_a) av = gload<XT>(aval + pa);
            }
            int inc = (int)len;
            for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
            const int off = F + inc - (int)len;
            for (uint32_t t = 0; t < len; ++t) {
                const int pos = off + (int)t;
                if (pos < CAP) {
                    const uint32_t j = __ldg(p.b_col + bs + t);
                    const XT bv = p.need_b ? gload<XT>(bval + bs + t) : (XT)1;
                    keys[pos] = ((unsigned long long)j << 32) | (unsigned)pos;
                    vals[pos] = pack_slot<ZT>(MulApply<XT, ZT>::f(mul, av, bv));
                }
            }
            F += __shfl_sync(0xffffffffu, inc, 31);
        }
    } else {
        uint32_t *s_off = reinterpret_cast<uint32_t *>(smem_raw + (size_t)CAP * 16);
        BT *s_bs = reinterpret_cast<BT *>(s_off + 256);
        uint32_t *s_len = reinterpret_cast<uint32_t *>(s_bs + 256);
        XT *s_av = reinterpret_cast<XT *>(s_len + 256);
        for (uint32_t pa0 = as; pa0 < ae; pa0 += 256) {         // a thread per A entry of the chunk, then a warp per entry, lanes along its B row
            const uint32_t pa = pa0 + threadIdx.x;
            BT bs = 0; uint32_t len = 0; XT av = (XT)1;
            if (pa < ae) {
                const uint32_t k = p.a_col[pa];
                bs = p.b_ptr[k]; len = (uint32_t)(p.b_ptr[k + 1] - bs);
                if (p.need_a) av = gload<XT>(aval + pa);
            }
            int total = 0;
            const int off = block_exclusive_scan((int)len, s_warp, &total);
            s_off[threadIdx.x] = (uint32_t)(F + off); s_bs[threadIdx.x] = bs; s_len[threadIdx.x] = len; s_av[threadIdx.x] = av;
            __syncthreads();
            const int nent = (int)min(256u, ae - pa0);
            for (int e = warp; e < nent; e += nwarps) {
                const uint32_t o = s_off[e], l = s_len[e];
                const BT b0 = s_bs[e];
                const XT a = s_av[e];
                for (uint32_t t = lane; t < l; t += 32) {
                    const uint32_t pos = o + t;
                    if (pos < (uint32_t)CAP) {
                        const uint32_t j = __ldg(p.b_col + b0 + t);
                        const XT bv = p.need_b ? gload<XT>(bval + b0 + t) : (XT)1;
                        keys[pos] = ((unsigned long long)j << 32) | pos;
                        vals[pos] = pack_slot<ZT>(MulApply<XT, ZT>::f(mul, a, bv));
                    }
                }
            }
            F += total;
            __syncthreads();
        }
    }
    if (F > CAP) F = CAP;                       // cannot happen: the bins are cut by the row's product count

    // ---- sort the keys (padding sorts last)
    int n2 = 2;
    while (n2 < F) n2 <<= 1;
    for (int s = F + tid; s < n2; s += gsize) keys[s] = ~0ull;
    group_sync<WARP>();
    bitonic_sort_u64<WARP>(keys, n2, tid, gsize);

    // ---- compress: the first key of every column folds the values of its run, in position order
    const int64_t base = p.c_ptr[row];
    ZT *cval = static_cast<ZT *>(p.c_val);
    int cnt = 0;
    for (int i0 = 0; i0 < F; i0 += gsize) {
        const int i = i0 + tid;
        const bool valid = i < F;
        const unsigned long long e = valid ? keys[i] : 0ull;
        const uint32_t col = (uint32_t)(e >> 32);
        bool head = valid && (i == 0 || (uint32_t)(keys[i - 1] >> 32) != col);
        if (COMP && head) head = !mask_blocks(p.m_col, p.m_ptr[row], p.m_ptr[row + 1], col);
        int rank = 0, total = 0;
        if constexpr (WARP) {
            const unsigned m = __ballot_sync(0xffffffffu, head);
            rank = cnt + __popc(m & ((1u << lane) - 1u)); total = __popc(m);
        } else {
            rank = cnt + block_exclusive_scan(head ? 1 : 0, s_warp, &total);
        }
        if (head) {
            ZT acc = unpack_slot<ZT>(vals[(uint32_t)e]);
            for (int t = i + 1; t < F; ++t) {
                const unsigned long long x = keys[t];
                if ((uint32_t)(x >> 32) != col) break;
                acc = MulApply<ZT, ZT>::f(add, acc, unpack_slot<ZT>(vals[(uint32_t)x]));
            }
            p.c_col[base + rank] = col; cval[base + rank] = acc;
        }
        cnt += total;
    }
}

// COMP: each CTA owns a second bitmap, the slice gridDim.x slices further on in spa_bits.  M'(row,:) is set into it when the
// row starts and a product tests it before its atomics, so a blocked column costs no atomic; the sweep clears it.
template <typename XT, typename ZT, int ADD, int MUL, bool NUMERIC, bool COMP, typename BT>
__global__ void __launch_bounds__(512) spa_kernel(const GemmArgsT<BT> p) {
    typedef typename SlotWord<ZT>::W W;
    __shared__ int s_warp[33];
    __shared__ unsigned int s_next;
    const int add = ADD >= 0 ? ADD : p.add_op;
    const int mul = MUL >= 0 ? MUL : p.mul_op;
    uint32_t *bits = p.spa_bits + (size_t)blockIdx.x * p.spa_words;
    uint32_t *mbits = COMP ? p.spa_bits + (size_t)(gridDim.x + blockIdx.x) * p.spa_words : nullptr;
    W *spa = NUMERIC ? static_cast<W *>(p.spa_val) + (size_t)blockIdx.x * p.ncols : nullptr;
    const W ident = pack_slot<ZT>(accum_init<ZT>(add));
    const XT *aval = static_cast<const XT *>(p.a_val), *bval = static_cast<const XT *>(p.b_val);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    while (true) {
        if (threadIdx.x == 0) s_next = atomicAdd(p.queue, 1u);
        __syncthreads();
        const unsigned int idx = s_next;
        __syncthreads();
        if (idx >= p.nbin) break;
        const int64_t row = p.rows[idx];
        const uint32_t as = p.a_ptr[row], ae = p.a_ptr[row + 1];
        if (COMP) {
            for (uint32_t q = p.m_ptr[row] + threadIdx.x; q < p.m_ptr[row + 1]; q += blockDim.x) {
                const uint32_t j = __ldg(p.m_col + q);
                atomicOr(&mbits[j >> 5], 1u << (j & 31));
            }
            __syncthreads();
        }
        for (uint32_t pa = as + warp; pa < ae; pa += nwarps) {
            const uint32_t k = p.a_col[pa];
            XT av = (XT)1;
            if (NUMERIC && p.need_a) av = gload<XT>(aval + pa);
            for (BT pb = p.b_ptr[k] + lane; pb < p.b_ptr[k + 1]; pb += 32) {
                const uint32_t j = __ldg(p.b_col + pb);
                const uint32_t bit = 1u << (j & 31);
                if (COMP && (mbits[j >> 5] & bit)) continue;
                if (!(bits[j >> 5] & bit)) atomicOr(&bits[j >> 5], bit);
                if (NUMERIC) {
                    const XT bv = p.need_b ? gload<XT>(bval + pb) : (XT)1;
                    atomic_combine<ZT>(&spa[j], MulApply<XT, ZT>::f(mul, av, bv), add);
                }
            }
        }
        __syncthreads();
        // ordered sweep: each thread owns a contiguous run of bitmap words
        const int64_t per = ceil_div(p.spa_words, (int64_t)blockDim.x);
        const int64_t w0 = (int64_t)threadIdx.x * per, w1 = min(w0 + per, p.spa_words);
        int cnt = 0;
        for (int64_t w = w0; w < w1; ++w) cnt += __popc(bits[w]);
        if (COMP) for (int64_t w = w0; w < w1; ++w) if (mbits[w]) mbits[w] = 0;
        int total = 0;
        int off = block_exclusive_scan(cnt, s_warp, &total);
        if (NUMERIC) {
            const int64_t base = p.c_ptr[row];
            ZT *cval = static_cast<ZT *>(p.c_val);
            for (int64_t w = w0; w < w1; ++w) {
                uint32_t m = bits[w];
                if (!m) continue;
                bits[w] = 0;
                while (m) {
                    const int b = __ffs(m) - 1; m &= m - 1;
                    const uint32_t j = (uint32_t)(w * 32 + b);
                    p.c_col[base + off] = j;
                    cval[base + off] = unpack_slot<ZT>(spa[j]);
                    spa[j] = ident;
                    ++off;
                }
            }
        } else {
            for (int64_t w = w0; w < w1; ++w) if (bits[w]) bits[w] = 0;
            if (threadIdx.x == 0) p.c_cnt[row] = total;
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------ complemented mask: split dense accumulators (spa-split)
// Rows with more than SPLIT_FLOPS products are spread over the whole GPU instead of owning one CTA of spa_kernel.  They are
// processed in groups; each row of a group (its slot) owns a dense accumulator, a presence bitmap and a bitmap of M'(row,:) in
// HBM.  A(row,:) is cut into chunks of about CHUNK_FLOPS products (equal runs of A entries) that persistent CTAs take from a
// queue.  The sweeps split each row into ranges of SPLIT_RANGE_WORDS bitmap words, one CTA per (range, slot).
// BT: the type of B's row offsets, as in GemmArgsT; A's positions in the chunk list are relative to the row panel
template <typename BT> struct SplitArgsT {
    const uint32_t *a_col; const void *a_val; const BT *b_ptr; const uint32_t *b_col; const void *b_val;
    const uint32_t *m_ptr, *m_col;
    const int32_t *rows;                 // the rows of the group, by slot
    const uint32_t *chunks;              // per chunk: slot, first A entry, end A entry
    int64_t nchunks; unsigned int *queue;
    uint32_t *pres, *mbit; void *acc;    // per slot: words bitmap words, ncols accumulator words
    int64_t words, ncols, nrange;
    int add_op, mul_op, need_a, need_b;
    int64_t *c_cnt; const int64_t *c_ptr; uint32_t *c_col; void *c_val;
    int64_t *range_cnt;                  // numeric: per (slot, range) count, then its exclusive scan
};
static constexpr int64_t SPLIT_RANGE_WORDS = 2048;

// M'(row,:) into the mask bitmap of every slot (blockIdx.y = slot)
template <typename BT> __global__ void split_mask_kernel(const SplitArgsT<BT> s) {
    const int64_t row = s.rows[blockIdx.y];
    uint32_t *mb = s.mbit + (size_t)blockIdx.y * s.words;
    for (uint32_t q = s.m_ptr[row] + blockIdx.x * blockDim.x + threadIdx.x; q < s.m_ptr[row + 1]; q += gridDim.x * blockDim.x) {
        const uint32_t j = __ldg(s.m_col + q);
        atomicOr(&mb[j >> 5], 1u << (j & 31));
    }
}

template <typename XT, typename ZT, int ADD, int MUL, bool NUMERIC, typename BT>
__global__ void __launch_bounds__(512) split_chunk_kernel(const SplitArgsT<BT> s) {
    typedef typename SlotWord<ZT>::W W;
    __shared__ unsigned int s_next;
    const int add = ADD >= 0 ? ADD : s.add_op;
    const int mul = MUL >= 0 ? MUL : s.mul_op;
    const XT *aval = static_cast<const XT *>(s.a_val), *bval = static_cast<const XT *>(s.b_val);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    while (true) {
        if (threadIdx.x == 0) s_next = atomicAdd(s.queue, 1u);
        __syncthreads();
        const unsigned int idx = s_next;
        __syncthreads();
        if (idx >= s.nchunks) break;
        const uint32_t slot = s.chunks[3 * (size_t)idx], pa0 = s.chunks[3 * (size_t)idx + 1], pa1 = s.chunks[3 * (size_t)idx + 2];
        uint32_t *bits = s.pres + (size_t)slot * s.words;
        const uint32_t *mb = s.mbit + (size_t)slot * s.words;
        W *acc = NUMERIC ? static_cast<W *>(s.acc) + (size_t)slot * s.ncols : nullptr;
        for (uint32_t pa = pa0 + warp; pa < pa1; pa += nwarps) {
            const uint32_t k = s.a_col[pa];
            XT av = (XT)1;
            if (NUMERIC && s.need_a) av = gload<XT>(aval + pa);
            for (BT pb = s.b_ptr[k] + lane; pb < s.b_ptr[k + 1]; pb += 32) {
                const uint32_t j = __ldg(s.b_col + pb);
                const uint32_t bit = 1u << (j & 31);
                if (mb[j >> 5] & bit) continue;
                if (!(bits[j >> 5] & bit)) atomicOr(&bits[j >> 5], bit);
                if (NUMERIC) {
                    const XT bv = s.need_b ? gload<XT>(bval + pb) : (XT)1;
                    atomic_combine<ZT>(&acc[j], MulApply<XT, ZT>::f(mul, av, bv), add);
                }
            }
        }
    }
}

// popcount of one (range, slot): symbolic (CLEAR) adds it to c_cnt[row] and clears both bitmaps of the range; numeric stores it
template <bool CLEAR, typename BT>
__global__ void __launch_bounds__(256) split_count_kernel(const SplitArgsT<BT> s) {
    __shared__ int s_warp[33];
    const int64_t slot = blockIdx.y, r = blockIdx.x;
    const int64_t w0 = r * SPLIT_RANGE_WORDS, w1 = min(w0 + SPLIT_RANGE_WORDS, s.words);
    uint32_t *bits = s.pres + (size_t)slot * s.words, *mb = s.mbit + (size_t)slot * s.words;
    int cnt = 0;
    for (int64_t w = w0 + threadIdx.x; w < w1; w += blockDim.x) {
        const uint32_t m = bits[w];
        cnt += __popc(m);
        if (CLEAR) { if (m) bits[w] = 0; if (mb[w]) mb[w] = 0; }
    }
    int total = 0;
    block_exclusive_scan(cnt, s_warp, &total);
    if (threadIdx.x == 0) {
        if (CLEAR) { if (total) atomicAdd(reinterpret_cast<unsigned long long *>(&s.c_cnt[s.rows[slot]]), (unsigned long long)total); }
        else s.range_cnt[slot * s.nrange + r] = total;
    }
}

// ordered sweep of one (range, slot): the entries go out sorted at c_ptr[row] + (their range's offset within the row), the
// accumulator words are reset to ident and both bitmaps cleared
template <typename ZT, typename BT>
__global__ void __launch_bounds__(256) split_fill_kernel(const SplitArgsT<BT> s, typename SlotWord<ZT>::W ident) {
    typedef typename SlotWord<ZT>::W W;
    __shared__ int s_warp[33];
    const int64_t slot = blockIdx.y, r = blockIdx.x;
    const int64_t w0r = r * SPLIT_RANGE_WORDS, w1r = min(w0r + SPLIT_RANGE_WORDS, s.words);
    uint32_t *bits = s.pres + (size_t)slot * s.words, *mb = s.mbit + (size_t)slot * s.words;
    W *acc = static_cast<W *>(s.acc) + (size_t)slot * s.ncols;
    const int64_t per = ceil_div(w1r - w0r, (int64_t)blockDim.x);
    const int64_t w0 = w0r + (int64_t)threadIdx.x * per, w1 = min(w0 + per, w1r);
    int cnt = 0;
    for (int64_t w = w0; w < w1; ++w) cnt += __popc(bits[w]);
    int total = 0;
    int off = block_exclusive_scan(cnt, s_warp, &total);
    const int64_t row = s.rows[slot];
    const int64_t base = s.c_ptr[row] + s.range_cnt[slot * s.nrange + r] - s.range_cnt[slot * s.nrange];
    ZT *cval = static_cast<ZT *>(s.c_val);
    for (int64_t w = w0; w < w1; ++w) {
        if (mb[w]) mb[w] = 0;
        uint32_t m = bits[w];
        if (!m) continue;
        bits[w] = 0;
        while (m) {
            const int b = __ffs(m) - 1; m &= m - 1;
            const uint32_t j = (uint32_t)(w * 32 + b);
            s.c_col[base + off] = j;
            cval[base + off] = unpack_slot<ZT>(acc[j]);
            acc[j] = ident;
            ++off;
        }
    }
}

// the rows of the dense-accumulator bin with more than split_flops products leave it: (row, flops, A range) into the split list
__global__ void split_pick_kernel(const int32_t *rows, int64_t n, const int64_t *flops, int64_t split_flops, const uint32_t *a_ptr,
                                  int32_t *keep, int64_t *split, unsigned int *counters) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        const int32_t row = rows[r];
        const int64_t f = flops[row];
        if (f > split_flops) {
            const unsigned int q = atomicAdd(&counters[1], 1u);
            split[4 * (size_t)q] = row; split[4 * (size_t)q + 1] = f; split[4 * (size_t)q + 2] = a_ptr[row]; split[4 * (size_t)q + 3] = a_ptr[row + 1];
        } else keep[atomicAdd(&counters[0], 1u)] = row;
    }
}

template <typename W> __global__ void fill_words_kernel(W *a, W v, int64_t n) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) a[k] = v;
}

// ------------------------------------------------------------------ masked: shared-memory hash of the mask row
// Rows whose products and mask row are both short (the warp class): one warp per row hashes the mask row M(i,:)
// (keys -> position inside the row), then streams the B rows named by A(i,:) and accumulates the products that hit it.
// The warp handles 32 A entries at a time: each lane fetches one (k, B row range) up front, the ranges are broadcast by
// shuffle and the lanes stride the B row -- the dependent-load chain per A entry is paid once per 32 entries.
// Heavier rows are cut into chunks and go to the streaming kernel (spgemm_stream.cuh).
template <typename BT> struct MaskedArgsT {
    GemmArgsT<BT> g;
    void *t_words;     // nnz(M) accumulator words
};

template <typename XT, typename ZT, typename BT, typename Hit>
__device__ __forceinline__ void stream_b_rows(const GemmArgsT<BT> &p, uint32_t pa0, uint32_t pa1, int lane, Hit &&hit) {
    const XT *aval = static_cast<const XT *>(p.a_val);
    for (uint32_t base = pa0; base < pa1; base += 32) {
        const uint32_t pa = base + lane;
        const bool valid = pa < pa1;
        const uint32_t k = valid ? __ldg(p.a_col + pa) : 0u;
        const BT bs = valid ? __ldg(p.b_ptr + k) : (BT)0, be = valid ? __ldg(p.b_ptr + k + 1) : (BT)0;
        XT av = (XT)1;
        if (p.need_a && valid) av = gload<XT>(aval + pa);
        const int cnt = min(32u, pa1 - base);
        for (int l = 0; l < cnt; ++l) {
            const BT s = __shfl_sync(0xffffffffu, bs, l), e = __shfl_sync(0xffffffffu, be, l);
            XT a;
            if constexpr (sizeof(XT) == 8) { long long t = __shfl_sync(0xffffffffu, reinterpret_cast<long long &>(av), l); a = reinterpret_cast<XT &>(t); }
            else if constexpr (sizeof(XT) == 4) { int t = __shfl_sync(0xffffffffu, reinterpret_cast<int &>(av), l); a = reinterpret_cast<XT &>(t); }
            else { int t = __shfl_sync(0xffffffffu, (int)av, l); a = (XT)t; }
            for (BT pb = s + lane; pb < e; pb += 32) hit(__ldg(p.b_col + pb), a, pb);
        }
    }
}

template <typename XT, typename ZT, int ADD, int MUL, typename BT>
__global__ void __launch_bounds__(256) masked_hash_kernel(const MaskedArgsT<BT> ma) {
    typedef typename SlotWord<ZT>::W W;
    const GemmArgsT<BT> &p = ma.g;
    extern __shared__ unsigned char smem_raw[];
    const int add = ADD >= 0 ? ADD : p.add_op;
    const int mul = MUL >= 0 ? MUL : p.mul_op;
    const int gid = threadIdx.x >> 5, lane = threadIdx.x & 31, groups = blockDim.x >> 5;
    const int half = p.table >> 1;                                    // max mask-row length
    // layout per warp: keys[table] u32 | slot[table] u32 | vals[half] W | found[half] u8
    const size_t per_group = (size_t)p.table * 8 + (size_t)half * sizeof(W) + (size_t)half;
    unsigned char *basep = smem_raw + (size_t)gid * ((per_group + 15) & ~(size_t)15);
    uint32_t *keys = reinterpret_cast<uint32_t *>(basep);
    uint32_t *slot = keys + p.table;
    W *vals = reinterpret_cast<W *>(slot + p.table);
    uint8_t *found = reinterpret_cast<uint8_t *>(vals + half);
    const int64_t idx = (int64_t)blockIdx.x * groups + gid;
    if (idx >= p.nbin) return;                                        // a whole warp
    const uint32_t tmask = (uint32_t)p.table - 1;
    const int hshift = __clz(p.table) + 1;                            // 32 - log2(table)
    const W ident = pack_slot<ZT>(accum_init<ZT>(add));
    const int64_t row = p.rows[idx];
    const uint32_t ms = p.m_ptr[row], me = p.m_ptr[row + 1];
    const int mlen = (int)(me - ms);
    for (int s = lane; s < p.table; s += 32) keys[s] = EMPTY_KEY;
    for (int s = lane; s < mlen; s += 32) { vals[s] = ident; found[s] = 0; }
    __syncwarp();
    for (uint32_t q = ms + lane; q < me; q += 32) {
        bool on = true;
        if (!p.m_struct) on = sc_cast(sc_load(p.m_tc, p.m_val, q), p.m_tc, TC_BOOL).u != 0;
        if (!on) continue;
        const uint32_t j = p.m_col[q];
        uint32_t s = hash_col(j, hshift);
        while (atomicCAS(&keys[s], EMPTY_KEY, j) != EMPTY_KEY) s = (s + 1) & tmask;   // mask columns are unique
        slot[s] = q - ms;
    }
    __syncwarp();
    const XT *bval = static_cast<const XT *>(p.b_val);
    auto hit = [&](uint32_t j, XT av, BT pb) {
        uint32_t s = hash_col(j, hshift);
        while (true) {
            const uint32_t kk = keys[s];
            if (kk == j) {
                const uint32_t q = slot[s];
                const XT bv = p.need_b ? gload<XT>(bval + pb) : (XT)1;
                atomic_combine<ZT>(&vals[q], MulApply<XT, ZT>::f(mul, av, bv), add);
                found[q] = 1;
                return;
            }
            if (kk == EMPTY_KEY) return;
            s = (s + 1) & tmask;
        }
    };
    stream_b_rows<XT, ZT, BT>(p, p.a_ptr[row], p.a_ptr[row + 1], lane, hit);
    __syncwarp();
    W *tw = static_cast<W *>(ma.t_words);
    for (int q = lane; q < mlen; q += 32) { tw[ms + q] = vals[q]; p.t_found[ms + q] = found[q]; }
}

// per-row chunk counts: class 1 rows (warp kernel) get 0 chunks
__global__ void chunk_count_kernel(const int64_t *flops, const uint32_t *m_ptr, int64_t nrows, int64_t chunk_flops,
                                   int warp_flops, int warp_mlen, int small_mlen, int medium_mlen, int64_t *cnt_small, int64_t *cnt_medium, int64_t *cnt_long, int64_t *cls1) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += (int64_t)gridDim.x * blockDim.x) {
        const int64_t f = flops[r]; const int64_t ml = m_ptr[r + 1] - m_ptr[r];
        int64_t cs = 0, cm = 0, cl = 0, c1 = 0;
        if (f > 0 && ml > 0) {
            if (f <= warp_flops && ml <= warp_mlen) c1 = 1;
            else if (ml <= small_mlen) cs = (f + chunk_flops - 1) / chunk_flops;
            else if (ml <= medium_mlen) cm = (f + chunk_flops - 1) / chunk_flops;
            else cl = (f + chunk_flops - 1) / chunk_flops;
        }
        cnt_small[r] = cs; cnt_medium[r] = cm; cnt_long[r] = cl; cls1[r] = c1;
    }
}
// after exclusive scans of the three arrays: emit the chunk lists and the class-1 row list
__global__ void chunk_fill_kernel(const int64_t *off_small, const int64_t *off_medium, const int64_t *off_long, const int64_t *off_cls1, int64_t nrows,
                                  int32_t *s_row, uint32_t *s_idx, uint32_t *s_cnt,
                                  int32_t *m_row, uint32_t *m_idx, uint32_t *m_cnt,
                                  int32_t *l_row, uint32_t *l_idx, uint32_t *l_cnt, int32_t *w_rows) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += (int64_t)gridDim.x * blockDim.x) {
        const int64_t cs = off_small[r + 1] - off_small[r], cm = off_medium[r + 1] - off_medium[r], cl = off_long[r + 1] - off_long[r];
        for (int64_t c = 0; c < cs; ++c) { const int64_t o = off_small[r] + c; s_row[o] = (int32_t)r; s_idx[o] = (uint32_t)c; s_cnt[o] = (uint32_t)cs; }
        for (int64_t c = 0; c < cm; ++c) { const int64_t o = off_medium[r] + c; m_row[o] = (int32_t)r; m_idx[o] = (uint32_t)c; m_cnt[o] = (uint32_t)cm; }
        for (int64_t c = 0; c < cl; ++c) { const int64_t o = off_long[r] + c; l_row[o] = (int32_t)r; l_idx[o] = (uint32_t)c; l_cnt[o] = (uint32_t)cl; }
        if (off_cls1[r + 1] > off_cls1[r]) w_rows[off_cls1[r]] = (int32_t)r;
    }
}

template <typename ZT> static void fill_accum_init(void *words, int64_t n, int add) {
    typedef typename SlotWord<ZT>::W W;
    fill_words_kernel<W><<<grid_for(n), 256, 0, G.stream>>>(static_cast<W *>(words), pack_slot<ZT>(accum_init<ZT>(add)), n);
}

// accumulator words (32-bit) -> 1- or 2-byte typed values
__global__ void narrow_words_kernel(const uint32_t *words, uint8_t *out, int vsize, int64_t n) {
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (int64_t)gridDim.x * blockDim.x) {
        if (vsize == 1) out[q] = (uint8_t)words[q]; else ((uint16_t *)out)[q] = (uint16_t)words[q];
    }
}
__global__ void row_len_kernel(const uint32_t *ptr, int64_t n, int64_t *out) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) out[r] = ptr[r + 1] - ptr[r];
}

// ------------------------------------------------------------------ masked dot:  T(i,j) = A(i,:) . B(j,:) for (i,j) in M
// One warp per mask row; lanes take mask entries; sorted-merge intersection of the two rows.
template <typename XT, typename ZT, int ADD, int MUL, typename BT>
__global__ void __launch_bounds__(256) masked_dot_kernel(const GemmArgsT<BT> p) {
    const int add = ADD >= 0 ? ADD : p.add_op;
    const int mul = MUL >= 0 ? MUL : p.mul_op;
    const XT *aval = static_cast<const XT *>(p.a_val), *bval = static_cast<const XT *>(p.b_val);
    ZT *tval = static_cast<ZT *>(p.c_val);
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const ZT ident = monoid_identity<ZT>(add);
    for (int64_t i = warp; i < p.nrows; i += nwarps) {
        const uint32_t as = p.a_ptr[i], ae = p.a_ptr[i + 1];
        for (uint32_t q = p.m_ptr[i] + lane; q < p.m_ptr[i + 1]; q += 32) {
            bool on = true;
            if (!p.m_struct) on = sc_cast(sc_load(p.m_tc, p.m_val, q), p.m_tc, TC_BOOL).u != 0;
            ZT acc = ident; uint8_t has = 0;
            if (on) {
                const uint32_t j = p.m_col[q];
                uint32_t x = as; BT y = p.b_ptr[j]; const BT ye = p.b_ptr[j + 1];
                while (x < ae && y < ye) {
                    const uint32_t cx = __ldg(p.a_col + x), cy = __ldg(p.b_col + y);
                    if (cx == cy) {
                        const XT av = p.need_a ? gload<XT>(aval + x) : (XT)1;
                        const XT bv = p.need_b ? gload<XT>(bval + y) : (XT)1;
                        const ZT prod = MulApply<XT, ZT>::f(mul, av, bv);
                        acc = has ? MulApply<ZT, ZT>::f(add, acc, prod) : prod;
                        has = 1; ++x; ++y;
                    } else if (cx < cy) ++x; else ++y;
                }
            }
            tval[q] = acc; p.t_found[q] = has;
        }
    }
}

// ------------------------------------------------------------------ compaction of a masked result (pattern of M, found flags) into CSR
// OT: the type of M's row offsets (uint32_t: rowptr32; int64_t: rowptr, the wide route of SDDMM)
template <typename OT> __global__ void row_found_count_kernel(const OT *m_ptr, const uint8_t *found, int64_t nrows, int64_t *cnt) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < nrows; r += nwarps) {
        int c = 0;
        for (OT q = m_ptr[r] + lane; q < m_ptr[r + 1]; q += 32) c += found[q] != 0;
        for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
        if (lane == 0) cnt[r] = c;
    }
}
template <typename OT>
__global__ void row_found_fill_kernel(const OT *m_ptr, const uint32_t *m_col, const uint8_t *found, const uint8_t *tval, int vsize,
                                      int64_t nrows, const int64_t *c_ptr, uint32_t *c_col, uint8_t *c_val) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < nrows; r += nwarps) {
        int64_t out = c_ptr[r];
        for (OT q0 = m_ptr[r]; q0 < m_ptr[r + 1]; q0 += 32) {
            const OT q = q0 + lane;
            const bool f = q < m_ptr[r + 1] && found[q] != 0;
            const unsigned ball = __ballot_sync(0xffffffffu, f);
            if (f) {
                const int64_t o = out + __popc(ball & ((1u << lane) - 1));
                c_col[o] = m_col[q];
                switch (vsize) {
                    case 1: c_val[o] = tval[q]; break;
                    case 2: ((uint16_t *)c_val)[o] = ((const uint16_t *)tval)[q]; break;
                    case 4: ((uint32_t *)c_val)[o] = ((const uint32_t *)tval)[q]; break;
                    default: ((uint64_t *)c_val)[o] = ((const uint64_t *)tval)[q]; break;
                }
            }
            out += __popc(ball);
        }
    }
}

// ------------------------------------------------------------------ C<M> = accum(C, T): row-wise three-way merge
struct MatFinalizeArgs {
    int64_t nrows;
    const int64_t *c_ptr; const uint32_t *c_col; const void *c_val; int ctc; int c_exists;
    const int64_t *t_ptr; const uint32_t *t_col; const void *t_val; int ttc;
    const int64_t *m_ptr; const uint32_t *m_col; const void *m_val; int mtc; int has_mask, mask_comp, mask_struct, replace;
    int accum_op, accum_tc, accum_ztc;
    int64_t *o_cnt; const int64_t *o_ptr; uint32_t *o_col; void *o_val;
};
template <bool FILL> __global__ void mat_finalize_kernel(const MatFinalizeArgs a) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < a.nrows; r += (int64_t)gridDim.x * blockDim.x) {
        int64_t pc = a.c_exists ? a.c_ptr[r] : 0, pce = a.c_exists ? a.c_ptr[r + 1] : 0;
        int64_t pt = a.t_ptr[r], pte = a.t_ptr[r + 1];
        int64_t pm = a.has_mask ? a.m_ptr[r] : 0, pme = a.has_mask ? a.m_ptr[r + 1] : 0;
        int64_t out = FILL ? a.o_ptr[r] : 0;
        while (pc < pce || pt < pte) {
            const uint32_t jc = pc < pce ? a.c_col[pc] : 0xFFFFFFFFu, jt = pt < pte ? a.t_col[pt] : 0xFFFFFFFFu;
            const uint32_t j = jc < jt ? jc : jt;
            const bool cp = jc == j, tp = jt == j;
            bool m = true;
            if (a.has_mask) {
                while (pm < pme && a.m_col[pm] < j) ++pm;
                m = pm < pme && a.m_col[pm] == j;
                if (m && !a.mask_struct) m = sc_cast(sc_load(a.mtc, a.m_val, pm), a.mtc, TC_BOOL).u != 0;
                if (a.mask_comp) m = !m;
            }
            bool keep = false; Sc v; v.u = 0;
            if (m) {
                if (a.accum_op >= 0) {
                    keep = true;
                    if (FILL) {
                        if (cp && tp) {
                            const Sc x = sc_cast(sc_load(a.ctc, a.c_val, pc), a.ctc, a.accum_tc);
                            const Sc y = sc_cast(sc_load(a.ttc, a.t_val, pt), a.ttc, a.accum_tc);
                            v = sc_cast(sc_binop(a.accum_op, a.accum_tc, x, y), a.accum_ztc, a.ctc);
                        } else if (cp) v = sc_load(a.ctc, a.c_val, pc);
                        else v = sc_cast(sc_load(a.ttc, a.t_val, pt), a.ttc, a.ctc);
                    }
                } else if (tp) { keep = true; if (FILL) v = sc_cast(sc_load(a.ttc, a.t_val, pt), a.ttc, a.ctc); }
            } else if (!a.replace && cp) { keep = true; if (FILL) v = sc_load(a.ctc, a.c_val, pc); }
            if (keep) { if (FILL) { a.o_col[out] = j; sc_store(a.ctc, a.o_val, out, v); } ++out; }
            if (cp) ++pc;
            if (tp) ++pt;
        }
        if (!FILL) a.o_cnt[r] = out;
    }
}

#include "spgemm_stream.cuh"

// ------------------------------------------------------------------ host side
static GrB_Info read_counts(const unsigned int *d, unsigned int *h, int n, std::string *err) {
    CU_TRY(cudaMemcpyAsync(h, d, n * sizeof(unsigned int), cudaMemcpyDeviceToHost, G.stream), err);
    CU_TRY(cudaStreamSynchronize(G.stream), err);
    return GrB_SUCCESS;
}
static constexpr int SMALL_TABLE = 256, SMALL_FLOPS = 128;      // warp per row
static constexpr int MEDIUM_TABLE = 4096, MEDIUM_FLOPS = 2048;  // CTA per row
static constexpr int MIDSMALL_TABLE = 1024;                       // masked: CTA per chunk, mask rows up to 512 entries
static constexpr int64_t CHUNK_FLOPS = 32768;     // flop budget of one CTA-level work unit
// complemented mask: rows with more products go to spa-split (DESIGN.md section 3.2); the HBM buffers of one group of split rows
static constexpr int64_t SPLIT_FLOPS = (int64_t)1 << 18;
static constexpr int64_t SPLIT_BUDGET = (int64_t)1 << 28;

// dispatch helpers: KERNEL is a macro taking (XT, ZT, ADD, MUL)
#define GB_FOR_SEMIRING(xt, zt, add, mul, KERNEL, err)                                                        \
    do {                                                                                                       \
        bool done_ = false;                                                                                    \
        if (xt == zt) {                                                                                        \
            if (xt == TC_FP32 && add == OP_PLUS && mul == OP_TIMES) { KERNEL(float, float, OP_PLUS, OP_TIMES); done_ = true; }    \
            else if (xt == TC_FP32 && add == OP_PLUS && mul == OP_SECOND) { KERNEL(float, float, OP_PLUS, OP_SECOND); done_ = true; } \
            else if (xt == TC_FP64 && add == OP_PLUS && mul == OP_TIMES) { KERNEL(double, double, OP_PLUS, OP_TIMES); done_ = true; } \
            else if (xt == TC_INT64 && add == OP_PLUS && mul == OP_PAIR) { KERNEL(int64_t, int64_t, OP_PLUS, OP_PAIR); done_ = true; } \
            else if (xt == TC_INT64 && add == OP_PLUS && mul == OP_TIMES) { KERNEL(int64_t, int64_t, OP_PLUS, OP_TIMES); done_ = true; } \
            else if (xt == TC_UINT32 && add == OP_PLUS && mul == OP_PAIR) { KERNEL(uint32_t, uint32_t, OP_PLUS, OP_PAIR); done_ = true; } \
            else if (xt == TC_BOOL && add == OP_LOR && mul == OP_LAND) { KERNEL(bool, bool, OP_LOR, OP_LAND); done_ = true; } \
        }                                                                                                      \
        if (!done_) GB_FOR_DOMAINS(xt, zt, done_, KERNEL(XT_, ZT_, -1, -1));                                   \
        if (!done_) return gb_fail(GrB_DOMAIN_MISMATCH, err, "mxm: unsupported semiring domains (x=%d, z=%d)", xt, zt); \
    } while (0)

struct RowBins { DevBuf<int32_t> rows; unsigned int count[4] = {0, 0, 0, 0}; unsigned int offset[4] = {0, 0, 0, 0}; };

static GrB_Info make_bins(const int64_t *work, int64_t nrows, BinLimits lim, RowBins &b, std::string *err) {
    DevBuf<unsigned int> d;
    GB_TRY(d.alloc(12, err));                          // counts[4] | offsets[4] | cursor[4]
    CU_TRY(cudaMemsetAsync(d, 0, 12 * sizeof(unsigned int), G.stream), err);
    bin_count_kernel<<<grid_for(nrows), 256, 0, G.stream>>>(work, nrows, lim, d); GB_LAUNCHED();
    GB_TRY(read_counts(d, b.count, 4, err));
    b.offset[0] = 0;
    for (int k = 1; k < 4; ++k) b.offset[k] = b.offset[k - 1] + b.count[k - 1];
    CU_TRY(cudaMemcpyAsync(d + 4, b.offset, 4 * sizeof(unsigned int), cudaMemcpyHostToDevice, G.stream), err);
    GB_TRY(b.rows.alloc((size_t)nrows, err));
    bin_fill_kernel<<<grid_for(nrows), 256, 0, G.stream>>>(work, nrows, lim, d + 4, d + 8, b.rows); GB_LAUNCHED();
    CU_TRY(cudaStreamSynchronize(G.stream), err);      // b.offset (host) was the source of an async copy
    return GrB_SUCCESS;
}

static size_t masked_smem(int table, int groups, size_t wsize) {
    const size_t per = (size_t)table * 8 + (size_t)(table / 2) * wsize + (size_t)(table / 2);
    return (size_t)groups * ((per + 15) & ~(size_t)15);
}

// The split rows of a complemented product: slots in row order, groups of `group` rows, the chunk list of each group
struct SplitPlan {
    int64_t nsplit = 0, nkeep = 0, group = 0, ncols = 0, words = 0, nrange = 0;
    DevBuf<int32_t> keep;                        // the rows that stay in spa_kernel
    std::vector<int64_t> chunk_off;              // per group: its first chunk; one more entry at the end
    int32_t *rows = nullptr; uint32_t *chunks = nullptr;
    void *acc = nullptr; uint32_t *pres = nullptr, *mbit = nullptr; int64_t *range_cnt = nullptr;
    DevBuf<unsigned int> queue;
};

// a_ptr: the 32-bit offsets of the row panel; the chunks' A positions are relative to it
static GrB_Info split_prepare(const RowBins &bins, const int64_t *flops, const uint32_t *a_ptr, int64_t ncols, size_t wsize, SplitPlan &sp,
                              std::string *err) {
    const unsigned int n3 = bins.count[3];
    DevBuf<unsigned int> cnt; DevBuf<int64_t> picked;
    GB_TRY(cnt.alloc(2, err));
    CU_TRY(cudaMemsetAsync(cnt, 0, 8, G.stream), err);
    GB_TRY(sp.keep.alloc(n3, err)); GB_TRY(picked.alloc((size_t)4 * n3, err));
    split_pick_kernel<<<grid_for(n3), 256, 0, G.stream>>>(bins.rows + bins.offset[3], n3, flops, SPLIT_FLOPS, a_ptr, sp.keep, picked, cnt);
    GB_LAUNCHED();
    unsigned int h[2];
    GB_TRY(read_counts(cnt, h, 2, err));
    sp.nkeep = h[0]; sp.nsplit = h[1];
    if (!sp.nsplit) { sp.keep.reset(); return GrB_SUCCESS; }
    std::vector<int64_t> hs((size_t)4 * sp.nsplit);
    CU_TRY(cudaMemcpyAsync(hs.data(), picked, hs.size() * 8, cudaMemcpyDeviceToHost, G.stream), err);
    CU_TRY(cudaStreamSynchronize(G.stream), err);
    std::vector<int64_t> ord((size_t)sp.nsplit);
    for (int64_t q = 0; q < sp.nsplit; ++q) ord[q] = q;
    std::sort(ord.begin(), ord.end(), [&](int64_t x, int64_t y) { return hs[4 * x] < hs[4 * y]; });
    sp.ncols = ncols; sp.words = ceil_div(ncols, 32); sp.nrange = ceil_div(sp.words, SPLIT_RANGE_WORDS);
    const int64_t per_row = ncols * (int64_t)wsize + 2 * sp.words * 4;
    sp.group = std::max<int64_t>(1, std::min<int64_t>(sp.nsplit, SPLIT_BUDGET / per_row));
    std::vector<int32_t> rows;
    std::vector<uint32_t> chunks;
    sp.chunk_off.assign(1, 0);
    for (int64_t q = 0; q < sp.nsplit; ++q) {
        const int64_t *e = &hs[4 * ord[q]];
        rows.push_back((int32_t)e[0]);
        const int64_t as = e[2], len = e[3] - e[2];
        const int64_t n = std::max<int64_t>(1, std::min<int64_t>(len, ceil_div(e[1], CHUNK_FLOPS)));
        for (int64_t c = 0; c < n; ++c) {
            chunks.push_back((uint32_t)(q % sp.group));
            chunks.push_back((uint32_t)(as + len * c / n)); chunks.push_back((uint32_t)(as + len * (c + 1) / n));
        }
        if ((q + 1) % sp.group == 0 || q + 1 == sp.nsplit) sp.chunk_off.push_back((int64_t)chunks.size() / 3);
    }
    GB_TRY(ws_array(WS_SPLIT_ROWS, &sp.rows, rows.size(), err));
    GB_TRY(ws_array(WS_SPLIT_CHUNKS, &sp.chunks, chunks.size(), err));
    GB_TRY(ws_array(WS_SPLIT_RANGES, &sp.range_cnt, (size_t)(sp.group * sp.nrange + 1), err));
    void *buf = nullptr;
    GB_TRY(ws_get(WS_SPLIT_BUF, &buf, (size_t)(sp.group * per_row) + 16, err));
    sp.acc = buf;
    sp.pres = reinterpret_cast<uint32_t *>(static_cast<char *>(buf) + (size_t)sp.group * ncols * wsize);
    sp.mbit = sp.pres + (size_t)sp.group * sp.words;
    CU_TRY(cudaMemsetAsync(sp.pres, 0, (size_t)sp.group * sp.words * 8, G.stream), err);       // both bitmaps
    GB_TRY(sp.queue.alloc(1, err));
    CU_TRY(cudaMemcpyAsync(sp.rows, rows.data(), rows.size() * 4, cudaMemcpyHostToDevice, G.stream), err);
    CU_TRY(cudaMemcpyAsync(sp.chunks, chunks.data(), chunks.size() * 4, cudaMemcpyHostToDevice, G.stream), err);
    CU_TRY(cudaStreamSynchronize(G.stream), err);      // the host vectors are the sources of the copies
    return GrB_SUCCESS;
}

// the launches of group g: its mask bitmaps, then the chunk kernel on a fresh queue; returns the group's argument block
template <typename BT>
static SplitArgsT<BT> split_group(const SplitPlan &sp, const SplitArgsT<BT> &base, int64_t g, int64_t *ng, std::string *err) {
    SplitArgsT<BT> s = base;
    s.rows = sp.rows + g * sp.group;
    *ng = std::min(sp.group, sp.nsplit - g * sp.group);
    s.chunks = sp.chunks + 3 * sp.chunk_off[g];
    s.nchunks = sp.chunk_off[g + 1] - sp.chunk_off[g];
    split_mask_kernel<BT><<<dim3((unsigned)std::min<int64_t>(ceil_div(sp.ncols, 256), 128), (unsigned)*ng), 256, 0, G.stream>>>(s);
    GB_LAUNCHED();
    cudaMemsetAsync(s.queue, 0, 4, G.stream);          // errors surface at the caller's cudaGetLastError
    return s;
}
static int split_ctas(int64_t nchunks) { return (int)std::max<int64_t>(1, std::min<int64_t>(nchunks, (int64_t)G.num_sms * 2)); }

template <typename XT, typename ZT, int ADD, int MUL, typename BT>
static GrB_Info split_numeric(const SplitPlan &sp, const SplitArgsT<BT> &base, std::string *err) {
    typedef typename SlotWord<ZT>::W W;
    const int add = ADD >= 0 ? ADD : base.add_op;
    fill_words_kernel<W><<<grid_for(sp.group * sp.ncols), 256, 0, G.stream>>>(static_cast<W *>(sp.acc), pack_slot<ZT>(accum_init<ZT>(add)),
                                                                                 sp.group * sp.ncols);
    GB_LAUNCHED();
    for (int64_t g = 0; g + 1 < (int64_t)sp.chunk_off.size(); ++g) {
        int64_t ng = 0;
        const SplitArgsT<BT> s = split_group<BT>(sp, base, g, &ng, err);
        split_chunk_kernel<XT, ZT, ADD, MUL, true, BT><<<split_ctas(s.nchunks), 512, 0, G.stream>>>(s);
        split_count_kernel<false, BT><<<dim3((unsigned)sp.nrange, (unsigned)ng), 256, 0, G.stream>>>(s);
        CU_TRY(cudaMemsetAsync(sp.range_cnt + ng * sp.nrange, 0, 8, G.stream), err);
        GB_TRY(dev_exclusive_scan(sp.range_cnt, ng * sp.nrange + 1, err));
        split_fill_kernel<ZT, BT><<<dim3((unsigned)sp.nrange, (unsigned)ng), 256, 0, G.stream>>>(s, pack_slot<ZT>(accum_init<ZT>(add)));
        G.launches += 4;
    }
    CU_TRY(cudaGetLastError(), err);
    return GrB_SUCCESS;
}

// One row panel of a CSR x CSR product: nrows rows of A and of the mask -- M, or M' (the entries of a complemented mask that
// block, see mask_true_pattern) -- with 32-bit offsets relative to the panel's first entries (the narrow route: the whole
// matrices, their rowptr32).  m_ptr is null when no mask entry applies.  The unmasked bins leave m_val and mnnz unused.
struct RowPanel {
    const uint32_t *a_ptr, *a_col; const void *a_val;
    const uint32_t *m_ptr, *m_col; const void *m_val;
    int64_t nrows, mnnz;
};
// the bins a call ran (esc-small, esc-medium, spa, spa-split, pull): reported once each, in this order, however many panels ran them
struct UnmaskedUse { bool bin[5] = {false, false, false, false, false}; bool pull_dot = false; };
// The pull route of an eligible call (spgemm_pull.cu): the rule's mode, and op(B)' with its values, formed by `ensure` only
// once a row pulls.  rows: the rows that pulled.
struct PullSide {
    bool dot = false; double alpha = 0.0;
    std::function<GrB_Info(PullOperands &)> ensure;
    int64_t rows = 0;
};
// the wide route's size rule, counted over the panels: the entries of T formed so far, refused on reaching `limit`
struct ResultCount { int64_t limit = 0, total = 0; };
static const char *const WIDE_RESULT_REFUSAL = "GrB_mxm: results of >= 2^32 entries are not supported with an operand of >= 2^32 entries";

// T = A (+).(x) B on one panel, unmasked.  A and B values already of the multiply's operand type.  With P.m_ptr set,
// T = (A (+).(x) B)<!M'>: the same bins, chosen by the unfiltered product counts, run their COMP instantiations, which never form
// a blocked entry.  pull (the narrow route of an eligible call, else null): the rows its rule picks leave the bins for the pull
// route, one more participant of the count - scan - fill.  BT: the type of B's row offsets (b_ptr).  spa_budget > 0 caps the
// dense-accumulator CTAs at that many bytes of accumulators and bitmaps (the wide route; the narrow one runs 2 per SM).  rc (the wide route, when the size rule counts):
// the panel is refused, before its entries are allocated, when T would reach rc->limit entries.  G.last_flops grows by the panel's products.
template <typename BT>
static GrB_Info spgemm_unmasked(const RowPanel &P, const Csr &B, const BT *b_ptr, const void *bval, int xt, int zt, int add, int mul,
                                bool need_a, bool need_b, int64_t spa_budget, UnmaskedUse &use, ResultCount *rc, PullSide *pull, Csr &T,
                                std::string *err) {
    const int64_t nrows = P.nrows, ncols = B.ncols;
    const bool comp = P.m_ptr != nullptr;
    const size_t wsize = tc_size(zt) == 8 ? 8 : 4;
    RowBins bins;
    SplitPlan sp;
    GemmArgsT<BT> g{};
    SplitArgsT<BT> sa{};
    const int32_t *spa_rows = nullptr;
    int64_t spa_n = 0;
    int spa_ctas = 1;
    DevBuf<unsigned int> queue; DevBuf<uint32_t> spa_bits;
    PullOperands po{P.a_ptr, P.a_col, P.a_val, P.m_ptr, P.m_col, nullptr, nullptr, nullptr, nrows, ncols, B.nrows, xt, zt, add, mul, need_a, need_b};
    PullPlan pp;
    // ---- symbolic: the bins count the entries of their rows
    auto symbolic = [&](int64_t *cnt) {
        CU_TRY(cudaMemsetAsync(cnt, 0, ((size_t)nrows + 1) * 8, G.stream), err);
        DevBuf<int64_t> flops; DevBuf<unsigned long long> total;
        GB_TRY(flops.alloc((size_t)nrows, err)); GB_TRY(total.alloc(1, err));
        CU_TRY(cudaMemsetAsync(total, 0, 8, G.stream), err);
        flops_kernel<BT><<<grid_for(nrows * 32), 256, 0, G.stream>>>(P.a_ptr, P.a_col, b_ptr, nrows, flops, total); GB_LAUNCHED();
        if (pull && (pull->dot || pull->alpha > 0)) {      // the pull rows get no products in the bins' flops
            GB_TRY(pull_plan(po, flops, pull->dot, pull->alpha, B.nnz, pp, err));
            if (pp.n) GB_TRY(pull->ensure(po));
        }
        GB_TRY(make_bins(flops, nrows, BinLimits{SMALL_FLOPS, MEDIUM_FLOPS}, bins, err));
        int64_t total_flops = 0; GB_TRY(read_i64((const int64_t *)total, &total_flops, err));
        G.last_flops += (uint64_t)total_flops;
        // the dense-accumulator bin: with a complemented mask its rows above SPLIT_FLOPS go to spa-split
        if (comp && bins.count[3]) GB_TRY(split_prepare(bins, flops, P.a_ptr, ncols, wsize, sp, err));
        spa_rows = sp.nsplit ? sp.keep.get() : bins.rows + bins.offset[3];
        spa_n = sp.nsplit ? sp.nkeep : (int64_t)bins.count[3];
        flops.reset(); total.reset();

        g.a_ptr = P.a_ptr; g.a_col = P.a_col; g.a_val = P.a_val; g.b_ptr = b_ptr; g.b_col = B.col; g.b_val = bval;
        g.nrows = nrows; g.ncols = ncols; g.add_op = add; g.mul_op = mul; g.need_a = need_a; g.need_b = need_b;
        g.c_cnt = cnt;
        if (comp) { g.m_ptr = P.m_ptr; g.m_col = P.m_col; }
        sa.a_col = P.a_col; sa.a_val = P.a_val; sa.b_ptr = b_ptr; sa.b_col = B.col; sa.b_val = bval; sa.m_ptr = g.m_ptr; sa.m_col = g.m_col;
        sa.queue = sp.queue; sa.pres = sp.pres; sa.mbit = sp.mbit; sa.acc = sp.acc; sa.words = sp.words; sa.ncols = ncols; sa.nrange = sp.nrange;
        sa.add_op = add; sa.mul_op = mul; sa.need_a = need_a; sa.need_b = need_b; sa.c_cnt = cnt; sa.range_cnt = sp.range_cnt;
        spa_ctas = std::max(1, std::min<int>((int)spa_n, G.num_sms * 2));
        if (spa_budget > 0 && spa_n) {  // one CTA's accumulator, presence bitmap and (comp) mask bitmap: ncols > 0 here
            const int64_t per_cta = ncols * (int64_t)wsize + ceil_div(ncols, 32) * 4 * (comp ? 2 : 1);
            spa_ctas = (int)std::max<int64_t>(1, std::min<int64_t>(spa_budget / per_cta, spa_ctas));
        }
        if (spa_n) {
            g.spa_words = ceil_div(ncols, 32);
            const size_t words = (size_t)spa_ctas * g.spa_words * (comp ? 2 : 1);     // comp: + the mask bitmaps
            GB_TRY(spa_bits.alloc(words, err));
            g.spa_bits = spa_bits;
            CU_TRY(cudaMemsetAsync(g.spa_bits, 0, words * 4, G.stream), err);
            GB_TRY(queue.alloc(2, err));
            CU_TRY(cudaMemsetAsync(queue, 0, 8, G.stream), err);
        }
        // the bins are recorded here: a complemented mask may block every product, and then the numeric pass does not run
        if (bins.count[1]) {
            g.rows = bins.rows + bins.offset[1]; g.nbin = bins.count[1]; g.table = SMALL_TABLE;
            (comp ? hash_symbolic_kernel<true, true, BT> : hash_symbolic_kernel<true, false, BT>)
                <<<(unsigned)ceil_div(g.nbin, 8), 256, 8 * SMALL_TABLE * 4, G.stream>>>(g);
            GB_LAUNCHED(); use.bin[0] = true;
        }
        if (bins.count[2]) {
            g.rows = bins.rows + bins.offset[2]; g.nbin = bins.count[2]; g.table = MEDIUM_TABLE;
            (comp ? hash_symbolic_kernel<false, true, BT> : hash_symbolic_kernel<false, false, BT>)
                <<<(unsigned)g.nbin, 256, MEDIUM_TABLE * 4, G.stream>>>(g);
            GB_LAUNCHED(); use.bin[1] = true;
        }
        if (spa_n) {
            g.rows = spa_rows; g.nbin = spa_n; g.queue = queue;
            (comp ? spa_kernel<bool, bool, -1, -1, false, true, BT> : spa_kernel<bool, bool, -1, -1, false, false, BT>)<<<spa_ctas, 512, 0, G.stream>>>(g);
            GB_LAUNCHED(); use.bin[2] = true;
        }
        for (int64_t k = 0; k + 1 < (int64_t)sp.chunk_off.size(); ++k) {
            int64_t ng = 0;
            const SplitArgsT<BT> s = split_group<BT>(sp, sa, k, &ng, err);
            split_chunk_kernel<bool, bool, -1, -1, false, BT><<<split_ctas(s.nchunks), 512, 0, G.stream>>>(s);
            split_count_kernel<true, BT><<<dim3((unsigned)sp.nrange, (unsigned)ng), 256, 0, G.stream>>>(s);
            G.launches += 2;
        }
        if (sp.nsplit) use.bin[3] = true;
        if (pp.n) {
            GB_TRY(pull_count(po, pp, cnt, err));
            use.bin[4] = true; use.pull_dot = pull->dot; pull->rows += pp.n;
        }
        return GrB_SUCCESS;
    };
    // ---- numeric (shared-memory bins: expand-sort-compress)
    auto numeric = [&](Csr &t) {
        g.c_ptr = t.rowptr; g.c_col = t.col; g.c_val = t.val;
        if (bins.count[1]) {
            g.rows = bins.rows + bins.offset[1]; g.nbin = bins.count[1];
#define K_ESC_SMALL(XT, ZT, A_, M_) (comp ? esc_numeric_kernel<XT, ZT, A_, M_, true, true, BT> : esc_numeric_kernel<XT, ZT, A_, M_, true, false, BT>) \
                <<<(unsigned)ceil_div(g.nbin, 8), 256, ESC_SMEM_SMALL, G.stream>>>(g)
            GB_FOR_SEMIRING(xt, zt, add, mul, K_ESC_SMALL, err); GB_LAUNCHED();
        }
        if (bins.count[2]) {
            g.rows = bins.rows + bins.offset[2]; g.nbin = bins.count[2];
#define K_ESC_MEDIUM(XT, ZT, A_, M_) (comp ? esc_numeric_kernel<XT, ZT, A_, M_, false, true, BT> : esc_numeric_kernel<XT, ZT, A_, M_, false, false, BT>) \
                <<<(unsigned)g.nbin, 256, esc_smem_medium<BT>(), G.stream>>>(g)
            GB_FOR_SEMIRING(xt, zt, add, mul, K_ESC_MEDIUM, err); GB_LAUNCHED();
        }
        if (spa_n) {
            g.rows = spa_rows; g.nbin = spa_n; g.queue = queue + 1;
            DevBuf<void> spa_val;
            GB_TRY(spa_val.alloc((size_t)spa_ctas * ncols * wsize + 16, err));
            g.spa_val = spa_val;
#define K_SPA(XT, ZT, A_, M_) do { \
            fill_accum_init<ZT>(g.spa_val, (int64_t)spa_ctas * ncols, (A_) >= 0 ? (A_) : add); \
            (comp ? spa_kernel<XT, ZT, A_, M_, true, true, BT> : spa_kernel<XT, ZT, A_, M_, true, false, BT>)<<<spa_ctas, 512, 0, G.stream>>>(g); } while (0)
            GB_FOR_SEMIRING(xt, zt, add, mul, K_SPA, err); G.launches += 2;
        }
        if (sp.nsplit) {
            sa.c_ptr = t.rowptr; sa.c_col = t.col; sa.c_val = t.val;
#define K_SPLIT(XT, ZT, A_, M_) GB_TRY((split_numeric<XT, ZT, A_, M_, BT>(sp, sa, err)))
            GB_FOR_SEMIRING(xt, zt, add, mul, K_SPLIT, err);
        }
        if (pp.n) GB_TRY(pull_fill(po, pp, t.rowptr, t.col, t.val, err));
        spa_bits.reset(); queue.reset(); bins.rows.reset();
        return GrB_SUCCESS;
    };
    // the size rule: checked on the panel's entry count after the scan, before its arrays are allocated
    auto check = [&](int64_t nnz) {
        if (rc) {
            rc->total += nnz;
            if (rc->total >= rc->limit) return gb_fail(GrB_INVALID_VALUE, err, "%s", WIDE_RESULT_REFUSAL);
        }
        return GrB_SUCCESS;
    };
    return csr_from_row_counts(nrows, ncols, tc_size(zt), T, err, symbolic, numeric, check);
}

// T<M> = A (+).(x) B restricted to a non-complemented mask M (pattern of T is a subset of M's).
// dot == true computes A (+).(x) B' by row intersections instead (B given un-transposed).
static constexpr int WARP_FLOPS = 2048;          // rows at most this heavy (and with short mask rows) run warp-per-row

// B200GRB_SPGEMM_TRACE=1: device time of the phases of one masked call (events on the compute stream), printed to stderr
struct PhaseTrace {
    bool on; std::vector<cudaEvent_t> ev; std::vector<const char *> name;
    PhaseTrace() : on(tunables().spgemm_trace) { mark("start"); }
    void mark(const char *n) { if (!on) return; cudaEvent_t e; cudaEventCreate(&e); cudaEventRecord(e, G.stream); ev.push_back(e); name.push_back(n); }
    ~PhaseTrace() {
        if (!on) return;
        cudaStreamSynchronize(G.stream);
        fprintf(stderr, "[mxm phases]");
        for (size_t k = 1; k < ev.size(); ++k) { float ms = 0; cudaEventElapsedTime(&ms, ev[k - 1], ev[k]); fprintf(stderr, " %s %.2f ms |", name[k], ms); }
        float tot = 0; cudaEventElapsedTime(&tot, ev.front(), ev.back()); fprintf(stderr, " total %.2f ms\n", tot);
        for (auto e : ev) cudaEventDestroy(e);
    }
};

// the methods a masked call ran: reported once each, in the same order, however many panels ran them
struct MaskedUse { bool dot = false, warp = false, cls[3] = {false, false, false}, exact[3] = {false, false, false}; };

// The masked methods on one panel: the accumulator word and the found flag of each of its mask entries, in the workspace
// (*tval, *tfound; 1- and 2-byte types are narrowed into `typed`).  BT: the type of B's row offsets.
template <typename BT>
static GrB_Info masked_panel(const RowPanel &P, const Csr &B, const BT *b_ptr, const void *bval, int xt, int zt, int add, int mul,
                             bool need_a, bool need_b, int mtc, bool m_struct, bool dot, int64_t ncols, PhaseTrace &trace,
                             MaskedUse &use, void **tval, uint8_t **tfound, DevBuf<void> &typed, std::string *err) {
    const int64_t nrows = P.nrows;
    const size_t zsz = (size_t)tc_size(zt), wsize = zsz == 8 ? 8 : 4;
    MaskedArgsT<BT> ma{};
    GemmArgsT<BT> &g = ma.g;
    g.a_ptr = P.a_ptr; g.a_col = P.a_col; g.a_val = P.a_val; g.b_ptr = b_ptr; g.b_col = B.col; g.b_val = bval;
    g.m_ptr = P.m_ptr; g.m_col = P.m_col; g.m_val = P.m_val; g.m_tc = mtc; g.m_struct = m_struct;
    g.nrows = nrows; g.ncols = ncols; g.add_op = add; g.mul_op = mul; g.need_a = need_a; g.need_b = need_b;
    void *words = nullptr; uint8_t *found = nullptr;          // per mask entry: accumulator word, "has a value"
    GB_TRY(ws_get(WS_WORDS, &words, (size_t)P.mnnz * wsize + 16, err));
    GB_TRY(ws_get(WS_FOUND, (void **)&found, (size_t)P.mnnz + 16, err));
    g.c_val = words; g.t_found = found; ma.t_words = words;
    *tval = words; *tfound = found;
    if (P.mnnz > 0 && dot) {
        // the dot kernel writes typed values directly
#define K_DOT(XT, ZT, A_, M_) masked_dot_kernel<XT, ZT, A_, M_, BT><<<grid_for(nrows * 32), 256, 0, G.stream>>>(g)
        GB_FOR_SEMIRING(xt, zt, add, mul, K_DOT, err); GB_LAUNCHED(); use.dot = true;
    } else if (P.mnnz > 0) {
        int64_t *flops = nullptr; unsigned long long *total = nullptr;
        GB_TRY(ws_array(WS_FLOPS, &flops, (size_t)nrows, err)); GB_TRY(ws_array(WS_TOTAL, &total, 1, err));
        CU_TRY(cudaMemsetAsync(total, 0, 8, G.stream), err);
        flops_kernel<<<grid_for(nrows * 32), 256, 0, G.stream>>>(P.a_ptr, P.a_col, b_ptr, nrows, flops, total); GB_LAUNCHED();
        // accumulators start at accum_init, flags at 0
        CU_TRY(cudaMemsetAsync(found, 0, (size_t)P.mnnz, G.stream), err);
#define K_IDENT(XT, ZT, A_, M_) fill_accum_init<ZT>(words, P.mnnz, (A_) >= 0 ? (A_) : add)
        GB_FOR_SEMIRING(xt, zt, add, mul, K_IDENT, err); GB_LAUNCHED();
        // classify rows and cut heavy ones into flop-bounded chunks
        int64_t *cs = nullptr, *cm = nullptr, *cl = nullptr, *c1 = nullptr;
        GB_TRY(ws_array(WS_CS, &cs, (size_t)nrows + 1, err));
        GB_TRY(ws_array(WS_CM, &cm, (size_t)nrows + 1, err)); GB_TRY(ws_array(WS_CL, &cl, (size_t)nrows + 1, err)); GB_TRY(ws_array(WS_C1, &c1, (size_t)nrows + 1, err));
        CU_TRY(cudaMemsetAsync(cs + nrows, 0, 8, G.stream), err);
        CU_TRY(cudaMemsetAsync(cm + nrows, 0, 8, G.stream), err); CU_TRY(cudaMemsetAsync(cl + nrows, 0, 8, G.stream), err);
        CU_TRY(cudaMemsetAsync(c1 + nrows, 0, 8, G.stream), err);
        chunk_count_kernel<<<grid_for(nrows), 256, 0, G.stream>>>(flops, P.m_ptr, nrows, CHUNK_FLOPS, WARP_FLOPS, SMALL_TABLE / 2,
                                                                  MIDSMALL_TABLE / 2, MEDIUM_TABLE / 2, cs, cm, cl, c1); GB_LAUNCHED();
        GB_TRY(dev_exclusive_scan(cs, nrows + 1, err));
        GB_TRY(dev_exclusive_scan(cm, nrows + 1, err)); GB_TRY(dev_exclusive_scan(cl, nrows + 1, err)); GB_TRY(dev_exclusive_scan(c1, nrows + 1, err));
        int64_t n_small = 0, n_medium = 0, n_long = 0, n_warp = 0, tf = 0;
        GB_TRY(read_i64(cs + nrows, &n_small, err));
        GB_TRY(read_i64(cm + nrows, &n_medium, err)); GB_TRY(read_i64(cl + nrows, &n_long, err)); GB_TRY(read_i64(c1 + nrows, &n_warp, err));
        GB_TRY(read_i64((const int64_t *)total, &tf, err));
        G.last_flops += (uint64_t)tf;
        int32_t *s_row = nullptr, *m_row = nullptr, *l_row = nullptr, *w_rows = nullptr;
        uint32_t *s_idx = nullptr, *s_cnt = nullptr, *m_idx = nullptr, *m_cnt = nullptr, *l_idx = nullptr, *l_cnt = nullptr;
        GB_TRY(ws_array(WS_SROW, &s_row, (size_t)n_small, err)); GB_TRY(ws_array(WS_SIDX, &s_idx, (size_t)n_small, err)); GB_TRY(ws_array(WS_SCNT, &s_cnt, (size_t)n_small, err));
        GB_TRY(ws_array(WS_MROW, &m_row, (size_t)n_medium, err)); GB_TRY(ws_array(WS_MIDX, &m_idx, (size_t)n_medium, err)); GB_TRY(ws_array(WS_MCNT, &m_cnt, (size_t)n_medium, err));
        GB_TRY(ws_array(WS_LROW, &l_row, (size_t)n_long, err)); GB_TRY(ws_array(WS_LIDX, &l_idx, (size_t)n_long, err)); GB_TRY(ws_array(WS_LCNT, &l_cnt, (size_t)n_long, err));
        GB_TRY(ws_array(WS_WROWS, &w_rows, (size_t)n_warp, err));
        chunk_fill_kernel<<<grid_for(nrows), 256, 0, G.stream>>>(cs, cm, cl, c1, nrows, s_row, s_idx, s_cnt, m_row, m_idx, m_cnt, l_row, l_idx, l_cnt, w_rows); GB_LAUNCHED();
        trace.mark("flops + chunk lists");
        if (n_warp) {
            g.rows = w_rows; g.nbin = n_warp; g.table = SMALL_TABLE;
            const size_t sm = masked_smem(SMALL_TABLE, 8, wsize);
#define K_MSMALL(XT, ZT, A_, M_) masked_hash_kernel<XT, ZT, A_, M_, BT><<<(unsigned)ceil_div(n_warp, 8), 256, sm, G.stream>>>(ma)
            GB_FOR_SEMIRING(xt, zt, add, mul, K_MSMALL, err); GB_LAUNCHED(); use.warp = true;
        }
        // chunked classes: the streaming kernel (spgemm_stream.cuh), persistent CTAs over blocks of consecutive chunks
        {
            unsigned int *queues = nullptr;
            GB_TRY(ws_array(WS_QUEUES, &queues, 4, err));
            CU_TRY(cudaMemsetAsync(queues, 0, 16, G.stream), err);
            // The 128-bit loads of a trip reach up to 3 positions past B's last entry, into the padding of its allocation (dmalloc
            // rounds to 256 bytes).  The filter indexes its bitmap with a loaded id before the position test drops it, so with an
            // exact bitmap a stray id there would read shared memory out of range: those positions must hold valid ids (0).
            if (B.nnz % 4 && (n_small || n_medium || n_long))
                CU_TRY(cudaMemsetAsync(B.col.get() + B.nnz, 0, (size_t)(4 - B.nnz % 4) * sizeof(uint32_t), G.stream), err);
            StreamArgsT<BT> sa{}; sa.g = g; sa.t_words = words;
            struct Cls { int64_t n; const int32_t *row; const uint32_t *idx, *cnt; int nt, bm_log2, vals_cap, grab; };
            const Cls cls[3] = {{n_small, s_row, s_idx, s_cnt, 256, 14, MIDSMALL_TABLE / 2, 8},
                                {n_medium, m_row, m_idx, m_cnt, 256, 16, MEDIUM_TABLE / 2, 4},
                                {n_long, l_row, l_idx, l_cnt, 1024, 20, 0, 4}};
            trace.mark("warp class");
            for (int k = 0; k < 3; ++k) {
                if (!cls[k].n) continue;
                sa.chunk_row = cls[k].row; sa.chunk_idx = cls[k].idx; sa.chunk_cnt = cls[k].cnt; sa.nchunks = cls[k].n;
                sa.queue = queues + k; sa.bm_log2 = cls[k].bm_log2; sa.exact = ncols <= ((int64_t)1 << cls[k].bm_log2) ? 1 : 0;
                sa.vals_cap = cls[k].vals_cap; sa.table = cls[k].vals_cap * 2; sa.grab = cls[k].grab; sa.spa_slot = nullptr;
                sa.blk_log2 = tunables().stream_blk_log2;
                const size_t sm_var = stream_var_smem(sa.bm_log2, sa.table, sa.vals_cap, wsize);
                const bool big = cls[k].nt == 1024;
                int ctas_big = 0;
                if (big) {      // hub mask rows: the column -> position map of each persistent CTA lives in HBM
                    ctas_big = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(sa.nchunks, sa.grab), G.num_sms));
                    bool fresh = false;          // the kernel resets every entry it sets: the maps stay all -1 between calls
                    GB_TRY(ws_array(WS_SPA_SLOT, &sa.spa_slot, (size_t)ctas_big * ncols, err, &fresh));
                    if (fresh) CU_TRY(cudaMemsetAsync(sa.spa_slot, 0xFF, ((size_t)ctas_big * ncols + ((size_t)ctas_big * ncols) / 4) * 4, G.stream), err);
                }
#define K_MSTREAM(XT, ZT, A_, M_) do { \
                const int nt = big ? 1024 : 256; \
                const size_t sm = sm_var + stream_fixed_smem<XT, BT>(nt); \
                auto kern = masked_stream_kernel<XT, ZT, A_, M_, BT>; \
                cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm); \
                int ctas = ctas_big; \
                if (!big) { int per_sm = 1; cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, 256, sm); \
                            ctas = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(sa.nchunks, sa.grab), (int64_t)G.num_sms * std::max(per_sm, 1))); } \
                kern<<<ctas, nt, sm, G.stream>>>(sa); } while (0)
                GB_FOR_SEMIRING(xt, zt, add, mul, K_MSTREAM, err); GB_LAUNCHED();
                use.cls[k] = true; use.exact[k] = sa.exact != 0;
                trace.mark(k == 0 ? "stream S" : (k == 1 ? "stream M" : "stream L"));
            }
        }
        if (zsz < 4) {      // narrow 32-bit accumulator words to the 1- or 2-byte type, in a second buffer
            GB_TRY(typed.alloc((size_t)P.mnnz * zsz + 16, err));
            narrow_words_kernel<<<grid_for(P.mnnz), 256, 0, G.stream>>>((const uint32_t *)words, (uint8_t *)typed, (int)zsz, P.mnnz); GB_LAUNCHED();
            *tval = typed;
        }
    }
    return GrB_SUCCESS;
}

template <typename OT>
static GrB_Info masked_compact_t(int64_t nrows, int64_t ncols, int64_t mnnz, const OT *m_ptr, const uint32_t *m_col, const uint8_t *found,
                                 const void *tval, size_t vsize, Csr &T, std::string *err);

// ------------------------------------------------------------------ the row panels of the CSR x CSR products
// Rows of T = A (+).(x) B, under a mask M or M' or none, depend on the same rows of A and of the mask only, so the wide route walks
// A and the mask in row panels of at most `bound` entries of each (a longer row is a panel of its own: every row has fewer than
// 2^31 entries), with their offsets rebased to 32 bits: the kernels keep 32-bit positions in A and the mask, and the per-mask-entry
// scratch and the per-row arrays are those of one panel.  B's rows are gathered by A's column ids and cannot be cut: the kernels
// read B's 64-bit offsets when B is wide.  Each panel is formed on its own; T is formed from the panels' row counts and entries.
static constexpr int64_t WIDE_PANEL = (int64_t)1 << 30;
static constexpr int64_t WIDE_PANEL_ROWS = (int64_t)1 << 26;       // and at most this many rows: the per-row arrays (40 B a row)

// the panel that starts at row r0: out = {r1, A's and M's first entries, M's end}, r1 the last row r <= r0 + max_rows with at most
// `bound` entries of A and of M in rows [r0, r), and at least r0 + 1
__global__ void panel_end_kernel(const int64_t *a_ptr, const int64_t *m_ptr, int64_t r0, int64_t nrows, int64_t bound, int64_t max_rows,
                                 int64_t *out) {
    const int64_t a0 = a_ptr[r0], m0 = m_ptr[r0];
    int64_t lo = r0 + 1, hi = min(nrows, r0 + max_rows);
    while (lo < hi) {
        const int64_t mid = lo + (hi - lo + 1) / 2;
        if (a_ptr[mid] - a0 <= bound && m_ptr[mid] - m0 <= bound) lo = mid; else hi = mid - 1;
    }
    out[0] = lo; out[1] = a0; out[2] = m0; out[3] = m_ptr[lo];
}
// out[r] = ptr[r0 + r] - ptr[r0], r = 0 .. n: the 32-bit offsets of a panel of n rows
__global__ void panel_rowptr_kernel(const int64_t *ptr, int64_t r0, int64_t n, uint32_t *out) {
    const int64_t base = ptr[r0];
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r <= n; r += (int64_t)gridDim.x * blockDim.x) out[r] = (uint32_t)(ptr[r0 + r] - base);
}

// The size rule of the unmasked wide route, in one pass over A's 64-bit offsets: total[0] += the products of every row (U, an upper
// bound on nnz(T)), total[1] += max(0, nnz of the longest B row named by A(i,:) - nnz(M'(i,:))) (L: that B row lies in T(i,:) but
// for what M' blocks, so L is a lower bound on nnz(T)).  m_ptr: M''s offsets, null without a complemented mask.  Warp per row.
template <typename BT>
__global__ void gemm_bound_kernel(const int64_t *a_ptr, const uint32_t *a_col, const BT *b_ptr, const int64_t *m_ptr, int64_t nrows,
                                  unsigned long long *total) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    unsigned long long u = 0, l = 0;
    for (int64_t r = warp; r < nrows; r += nwarps) {
        int64_t f = 0, longest = 0;
        for (int64_t p = a_ptr[r] + lane; p < a_ptr[r + 1]; p += 32) {
            const uint32_t k = a_col[p];
            const int64_t len = (int64_t)(b_ptr[k + 1] - b_ptr[k]);
            f += len; longest = max(longest, len);
        }
        for (int o = 16; o > 0; o >>= 1) {
            f += __shfl_xor_sync(0xffffffffu, f, o);
            longest = max(longest, (int64_t)__shfl_xor_sync(0xffffffffu, longest, o));
        }
        if (m_ptr) longest -= m_ptr[r + 1] - m_ptr[r];
        if (lane == 0) { u += (unsigned long long)f; if (longest > 0) l += (unsigned long long)longest; }
    }
    if (lane == 0 && u) atomicAdd(&total[0], u);
    if (lane == 0 && l) atomicAdd(&total[1], l);
}

// T (ncols columns, zsz bytes a value) = body(P, part) on the row panels P of A and of the mask M (null: no mask entry applies).
// aval: A's values as the multiply reads them; asz, msz: the bytes of one value of A and of M in the panel (0: not read).  The
// narrow route (!wide) is one panel, the whole of A and M through their rowptr32, formed straight into T; the wide route cuts
// panels of at most `bound` entries of A and of M.
template <typename Body>
static GrB_Info spgemm_panels(const Csr &A, const void *aval, size_t asz, const Csr *M, size_t msz, bool wide, int64_t bound,
                              int64_t ncols, size_t zsz, Csr &T, std::string *err, Body &&body) {
    const int64_t nrows = A.nrows;
    if (!wide)
        return body(RowPanel{A.rowptr32, A.col, aval, M ? M->rowptr32.get() : nullptr, M ? M->col.get() : nullptr,
                             M && msz ? M->val.get() : nullptr, nrows, M ? M->nnz : 0}, T);
    std::vector<Csr> parts;
    DevBuf<int64_t> ends;
    GB_TRY(ends.alloc(4, err));
    // the panel that starts at row r0, formed into `part`; *r1 = its end.  Without M, A's offsets stand in for panel_end_kernel's M.
    auto panel = [&](int64_t r0, int64_t *r1, Csr &part) -> GrB_Info {
        panel_end_kernel<<<1, 1, 0, G.stream>>>(A.rowptr, M ? M->rowptr.get() : A.rowptr.get(), r0, nrows, bound, WIDE_PANEL_ROWS, ends);
        GB_LAUNCHED();
        int64_t h[4];
        CU_TRY(cudaMemcpyAsync(h, ends, sizeof(h), cudaMemcpyDeviceToHost, G.stream), err);
        CU_TRY(cudaStreamSynchronize(G.stream), err);
        *r1 = h[0];
        const int64_t a0 = h[1], m0 = h[2], m1 = h[3], pn = *r1 - r0;
        uint32_t *ap = nullptr, *mp = nullptr;
        GB_TRY(ws_array(WS_PANEL_A, &ap, (size_t)pn + 1, err));
        panel_rowptr_kernel<<<grid_for(pn + 1), 256, 0, G.stream>>>(A.rowptr, r0, pn, ap); GB_LAUNCHED();
        if (M) {
            GB_TRY(ws_array(WS_PANEL_M, &mp, (size_t)pn + 1, err));
            panel_rowptr_kernel<<<grid_for(pn + 1), 256, 0, G.stream>>>(M->rowptr, r0, pn, mp); GB_LAUNCHED();
        }
        const RowPanel P{ap, A.col + a0, aval ? static_cast<const uint8_t *>(aval) + a0 * asz : nullptr, mp, M ? M->col + m0 : nullptr,
                         M && msz ? static_cast<const uint8_t *>(M->val.get()) + m0 * msz : nullptr, pn, M ? m1 - m0 : 0};
        return body(P, part);
    };
    int64_t r1 = 0;
    if (nrows > 0) {
        parts.emplace_back();
        GB_TRY(panel(0, &r1, parts[0]));
        if (r1 == nrows) {                      // one panel: it is T
            T = std::move(parts[0]);
            return GrB_SUCCESS;
        }
    }
    return csr_from_row_counts(nrows, ncols, zsz, T, err,
        [&](int64_t *rowptr) {
            CU_TRY(cudaMemsetAsync(rowptr + nrows, 0, 8, G.stream), err);
            for (int64_t r0 = 0, q = 0; r0 < nrows; r0 = r1, ++q) {
                if (q > 0) { parts.emplace_back(); GB_TRY(panel(r0, &r1, parts.back())); }
                else r1 = parts[0].nrows;
                row_len_kernel<<<grid_for(r1 - r0), 256, 0, G.stream>>>(parts.back().rowptr32, r1 - r0, rowptr + r0); GB_LAUNCHED();
            }
            return GrB_SUCCESS;
        },
        [&](Csr &t) {
            int64_t at = 0;
            for (Csr &part : parts) {
                if (part.nnz) {
                    CU_TRY(cudaMemcpyAsync(t.col.get() + at, part.col, (size_t)part.nnz * 4, cudaMemcpyDeviceToDevice, G.stream), err);
                    CU_TRY(cudaMemcpyAsync(static_cast<uint8_t *>(t.val.get()) + at * zsz, part.val, (size_t)part.nnz * zsz,
                                           cudaMemcpyDeviceToDevice, G.stream), err);
                }
                at += part.nnz;
                part = Csr();
            }
            return GrB_SUCCESS;
        });
}

static void masked_report(const MaskedUse &u, bool wide) {
    bool first = true;
    auto entry = [&](const char *k) { gb_kernel_used(k); if (first && wide) gb_kernel_used("offsets=64"); first = false; };
    if (u.dot) entry("dot");
    if (u.warp) entry("masked-warp");
    for (int k = 0; k < 3; ++k) {
        if (!u.cls[k]) continue;
        entry(k == 0 ? "stream-S" : (k == 1 ? "stream-M" : "stream-L"));
        gb_kernel_used(u.exact[k] ? "filter=exact" : "filter=bloom");
    }
}

// ------------------------------------------------------------------ the wide route of the unmasked and complemented-mask bins
// The masked route's row panels (spgemm_panels, of A and M', the entries of a complemented mask that block): each panel runs the
// whole pipeline (flops, bins, symbolic, scan, numeric) into a CSR of its rows; T is the one panel, or is formed from the panels'
// row counts and entries.  B is read through its 64-bit offsets when it is wide.  The route forms results of fewer than 2^32
// entries: T would take 34 GB or more in FP32 (twice that while the panels are joined), which does not fit beside a wide operand
// on an 80 GB card.  gemm_bound_kernel bounds nnz(T) before any panel runs: L >= the limit is refused at once; U < the limit
// needs no further check; otherwise the panels' symbolic counts are added up and the call refused as soon as the scan of a
// panel's counts reaches the limit, before that panel's entries are allocated or formed.  The dense accumulators of a panel are capped at WIDE_SPA_BUDGET bytes (one FP32 accumulator is
// 1 GB at n = 2^28).
static constexpr int64_t WIDE_RESULT = (int64_t)1 << 32;
static constexpr int64_t WIDE_SPA_BUDGET = (int64_t)1 << 32;
// the route of a CSR x CSR product without a (non-complemented) mask: a CSR without rowptr32, or any CSR under B200_debug_wide_gemm
static inline bool gemm_wide(const Csr &c) { return !c.rowptr32 || G.debug_wide_gemm > 0; }

static void unmasked_report(const UnmaskedUse &u, bool wide) {
    static const char *const names[5] = {"esc-small", "esc-medium", "spa", "spa-split", "pull"};
    bool first = true;
    for (int k = 0; k < 5; ++k) {
        if (!u.bin[k]) continue;
        gb_kernel_used(names[k]);
        if (first && wide) gb_kernel_used("offsets=64");
        first = false;
    }
    if (u.bin[4]) gb_kernel_used(u.pull_dot ? "pull=dot" : "pull=auto");
}

// T = A (+).(x) B, unmasked, or (A (+).(x) B)<!Mb> with Mb the entries of a complemented mask that block.  The narrow route runs
// the bins once on the whole of A and Mb; the wide route (an operand or the mask of 2^32 or more entries, or B200_debug_wide_gemm)
// on row panels, with B's 64-bit offsets when B is wide.  pull: the pull route of an eligible call, or null.
static GrB_Info spgemm_unmasked_call(const Csr &A, const Csr &B, const void *aval, const void *bval, int xt, int zt, int add, int mul,
                                     bool need_a, bool need_b, const Csr *Mb, bool wide, PullSide *pull, Csr &T, std::string *err) {
    const Csr *M = Mb && Mb->nnz > 0 ? Mb : nullptr;
    const int64_t nrows = A.nrows;
    const bool seam = G.debug_wide_gemm > 0;
    const int64_t bound = std::min(seam ? G.debug_wide_gemm : WIDE_PANEL, WIDE_PANEL);
    const int64_t budget = !wide ? 0 : seam && G.debug_spa_budget > 0 ? G.debug_spa_budget : WIDE_SPA_BUDGET;
    ResultCount rc;
    rc.limit = seam && G.debug_gemm_limit > 0 ? G.debug_gemm_limit : WIDE_RESULT;
    UnmaskedUse use;
    G.last_flops = 0;
    auto run = [&](auto b_ptr) -> GrB_Info {
        bool counting = false;
        if (wide && nrows > 0) {
            DevBuf<unsigned long long> tot;
            GB_TRY(tot.alloc(2, err));
            CU_TRY(cudaMemsetAsync(tot, 0, 16, G.stream), err);
            gemm_bound_kernel<<<grid_for(nrows * 32), 256, 0, G.stream>>>(A.rowptr, A.col, b_ptr, M ? M->rowptr.get() : nullptr, nrows, tot);
            GB_LAUNCHED();
            unsigned long long h[2];
            CU_TRY(cudaMemcpyAsync(h, tot, sizeof(h), cudaMemcpyDeviceToHost, G.stream), err);
            CU_TRY(cudaStreamSynchronize(G.stream), err);
            if (h[1] >= (unsigned long long)rc.limit) return gb_fail(GrB_INVALID_VALUE, err, "%s", WIDE_RESULT_REFUSAL);
            counting = h[0] >= (unsigned long long)rc.limit;
        }
        return spgemm_panels(A, aval, need_a ? tc_size(xt) : 0, M, 0, wide, bound, B.ncols, tc_size(zt), T, err,
                             [&](const RowPanel &P, Csr &part) {
                                 // the pull runs on the narrow route only
                                 return spgemm_unmasked(P, B, b_ptr, bval, xt, zt, add, mul, need_a, need_b, budget, use,
                                                        counting ? &rc : nullptr, wide ? nullptr : pull, part, err);
                             });
    };
    GB_TRY(gemm_wide(B) ? run(B.rowptr.get()) : run(B.rowptr32.get()));
    G.last_nnz_out = (uint64_t)T.nnz;
    unmasked_report(use, wide);
    return GrB_SUCCESS;
}

// The narrow route runs the masked methods once on the whole of A and M; the wide route (csr_wide: an operand of 2^32 or more
// entries, or B200_debug_wide) on row panels, with B's 64-bit offsets when B is wide.
static GrB_Info spgemm_masked(const Csr &A, const Csr &B, const void *aval, const void *bval, int xt, int zt,
                              int add, int mul, bool need_a, bool need_b, const Csr &M, int mtc, bool m_struct,
                              bool dot, Csr &T, std::string *err) {
    const int64_t nrows = A.nrows, ncols = dot ? B.nrows : B.ncols;
    T = Csr(); T.nrows = nrows; T.ncols = ncols;
    const size_t zsz = (size_t)tc_size(zt);
    PhaseTrace trace;
    MaskedUse use;
    G.last_flops = 0;
    const bool wide = csr_wide(A) || csr_wide(B) || csr_wide(M);
    const int64_t bound = std::min(G.debug_wide > 0 ? wide_chunk() : WIDE_PANEL, WIDE_PANEL);
    auto run = [&](auto b_ptr) {
        return spgemm_panels(A, aval, need_a ? tc_size(xt) : 0, &M, M.val.get() ? tc_size(mtc) : 0, wide, bound, ncols, zsz, T, err,
                             [&](const RowPanel &P, Csr &part) -> GrB_Info {
                                 void *tval = nullptr; uint8_t *found = nullptr;
                                 DevBuf<void> typed;
                                 GB_TRY(masked_panel(P, B, b_ptr, bval, xt, zt, add, mul, need_a, need_b, mtc, m_struct, dot, ncols,
                                                     trace, use, &tval, &found, typed, err));
                                 return masked_compact_t<uint32_t>(P.nrows, ncols, P.mnnz, P.m_ptr, P.m_col, found, tval, zsz, part, err);
                             });
    };
    GB_TRY(csr_wide(B) ? run(B.rowptr.get()) : run(B.rowptr32.get()));
    G.last_nnz_out = (uint64_t)T.nnz;
    masked_report(use, wide);
    trace.mark("compaction");
    CU_TRY(cudaGetLastError(), err);
    return GrB_SUCCESS;
}

template <typename OT>
static GrB_Info masked_compact_t(int64_t nrows, int64_t ncols, int64_t mnnz, const OT *m_ptr, const uint32_t *m_col, const uint8_t *found,
                                 const void *tval, size_t vsize, Csr &T, std::string *err) {
    return csr_from_row_counts(nrows, ncols, vsize, T, err,
        [&](int64_t *rowptr) {
            CU_TRY(cudaMemsetAsync(rowptr, 0, ((size_t)nrows + 1) * 8, G.stream), err);
            if (mnnz > 0) { row_found_count_kernel<<<grid_for(nrows * 32), 256, 0, G.stream>>>(m_ptr, found, nrows, rowptr); GB_LAUNCHED(); }
            return GrB_SUCCESS;
        },
        [&](Csr &t) {
            row_found_fill_kernel<<<grid_for(nrows * 32), 256, 0, G.stream>>>(m_ptr, m_col, found, (const uint8_t *)tval, (int)vsize,
                                                                              nrows, t.rowptr, t.col, (uint8_t *)t.val); GB_LAUNCHED();
            return GrB_SUCCESS;
        });
}
GrB_Info masked_compact(const Csr &M, const uint8_t *found, const void *tval, size_t vsize, Csr &T, std::string *err) {
    GB_TRY(csr_wide(M) ? masked_compact_t<int64_t>(M.nrows, M.ncols, M.nnz, M.rowptr.get(), M.col, found, tval, vsize, T, err)
                       : masked_compact_t<uint32_t>(M.nrows, M.ncols, M.nnz, M.rowptr32.get(), M.col, found, tval, vsize, T, err));
    G.last_nnz_out = (uint64_t)T.nnz;
    return GrB_SUCCESS;
}

// C<M> = accum(C, T) into a fresh CSR `out` of C's type (T has type ttc)
static GrB_Info matrix_finalize(const Csr *C, int ctc, const Csr &T, int ttc, const Csr *M, int mtc, const DescFlags &f,
                                const GrB_BinaryOp accum, Csr &out, std::string *err) {
    const int64_t nrows = T.nrows;
    MatFinalizeArgs a{};
    a.nrows = nrows;
    if (C) { a.c_ptr = C->rowptr; a.c_col = C->col; a.c_val = C->val; a.c_exists = 1; }
    a.ctc = ctc;
    a.t_ptr = T.rowptr; a.t_col = T.col; a.t_val = T.val; a.ttc = ttc;
    if (M) { a.m_ptr = M->rowptr; a.m_col = M->col; a.m_val = M->val; a.mtc = mtc; a.has_mask = 1; }
    a.mask_comp = f.mask_comp; a.mask_struct = f.mask_struct; a.replace = f.replace;
    a.accum_op = accum ? accum->opcode : -1;
    a.accum_tc = accum ? accum->xtype->code : 0; a.accum_ztc = accum ? accum->ztype->code : 0;
    return csr_from_row_counts(nrows, T.ncols, tc_size(ctc), out, err,
        [&](int64_t *rowptr) {
            CU_TRY(cudaMemsetAsync(rowptr, 0, ((size_t)nrows + 1) * 8, G.stream), err);
            a.o_cnt = rowptr;
            mat_finalize_kernel<false><<<grid_for(nrows, 128), 128, 0, G.stream>>>(a); GB_LAUNCHED();
            return GrB_SUCCESS;
        },
        [&](Csr &t) {
            a.o_ptr = t.rowptr; a.o_col = t.col; a.o_val = t.val;
            mat_finalize_kernel<true><<<grid_for(nrows, 128), 128, 0, G.stream>>>(a); GB_LAUNCHED();
            return GrB_SUCCESS;
        });
}

// write T (type ttc) back into C under mask / accum / replace; consumes T
GrB_Info matrix_writeback(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const DescFlags &f,
                          Csr &&t_in, int ttc, bool t_already_masked, std::string *err) {
    Csr T = std::move(t_in);
    const int ctc = C->type->code;
    if (!Mask && f.mask_comp) {
        // C<!NULL>: nothing is written; GrB_REPLACE clears C (C API 1.3 section 4.3, SuiteSparse's quick-mask exit)
        T = Csr();
        if (f.replace) {
            matrix_invalidate_device(C);
            C->hi.clear(); C->hj.clear(); C->hx.clear(); C->pi.clear(); C->pj.clear(); C->px.clear(); C->host_valid = true;
        }
        return GrB_SUCCESS;
    }
    const bool c_empty = matrix_known_empty(C);
    // fast exits: the result is exactly T
    const bool plain = !accum && (!Mask || (t_already_masked && (f.replace || c_empty)));
    if (plain || (accum && !Mask && c_empty)) {
        if (ttc != ctc) {
            DevBuf<void> cv;
            GB_TRY(dev_cast_values(cv, ctc, T.val, ttc, T.nnz, err));
            T.val = std::move(cv);
        }
        matrix_adopt_device(C, std::move(T));
        return GrB_SUCCESS;
    }
    if (!c_empty) GB_TRY(matrix_ensure_device(C));
    if (Mask) GB_TRY(matrix_ensure_device(Mask));
    Csr out;
    GrB_Info r = matrix_finalize(c_empty ? nullptr : &C->dev, ctc, T, ttc, Mask ? &Mask->dev : nullptr,
                                 Mask ? Mask->type->code : 0, f, accum, out, err);
    T = Csr();
    if (r != GrB_SUCCESS) return r;
    matrix_adopt_device(C, std::move(out));
    return GrB_SUCCESS;
}

// Values one operand gets in place of its own (the inner form of a positional multiply): side 1 = each entry of op(A) its column
// index, side 2 = each entry of op(B) its row index; through ids (hypersparse operands) when given, plus off, of type tc
struct MxmPos { int side = 0; int tc = 0; int64_t off = 0; const uint64_t *ids = nullptr; };
// *out = the values of c (op(A) on side 1, op(B) or op(B)' on side 2; of type tc) as the multiply reads them: pos's index of each
// entry, its column when by_col, else its row, when pos.side is this side; else mxm_values.  The buffer belongs to the caller.
static GrB_Info mxm_csr_values(DevBuf<void> &cast, const void **out, const Csr &c, int tc, bool reads, int xt, const MxmPos &pos,
                               int side, bool by_col, std::string *err) {
    if (pos.side != side) return mxm_values(cast, out, reads, xt, c.val, tc, c.nnz, err);
    GB_TRY(cast.alloc((size_t)c.nnz * tc_size(pos.tc) + 16, err));
    GB_TRY(pos_csr_values(cast, pos.tc, nullptr, OP_ANY, c, by_col, pos.ids, pos.off, err));
    *out = cast;
    return GrB_SUCCESS;
}

// T = op(A) (+).(x) op(B) under Mask (*masked tells the write-back): a mask that is not complemented selects the masked
// methods; a complemented one runs the unmasked bins with the filter of the entries that block (DESIGN.md section 3.2)
static GrB_Info mxm_product(const GrB_Matrix Mask, const DescFlags &f, int xt, int zt, int add, int mul, const GrB_Matrix A, const GrB_Matrix B,
                            const MxmPos &pos, GbBurble &burble, Csr &T, bool *masked, std::string *err) {
    const bool need_a = mul_reads_x(mul), need_b = mul_reads_y(mul);
    const bool use_mask = Mask && !f.mask_comp;
    *masked = Mask != nullptr;
    Csr *pa; GB_TRY(source_csr(A, f.tran0, &pa));
    GB_TRY(matrix_ensure_device(B));
    // C<M> = A*B': small problems intersect rows of A and B directly (no transpose); large ones
    // go through the cached transpose and the load-balanced masked hash kernels
    const bool dot = use_mask && f.tran1 && B->dev.nnz < ((int64_t)1 << 18);
    if (f.tran1 && !dot) GB_TRY(matrix_ensure_transpose(B));
    if (Mask) GB_TRY(matrix_ensure_device(Mask));
    const Csr &a = *pa;
    const Csr &b = (f.tran1 && !dot) ? B->devT : B->dev;
    // the unmasked and complemented-mask bins take their wide route when an operand or the mask is wide (spgemm_unmasked_call);
    // the masked methods choose theirs in spgemm_masked
    const bool wide = !use_mask && (gemm_wide(a) || gemm_wide(b) || (Mask && gemm_wide(Mask->dev)));
    if (wide && burble.on)
        burble.note("spgemm, 64-bit offsets", (double)a.nnz * (4.0 + (need_a ? tc_size(xt) : 0)) + (double)b.nnz * (4.0 + (need_b ? tc_size(xt) : 0)) +
                                              (double)(a.nrows + b.nrows + 2) * 8);

    DevBuf<void> a_cast, b_cast;
    const void *aval = nullptr, *bval = nullptr;
    GB_TRY(mxm_csr_values(a_cast, &aval, a, A->type->code, need_a, xt, pos, 1, /*by_col=*/true, err));
    // op(B)'s row index: the row of b, or its column when b is B itself standing for B' (the dot method)
    GB_TRY(mxm_csr_values(b_cast, &bval, b, B->type->code, need_b, xt, pos, 2, /*by_col=*/f.tran1 && dot, err));

    GrB_Info r;
    if (use_mask) r = spgemm_masked(a, b, aval, bval, xt, zt, add, mul, need_a, need_b, Mask->dev, Mask->type->code, f.mask_struct, dot, T, err);
    else {
        Csr mtrue;                              // a valued complemented mask: its true entries
        const Csr *mb = nullptr;
        if (Mask && f.mask_struct) mb = &Mask->dev;
        else if (Mask) { GB_TRY(mask_true_pattern(Mask->dev, Mask->type->code, mtrue, err)); mb = &mtrue; }
        // a complemented mask and a saturating monoid (on the narrow route: spgemm_unmasked_call): GxB_AxB_DOT pulls every row
        // with products, the default descriptor the rows the B200GRB_MXM_PULL rule picks (DESIGN.md section 3.2)
        PullSide ps;
        DevBuf<void> bt_cast;
        const bool eligible = Mask && (add == OP_LOR || add == OP_LAND || add == OP_ANY);
        if (eligible) {
            ps.dot = f.axb == GxB_AxB_DOT;
            ps.alpha = f.axb == GxB_DEFAULT ? tunables().mxm_pull : 0.0;
            // op(B)': B itself under INP1 = TRAN, else B's cached transpose; its values of the multiply's x type, or op(B)'s
            // row index p (the column in op(B)') for the positional inner form on op(B)
            ps.ensure = [&](PullOperands &o) -> GrB_Info {
                if (!f.tran1) GB_TRY(matrix_ensure_transpose(B));
                const Csr &bt = f.tran1 ? B->dev : B->devT;
                if (!bt.rowptr32) return gb_fail(GrB_PANIC, err, "GrB_mxm: the pull route needs 32-bit offsets of op(B)'");
                o.bt_ptr = bt.rowptr32; o.bt_col = bt.col;
                return mxm_csr_values(bt_cast, &o.bt_val, bt, B->type->code, need_b, xt, pos, 2, /*by_col=*/true, err);
            };
        }
        r = spgemm_unmasked_call(a, b, aval, bval, xt, zt, add, mul, need_a, need_b, mb, wide, eligible ? &ps : nullptr, T, err);
        if (r == GrB_SUCCESS && ps.rows && burble.on) {
            static std::string note;                    // outlives the call's burble line (calls are serialised under GB_LOCK)
            note = "spgemm pull, " + std::to_string(ps.rows) + " rows" + (ps.dot ? " (GxB_AxB_DOT)" : " (auto)");
            burble.note(note.c_str(), burble.bytes);
        }
    }
    a_cast.reset(); b_cast.reset();
    return r;
}

extern "C" GrB_Info GrB_mxm(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const GrB_Semiring semiring,
                            const GrB_Matrix A, const GrB_Matrix B, const GrB_Descriptor desc) {
    GB_LOCK; GB_CHECK_INIT;
    if (!C || !semiring || !A || !B) return gb_fail(GrB_NULL_POINTER, nullptr, "GrB_mxm: NULL argument");
    if (!gb_valid_matrix(C) || !gb_valid_matrix(A) || !gb_valid_matrix(B) || (Mask && !gb_valid_matrix(Mask)) || semiring->magic != GB_MAGIC)
        return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "GrB_mxm: invalid object");
    std::string *err = &C->err;
    GB_TRY(gb_refuse_positional_accum(accum, "GrB_mxm"));
    GB_TRY(gb_refuse_user_with_positional(semiring, accum, "GrB_mxm"));
    if (gb_hyper_matrix(A) || gb_hyper_matrix(B) || gb_hyper_matrix(C)) return hyper_mxm(C, Mask, accum, semiring, A, B, desc);
    const DescFlags f = desc_flags(desc);
    const GrB_BinaryOp mulop = semiring->mul, addop = semiring->add->op;
    if (mulop->opcode == OP_USER || addop->opcode == OP_USER || (accum && accum->opcode == OP_USER))
        return gb_fail(GrB_INVALID_VALUE, err, "GrB_mxm: user-defined operators are host function pointers and cannot run on the GPU (no CPU fallback)");
    const uint64_t am = f.tran0 ? A->ncols : A->nrows, ak = f.tran0 ? A->nrows : A->ncols;
    const uint64_t bk = f.tran1 ? B->ncols : B->nrows, bn = f.tran1 ? B->nrows : B->ncols;
    if (ak != bk || C->nrows != am || C->ncols != bn || (Mask && (Mask->nrows != am || Mask->ncols != bn)))
        return gb_fail(GrB_DIMENSION_MISMATCH, err, "GrB_mxm: dimensions do not match (op(A) %llux%llu, op(B) %llux%llu, C %llux%llu)",
                       (unsigned long long)am, (unsigned long long)ak, (unsigned long long)bk, (unsigned long long)bn,
                       (unsigned long long)C->nrows, (unsigned long long)C->ncols);
    if (!G.have_device) return gb_fail(GrB_PANIC, err, "GrB_mxm: no CUDA device: libb200grb computes only on the GPU (no CPU fallback)");
    if (op_is_positional(mulop->opcode)) return positional_mxm(C, Mask, accum, semiring, A, B, f, nullptr, nullptr, nullptr);
    const int xt = mulop->xtype->code, zt = addop->ztype->code, add = addop->opcode, mul = mulop->opcode;
    GbBurble burble("GrB_mxm");
    G.last_kernel.clear();
    if (!Mask && f.mask_comp) return matrix_writeback(C, nullptr, accum, f, Csr(), zt, false, err);   // C<!NULL>: no product needed
    if (A->dn.valid && B->dn.valid && Mask && !f.mask_comp && !Mask->dn.valid) {                   // two dense operands under a sparse mask
        GB_TRY(matrix_ensure_device(Mask));
        return sddmm_mxm(C, Mask, accum, semiring, A, B, f, burble);
    }
    if (A->dn.valid && B->dn.valid && !A->dn.pres && !B->dn.pres && (bn == 0 || am <= (uint64_t)INT32_MAX / bn))
        return gemm_mxm(C, Mask, accum, semiring, A, B, f, burble);                                 // two full dense operands
    if (B->dn.valid && !f.tran1) return spmm_mxm(C, Mask, accum, semiring, A, B, f, burble);         // dense X: DESIGN.md section 3.6
    if (A->dn.valid && !B->dn.valid && op_mirror(mul) >= 0 && (bn == 0 || am <= (uint64_t)INT32_MAX / bn))
        return spmm_left_mxm(C, Mask, accum, semiring, A, B, f, burble);                            // dense X on the left
    Csr T; bool masked = false;
    GB_TRY(mxm_product(Mask, f, xt, zt, add, mul, A, B, MxmPos(), burble, T, &masked, err));
    return matrix_writeback(C, Mask, accum, f, std::move(T), zt, masked, err);
}

// C<Mask> = accum(C, op(A) (+).(x) op(B)) with a positional multiply (DESIGN.md section 3.5).  FIRSTJ / SECONDI give the inner index
// k: the values of op(A) become their column index and the call runs on (+).FIRST, or those of op(B) their row index with
// (+).SECOND, whichever operand has fewer entries.  FIRSTI / SECONDJ give the row i / column j of C: (+).PAIR in INT64 counts the
// products of every entry under the same mask, and one kernel turns each count into the fold of that many copies of i or j.
GrB_Info positional_mxm(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const GrB_Semiring s, const GrB_Matrix A,
                        const GrB_Matrix B, const DescFlags &f, const uint64_t *ids_m, const uint64_t *ids_k, const uint64_t *ids_n) {
    std::string *err = &C->err;
    const PosOp p = pos_binop(s->mul->opcode);
    const int zt = s->add->op->ztype->code, add = s->add->op->opcode;
    GbBurble burble("GrB_mxm");
    G.last_kernel.clear();
    if (!Mask && f.mask_comp) return matrix_writeback(C, nullptr, accum, f, Csr(), zt, false, err);   // C<!NULL>: no product needed
    Csr T; bool masked = false;
    if (p.second != p.col) {
        // ---- inner form: product = k (+ off)
        GB_TRY(matrix_ensure_device(A)); GB_TRY(matrix_ensure_device(B));
        MxmPos pos; pos.tc = zt; pos.off = p.off; pos.ids = ids_k;
        pos.side = A->dev.nnz <= B->dev.nnz ? 1 : 2;
        const int mul = pos.side == 1 ? OP_FIRST : OP_SECOND;
        GB_TRY(mxm_product(Mask, f, zt, zt, add, mul, A, B, pos, burble, T, &masked, err));
        gb_kernel_used("positional=inner");
        gb_kernel_used(pos.side == 1 ? "positional-operand=A" : "positional-operand=B");
        return matrix_writeback(C, Mask, accum, f, std::move(T), zt, masked, err);
    }
    // ---- count form: product = i (FIRSTI) or j (SECONDJ), + off
    const bool idem = add == OP_MIN || add == OP_MAX || add == OP_ANY;       // the count is not needed, only the pattern
    GB_TRY(mxm_product(Mask, f, TC_INT64, TC_INT64, idem ? OP_ANY : OP_PLUS, OP_PAIR, A, B, MxmPos(), burble, T, &masked, err));
    DevBuf<void> v;
    GB_TRY(v.alloc((size_t)T.nnz * tc_size(zt) + 16, err));
    GB_TRY(pos_csr_values(v, zt, (const int64_t *)T.val.get(), add, T, /*by_col=*/p.second, p.second ? ids_n : ids_m, p.off, err));
    T.val = std::move(v);
    gb_kernel_used("positional=count");
    return matrix_writeback(C, Mask, accum, f, std::move(T), zt, masked, err);
}

// C<M> = accum(C, A')  -- used by the reference around the hot path (Matrix.transpose,
// reference: pygraphblas/matrix.py:1003-1061; tests/test_matrix.py:299 `m.transpose().mxv(...)`)
extern "C" GrB_Info GrB_transpose(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const GrB_Matrix A, const GrB_Descriptor desc) {
    GB_LOCK; GB_CHECK_INIT;
    if (!C || !A) return gb_fail(GrB_NULL_POINTER, nullptr, "GrB_transpose: NULL argument");
    if (!gb_valid_matrix(C) || !gb_valid_matrix(A) || (Mask && !gb_valid_matrix(Mask))) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "GrB_transpose: invalid object");
    std::string *err = &C->err;
    const DescFlags f = desc_flags(desc);
    GB_TRY(gb_refuse_positional_accum(accum, "GrB_transpose"));
    if (accum && accum->opcode == OP_USER) return gb_fail(GrB_INVALID_VALUE, err, "GrB_transpose: user-defined accumulators cannot run on the GPU");
    const uint64_t tn = f.tran0 ? A->nrows : A->ncols, tm = f.tran0 ? A->ncols : A->nrows;
    if (C->nrows != tn || C->ncols != tm || (Mask && (Mask->nrows != tn || Mask->ncols != tm)))
        return gb_fail(GrB_DIMENSION_MISMATCH, err, "GrB_transpose: dimensions do not match");
    if (!G.have_device) return gb_fail(GrB_PANIC, err, "GrB_transpose: no CUDA device: libb200grb computes only on the GPU (no CPU fallback)");
    Csr *src; GB_TRY(source_csr(A, !f.tran0, &src));
    Csr T; GB_TRY(csr_copy(*src, A->type->size, true, T, err));      // a copy: C may alias A
    GB_TRY(dev_build_rowptr32(T, err));
    return matrix_writeback(C, Mask, accum, f, std::move(T), A->type->code, false, err);
}
