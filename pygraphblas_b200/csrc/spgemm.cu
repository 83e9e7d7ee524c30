// spgemm.cu -- GrB_mxm on sm_90a:  C<M> = accum(C, op(A) (+).(x) op(B))
//
// Replaces the SuiteSparse call behind reference: pygraphblas/matrix.py:2574
// (Matrix.mxm, `@`, `@=`, `**`).  Gustavson row-wise formulation, three methods:
//
//   unmasked    per-row flop count -> rows binned by flops -> symbolic pass (distinct
//               columns per row) -> scan -> numeric pass.  Small / medium rows use a hash
//               table in shared memory (atomicCAS probing), rows beyond the shared-memory
//               budget a dense accumulator in HBM owned by a persistent CTA.  Rows come out
//               sorted (in-smem bitonic sort / ordered bitmap sweep).
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
#include <algorithm>
#include <limits>
#include <type_traits>

static inline int grid_for(int64_t n, int threads = 256) {
    return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n, threads), (int64_t)G.num_sms * 16));
}

static constexpr uint32_t EMPTY_KEY = 0xFFFFFFFFu;

// ------------------------------------------------------------------ device helpers
template <typename T> __device__ __forceinline__ T gload(const T *p) {
    if constexpr (sizeof(T) == 1) { const unsigned char v = __ldg(reinterpret_cast<const unsigned char *>(p)); return reinterpret_cast<const T &>(v); }
    else return __ldg(p);
}

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

struct GemmArgs {
    const uint32_t *a_ptr, *a_col; const void *a_val;
    const uint32_t *b_ptr, *b_col; const void *b_val;
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

// ------------------------------------------------------------------ flop count + binning
__global__ void flops_kernel(const uint32_t *a_ptr, const uint32_t *a_col, const uint32_t *b_ptr, int64_t nrows,
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

// bins: 0 = nothing to do, 1 = warp/smem hash, 2 = CTA/smem hash, 3 = dense accumulator
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

// ------------------------------------------------------------------ unmasked: shared-memory hash
// One row per group (a warp, or the whole CTA).  Symbolic: count distinct columns.
template <bool WARP>
__global__ void __launch_bounds__(256) hash_symbolic_kernel(const GemmArgs p) {
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
        if (WARP) {       // lane per A entry, each lane walks its B row
            for (uint32_t pa = as + tid; pa < ae; pa += 32) {
                const uint32_t k = p.a_col[pa];
                for (uint32_t pb = p.b_ptr[k]; pb < p.b_ptr[k + 1]; ++pb) {
                    const uint32_t j = __ldg(p.b_col + pb);
                    uint32_t s = hash_col(j, hshift);
                    while (true) {
                        const uint32_t seen = atomicCAS(&keys[s], EMPTY_KEY, j);
                        if (seen == EMPTY_KEY) { ++mine; break; }
                        if (seen == j) break;
                        s = (s + 1) & tmask;
                    }
                }
            }
        } else {          // warp per A entry, lanes stride the B row
            const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
            for (uint32_t pa = as + warp; pa < ae; pa += nwarps) {
                const uint32_t k = p.a_col[pa];
                for (uint32_t pb = p.b_ptr[k] + lane; pb < p.b_ptr[k + 1]; pb += 32) {
                    const uint32_t j = __ldg(p.b_col + pb);
                    uint32_t s = hash_col(j, hshift);
                    while (true) {
                        const uint32_t seen = atomicCAS(&keys[s], EMPTY_KEY, j);
                        if (seen == EMPTY_KEY) { ++mine; break; }
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

// Numeric: packed[s] = (column << 32 | slot), vals[s] = accumulator.  After the products are in,
// the packed array is bitonic-sorted (empty keys sort last) and the first nnz entries written out.
template <typename XT, typename ZT, int ADD, int MUL, bool WARP>
__global__ void __launch_bounds__(256) hash_numeric_kernel(const GemmArgs p) {
    typedef typename SlotWord<ZT>::W W;
    extern __shared__ unsigned char smem_raw[];
    const int add = ADD >= 0 ? ADD : p.add_op;
    const int mul = MUL >= 0 ? MUL : p.mul_op;
    const int gsize = WARP ? 32 : blockDim.x;
    const int gid = WARP ? (threadIdx.x >> 5) : 0;
    const int tid = WARP ? (threadIdx.x & 31) : threadIdx.x;
    const int groups = WARP ? (blockDim.x >> 5) : 1;
    unsigned long long *packed = reinterpret_cast<unsigned long long *>(smem_raw) + (size_t)gid * p.table;
    W *vals = reinterpret_cast<W *>(smem_raw + (size_t)groups * p.table * 8) + (size_t)gid * p.table;
    const int64_t idx = (int64_t)blockIdx.x * groups + gid;
    const bool active = idx < p.nbin;
    const uint32_t tmask = (uint32_t)p.table - 1;
    const int hshift = __clz(p.table) + 1;                            // 32 - log2(table)
    const W ident = pack_slot<ZT>(accum_init<ZT>(add));
    for (int s = tid; s < p.table; s += gsize) { packed[s] = ((unsigned long long)EMPTY_KEY << 32) | (unsigned)s; vals[s] = ident; }
    group_sync<WARP>();
    const XT *aval = static_cast<const XT *>(p.a_val), *bval = static_cast<const XT *>(p.b_val);
    int64_t row = 0;
    if (active) {
        row = p.rows[idx];
        const uint32_t as = p.a_ptr[row], ae = p.a_ptr[row + 1];
        auto insert = [&](uint32_t j, ZT prod) {
            uint32_t s = hash_col(j, hshift);
            while (true) {
                uint32_t *kp = reinterpret_cast<uint32_t *>(&packed[s]) + 1;   // high word = key
                const uint32_t seen = atomicCAS(kp, EMPTY_KEY, j);
                if (seen == EMPTY_KEY || seen == j) break;
                s = (s + 1) & tmask;
            }
            atomic_combine<ZT>(&vals[s], prod, add);
        };
        if (WARP) {
            for (uint32_t pa = as + tid; pa < ae; pa += 32) {
                const uint32_t k = p.a_col[pa];
                const XT av = p.need_a ? gload<XT>(aval + pa) : (XT)1;
                for (uint32_t pb = p.b_ptr[k]; pb < p.b_ptr[k + 1]; ++pb) {
                    const XT bv = p.need_b ? gload<XT>(bval + pb) : (XT)1;
                    insert(__ldg(p.b_col + pb), MulApply<XT, ZT>::f(mul, av, bv));
                }
            }
        } else {
            const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
            for (uint32_t pa = as + warp; pa < ae; pa += nwarps) {
                const uint32_t k = p.a_col[pa];
                const XT av = p.need_a ? gload<XT>(aval + pa) : (XT)1;
                for (uint32_t pb = p.b_ptr[k] + lane; pb < p.b_ptr[k + 1]; pb += 32) {
                    const XT bv = p.need_b ? gload<XT>(bval + pb) : (XT)1;
                    insert(__ldg(p.b_col + pb), MulApply<XT, ZT>::f(mul, av, bv));
                }
            }
        }
    }
    group_sync<WARP>();
    bitonic_sort_u64<WARP>(packed, p.table, tid, gsize);
    if (active) {
        const int64_t base = p.c_ptr[row];
        const int n = (int)(p.c_ptr[row + 1] - base);
        ZT *cval = static_cast<ZT *>(p.c_val);
        for (int k = tid; k < n; k += gsize) {
            const unsigned long long e = packed[k];
            p.c_col[base + k] = (uint32_t)(e >> 32);
            cval[base + k] = unpack_slot<ZT>(vals[(uint32_t)e]);
        }
    }
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
// The numeric pass of the two shared-memory bins without a hash table.  The products of a row are EXPANDED into shared memory in
// their Gustavson order (key = column << 32 | position, the value stays at its position), the keys are SORTED by a bitonic
// network over the next power of two of the row's OWN product count (the hash path sorts its whole table -- 256 or 4096 slots --
// whatever the row holds), and equal columns are COMPRESSED by folding their values in position order.  No atomics and no table
// to clear; a floating-point PLUS monoid gives the same bit pattern on every run (the hash path adds in arrival order).  One
// warp per row of the small bin (<= 128 products), one CTA per row of the medium bin (<= 2048).  The row's output count comes
// from the symbolic pass (c_ptr), as for the hash kernels.
static constexpr int ESC_SMALL = 128, ESC_MEDIUM = 2048;
static constexpr size_t ESC_SMEM_SMALL = (size_t)8 * ESC_SMALL * 16;                       // 8 warps x (keys 8 B + value words 8 B)
static constexpr size_t ESC_SMEM_MEDIUM = (size_t)ESC_MEDIUM * 16 + 3 * 256 * 4 + 256 * 8;   // + offsets, starts, lengths, A values of a chunk

template <typename XT, typename ZT, int ADD, int MUL, bool WARP>
__global__ void __launch_bounds__(256) esc_numeric_kernel(const GemmArgs p) {
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
            uint32_t bs = 0, len = 0; XT av = (XT)1;
            if (pa < ae) {
                const uint32_t k = p.a_col[pa];
                bs = p.b_ptr[k]; len = p.b_ptr[k + 1] - bs;
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
        uint32_t *s_bs = s_off + 256, *s_len = s_bs + 256;
        XT *s_av = reinterpret_cast<XT *>(s_len + 256);
        for (uint32_t pa0 = as; pa0 < ae; pa0 += 256) {         // a thread per A entry of the chunk, then a warp per entry, lanes along its B row
            const uint32_t pa = pa0 + threadIdx.x;
            uint32_t bs = 0, len = 0; XT av = (XT)1;
            if (pa < ae) {
                const uint32_t k = p.a_col[pa];
                bs = p.b_ptr[k]; len = p.b_ptr[k + 1] - bs;
                if (p.need_a) av = gload<XT>(aval + pa);
            }
            int total = 0;
            const int off = block_exclusive_scan((int)len, s_warp, &total);
            s_off[threadIdx.x] = (uint32_t)(F + off); s_bs[threadIdx.x] = bs; s_len[threadIdx.x] = len; s_av[threadIdx.x] = av;
            __syncthreads();
            const int nent = (int)min(256u, ae - pa0);
            for (int e = warp; e < nent; e += nwarps) {
                const uint32_t o = s_off[e], b0 = s_bs[e], l = s_len[e];
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
        const bool head = valid && (i == 0 || (uint32_t)(keys[i - 1] >> 32) != col);
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

template <typename XT, typename ZT, int ADD, int MUL, bool NUMERIC>
__global__ void __launch_bounds__(512) spa_kernel(const GemmArgs p) {
    typedef typename SlotWord<ZT>::W W;
    __shared__ int s_warp[33];
    __shared__ unsigned int s_next;
    const int add = ADD >= 0 ? ADD : p.add_op;
    const int mul = MUL >= 0 ? MUL : p.mul_op;
    uint32_t *bits = p.spa_bits + (size_t)blockIdx.x * p.spa_words;
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
        for (uint32_t pa = as + warp; pa < ae; pa += nwarps) {
            const uint32_t k = p.a_col[pa];
            XT av = (XT)1;
            if (NUMERIC && p.need_a) av = gload<XT>(aval + pa);
            for (uint32_t pb = p.b_ptr[k] + lane; pb < p.b_ptr[k + 1]; pb += 32) {
                const uint32_t j = __ldg(p.b_col + pb);
                const uint32_t bit = 1u << (j & 31);
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

template <typename W> __global__ void fill_words_kernel(W *a, W v, int64_t n) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) a[k] = v;
}

// ------------------------------------------------------------------ masked: shared-memory hash of the mask row
// Rows whose products and mask row are both short (the warp class): one warp per row hashes the mask row M(i,:)
// (keys -> position inside the row), then streams the B rows named by A(i,:) and accumulates the products that hit it.
// The warp handles 32 A entries at a time: each lane fetches one (k, B row range) up front, the ranges are broadcast by
// shuffle and the lanes stride the B row -- the dependent-load chain per A entry is paid once per 32 entries.
// Heavier rows are cut into chunks and go to the streaming kernel (spgemm_stream.cuh).
struct MaskedArgs {
    GemmArgs g;
    void *t_words;     // nnz(M) accumulator words
};

template <typename XT, typename ZT, typename Hit>
__device__ __forceinline__ void stream_b_rows(const GemmArgs &p, uint32_t pa0, uint32_t pa1, int lane, Hit &&hit) {
    const XT *aval = static_cast<const XT *>(p.a_val);
    for (uint32_t base = pa0; base < pa1; base += 32) {
        const uint32_t pa = base + lane;
        const bool valid = pa < pa1;
        const uint32_t k = valid ? __ldg(p.a_col + pa) : 0u;
        const uint32_t bs = valid ? __ldg(p.b_ptr + k) : 0u, be = valid ? __ldg(p.b_ptr + k + 1) : 0u;
        XT av = (XT)1;
        if (p.need_a && valid) av = gload<XT>(aval + pa);
        const int cnt = min(32u, pa1 - base);
        for (int l = 0; l < cnt; ++l) {
            const uint32_t s = __shfl_sync(0xffffffffu, bs, l), e = __shfl_sync(0xffffffffu, be, l);
            XT a;
            if constexpr (sizeof(XT) == 8) { long long t = __shfl_sync(0xffffffffu, reinterpret_cast<long long &>(av), l); a = reinterpret_cast<XT &>(t); }
            else if constexpr (sizeof(XT) == 4) { int t = __shfl_sync(0xffffffffu, reinterpret_cast<int &>(av), l); a = reinterpret_cast<XT &>(t); }
            else { int t = __shfl_sync(0xffffffffu, (int)av, l); a = (XT)t; }
            for (uint32_t pb = s + lane; pb < e; pb += 32) hit(__ldg(p.b_col + pb), a, pb);
        }
    }
}

template <typename XT, typename ZT, int ADD, int MUL>
__global__ void __launch_bounds__(256) masked_hash_kernel(const MaskedArgs ma) {
    typedef typename SlotWord<ZT>::W W;
    const GemmArgs &p = ma.g;
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
    auto hit = [&](uint32_t j, XT av, uint32_t pb) {
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
    stream_b_rows<XT, ZT>(p, p.a_ptr[row], p.a_ptr[row + 1], lane, hit);
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
template <typename XT, typename ZT, int ADD, int MUL>
__global__ void __launch_bounds__(256) masked_dot_kernel(const GemmArgs p) {
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
                uint32_t x = as, y = p.b_ptr[j]; const uint32_t ye = p.b_ptr[j + 1];
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
__global__ void row_found_count_kernel(const uint32_t *m_ptr, const uint8_t *found, int64_t nrows, int64_t *cnt) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < nrows; r += nwarps) {
        int c = 0;
        for (uint32_t q = m_ptr[r] + lane; q < m_ptr[r + 1]; q += 32) c += found[q] != 0;
        for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
        if (lane == 0) cnt[r] = c;
    }
}
__global__ void row_found_fill_kernel(const uint32_t *m_ptr, const uint32_t *m_col, const uint8_t *found, const uint8_t *tval, int vsize,
                                      int64_t nrows, const int64_t *c_ptr, uint32_t *c_col, uint8_t *c_val) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < nrows; r += nwarps) {
        int64_t out = c_ptr[r];
        for (uint32_t q0 = m_ptr[r]; q0 < m_ptr[r + 1]; q0 += 32) {
            const uint32_t q = q0 + lane;
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
static GrB_Info read_i64(const int64_t *d, int64_t *h, std::string *err) {
    CU_TRY(cudaMemcpyAsync(h, d, 8, cudaMemcpyDeviceToHost, G.stream), err);
    CU_TRY(cudaStreamSynchronize(G.stream), err);
    return GrB_SUCCESS;
}

static bool op_uses_x(int op) { return !(op == OP_SECOND || op == OP_PAIR); }
static bool op_uses_y(int op) { return !(op == OP_FIRST || op == OP_PAIR || op == OP_ANY); }

static constexpr int SMALL_TABLE = 256, SMALL_FLOPS = 128;      // warp per row
static constexpr int MEDIUM_TABLE = 4096, MEDIUM_FLOPS = 2048;  // CTA per row
static constexpr int MIDSMALL_TABLE = 1024;                       // masked: CTA per chunk, mask rows up to 512 entries

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
            else switch (xt) {                                                                                 \
                case TC_BOOL: KERNEL(bool, bool, -1, -1); done_ = true; break;                                 \
                case TC_INT8: KERNEL(int8_t, int8_t, -1, -1); done_ = true; break;                             \
                case TC_INT16: KERNEL(int16_t, int16_t, -1, -1); done_ = true; break;                          \
                case TC_INT32: KERNEL(int32_t, int32_t, -1, -1); done_ = true; break;                          \
                case TC_INT64: KERNEL(int64_t, int64_t, -1, -1); done_ = true; break;                          \
                case TC_UINT8: KERNEL(uint8_t, uint8_t, -1, -1); done_ = true; break;                          \
                case TC_UINT16: KERNEL(uint16_t, uint16_t, -1, -1); done_ = true; break;                       \
                case TC_UINT32: KERNEL(uint32_t, uint32_t, -1, -1); done_ = true; break;                       \
                case TC_UINT64: KERNEL(uint64_t, uint64_t, -1, -1); done_ = true; break;                       \
                case TC_FP32: KERNEL(float, float, -1, -1); done_ = true; break;                               \
                case TC_FP64: KERNEL(double, double, -1, -1); done_ = true; break;                             \
            }                                                                                                  \
        } else if (zt == TC_BOOL) switch (xt) {                                                                \
            case TC_INT8: KERNEL(int8_t, bool, -1, -1); done_ = true; break;                                   \
            case TC_INT16: KERNEL(int16_t, bool, -1, -1); done_ = true; break;                                 \
            case TC_INT32: KERNEL(int32_t, bool, -1, -1); done_ = true; break;                                 \
            case TC_INT64: KERNEL(int64_t, bool, -1, -1); done_ = true; break;                                 \
            case TC_UINT8: KERNEL(uint8_t, bool, -1, -1); done_ = true; break;                                 \
            case TC_UINT16: KERNEL(uint16_t, bool, -1, -1); done_ = true; break;                               \
            case TC_UINT32: KERNEL(uint32_t, bool, -1, -1); done_ = true; break;                               \
            case TC_UINT64: KERNEL(uint64_t, bool, -1, -1); done_ = true; break;                               \
            case TC_FP32: KERNEL(float, bool, -1, -1); done_ = true; break;                                    \
            case TC_FP64: KERNEL(double, bool, -1, -1); done_ = true; break;                                   \
        }                                                                                                      \
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

static size_t numeric_smem(int table, int groups, size_t wsize) { return (size_t)groups * table * (8 + wsize); }
static size_t masked_smem(int table, int groups, size_t wsize) {
    const size_t per = (size_t)table * 8 + (size_t)(table / 2) * wsize + (size_t)(table / 2);
    return (size_t)groups * ((per + 15) & ~(size_t)15);
}

// T = A (+).(x) B, unmasked.  A and B values already of the multiply's operand type.
static GrB_Info spgemm_unmasked(const Csr &A, const Csr &B, const void *aval, const void *bval, int xt, int zt,
                                int add, int mul, bool need_a, bool need_b, Csr &T, std::string *err) {
    const int64_t nrows = A.nrows, ncols = B.ncols;
    T = Csr(); T.nrows = nrows; T.ncols = ncols;
    GB_TRY(T.rowptr.alloc((size_t)nrows + 1, err));
    CU_TRY(cudaMemsetAsync(T.rowptr, 0, ((size_t)nrows + 1) * 8, G.stream), err);
    DevBuf<int64_t> flops; DevBuf<unsigned long long> total;
    GB_TRY(flops.alloc((size_t)nrows, err)); GB_TRY(total.alloc(1, err));
    CU_TRY(cudaMemsetAsync(total, 0, 8, G.stream), err);
    flops_kernel<<<grid_for(nrows * 32), 256, 0, G.stream>>>(A.rowptr32, A.col, B.rowptr32, nrows, flops, total); GB_LAUNCHED();
    RowBins bins;
    GB_TRY(make_bins(flops, nrows, BinLimits{SMALL_FLOPS, MEDIUM_FLOPS}, bins, err));
    int64_t total_flops = 0; GB_TRY(read_i64((const int64_t *)total, &total_flops, err));
    G.last_flops = (uint64_t)total_flops;
    flops.reset(); total.reset();

    GemmArgs g{};
    g.a_ptr = A.rowptr32; g.a_col = A.col; g.a_val = aval; g.b_ptr = B.rowptr32; g.b_col = B.col; g.b_val = bval;
    g.nrows = nrows; g.ncols = ncols; g.add_op = add; g.mul_op = mul; g.need_a = need_a; g.need_b = need_b;
    g.c_cnt = T.rowptr;
    const size_t wsize = tc_size(zt) == 8 ? 8 : 4;
    const int spa_ctas = std::max(1, std::min<int>((int)bins.count[3], G.num_sms * 2));
    DevBuf<unsigned int> queue; DevBuf<uint32_t> spa_bits;
    if (bins.count[3]) {
        g.spa_words = ceil_div(ncols, 32);
        GB_TRY(spa_bits.alloc((size_t)spa_ctas * g.spa_words, err));
        g.spa_bits = spa_bits;
        CU_TRY(cudaMemsetAsync(g.spa_bits, 0, (size_t)spa_ctas * g.spa_words * 4, G.stream), err);
        GB_TRY(queue.alloc(2, err));
        CU_TRY(cudaMemsetAsync(queue, 0, 8, G.stream), err);
    }
    // ---- symbolic
    if (bins.count[1]) {
        g.rows = bins.rows + bins.offset[1]; g.nbin = bins.count[1]; g.table = SMALL_TABLE;
        hash_symbolic_kernel<true><<<(unsigned)ceil_div(g.nbin, 8), 256, 8 * SMALL_TABLE * 4, G.stream>>>(g); GB_LAUNCHED();
    }
    if (bins.count[2]) {
        g.rows = bins.rows + bins.offset[2]; g.nbin = bins.count[2]; g.table = MEDIUM_TABLE;
        hash_symbolic_kernel<false><<<(unsigned)g.nbin, 256, MEDIUM_TABLE * 4, G.stream>>>(g); GB_LAUNCHED();
    }
    if (bins.count[3]) {
        g.rows = bins.rows + bins.offset[3]; g.nbin = bins.count[3]; g.queue = queue;
        spa_kernel<bool, bool, -1, -1, false><<<spa_ctas, 512, 0, G.stream>>>(g); GB_LAUNCHED();
    }
    GB_TRY(dev_exclusive_scan(T.rowptr, nrows + 1, err));
    int64_t nnz = 0; GB_TRY(read_i64(T.rowptr + nrows, &nnz, err));
    T.nnz = nnz; G.last_nnz_out = (uint64_t)nnz;
    GB_TRY(T.col.alloc((size_t)nnz, err));
    GB_TRY(T.val.alloc((size_t)nnz * tc_size(zt) + 16, err));
    g.c_ptr = T.rowptr; g.c_col = T.col; g.c_val = T.val;
    // ---- numeric (shared-memory bins: expand-sort-compress unless B200GRB_SPGEMM_ESC=0 selects the hash kernels)
    const bool esc = tunables().spgemm_esc;
    if (bins.count[1]) {
        g.rows = bins.rows + bins.offset[1]; g.nbin = bins.count[1]; g.table = SMALL_TABLE;
        const size_t sm = numeric_smem(SMALL_TABLE, 8, wsize);
#define K_SMALL(XT, ZT, A_, M_) hash_numeric_kernel<XT, ZT, A_, M_, true><<<(unsigned)ceil_div(g.nbin, 8), 256, sm, G.stream>>>(g)
#define K_ESC_SMALL(XT, ZT, A_, M_) esc_numeric_kernel<XT, ZT, A_, M_, true><<<(unsigned)ceil_div(g.nbin, 8), 256, ESC_SMEM_SMALL, G.stream>>>(g)
        if (esc) GB_FOR_SEMIRING(xt, zt, add, mul, K_ESC_SMALL, err); else GB_FOR_SEMIRING(xt, zt, add, mul, K_SMALL, err);
        GB_LAUNCHED(); gb_kernel_used(esc ? "esc-small" : "hash-small");
    }
    if (bins.count[2]) {
        g.rows = bins.rows + bins.offset[2]; g.nbin = bins.count[2]; g.table = MEDIUM_TABLE;
        const size_t sm = numeric_smem(MEDIUM_TABLE, 1, wsize);
#define K_MEDIUM(XT, ZT, A_, M_) do { \
        cudaFuncSetAttribute(hash_numeric_kernel<XT, ZT, A_, M_, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm); \
        hash_numeric_kernel<XT, ZT, A_, M_, false><<<(unsigned)g.nbin, 256, sm, G.stream>>>(g); } while (0)
#define K_ESC_MEDIUM(XT, ZT, A_, M_) esc_numeric_kernel<XT, ZT, A_, M_, false><<<(unsigned)g.nbin, 256, ESC_SMEM_MEDIUM, G.stream>>>(g)
        if (esc) GB_FOR_SEMIRING(xt, zt, add, mul, K_ESC_MEDIUM, err); else GB_FOR_SEMIRING(xt, zt, add, mul, K_MEDIUM, err);
        GB_LAUNCHED(); gb_kernel_used(esc ? "esc-medium" : "hash-medium");
    }
    if (bins.count[3]) {
        g.rows = bins.rows + bins.offset[3]; g.nbin = bins.count[3]; g.queue = queue + 1;
        DevBuf<void> spa_val;
        GB_TRY(spa_val.alloc((size_t)spa_ctas * ncols * wsize + 16, err));
        g.spa_val = spa_val;
#define K_SPA(XT, ZT, A_, M_) do { \
        fill_accum_init<ZT>(g.spa_val, (int64_t)spa_ctas * ncols, (A_) >= 0 ? (A_) : add); \
        spa_kernel<XT, ZT, A_, M_, true><<<spa_ctas, 512, 0, G.stream>>>(g); } while (0)
        GB_FOR_SEMIRING(xt, zt, add, mul, K_SPA, err); G.launches += 2; gb_kernel_used("spa");
    }
    spa_bits.reset(); queue.reset(); bins.rows.reset();
    GB_TRY(dev_build_rowptr32(T, err));
    CU_TRY(cudaGetLastError(), err);
    return GrB_SUCCESS;
}

// T<M> = A (+).(x) B restricted to a non-complemented mask M (pattern of T is a subset of M's).
// dot == true computes A (+).(x) B' by row intersections instead (B given un-transposed).
static constexpr int64_t CHUNK_FLOPS = 32768;     // flop budget of one CTA-level work unit
static constexpr int WARP_FLOPS = 2048;           // rows at most this heavy (and with short mask rows) run warp-per-row

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

static GrB_Info spgemm_masked(const Csr &A, const Csr &B, const void *aval, const void *bval, int xt, int zt,
                              int add, int mul, bool need_a, bool need_b, const Csr &M, int mtc, bool m_struct,
                              bool dot, Csr &T, std::string *err) {
    const int64_t nrows = A.nrows, ncols = dot ? B.nrows : B.ncols;
    T = Csr(); T.nrows = nrows; T.ncols = ncols;
    const size_t zsz = (size_t)tc_size(zt), wsize = zsz == 8 ? 8 : 4;
    MaskedArgs ma{};
    GemmArgs &g = ma.g;
    g.a_ptr = A.rowptr32; g.a_col = A.col; g.a_val = aval; g.b_ptr = B.rowptr32; g.b_col = B.col; g.b_val = bval;
    g.m_ptr = M.rowptr32; g.m_col = M.col; g.m_val = M.val; g.m_tc = mtc; g.m_struct = m_struct;
    g.nrows = nrows; g.ncols = ncols; g.add_op = add; g.mul_op = mul; g.need_a = need_a; g.need_b = need_b;
    PhaseTrace trace;
    DevBuf<void> typed;                                        // 1- and 2-byte types: the accumulator words narrowed
    void *words = nullptr; uint8_t *found = nullptr;          // per mask entry: accumulator word, "has a value"
    GB_TRY(ws_get(WS_WORDS, &words, (size_t)M.nnz * wsize + 16, err));
    GB_TRY(ws_get(WS_FOUND, (void **)&found, (size_t)M.nnz + 16, err));
    g.c_val = words; g.t_found = found; ma.t_words = words;
    G.last_flops = 0;
    if (M.nnz > 0 && dot) {
        // the dot kernel writes typed values directly
#define K_DOT(XT, ZT, A_, M_) masked_dot_kernel<XT, ZT, A_, M_><<<grid_for(nrows * 32), 256, 0, G.stream>>>(g)
        GB_FOR_SEMIRING(xt, zt, add, mul, K_DOT, err); GB_LAUNCHED(); gb_kernel_used("dot");
    } else if (M.nnz > 0) {
        int64_t *flops = nullptr; unsigned long long *total = nullptr;
        GB_TRY(ws_array(WS_FLOPS, &flops, (size_t)nrows, err)); GB_TRY(ws_array(WS_TOTAL, &total, 1, err));
        CU_TRY(cudaMemsetAsync(total, 0, 8, G.stream), err);
        flops_kernel<<<grid_for(nrows * 32), 256, 0, G.stream>>>(A.rowptr32, A.col, B.rowptr32, nrows, flops, total); GB_LAUNCHED();
        // accumulators start at accum_init, flags at 0
        CU_TRY(cudaMemsetAsync(found, 0, (size_t)M.nnz, G.stream), err);
#define K_IDENT(XT, ZT, A_, M_) fill_accum_init<ZT>(words, M.nnz, (A_) >= 0 ? (A_) : add)
        GB_FOR_SEMIRING(xt, zt, add, mul, K_IDENT, err); GB_LAUNCHED();
        // classify rows and cut heavy ones into flop-bounded chunks
        int64_t *cs = nullptr, *cm = nullptr, *cl = nullptr, *c1 = nullptr;
        GB_TRY(ws_array(WS_CS, &cs, (size_t)nrows + 1, err));
        GB_TRY(ws_array(WS_CM, &cm, (size_t)nrows + 1, err)); GB_TRY(ws_array(WS_CL, &cl, (size_t)nrows + 1, err)); GB_TRY(ws_array(WS_C1, &c1, (size_t)nrows + 1, err));
        CU_TRY(cudaMemsetAsync(cs + nrows, 0, 8, G.stream), err);
        CU_TRY(cudaMemsetAsync(cm + nrows, 0, 8, G.stream), err); CU_TRY(cudaMemsetAsync(cl + nrows, 0, 8, G.stream), err);
        CU_TRY(cudaMemsetAsync(c1 + nrows, 0, 8, G.stream), err);
        chunk_count_kernel<<<grid_for(nrows), 256, 0, G.stream>>>(flops, M.rowptr32, nrows, CHUNK_FLOPS, WARP_FLOPS, SMALL_TABLE / 2,
                                                                  MIDSMALL_TABLE / 2, MEDIUM_TABLE / 2, cs, cm, cl, c1); GB_LAUNCHED();
        GB_TRY(dev_exclusive_scan(cs, nrows + 1, err));
        GB_TRY(dev_exclusive_scan(cm, nrows + 1, err)); GB_TRY(dev_exclusive_scan(cl, nrows + 1, err)); GB_TRY(dev_exclusive_scan(c1, nrows + 1, err));
        int64_t n_small = 0, n_medium = 0, n_long = 0, n_warp = 0, tf = 0;
        GB_TRY(read_i64(cs + nrows, &n_small, err));
        GB_TRY(read_i64(cm + nrows, &n_medium, err)); GB_TRY(read_i64(cl + nrows, &n_long, err)); GB_TRY(read_i64(c1 + nrows, &n_warp, err));
        GB_TRY(read_i64((const int64_t *)total, &tf, err));
        G.last_flops = (uint64_t)tf;
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
#define K_MSMALL(XT, ZT, A_, M_) masked_hash_kernel<XT, ZT, A_, M_><<<(unsigned)ceil_div(n_warp, 8), 256, sm, G.stream>>>(ma)
            GB_FOR_SEMIRING(xt, zt, add, mul, K_MSMALL, err); GB_LAUNCHED(); gb_kernel_used("masked-warp");
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
            StreamArgs sa{}; sa.g = g; sa.t_words = words;
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
                const size_t sm = sm_var + stream_fixed_smem<XT>(nt); \
                auto kern = masked_stream_kernel<XT, ZT, A_, M_>; \
                cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm); \
                int ctas = ctas_big; \
                if (!big) { int per_sm = 1; cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, 256, sm); \
                            ctas = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(sa.nchunks, sa.grab), (int64_t)G.num_sms * std::max(per_sm, 1))); } \
                kern<<<ctas, nt, sm, G.stream>>>(sa); } while (0)
                GB_FOR_SEMIRING(xt, zt, add, mul, K_MSTREAM, err); GB_LAUNCHED();
                gb_kernel_used(k == 0 ? "stream-S" : (k == 1 ? "stream-M" : "stream-L"));
                gb_kernel_used(sa.exact ? "filter=exact" : "filter=bloom");
                trace.mark(k == 0 ? "stream S" : (k == 1 ? "stream M" : "stream L"));
            }
        }
        if (zsz < 4) {      // narrow 32-bit accumulator words to the 1- or 2-byte type, in a second buffer
            GB_TRY(typed.alloc((size_t)M.nnz * zsz + 16, err));
            narrow_words_kernel<<<grid_for(M.nnz), 256, 0, G.stream>>>((const uint32_t *)words, (uint8_t *)typed, (int)zsz, M.nnz); GB_LAUNCHED();
            words = typed;
        }
    }
    void *tval = words;
    // compact (pattern of M, found) -> CSR
    GB_TRY(T.rowptr.alloc((size_t)nrows + 1, err));
    CU_TRY(cudaMemsetAsync(T.rowptr, 0, ((size_t)nrows + 1) * 8, G.stream), err);
    if (M.nnz > 0) { row_found_count_kernel<<<grid_for(nrows * 32), 256, 0, G.stream>>>(M.rowptr32, found, nrows, T.rowptr); GB_LAUNCHED(); }
    GB_TRY(dev_exclusive_scan(T.rowptr, nrows + 1, err));
    int64_t nnz = 0; GB_TRY(read_i64(T.rowptr + nrows, &nnz, err));
    T.nnz = nnz; G.last_nnz_out = (uint64_t)nnz;
    GB_TRY(T.col.alloc((size_t)nnz, err));
    GB_TRY(T.val.alloc((size_t)nnz * zsz + 16, err));
    if (nnz > 0) {
        row_found_fill_kernel<<<grid_for(nrows * 32), 256, 0, G.stream>>>(M.rowptr32, M.col, found, (const uint8_t *)tval, (int)zsz,
                                                                          nrows, T.rowptr, T.col, (uint8_t *)T.val); GB_LAUNCHED();
    }
    typed.reset();
    GB_TRY(dev_build_rowptr32(T, err));
    trace.mark("compaction");
    CU_TRY(cudaGetLastError(), err);
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
    out = Csr(); out.nrows = T.nrows; out.ncols = T.ncols;
    GB_TRY(out.rowptr.alloc((size_t)nrows + 1, err));
    CU_TRY(cudaMemsetAsync(out.rowptr, 0, ((size_t)nrows + 1) * 8, G.stream), err);
    a.o_cnt = out.rowptr;
    mat_finalize_kernel<false><<<grid_for(nrows, 128), 128, 0, G.stream>>>(a); GB_LAUNCHED();
    GB_TRY(dev_exclusive_scan(out.rowptr, nrows + 1, err));
    int64_t nnz = 0; GB_TRY(read_i64(out.rowptr + nrows, &nnz, err));
    out.nnz = nnz;
    GB_TRY(out.col.alloc((size_t)nnz, err));
    GB_TRY(out.val.alloc((size_t)nnz * tc_size(ctc) + 16, err));
    a.o_ptr = out.rowptr; a.o_col = out.col; a.o_val = out.val;
    if (nnz > 0) { mat_finalize_kernel<true><<<grid_for(nrows, 128), 128, 0, G.stream>>>(a); GB_LAUNCHED(); }
    GB_TRY(dev_build_rowptr32(out, err));
    CU_TRY(cudaGetLastError(), err);
    return GrB_SUCCESS;
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
    const bool c_empty = C->host_valid ? (C->hi.empty() && C->pi.empty()) : (C->dev.nnz == 0);
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

extern "C" GrB_Info GrB_mxm(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const GrB_Semiring semiring,
                            const GrB_Matrix A, const GrB_Matrix B, const GrB_Descriptor desc) {
    GB_LOCK; GB_CHECK_INIT;
    if (!C || !semiring || !A || !B) return gb_fail(GrB_NULL_POINTER, nullptr, "GrB_mxm: NULL argument");
    if (!gb_valid_matrix(C) || !gb_valid_matrix(A) || !gb_valid_matrix(B) || (Mask && !gb_valid_matrix(Mask)) || semiring->magic != GB_MAGIC)
        return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "GrB_mxm: invalid object");
    std::string *err = &C->err;
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
    const int xt = mulop->xtype->code, zt = addop->ztype->code, add = addop->opcode, mul = mulop->opcode;
    const bool need_a = op_uses_x(mul), need_b = op_uses_y(mul);
    GbBurble burble("GrB_mxm");
    G.last_kernel.clear();
    if (!Mask && f.mask_comp) return matrix_writeback(C, nullptr, accum, f, Csr(), zt, false, err);   // C<!NULL>: no product needed

    // masked methods apply to non-complemented masks
    const bool use_mask = Mask && !f.mask_comp;
    if (f.tran0) GB_TRY(matrix_ensure_transpose(A)); else GB_TRY(matrix_ensure_device(A));
    GB_TRY(matrix_ensure_device(B));
    // C<M> = A*B': small problems intersect rows of A and B directly (no transpose); large ones
    // go through the cached transpose and the load-balanced masked hash kernels
    const bool dot = use_mask && f.tran1 && B->dev.nnz < ((int64_t)1 << 18);
    if (f.tran1 && !dot) GB_TRY(matrix_ensure_transpose(B));
    if (Mask) GB_TRY(matrix_ensure_device(Mask));
    const Csr &a = f.tran0 ? A->devT : A->dev;
    const Csr &b = (f.tran1 && !dot) ? B->devT : B->dev;
    if (!a.rowptr32 || !b.rowptr32 || (Mask && !Mask->dev.rowptr32))
        return gb_fail(GrB_INVALID_VALUE, err, "GrB_mxm: operands with >= 2^32 entries are not supported");

    DevBuf<void> a_cast, b_cast;
    const void *aval = a.val, *bval = b.val;
    if (need_a && A->type->code != xt) { GB_TRY(dev_cast_values(a_cast, xt, a.val, A->type->code, a.nnz, err)); aval = a_cast; }
    if (need_b && B->type->code != xt) { GB_TRY(dev_cast_values(b_cast, xt, b.val, B->type->code, b.nnz, err)); bval = b_cast; }

    Csr T; GrB_Info r;
    if (use_mask) r = spgemm_masked(a, b, aval, bval, xt, zt, add, mul, need_a, need_b, Mask->dev, Mask->type->code, f.mask_struct, dot, T, err);
    else r = spgemm_unmasked(a, b, aval, bval, xt, zt, add, mul, need_a, need_b, T, err);
    a_cast.reset(); b_cast.reset();
    if (r != GrB_SUCCESS) return r;
    return matrix_writeback(C, Mask, accum, f, std::move(T), zt, use_mask, err);
}

// C<M> = accum(C, A')  -- used by the reference around the hot path (Matrix.transpose,
// reference: pygraphblas/matrix.py:1003-1061; tests/test_matrix.py:299 `m.transpose().mxv(...)`)
extern "C" GrB_Info GrB_transpose(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const GrB_Matrix A, const GrB_Descriptor desc) {
    GB_LOCK; GB_CHECK_INIT;
    if (!C || !A) return gb_fail(GrB_NULL_POINTER, nullptr, "GrB_transpose: NULL argument");
    if (!gb_valid_matrix(C) || !gb_valid_matrix(A) || (Mask && !gb_valid_matrix(Mask))) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "GrB_transpose: invalid object");
    std::string *err = &C->err;
    const DescFlags f = desc_flags(desc);
    if (accum && accum->opcode == OP_USER) return gb_fail(GrB_INVALID_VALUE, err, "GrB_transpose: user-defined accumulators cannot run on the GPU");
    const uint64_t tn = f.tran0 ? A->nrows : A->ncols, tm = f.tran0 ? A->ncols : A->nrows;
    if (C->nrows != tn || C->ncols != tm || (Mask && (Mask->nrows != tn || Mask->ncols != tm)))
        return gb_fail(GrB_DIMENSION_MISMATCH, err, "GrB_transpose: dimensions do not match");
    if (!G.have_device) return gb_fail(GrB_PANIC, err, "GrB_transpose: no CUDA device: libb200grb computes only on the GPU (no CPU fallback)");
    if (f.tran0) GB_TRY(matrix_ensure_device(A)); else GB_TRY(matrix_ensure_transpose(A));
    const Csr &src = f.tran0 ? A->dev : A->devT;
    // T = copy of src (C may alias A)
    Csr T; T.nrows = src.nrows; T.ncols = src.ncols; T.nnz = src.nnz;
    const size_t sz = A->type->size;
    GB_TRY(T.rowptr.alloc((size_t)src.nrows + 1, err));
    GB_TRY(T.col.alloc((size_t)src.nnz, err));
    GB_TRY(T.val.alloc((size_t)src.nnz * sz + 16, err));
    CU_TRY(cudaMemcpyAsync(T.rowptr, src.rowptr, ((size_t)src.nrows + 1) * 8, cudaMemcpyDeviceToDevice, G.stream), err);
    if (src.nnz) {
        CU_TRY(cudaMemcpyAsync(T.col, src.col, (size_t)src.nnz * 4, cudaMemcpyDeviceToDevice, G.stream), err);
        CU_TRY(cudaMemcpyAsync(T.val, src.val, (size_t)src.nnz * sz, cudaMemcpyDeviceToDevice, G.stream), err);
    }
    GB_TRY(dev_build_rowptr32(T, err));
    return matrix_writeback(C, Mask, accum, f, std::move(T), A->type->code, false, err);
}
