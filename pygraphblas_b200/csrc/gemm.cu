// gemm.cu -- GrB_mxm with two full dense-form operands (DESIGN.md section 3.6, "Two full dense operands"): the tiled semiring
// GEMM
//
//   T = op(A) (+).(x) op(B),   op(A) m x k, op(B) k x n, both dense forms without presence bytes, T m x n formed dense
//
// A CTA of 256 threads owns a 64 x 64 tile of T at a time; each thread a 4 x 4 micro-tile in registers, so every value staged in
// shared memory serves four products.  op(A) and op(B) go through shared memory in k-tiles of gemm_bk() positions, two stages
// deep (cp.async for 4- and 8-byte values), read in place whatever the descriptor: the loader picks the coalesced order of each
// layout and writes k-major tiles.  The fold is SpMM's on a full row: k ascending in chunks of SPMM_SEG, each chunk folded left
// to right from its first product with the explicitly rounded add (never contracted with the multiply), the chunk partials
// folded pairwise in the fixed tree over chunk order of spmm_combine_kernel.  The tree lives in per-CTA scratch: the CTAs are
// persistent and each reuses its slot of levels tile after tile, so the scratch is independent of m and n.  No atomics.
#include "common.cuh"
#include "spmv_common.cuh"

static constexpr int GEMM_TILE = 64, GEMM_THREADS = 256, GEMM_MICRO = 4, GEMM_STAGES = 2;
static constexpr int GEMM_LD = GEMM_TILE + 4;         // row stride of a staged tile: 16-byte aligned micro-tile reads
// k positions per staged tile: one chunk for values up to 4 bytes, half of one for 8-byte values (the same shared memory)
template <typename XT> constexpr int gemm_bk() { return sizeof(XT) == 8 ? SPMM_SEG / 2 : SPMM_SEG; }
template <typename XT> constexpr size_t gemm_smem() { return (size_t)GEMM_STAGES * 2 * gemm_bk<XT>() * GEMM_LD * sizeof(XT); }

struct GemmArgs {
    const void *a, *b;          // A (m x k, or k x m under ta) and B (k x n, or n x k under tb), values of the multiply's x type
    int64_t m, n, k;
    int ta, tb;
    int add, mul;
    void *t;                    // T: m x n row-major
    void *lv;                   // tree levels: `levels` per CTA, 16 values per thread each (k > SPMM_SEG only)
    int levels;
    int64_t ntn;                // tiles across n
    int64_t ntiles;
};

// The monoid's operator in the fold: a floating-point PLUS is the explicitly rounded add (as sddmm_add)
template <typename ZT> __device__ __forceinline__ ZT gemm_add(int add, ZT a, ZT b) {
    if constexpr (std::is_same<ZT, float>::value) { if (add == OP_PLUS) return __fadd_rn(a, b); }
    if constexpr (std::is_same<ZT, double>::value) { if (add == OP_PLUS) return __dadd_rn(a, b); }
    return MulApply<ZT, ZT>::f(add, a, b);
}

__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
__device__ __forceinline__ void cp_async_wait_prev() { asm volatile("cp.async.wait_group %0;\n" :: "n"(GEMM_STAGES - 2)); }

// One k-tile of an operand into s[kk * GEMM_LD + c]: element (c, kk) of the tile at src[(c0 + c) * cs + (k0 + kk) * ks].
// kfast: consecutive threads take consecutive kk (the operand is contiguous along k), else consecutive c.  Positions past
// the operand's edges are not loaded (their products are never folded or never stored).
template <typename XT, int BK>
__device__ __forceinline__ void gemm_stage(XT *s, const XT *src, int64_t c0, int64_t cn, int64_t k0, int64_t kn, int64_t cs, int64_t ks,
                                           bool kfast) {
#pragma unroll 4
    for (int e = threadIdx.x; e < BK * GEMM_TILE; e += GEMM_THREADS) {
        const int kk = kfast ? e % BK : e / GEMM_TILE, c = kfast ? e / BK : e % GEMM_TILE;
        if (c0 + c >= cn || k0 + kk >= kn) continue;
        XT *d = s + kk * GEMM_LD + c;
        const XT *g = src + (c0 + c) * cs + (k0 + kk) * ks;
        if constexpr (sizeof(XT) >= 4) {
            const unsigned sa = (unsigned)__cvta_generic_to_shared(d);
            asm volatile("cp.async.ca.shared.global [%0], [%1], %2;\n" :: "r"(sa), "l"(g), "n"((int)sizeof(XT)));
        } else {
            *d = gload(g);
        }
    }
}

template <typename XT> struct alignas(GEMM_MICRO * sizeof(XT)) GemmVec { XT e[GEMM_MICRO]; };

template <typename XT, typename ZT, int ADD, int MUL>
__global__ void __launch_bounds__(GEMM_THREADS, ADD >= 0 ? 2 : 1) gemm_kernel(const GemmArgs p) {
    constexpr int BK = gemm_bk<XT>(), STAGE = 2 * BK * GEMM_LD;
    extern __shared__ __align__(16) unsigned char gemm_smem_raw[];
    XT *sm = reinterpret_cast<XT *>(gemm_smem_raw);
    const int add = ADD >= 0 ? ADD : p.add, mul = MUL >= 0 ? MUL : p.mul;
    const bool rx = mul_reads_x(mul), ry = mul_reads_y(mul);
    const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
    const XT *A = (const XT *)p.a, *B = (const XT *)p.b;
    const int64_t nch = ceil_div(p.k, SPMM_SEG), nkt = ceil_div(p.k, BK);
    // the thread's tree levels: level l, value e at lv[(l * 16 + e) * GEMM_THREADS]
    ZT *lv = (ZT *)p.lv + (size_t)blockIdx.x * p.levels * (GEMM_MICRO * GEMM_MICRO * GEMM_THREADS) + threadIdx.x;
    for (int64_t tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
        const int64_t i0 = tile / p.ntn * GEMM_TILE, j0 = tile % p.ntn * GEMM_TILE;
        auto issue = [&](int64_t kt) {
            if (kt < nkt) {
                XT *s = sm + (kt % GEMM_STAGES) * STAGE;
                const int64_t k0 = kt * BK;
                if (rx) gemm_stage<XT, BK>(s, A, i0, p.m, k0, p.k, p.ta ? 1 : p.k, p.ta ? p.m : 1, !p.ta);
                if (ry) gemm_stage<XT, BK>(s + BK * GEMM_LD, B, j0, p.n, k0, p.k, p.tb ? p.k : 1, p.tb ? 1 : p.n, p.tb);
            }
            cp_async_commit();
        };
#pragma unroll
        for (int s = 0; s < GEMM_STAGES - 1; ++s) issue(s);
        ZT acc[GEMM_MICRO][GEMM_MICRO];
        for (int64_t kt = 0; kt < nkt; ++kt) {
            cp_async_wait_prev();                   // k-tile kt has landed
            __syncthreads();
            issue(kt + GEMM_STAGES - 1);            // into the stage the previous k-tile was folded from
            const XT *as = sm + (kt % GEMM_STAGES) * STAGE + ty * GEMM_MICRO, *bs = as - ty * GEMM_MICRO + BK * GEMM_LD + tx * GEMM_MICRO;
            const int64_t k0 = kt * BK;
            const int kn = (int)min((int64_t)BK, p.k - k0);
            GemmVec<XT> a{}, b{};
            auto fetch = [&](int kk) {
                if (rx) a = *reinterpret_cast<const GemmVec<XT> *>(as + kk * GEMM_LD);
                if (ry) b = *reinterpret_cast<const GemmVec<XT> *>(bs + kk * GEMM_LD);
            };
            int kk = 0;
            if (k0 % SPMM_SEG == 0) {               // a chunk starts: its fold starts from its first product
                fetch(0);
#pragma unroll
                for (int i = 0; i < GEMM_MICRO; ++i)
#pragma unroll
                    for (int j = 0; j < GEMM_MICRO; ++j) acc[i][j] = MulApply<XT, ZT>::f(mul, a.e[i], b.e[j]);
                kk = 1;
            }
            auto step = [&](int kk) {
                fetch(kk);
#pragma unroll
                for (int i = 0; i < GEMM_MICRO; ++i)
#pragma unroll
                    for (int j = 0; j < GEMM_MICRO; ++j) acc[i][j] = gemm_add<ZT>(add, acc[i][j], MulApply<XT, ZT>::f(mul, a.e[i], b.e[j]));
            };
            if constexpr (ADD >= 0) {
#pragma unroll 8
                for (; kk < kn; ++kk) step(kk);
            } else {
#pragma unroll 1
                for (; kk < kn; ++kk) step(kk);
            }
            __syncthreads();                        // the stage is refilled by the next k-tile's issue
            const bool last = kt == nkt - 1;
            if (nch > 1 && (last || (k0 + BK) % SPMM_SEG == 0)) {
                // chunk c joins the tree (the binary counter of sddmm_kernel, every partial present): it merges with the held
                // groups of the set low bits of c, left operand first, and rests at the first free level; the last chunk merges
                // with every held group, smallest first
                const int64_t c = k0 / SPMM_SEG;
                int l = 0;
                for (; l < p.levels && (last || ((c >> l) & 1)); ++l) {
                    if (!((c >> l) & 1)) continue;
#pragma unroll
                    for (int e = 0; e < GEMM_MICRO * GEMM_MICRO; ++e)
                        acc[e / GEMM_MICRO][e % GEMM_MICRO] =
                            gemm_add<ZT>(add, lv[(size_t)(l * 16 + e) * GEMM_THREADS], acc[e / GEMM_MICRO][e % GEMM_MICRO]);
                }
                if (!last) {
#pragma unroll
                    for (int e = 0; e < GEMM_MICRO * GEMM_MICRO; ++e) lv[(size_t)(l * 16 + e) * GEMM_THREADS] = acc[e / GEMM_MICRO][e % GEMM_MICRO];
                }
            }
        }
        ZT *T = (ZT *)p.t;
#pragma unroll
        for (int i = 0; i < GEMM_MICRO; ++i) {
            const int64_t r = i0 + ty * GEMM_MICRO + i;
            if (r >= p.m) continue;
#pragma unroll
            for (int j = 0; j < GEMM_MICRO; ++j) {
                const int64_t cc = j0 + tx * GEMM_MICRO + j;
                if (cc < p.n) T[r * p.n + cc] = acc[i][j];
            }
        }
    }
}

// One launch: as many persistent CTAs as fit on the device, at most one per tile; the tree scratch is sized for that grid
template <typename XT, typename ZT, int ADD, int MUL>
static GrB_Info gemm_run(GemmArgs &p, std::string *err) {
    auto kern = gemm_kernel<XT, ZT, ADD, MUL>;
    constexpr size_t smem = gemm_smem<XT>();
    CU_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), err);
    int per_sm = 0;
    CU_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, GEMM_THREADS, smem), err);
    const int64_t grid = std::max<int64_t>(1, std::min<int64_t>(p.ntiles, (int64_t)G.num_sms * std::max(per_sm, 1)));
    if (p.levels > 0) {
        const size_t bytes = (size_t)grid * p.levels * GEMM_MICRO * GEMM_MICRO * GEMM_THREADS * sizeof(ZT);
        GB_TRY(ws_get(WS_GEMM_TREE, &p.lv, bytes + 16, err));
    }
    kern<<<(unsigned)grid, GEMM_THREADS, smem, G.stream>>>(p);
    GB_LAUNCHED();
    return GrB_SUCCESS;
}

// the specialised semirings (the SpMV list, spmv_common.cuh) on x = z = T
template <typename T> static bool gemm_launch_fast(GemmArgs &p, GrB_Info *r, std::string *err) {
#define GB_GEMM_FAST(A, M) if (p.add == A && p.mul == M) { *r = gemm_run<T, T, A, M>(p, err); return true; }
    GB_SPMV_FAST_PAIRS(T, GB_GEMM_FAST)
#undef GB_GEMM_FAST
    return false;
}
static GrB_Info gemm_launch(int xt, int zt, GemmArgs &p, bool *fast, std::string *err) {
    GrB_Info r = GrB_SUCCESS;
    *fast = false;
    if (xt == zt) switch (xt) {
        case TC_FP32: *fast = gemm_launch_fast<float>(p, &r, err); break;
        case TC_FP64: *fast = gemm_launch_fast<double>(p, &r, err); break;
        case TC_INT32: *fast = gemm_launch_fast<int32_t>(p, &r, err); break;
        case TC_INT64: *fast = gemm_launch_fast<int64_t>(p, &r, err); break;
        case TC_UINT32: *fast = gemm_launch_fast<uint32_t>(p, &r, err); break;
        case TC_UINT64: *fast = gemm_launch_fast<uint64_t>(p, &r, err); break;
        case TC_BOOL: *fast = gemm_launch_fast<bool>(p, &r, err); break;
        default: break;
    }
    if (*fast) return r;
    bool matched = false;
    GB_FOR_DOMAINS(xt, zt, matched, (r = gemm_run<XT_, ZT_, -1, -1>(p, err)));
    if (!matched) return gb_fail(GrB_DOMAIN_MISMATCH, err, "GrB_mxm: unsupported semiring domains (x=%d, z=%d)", xt, zt);
    return r;
}

GrB_Info gemm_mxm(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const GrB_Semiring s, const GrB_Matrix A,
                  const GrB_Matrix B, const DescFlags &f, GbBurble &burble) {
    std::string *err = &C->err;
    const GrB_BinaryOp mulop = s->mul, addop = s->add->op;
    const int xt = mulop->xtype->code, zt = addop->ztype->code, add = addop->opcode, mul = mulop->opcode;
    const size_t zsz = tc_size(zt);
    gb_kernel_used("gemm");
    const int64_t m = (int64_t)(f.tran0 ? A->ncols : A->nrows), k = (int64_t)(f.tran0 ? A->nrows : A->ncols);
    const int64_t n = (int64_t)(f.tran1 ? B->nrows : B->ncols);
    // operands cast to the multiply's input type where it reads them, as on the SpMM route
    DevBuf<void> a_cast, b_cast;
    const void *aval = nullptr, *bval = nullptr;
    GB_TRY(mxm_values(a_cast, &aval, mul_reads_x(mul), xt, A->dn.val, A->type->code, m * k, err));
    GB_TRY(mxm_values(b_cast, &bval, mul_reads_y(mul), xt, B->dn.val, B->type->code, k * n, err));
    // T in fresh buffers: C may alias A or B.  With k > 0 every position has a product and T needs no presence bytes; with
    // k = 0 none has one.
    DevBuf<void> tval; DevBuf<uint8_t> tpres;
    GB_TRY(tval.alloc((size_t)(m * n) * zsz + 16, err));
    if (k == 0) {
        GB_TRY(tpres.alloc((size_t)(m * n), err));
        if (m * n > 0) CU_TRY(cudaMemsetAsync(tpres, 0, (size_t)(m * n), G.stream), err);
    } else if (m > 0 && n > 0) {
        GemmArgs p{};
        p.a = aval; p.b = bval; p.m = m; p.n = n; p.k = k; p.ta = f.tran0; p.tb = f.tran1; p.add = add; p.mul = mul;
        p.t = tval;
        const int64_t nch = ceil_div(k, SPMM_SEG);
        while (nch > 1 && ((nch - 1) >> p.levels) != 0) ++p.levels;      // bit length of nch - 1: the highest level held
        p.ntn = ceil_div(n, GEMM_TILE);
        p.ntiles = ceil_div(m, GEMM_TILE) * p.ntn;
        bool fast = false;
        GB_TRY(gemm_launch(xt, zt, p, &fast, err));
        gb_kernel_used(fast ? "gemm-fast" : "gemm-generic");
        if (nch > 1) gb_kernel_used("gemm-tree");
        CU_TRY(cudaGetLastError(), err);
    }
    a_cast.reset(); b_cast.reset();
    G.last_flops = (uint64_t)m * (uint64_t)n * (uint64_t)k;
    // algorithmic bytes: op(A) and op(B) once, T (values, and presence bytes when k = 0)
    const double bytes = (double)(m * k) * tc_size(A->type->code) + (double)(k * n) * tc_size(B->type->code) +
                         (double)(m * n) * (zsz + (k == 0 ? 1 : 0));
    burble.note("gemm", bytes);
    return spmm_writeback(C, Mask, accum, f, std::move(tval), std::move(tpres), zt, err);
}
