// sddmm.cu -- GrB_mxm with two dense-form operands under a sparse mask (DESIGN.md section 3.6, "Two dense operands under a
// sparse mask"): the sampled dense-dense product
//
//   T<M> = X (+).(x) Y',   X = op(A) as m x d row-major, Y = op(B)' as n x d row-major, M a CSR m x n mask, not complemented
//
// One d-long dot product per entry of M the mask lets through, and nothing for any other position: the mask is applied first.
// One lane per mask entry (i, j): it walks X(i, :) and Y(j, :) in k order.  Consecutive entries of M share i, so a warp's loads
// of X are broadcasts; the rows of Y are the gather, d contiguous values each.  The fold is the SpMM kernel's: k ascending in
// chunks of SPMM_SEG, each chunk folded in order from its first present product, the chunk partials folded pairwise in the fixed
// tree over chunk order of spmm_combine_kernel.  T(i, j) depends on X(i, :), Y(j, :), d and the semiring only.  No atomics.
#include "common.cuh"
#include "spmv_common.cuh"

struct SddmmArgs {
    const uint32_t *mrow, *mcol;                // row and column of every entry of M
    const void *mval; int mtc, m_struct;        // M's values, read when the mask is valued
    const void *xval; const uint8_t *xpres;     // X: m x d row-major, values of the multiply's x type
    const void *yval; const uint8_t *ypres;     // Y: n x d row-major, values of the multiply's y type
    int64_t d, nnz;
    int add, mul;
    int vec;                                    // rows of X and Y start and end on 16-byte boundaries
    void *tval; uint8_t *found;                 // per mask entry; found NULL: every entry gets a value
};

// levels of the tree over chunk partials: 2^SDDMM_LEVELS chunks of SPMM_SEG cover every d a dense form can have (< 2^31)
static constexpr int SDDMM_LEVELS = 25;

// warp per row of M: the row id of each of its entries
__global__ void sddmm_rowid_kernel(const uint32_t *rowptr, int64_t m, uint32_t *mrow) {
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int lane = threadIdx.x & 31;
    for (int64_t r = warp; r < m; r += nwarps)
        for (uint32_t q = rowptr[r] + lane; q < rowptr[r + 1]; q += 32) mrow[q] = (uint32_t)r;
}

// the wide route: warp per row of M, the row id of each of its entries in the chunk [q0, q1), at mrow[q - q0].  Reads the 64-bit
// row offsets and keeps only a chunk's row ids; every row is visited once per chunk (16 bytes of offsets each).
__global__ void sddmm_rowid_wide_kernel(const int64_t *rowptr, int64_t m, int64_t q0, int64_t q1, uint32_t *mrow) {
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int lane = threadIdx.x & 31;
    for (int64_t r = warp; r < m; r += nwarps) {
        const int64_t e = min(rowptr[r + 1], q1);
        for (int64_t q = max(rowptr[r], q0) + lane; q < e; q += 32) mrow[q - q0] = (uint32_t)r;
    }
}

// The monoid's operator on two values of the fold.  A floating-point PLUS is the explicitly rounded add, which the compiler
// never contracts with the multiply before it into a fused multiply-add: the oracle rounds the product and the sum separately,
// and up to one chunk the result is its left-to-right fold bit for bit, whatever the values.
template <typename ZT> __device__ __forceinline__ ZT sddmm_add(int add, ZT a, ZT b) {
    if constexpr (std::is_same<ZT, float>::value) { if (add == OP_PLUS) return __fadd_rn(a, b); }
    if constexpr (std::is_same<ZT, double>::value) { if (add == OP_PLUS) return __dadd_rn(a, b); }
    return MulApply<ZT, ZT>::f(add, a, b);
}

// The kernels with run-time operator codes are bounded for one resident CTA, not two: under the 128-register cap of two, ptxas
// spills the tree levels of the INT64 and INT16 instances to local memory.
template <typename XT, typename ZT, int ADD, int MUL>
__global__ void __launch_bounds__(256, ADD >= 0 ? 2 : 1) sddmm_kernel(const SddmmArgs p) {
    const int add = ADD >= 0 ? ADD : p.add, mul = MUL >= 0 ? MUL : p.mul;
    const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= p.nnz) return;                             // lanes fold independently: no warp-wide operation follows
    ZT *tv = (ZT *)p.tval;
    if (!p.m_struct && sc_cast(sc_load(p.mtc, p.mval, q), p.mtc, TC_BOOL).u == 0) { tv[q] = (ZT)0; p.found[q] = 0; return; }
    const int64_t xo = (int64_t)p.mrow[q] * p.d, yo = (int64_t)__ldg(p.mcol + q) * p.d;
    const XT *xr = (const XT *)p.xval + xo, *yr = (const XT *)p.yval + yo;
    const uint8_t *xp = p.xpres ? p.xpres + xo : nullptr, *yp = p.ypres ? p.ypres + yo : nullptr;
    const bool rx = mul_reads_x(mul), ry = mul_reads_y(mul);
    // lv[l]: the fold of 2^l consecutive chunks, held while bit l of the number of finished chunks is set (hb: it has a value)
    ZT lv[SDDMM_LEVELS] = {};
    uint32_t hb = 0, nc = 0;
    for (int64_t k0 = 0; k0 < p.d; k0 += SPMM_SEG, ++nc) {
        const int64_t k1 = min(k0 + SPMM_SEG, p.d);
        ZT acc = (ZT)0; bool has = false;
        auto step = [&](int64_t k, XT x, XT y) {
            if ((xp && gload(xp + k) == 0) || (yp && gload(yp + k) == 0)) return;
            const ZT z = MulApply<XT, ZT>::f(mul, x, y);
            acc = has ? sddmm_add<ZT>(add, acc, z) : z; has = true;
        };
        int64_t k = k0;
        if constexpr (ADD >= 0) {
            // the specialised semirings: 128-bit loads, two per operand and trip, so both halves of a 32-byte sector are requested
            // together; the values are folded in k order afterwards
            constexpr int E = 16 / (int)sizeof(XT);
            auto trip = [&](auto nv) {
                constexpr int NV = decltype(nv)::value;
                union { uint4 v[NV]; XT e[NV * E]; } x, y;
#pragma unroll
                for (int u = 0; u < NV; ++u) {
                    if (rx) x.v[u] = __ldg(reinterpret_cast<const uint4 *>(xr + k) + u);
                    if (ry) y.v[u] = __ldg(reinterpret_cast<const uint4 *>(yr + k) + u);
                }
#pragma unroll
                for (int u = 0; u < NV * E; ++u) step(k + u, rx ? x.e[u] : (XT)0, ry ? y.e[u] : (XT)0);
                k += NV * E;
            };
            if (p.vec) {
                while (k + 2 * E <= k1) trip(std::integral_constant<int, 2>());
                if (k + E <= k1) trip(std::integral_constant<int, 1>());
            }
        }
        constexpr int U = 4;    // values whose loads are in flight together; folded in order afterwards
        for (; k + U <= k1; k += U) {
            XT x[U], y[U];
#pragma unroll
            for (int u = 0; u < U; ++u) { x[u] = rx ? gload(xr + k + u) : (XT)0; y[u] = ry ? gload(yr + k + u) : (XT)0; }
#pragma unroll
            for (int u = 0; u < U; ++u) step(k + u, x[u], y[u]);
        }
        for (; k < k1; ++k) step(k, rx ? gload(xr + k) : (XT)0, ry ? gload(yr + k) : (XT)0);
        // the chunk's partial joins the tree: it merges with every level that is held, left operand first, and rests at the
        // first free one
        bool placed = false;
#pragma unroll
        for (int l = 0; l < SDDMM_LEVELS; ++l) {
            if (placed) continue;
            if ((nc >> l) & 1) {
                if ((hb >> l) & 1) { acc = has ? sddmm_add<ZT>(add, lv[l], acc) : lv[l]; has = true; }
            } else {
                lv[l] = acc; hb = (hb & ~(1u << l)) | ((uint32_t)has << l); placed = true;
            }
        }
    }
    // what is held, from the last (smallest) group to the first: each is the left operand of everything after it
    ZT r = (ZT)0; bool rh = false;
#pragma unroll
    for (int l = 0; l < SDDMM_LEVELS; ++l)
        if (((nc >> l) & 1) && ((hb >> l) & 1)) { r = rh ? sddmm_add<ZT>(add, lv[l], r) : lv[l]; rh = true; }
    tv[q] = rh ? r : (ZT)0;
    if (p.found) p.found[q] = rh;
}

// the specialised semirings (the SpMV list, spmv_common.cuh) on x = z = T
template <typename T> static bool sddmm_launch_fast(int add, int mul, const SddmmArgs &p, unsigned grid) {
#define GB_SDDMM_FAST(A, M) if (add == A && mul == M) { sddmm_kernel<T, T, A, M><<<grid, 256, 0, G.stream>>>(p); return true; }
    GB_SPMV_FAST_PAIRS(T, GB_SDDMM_FAST)
#undef GB_SDDMM_FAST
    return false;
}
static bool sddmm_launch(int xt, int zt, const SddmmArgs &p, bool *fast) {
    const unsigned grid = (unsigned)ceil_div(p.nnz, 256);
    *fast = false;
    if (xt == zt) switch (xt) {
        case TC_FP32: *fast = sddmm_launch_fast<float>(p.add, p.mul, p, grid); break;
        case TC_FP64: *fast = sddmm_launch_fast<double>(p.add, p.mul, p, grid); break;
        case TC_INT32: *fast = sddmm_launch_fast<int32_t>(p.add, p.mul, p, grid); break;
        case TC_INT64: *fast = sddmm_launch_fast<int64_t>(p.add, p.mul, p, grid); break;
        case TC_UINT32: *fast = sddmm_launch_fast<uint32_t>(p.add, p.mul, p, grid); break;
        case TC_UINT64: *fast = sddmm_launch_fast<uint64_t>(p.add, p.mul, p, grid); break;
        case TC_BOOL: *fast = sddmm_launch_fast<bool>(p.add, p.mul, p, grid); break;
        default: break;
    }
    if (*fast) return true;
    bool matched = false;
    GB_FOR_DOMAINS(xt, zt, matched, (sddmm_kernel<XT_, ZT_, -1, -1><<<grid, 256, 0, G.stream>>>(p)));
    return matched;
}

// One operand in the kernel's layout: its dense form, cast to the multiply's input type where the multiply reads it and the
// types differ, and transposed (rows x cols -> cols x rows, per call, not cached) when `tr`.  The buffers it built live in `o`.
struct SddmmOperand {
    DevBuf<void> cast, tval; DevBuf<uint8_t> tpres;
    const void *val = nullptr; const uint8_t *pres = nullptr;
    double bytes = 0.0;                         // of the byte model: the operand once, and twice more for a transpose
};
static GrB_Info sddmm_operand(const GrB_Matrix A, bool reads, int xt, bool tr, const char *token, SddmmOperand &o, std::string *err) {
    const int64_t rows = (int64_t)A->nrows, cols = (int64_t)A->ncols, n = rows * cols;
    o.pres = A->dn.pres;
    o.bytes = (double)n * (tc_size(A->type->code) + (o.pres ? 1 : 0));
    GB_TRY(mxm_values(o.cast, &o.val, reads, xt, A->dn.val, A->type->code, n, err));
    const size_t b = tc_size(reads ? xt : A->type->code);      // the bytes of one value of o.val
    if (tr && (reads || o.pres)) {              // an operand that is neither read nor has absent entries has no layout
        GB_TRY(o.tval.alloc((size_t)n * b + 16, err));
        if (o.pres) GB_TRY(o.tpres.alloc((size_t)n, err));
        GB_TRY(dense_transpose(o.val, o.pres, rows, cols, b, o.tval, o.tpres, err));
        o.cast.reset();
        o.val = o.tval; o.pres = o.pres ? o.tpres.get() : nullptr;
        o.bytes += 2.0 * (double)n * (b + (o.pres ? 1 : 0));
        gb_kernel_used(token);
    }
    return GrB_SUCCESS;
}

GrB_Info sddmm_mxm(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const GrB_Semiring s, const GrB_Matrix A,
                   const GrB_Matrix B, const DescFlags &f, GbBurble &burble) {
    std::string *err = &C->err;
    const GrB_BinaryOp mulop = s->mul, addop = s->add->op;
    const int xt = mulop->xtype->code, zt = addop->ztype->code, add = addop->opcode, mul = mulop->opcode;
    const size_t zsz = tc_size(zt);
    gb_kernel_used("sddmm");
    const Csr &M = Mask->dev;                           // on the device (GrB_mxm)
    const int64_t m = M.nrows, n = M.ncols, d = (int64_t)(f.tran0 ? A->nrows : A->ncols);
    SddmmOperand X, Y;
    GB_TRY(sddmm_operand(A, mul_reads_x(mul), xt, f.tran0 && d > 1, "x-transpose", X, err));
    GB_TRY(sddmm_operand(B, mul_reads_y(mul), xt, !f.tran1 && d > 1, "y-transpose", Y, err));
    const bool full = !X.pres && !Y.pres;
    // with nothing absent and a structural mask, T has exactly M's pattern: the kernel writes T's values in place
    const bool pattern_mask = full && f.mask_struct && d > 0;
    Csr T;
    void *tval = nullptr; uint8_t *found = nullptr;
    if (pattern_mask) {
        GB_TRY(csr_copy(M, zsz, false, T, err));
        tval = T.val;
    } else {
        GB_TRY(ws_get(WS_WORDS, &tval, (size_t)M.nnz * zsz + 16, err));
        GB_TRY(ws_get(WS_FOUND, (void **)&found, (size_t)M.nnz + 16, err));
    }
    // the wide route (csr_wide: nnz(M) >= 2^32, or B200_debug_wide) takes M in chunks of entries: the row ids of one chunk
    // from the 64-bit row offsets, then the same kernel on that chunk's slice of M and T
    const bool wide = csr_wide(M);
    if (M.nnz > 0 && d > 0) {
        const int64_t chunk = !wide ? M.nnz : std::min(M.nnz, wide_chunk());
        uint32_t *mrow = nullptr;
        GB_TRY(ws_array(WS_MASK_ROW, &mrow, (size_t)chunk, err));
        if (!wide) { sddmm_rowid_kernel<<<grid_for(m * 32), 256, 0, G.stream>>>(M.rowptr32, m, mrow); GB_LAUNCHED(); }
        const size_t msz = tc_size(Mask->type->code);
        bool fast = false;
        for (int64_t q0 = 0; q0 < M.nnz; q0 += chunk) {
            const int64_t q1 = std::min(q0 + chunk, M.nnz);
            if (wide) { sddmm_rowid_wide_kernel<<<grid_for(m * 32), 256, 0, G.stream>>>(M.rowptr, m, q0, q1, mrow); GB_LAUNCHED(); }
            SddmmArgs p{};
            p.mrow = mrow; p.mcol = M.col + q0; p.mval = M.val.get() ? (const uint8_t *)M.val.get() + q0 * msz : nullptr;
            p.mtc = Mask->type->code; p.m_struct = f.mask_struct;
            p.xval = X.val; p.xpres = X.pres; p.yval = Y.val; p.ypres = Y.pres;
            p.d = d; p.nnz = q1 - q0; p.add = add; p.mul = mul;
            p.vec = (d * (int64_t)tc_size(xt)) % 16 == 0 && (uintptr_t)X.val % 16 == 0 && (uintptr_t)Y.val % 16 == 0;
            p.tval = (uint8_t *)tval + q0 * zsz; p.found = found ? found + q0 : nullptr;
            if (!sddmm_launch(xt, zt, p, &fast))
                return gb_fail(GrB_DOMAIN_MISMATCH, err, "GrB_mxm: unsupported semiring domains (x=%d, z=%d)", xt, zt);
            GB_LAUNCHED();
        }
        gb_kernel_used(fast ? "sddmm-fast" : "sddmm-generic");
        if (wide) gb_kernel_used("offsets=64");
    } else if (found && M.nnz > 0) {
        CU_TRY(cudaMemsetAsync(found, 0, (size_t)M.nnz, G.stream), err);      // d = 0: no entry has a product
    }
    if (pattern_mask) {
        GB_TRY(dev_build_rowptr32(T, err));
        G.last_nnz_out = (uint64_t)T.nnz;
    } else {
        GB_TRY(masked_compact(M, found, tval, zsz, T, err));
    }
    gb_kernel_used(pattern_mask ? "pattern=mask" : "pattern=compact");
    CU_TRY(cudaGetLastError(), err);
    const double operand_bytes = X.bytes + Y.bytes;
    X = SddmmOperand(); Y = SddmmOperand();
    G.last_flops = full ? (uint64_t)M.nnz * (uint64_t)d : 0;
    // algorithmic bytes: M (ids, row pointers, values when it is valued), X and Y once, T (ids, values, row pointers), and the
    // transposes built.  Left out: the gather, nnz(M) d b_Y -- rows of Y are read once per entry that names them, and how much of
    // that the caches absorb depends on M.
    const double bytes = (double)M.nnz * 4 + (double)(m + 1) * (wide ? 8 : 4) + (f.mask_struct ? 0.0 : (double)M.nnz * tc_size(Mask->type->code)) +
                         operand_bytes + (double)T.nnz * (4 + tc_size(C->type->code)) + (double)(m + 1) * 8;
    burble.note(wide ? "sddmm, 64-bit offsets" : "sddmm", bytes);
    return matrix_writeback(C, Mask, accum, f, std::move(T), zt, /*masked=*/true, err);
}
