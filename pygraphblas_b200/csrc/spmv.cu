// spmv.cu -- GrB_mxv / GrB_vxm on sm_90a:  w<mask> = accum(w, op(A) (+).(x) u)
//
// Replaces the SuiteSparse call behind reference: pygraphblas/matrix.py:2716
// (Matrix.mxv) and reference: pygraphblas/vector.py:961 (Vector.vxm).
//
// Layout in HBM: A is CSR (32-bit row offsets shadow, 32-bit column ids, values of
// the matrix type), vectors are dense value arrays + one presence byte per position
// (no presence array at all when every position is present).
//
// This file: the host logic of both calls (operand casts, kernel choice, write-back).
// Kernel choice, in order (DESIGN.md section 3.1):
//   mask + LOR/LAND/ANY monoid  -> masked push (small frontier, spmv_pull.cu) or masked pull with early exit
//   nnz == 0                    -> no kernel but clearing T's presence
//   otherwise                   -> run kernel (spmv_run*.cu): 256-entry runs per warp on a cached run plan,
//                                  compile-time semirings (+ shared-memory hot-column table), run-time
//                                  operator codes, dense or sparse u; rows that straddle runs are
//                                  combined by a fix-up kernel in a fixed order
// Every path is nnz-split (R-MAT hub rows cannot serialise a warp) and deterministic for a given matrix.
//
// Algorithmic bytes per call (DESIGN.md): nnz*(4 + sizeof(a)) + (nrows+1)*4
//   + ncols*sizeof(u) + nrows*(sizeof(t) + 1).
#include "spmv_args.cuh"

__global__ void clear_presence_kernel(uint8_t *p, int64_t n) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) p[k] = 0;
}

// w<mask> = accum(w, A' (+).(x) u) with `flip` selecting mul(u,a) (vxm) and `use_transpose`
// selecting the cached CSR of A' (so that the kernel always pulls along CSR rows).
static GrB_Info mxv_core(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_Semiring s,
                         const GrB_Matrix A, const GrB_Vector u, const DescFlags &f, bool use_transpose, bool flip,
                         const char *fn) {
    std::string *err = &w->err;
    // ---- domain / dimension checks (host, synchronous)
    const GrB_BinaryOp mulop = s->mul; const GrB_BinaryOp addop = s->add->op;
    if (mulop->opcode == OP_USER || addop->opcode == OP_USER || (accum && accum->opcode == OP_USER))
        return gb_fail(GrB_INVALID_VALUE, err, "%s: user-defined operators are host function pointers and cannot run on the GPU (no CPU fallback)", fn);
    const uint64_t out_n = use_transpose ? A->ncols : A->nrows, in_n = use_transpose ? A->nrows : A->ncols;
    if (u->n != in_n || w->n != out_n || (mask && mask->n != out_n))
        return gb_fail(GrB_DIMENSION_MISMATCH, err, "%s: dimensions do not match (A is %llux%llu%s, u %llu, w %llu)", fn,
                       (unsigned long long)A->nrows, (unsigned long long)A->ncols, use_transpose ? " transposed" : "",
                       (unsigned long long)u->n, (unsigned long long)w->n);
    if (!G.have_device) return gb_fail(GrB_PANIC, err, "%s: no CUDA device: libb200grb computes only on the GPU (no CPU fallback)", fn);
    const int xt = mulop->xtype->code, zt = addop->ztype->code;
    const int add = addop->opcode, mul = mulop->opcode;
    G.last_kernel.clear();
    if (!mask && f.mask_comp)      // w<!NULL>: nothing is let through, no product needed (vector_write clears w under REPLACE)
        return vector_write(w, nullptr, accum, f, DenseForm(), zt, false, nullptr);

    // ---- operands in HBM
    Csr *pc; GB_TRY(source_csr(A, use_transpose, &pc));
    Csr &c = *pc;
    GB_TRY(vector_ensure_device(u));
    if (mask) GB_TRY(vector_ensure_device(mask));
    const bool need_final = mask != nullptr || accum != nullptr;
    const bool w_empty = w->host_valid && w->hi.empty() && w->pi.empty();   // nothing to merge with
    if (need_final && !w_empty) GB_TRY(vector_ensure_device(w));
    // the multiply sees (x = matrix entry, y = u entry) for mxv and the reverse for vxm; for the
    // operators that ignore one side the flip folds into the operator itself
    int kmul = mul; bool kflip = flip;
    if (flip && (mul == OP_FIRST || mul == OP_SECOND)) { kmul = mul == OP_FIRST ? OP_SECOND : OP_FIRST; kflip = false; }
    if (flip && (mul == OP_TIMES || mul == OP_PLUS || mul == OP_MIN || mul == OP_MAX || mul == OP_PAIR || mul == OP_LAND || mul == OP_LOR ||
                 mul == OP_LXOR || mul == OP_EQ || mul == OP_NE || mul == OP_ISEQ || mul == OP_ISNE)) kflip = false;     // commutative
    const bool need_a = kflip ? mul_reads_y(kmul) : mul_reads_x(kmul);
    const bool need_u = kflip ? mul_reads_x(kmul) : mul_reads_y(kmul);
    const bool sparse_u = u->dv.pres != nullptr;
    const bool fast_sr = !kflip && spmv_is_fast(xt, zt, add, kmul, false);      // a compile-time specialised semiring
    const bool fast = fast_sr && !sparse_u;
    const Tunables &tn = tunables();
    std::string hot_note;                    // the burble line names the cluster; it is printed when `burble` is destroyed
    GbBurble burble(fn);
    // wide route (csr_wide: nnz >= 2^32, or B200_debug_wide): 64-bit row offsets in the run plan, pull and push kernels
    const bool wide = csr_wide(c);

    DevBuf<void> a_cast, u_cast;
    const void *aval = c.val, *uval = u->dv.val;
    if (need_a && A->type->code != xt) { GB_TRY(dev_cast_values(a_cast, xt, c.val, A->type->code, c.nnz, err)); aval = a_cast; }
    if (need_u && u->type->code != xt) { GB_TRY(dev_cast_values(u_cast, xt, u->dv.val, u->type->code, (int64_t)u->n, err)); uval = u_cast; }
    // run-time-operator kernels always read both operands: give them something readable of the right type
    if (!fast && !need_a && A->type->code != xt) { GB_TRY(dev_cast_values(a_cast, xt, c.val, A->type->code, c.nnz, err)); aval = a_cast; }
    if (!fast && !need_u && u->type->code != xt) { GB_TRY(dev_cast_values(u_cast, xt, u->dv.val, u->type->code, (int64_t)u->n, err)); uval = u_cast; }

    const int64_t n = (int64_t)out_n;
    const size_t zsz = (size_t)tc_size(zt);
    // T's buffers become w (no mask, no accumulator: w<-T).  When w already owns device buffers of the right shape and is not an
    // operand of this call, T is formed in place -- the iterated call `A.mxv(u, out=w)` then allocates nothing.
    void *tval = nullptr; uint8_t *tpres = nullptr;
    DevBuf<void> t_val; DevBuf<uint8_t> t_pres;      // T's own buffers when it is not formed in w's
    const bool w_reusable = !need_final && w != u && w->dv.valid && w->dv.val && w->dv.pres && !w->dv.val.borrowed() &&
                            w->type->code == zt && a_cast.get() != w->dv.val && u_cast.get() != w->dv.val;
    const bool in_place = w_reusable && (tn.mxv_inplace == 2 || (tn.mxv_inplace == 1 && !w->h2d_pending && !w->d2h_pending));
    if (in_place && tn.mxv_inplace == 2) {      // whatever the flags say: the kernels below start after w's last overlapped copies
        if (w->ev_h2d) { cudaStreamWaitEvent(G.stream, w->ev_h2d, 0); cudaStreamWaitEvent(G.stream, w->ev_d2h, 0); }
        w->h2d_pending = false; w->d2h_pending = false;
    }
    if (in_place) { tval = w->dv.val; tpres = w->dv.pres; }
    else {
        GB_TRY(t_val.alloc((size_t)n * zsz + 16, err));
        GB_TRY(t_pres.alloc((size_t)n, err));
        tval = t_val; tpres = t_pres;
    }

    // mask + saturating monoid (BFS-shaped): skip masked-out rows, stop rows at the first hit
    const bool use_pull = mask != nullptr && (add == OP_LOR || add == OP_LAND || add == OP_ANY) && c.nnz > 0 && !tn.no_pull;
    bool pushed = false;
    if (use_pull) {
        // the run-time-operator kernel reads both operands: make sure both are of the operand type
        if (aval == c.val && A->type->code != xt) { GB_TRY(dev_cast_values(a_cast, xt, c.val, A->type->code, c.nnz, err)); aval = a_cast; }
        if (uval == u->dv.val && u->type->code != xt) { GB_TRY(dev_cast_values(u_cast, xt, u->dv.val, u->type->code, (int64_t)u->n, err)); uval = u_cast; }
        // few frontier edges: push along the rows of the other orientation (already in HBM) instead of pulling every row
        const Csr &o = use_transpose ? A->dev : A->devT;
        if (sparse_u && o.valid && (wide || o.rowptr32) && o.nnz == c.nnz && A->type->code == xt && !tn.no_push) {
            auto push = [&](auto &ps, const auto *rowptr) {
                ps.rowptr = rowptr; ps.col = o.col; ps.aval = o.val; ps.nin = o.nrows; ps.uval = uval; ps.upres = u->dv.pres;
                ps.mval = mask->dv.val; ps.mpres = mask->dv.pres; ps.mtc = mask->type->code; ps.mask_comp = f.mask_comp; ps.mask_struct = f.mask_struct;
                ps.tval = tval; ps.tpres = tpres; ps.nout = n; ps.add_op = add; ps.mul_op = kmul; ps.flip = kflip;
                return spmv_masked_push_try(xt, zt, ps, c.nnz, &pushed, err);
            };
            PushArgs ps{}; PushArgsWide psw{};
            GB_TRY(wide ? push(psw, o.rowptr.get()) : push(ps, o.rowptr32.get()));
        }
        // rows longer than PULL_LONG: at most nnz / PULL_LONG of them
        const int64_t long_cap = c.nnz / (int64_t)PULL_LONG + 1;
        DevBuf<uint32_t> long_rows; DevBuf<int> long_count;
        GB_TRY(long_rows.alloc((size_t)long_cap + 1, err));
        GB_TRY(long_count.alloc(4, err));
        CU_TRY(cudaMemsetAsync(long_count, 0, sizeof(int), G.stream), err);
        auto pull = [&](auto &pa, const auto *rowptr) {
            pa.rowptr = rowptr; pa.col = c.col; pa.aval = aval; pa.nrows = c.nrows; pa.uval = uval; pa.upres = u->dv.pres;
            pa.mval = mask->dv.val; pa.mpres = mask->dv.pres; pa.mtc = mask->type->code; pa.mask_comp = f.mask_comp; pa.mask_struct = f.mask_struct;
            pa.tval = tval; pa.tpres = tpres; pa.add_op = add; pa.mul_op = kmul; pa.flip = kflip;
            pa.long_cap = long_cap; pa.has_long = c.nnz > (int64_t)PULL_LONG; pa.long_rows = long_rows; pa.long_count = long_count;
            return spmv_masked_pull_dispatch(xt, zt, pa, err);
        };
        PullArgs pa{}; PullArgsWide paw{};
        if (!pushed) GB_TRY(wide ? pull(paw, c.rowptr.get()) : pull(pa, c.rowptr32.get()));
    }
    const char *kernel_name = "pull";
    int hot_cluster = 0, hot_ctas = 0, hot_ids = 0; uint32_t hot_t0 = 0, hot_t1 = 0, hot_henc = 0;      // cluster size, grid, id width, tiers of the hot-table launch
    if (use_pull) {
        if (pushed) kernel_name = "push";
    } else if (c.nnz == 0) {
        clear_presence_kernel<<<grid_for(n), 256, 0, G.stream>>>(tpres, n); GB_LAUNCHED();
        kernel_name = "empty";
    } else {
        // the run kernel on the cached run plan: compile-time specialised semirings, or run-time operator codes on the (x, z)
        // domains GB_FOR_DOMAINS lists; dense or sparse u
        bool domains_ok; GB_FOR_DOMAINS(xt, zt, domains_ok, (void)0);      // the specialised semirings are among them
        if (!domains_ok) return gb_fail(GrB_DOMAIN_MISMATCH, err, "mxv: unsupported semiring domains (x=%d, z=%d)", xt, zt);
        GB_TRY(spmv_run_plan(c, err));
        RunArgs ra{};
        const RunPlan &rp = c.run;
        ra.col = c.col; ra.aval = aval; ra.uval = uval; ra.headw = rp.headw; ra.run_base = rp.base;
        ra.nzrow = rp.nzrow; ra.rowptr = c.rowptr32; ra.nruns = rp.nruns; ra.nnz = c.nnz; ra.tval = tval;
        ra.tail_row = rp.tail_row; ra.tail_last = rp.tail_last; ra.long_run = rp.long_run; ra.nlong = rp.nlong;
        ra.add_op = add; ra.mul_op = kmul; ra.flip = kflip;
        ra.head_val = rp.ws_head; ra.tail_val = rp.ws_tail;            // scratch kept with the plan (the library serialises calls)
        if (sparse_u) { ra.upres = u->dv.pres; ra.tpres = tpres; ra.head_has = rp.ws_head_has; ra.tail_has = rp.ws_tail_has; }
        // hot-column table: on by default for large matrices whose gathers are concentrated (R-MAT-like);
        // B200GRB_SPMV_HOT=0 disables it, =<KB> caps the table size (and forces the kernel whatever the coverage)
        int hot_kb = tn.spmv_hot_kb >= 0 ? tn.spmv_hot_kb : 128;     // stage + table stay inside the 196 KB carve-out: the 228 KB one leaves no L1
        if (fast && need_u && hot_kb > 0 && c.nnz >= ((int64_t)1 << 20) && c.ncols >= (1 << 16)) {
            GB_TRY(spmv_hot_plan(c, err));
            if (!c.hot.col || (tn.spmv_hot_kb < 0 && c.hot.cover < 0.25)) hot_kb = 0;
        } else hot_kb = 0;
        Hot2Args hot{};
        if (hot_kb > 0) {
            // the launch runs the prep kernel first: u at the hot columns, T cleared, T's presence from the plan
            hot.col = c.hot.col; hot.id_bytes = c.hot.id_bytes;
            hot.u_hot = c.hot.ws_uhot; hot.hperm = c.hot.perm; hot.henc = c.hot.henc; hot.u = uval; hot.vsize = tc_size(xt);
            hot.tval = tval; hot.tval_bytes = (size_t)n * zsz; hot.pres_tmpl = rp.pres_tmpl; hot.tpres = tpres; hot.nrows = c.nrows;
            hot.want_cluster = 1;
            while (hot.want_cluster < 16 && hot.want_cluster * 2 <= tn.spmv_cluster) hot.want_cluster *= 2;
            hot.want_repl = (uint32_t)(((size_t)tn.spmv_hot_repl_kb << 10) / tc_size(xt));
            kernel_name = "run+hot-table (TMA-staged)";
        } else {
            CU_TRY(cudaMemsetAsync(tval, 0, (size_t)n * zsz, G.stream), err);
            if (sparse_u) CU_TRY(cudaMemsetAsync(tpres, 0, (size_t)n, G.stream), err);     // presence follows u: written row by row
            else CU_TRY(cudaMemcpyAsync(tpres, rp.pres_tmpl, (size_t)n, cudaMemcpyDeviceToDevice, G.stream), err);
            kernel_name = sparse_u ? "run (sparse u)" : "run";
        }
        const bool ok = fast_sr ? spmv_run_dispatch(xt, add, kmul, ra, hot_kb > 0 ? &hot : nullptr, (size_t)hot_kb << 10) : spmv_run_generic(xt, zt, ra);
        if (!ok) return gb_fail(GrB_PANIC, err, "mxv: internal dispatch error");
        if (hot_kb > 0) { hot_cluster = hot.cluster; hot_ctas = hot.ctas; hot_t0 = hot.t0; hot_t1 = hot.t1; hot_henc = hot.henc; hot_ids = hot.id_bytes * 8; }
    }
    gb_kernel_used(kernel_name);
    if (wide) gb_kernel_used("offsets=64");
    if (in_place) gb_kernel_used("mxv=in-place");
    if (hot_cluster > 0) {
        gb_kernel_used(("hot-cluster=" + std::to_string(hot_cluster)).c_str());
        gb_kernel_used(("hot-ctas=" + std::to_string(hot_ctas)).c_str());
        gb_kernel_used(("hot-tiers=" + std::to_string(hot_t0) + "," + std::to_string(hot_t1) + "," + std::to_string(hot_henc)).c_str());
        gb_kernel_used(("ids=" + std::to_string(hot_ids)).c_str());
        if (burble.on) { hot_note = std::string(kernel_name) + " cluster " + std::to_string(hot_cluster) + ", T0 " + std::to_string(hot_t0); kernel_name = hot_note.c_str(); }
    }
    if (burble.on && wide) { hot_note = std::string(kernel_name) + ", 64-bit offsets"; kernel_name = hot_note.c_str(); }
    if (burble.on) burble.note(kernel_name,(double)c.nnz * (4.0 + (need_a ? tc_size(xt) : 0)) + (double)(c.nrows + 1) * (wide ? 8 : 4) + (double)c.ncols * (need_u ? tc_size(xt) : 0) + (double)n * (zsz + 1));
    a_cast.reset(); u_cast.reset();
    vector_mark_used(u); if (mask) vector_mark_used(mask);          // an overlapped import into u may start as soon as these kernels are done

    if (in_place) {                    // T was formed in w's own buffers: only the bookkeeping changes
        w->dev_nvals = -1; w->host_valid = false; w->hi.clear(); w->hx.clear(); w->pi.clear(); w->px.clear();
        w->use_recorded = false;       // the kernels above write w: an import into w waits for them
        CU_TRY(cudaGetLastError(), err);
        return GrB_SUCCESS;
    }
    // ---- w<mask> = accum(w, t)   (vector_ops.cu)
    return vector_write(w, mask, accum, f, DenseForm{std::move(t_val), std::move(t_pres)}, zt, /*t_scalar=*/false, /*region=*/nullptr);
}

// The value semiring the inner form runs on: the monoid of s, with FIRST (vxm) / SECOND (mxv) of the monoid's type
static GB_Semiring_opaque value_semiring(const GrB_Semiring s, bool vxm) {
    const bool i32 = s->add->op->ztype->code == TC_INT32;
    const GrB_BinaryOp m = vxm ? (i32 ? GrB_FIRST_INT32 : GrB_FIRST_INT64) : (i32 ? GrB_SECOND_INT32 : GrB_SECOND_INT64);
    return GB_Semiring_opaque{GB_MAGIC, s->add, m, s->name, true};
}

// w<mask> = accum(w, op(A) (+).(x) u) with a positional multiply (DESIGN.md section 3.5).  FIRSTJ / SECONDI give the inner index k:
// u's values are replaced by k (a dense iota of the monoid type, u's presence kept) and the call runs on (+).SECOND (mxv) or
// (+).FIRST (vxm), with A's plans as they are.  FIRSTI / SECONDJ give the output position (or 0): the number of products per
// position comes from (+).PAIR in INT64 under the same mask, and one kernel turns it into the fold of that many copies.
GrB_Info positional_mxv(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_Semiring s, const GrB_Matrix A,
                        const GrB_Vector u, const DescFlags &f, bool vxm, const uint64_t *ids_in, const uint64_t *ids_out) {
    const char *fn = vxm ? "GrB_vxm" : "GrB_mxv";
    const bool use_transpose = vxm ? !f.tran1 : f.tran0;
    std::string *err = &w->err;
    const PosOp p = pos_binop(s->mul->opcode);
    const int zt = s->add->op->ztype->code, add = s->add->op->opcode;
    const uint64_t out_n = use_transpose ? A->ncols : A->nrows, in_n = use_transpose ? A->nrows : A->ncols;
    if (u->n != in_n || w->n != out_n || (mask && mask->n != out_n))
        return mxv_core(w, mask, accum, s, A, u, f, use_transpose, vxm, fn);           // reports the mismatch
    if (!G.have_device) return gb_fail(GrB_PANIC, err, "%s: no CUDA device: libb200grb computes only on the GPU (no CPU fallback)", fn);
    if (!mask && f.mask_comp) return mxv_core(w, mask, accum, s, A, u, f, use_transpose, vxm, fn);   // w<!NULL>: no product
    if (p.second != p.col) {
        // ---- inner form: product = k (+ off)
        GB_TRY(vector_ensure_device(u));
        DevBuf<void> iota; DevBuf<uint8_t> pres;
        GB_TRY(iota.alloc((size_t)in_n * tc_size(zt) + 16, err));
        GB_TRY(pos_vector_values(iota, zt, nullptr, OP_ANY, (int64_t)in_n, false, ids_in, p.off, err));
        const uint8_t *upres = u->dv.pres;
        if (upres && w == u) {      // T may be formed in w's buffers: the kernels must not read the presence they write
            GB_TRY(pres.alloc((size_t)in_n, err));
            CU_TRY(cudaMemcpyAsync(pres, upres, (size_t)in_n, cudaMemcpyDeviceToDevice, G.stream), err);
            upres = pres;
        }
        GB_Vector_opaque k{};      // u with the values k
        k.magic = GB_MAGIC; k.type = s->add->op->ztype; k.n = in_n; k.host_valid = false;
        k.dv = DenseForm::borrow(iota, (uint8_t *)upres); k.dev_nvals = u->dev_nvals;
        GB_Semiring_opaque sr = value_semiring(s, vxm);
        GB_TRY(mxv_core(w, mask, accum, &sr, A, &k, f, use_transpose, vxm, fn));
        vector_mark_used(u);
        gb_kernel_used("positional=inner");
        return GrB_SUCCESS;
    }
    // ---- count form: product = the output position (mxv FIRSTI, vxm SECONDJ) or 0 (mxv SECONDJ, vxm FIRSTI), + off
    const bool zero = vxm ? !p.second : p.second;
    GrB_Vector t = nullptr;
    GB_TRY(GrB_Vector_new(&t, GrB_INT64, out_n));
    const bool idem = add == OP_MIN || add == OP_MAX || add == OP_ANY;     // the count is not needed, only the pattern
    DescFlags fc = f; fc.replace = false;
    GrB_Info r = mxv_core(t, mask, nullptr, idem ? GxB_ANY_PAIR_INT64 : GxB_PLUS_PAIR_INT64, A, u, fc, use_transpose, vxm, fn);
    if (r == GrB_SUCCESS) r = vector_ensure_device(t);
    // T = the values from the counts, with the counts' presence (its own copy: w may adopt T's buffers)
    DevBuf<void> tval; DevBuf<uint8_t> tpres;
    if (r == GrB_SUCCESS) r = tval.alloc((size_t)out_n * tc_size(zt) + 16, err);
    if (r == GrB_SUCCESS) r = pos_vector_values(tval, zt, (const int64_t *)t->dv.val, add, (int64_t)out_n, zero, ids_out, p.off, err);
    if (r == GrB_SUCCESS && t->dv.pres) {
        r = tpres.alloc((size_t)out_n, err);
        if (r == GrB_SUCCESS && cudaMemcpyAsync(tpres, t->dv.pres, (size_t)out_n, cudaMemcpyDeviceToDevice, G.stream) != cudaSuccess)
            r = gb_fail(GrB_PANIC, err, "%s: copy of the count presence failed", fn);
    }
    if (r == GrB_SUCCESS) {
        gb_kernel_used("positional=count");
        r = vector_write(w, mask, accum, f, DenseForm{std::move(tval), std::move(tpres)}, zt, false, nullptr);
    } else if (t->err.size()) *err = t->err;
    GrB_Vector_free(&t);
    return r;
}

static GrB_Info mxv_check(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_Semiring s, const GrB_Matrix A, const GrB_Vector u,
                          const char *fn) {
    if (!w || !s || !A || !u) return gb_fail(GrB_NULL_POINTER, nullptr, "%s: NULL argument", fn);
    if (!gb_valid_vector(w) || !gb_valid_vector(u) || !gb_valid_matrix(A) || (mask && !gb_valid_vector(mask)) || s->magic != GB_MAGIC)
        return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "%s: invalid object", fn);
    GB_TRY(gb_refuse_positional_accum(accum, fn));
    return gb_refuse_user_with_positional(s, accum, fn);
}

extern "C" GrB_Info GrB_mxv(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_Semiring semiring,
                            const GrB_Matrix A, const GrB_Vector u, const GrB_Descriptor desc) {
    GB_LOCK; GB_CHECK_INIT;
    GB_TRY(mxv_check(w, mask, accum, semiring, A, u, "GrB_mxv"));
    if (gb_hyper_matrix(A) || gb_hyper_vector(u) || gb_hyper_vector(w)) return hyper_mxv(w, mask, accum, semiring, A, u, desc, false);
    const DescFlags f = desc_flags(desc);
    if (op_is_positional(semiring->mul->opcode)) return positional_mxv(w, mask, accum, semiring, A, u, f, false, nullptr, nullptr);
    return mxv_core(w, mask, accum, semiring, A, u, f, /*use_transpose=*/f.tran0, /*flip=*/false, "GrB_mxv");
}

extern "C" GrB_Info GrB_vxm(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_Semiring semiring,
                            const GrB_Vector u, const GrB_Matrix A, const GrB_Descriptor desc) {
    GB_LOCK; GB_CHECK_INIT;
    GB_TRY(mxv_check(w, mask, accum, semiring, A, u, "GrB_vxm"));
    if (gb_hyper_matrix(A) || gb_hyper_vector(u) || gb_hyper_vector(w)) return hyper_mxv(w, mask, accum, semiring, A, u, desc, true);
    const DescFlags f = desc_flags(desc);
    if (op_is_positional(semiring->mul->opcode)) return positional_mxv(w, mask, accum, semiring, A, u, f, true, nullptr, nullptr);
    // w' = u'A  <=>  w = A'u: pull along the rows of A' (INP1 = TRAN cancels the transpose)
    return mxv_core(w, mask, accum, semiring, A, u, f, /*use_transpose=*/!f.tran1, /*flip=*/true, "GrB_vxm");
}

