// Vector "loop glue" on the device: the element-wise operations that sit between two mxv / vxm calls in the
// reference's algorithms, so that a whole BFS / SSSP / PageRank iteration stays in HBM
// (SURVEY.md section 8(f)1):
//
//   GrB_Vector_eWiseAdd_{BinaryOp,Monoid,Semiring}, GrB_Vector_eWiseMult_{BinaryOp,Monoid,Semiring}
//                                    reference: pygraphblas/vector.py:604-735 (eadd / emult, operators + - * / | &)
//   GrB_Vector_apply, GrB_Vector_apply_BinaryOp1st/2nd_<T>, GxB_Vector_apply_BinaryOp1st/2nd
//                                    vector.py:1101-1178 (apply, apply_first, apply_second)
//   GrB_Vector_assign_<T>, GrB_Vector_assign, GrB_Vector_extract
//                                    vector.py:1436-1524, 1526-1560 (assign_scalar, assign, extract; slices)
//   GrB_Vector_reduce_<T>            vector.py:533-593 (reduce_bool / reduce_int / reduce_float)
//
// Vectors live in HBM as a dense value array plus presence bytes (NULL = every position present), so every
// operation is one streaming kernel that forms T followed by the common write-back
// w<mask> = accum(w, T) (vector_write, also the last step of GrB_mxv / GrB_vxm).  All kernels work on the
// 64-bit scalar carrier (common.cuh: Sc), i.e. one code path for the 11 builtin types and every typecast the
// API allows; they move <= 30 bytes per position and are HBM-bound at a few million positions.
#include "common.cuh"
#include <algorithm>
#include <vector>
#include "../../include/b200grb_compat.h"

static inline int vgrid(int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n, 256), (int64_t)G.num_sms * 16)); }

// ------------------------------------------------------------------ write-back:  w<mask> = accum(w, t)
struct VecFinalizeArgs {
    int64_t n;
    const void *wval; const uint8_t *wpres; int wtc; int w_exists;
    const void *tval; const uint8_t *tpres; int ttc; int t_scalar;
    const void *mval; const uint8_t *mpres; int mtc; int has_mask, mask_comp, mask_struct, replace;
    int accum_op, accum_tc, accum_ztc;   // accum_op < 0: none
    const uint8_t *region;               // GrB_assign: positions outside the region keep w
    void *oval; uint8_t *opres;          // opres NULL: the result is known to be full
};
__global__ void vec_finalize_kernel(const VecFinalizeArgs a) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * blockDim.x) {
        const bool tp = a.tpres ? a.tpres[i] != 0 : true;
        const bool wp = a.w_exists ? (a.wpres ? a.wpres[i] != 0 : true) : false;
        const size_t ti = a.t_scalar ? 0 : (size_t)i;
        bool m = true;
        if (a.has_mask) {
            m = a.mpres ? a.mpres[i] != 0 : true;
            if (m && !a.mask_struct) { const Sc mv = sc_cast(sc_load(a.mtc, a.mval, i), a.mtc, TC_BOOL); m = mv.u != 0; }
            if (a.mask_comp) m = !m;
        }
        Sc out; out.u = 0; bool op = false;
        if (m) {
            if (a.region && !a.region[i]) { if (wp) { out = sc_load(a.wtc, a.wval, i); op = true; } }
            else if (a.accum_op >= 0) {
                if (wp && tp) {
                    const Sc x = sc_cast(sc_load(a.wtc, a.wval, i), a.wtc, a.accum_tc);
                    const Sc y = sc_cast(sc_load(a.ttc, a.tval, ti), a.ttc, a.accum_tc);
                    out = sc_cast(sc_binop(a.accum_op, a.accum_tc, x, y), a.accum_ztc, a.wtc); op = true;
                } else if (wp) { out = sc_load(a.wtc, a.wval, i); op = true; }
                else if (tp) { out = sc_cast(sc_load(a.ttc, a.tval, ti), a.ttc, a.wtc); op = true; }
            } else if (tp) { out = sc_cast(sc_load(a.ttc, a.tval, ti), a.ttc, a.wtc); op = true; }
        } else if (!a.replace && wp) { out = sc_load(a.wtc, a.wval, i); op = true; }
        if (op) sc_store(a.wtc, a.oval, i, out);
        if (a.opres) a.opres[i] = op;
    }
}

// The same write-back when w, T and the accumulator share one type T (the iterated cases: SSSP's
// v = min(v, t), BFS's q<!visited> = t, PageRank's r += t): no carrier, no casts, the operator applied on T.
template <typename T> struct VecFinalizeTyped {
    int64_t n;
    const T *wval; const uint8_t *wpres; int w_exists;
    const T *tval; const uint8_t *tpres;
    const void *mval; const uint8_t *mpres; int mtc; int has_mask, mask_comp, mask_struct, replace;
    int accum_op;                        // < 0: none
    T *oval; uint8_t *opres;
};
template <typename T>
__global__ void __launch_bounds__(256) vec_finalize_typed_kernel(const VecFinalizeTyped<T> a) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * blockDim.x) {
        const bool tp = a.tpres ? a.tpres[i] != 0 : true;
        const bool wp = a.w_exists ? (a.wpres ? a.wpres[i] != 0 : true) : false;
        bool m = true;
        if (a.has_mask) {
            m = a.mpres ? a.mpres[i] != 0 : true;
            if (m && !a.mask_struct) m = mask_value_true(a.mtc, a.mval, i);
            if (a.mask_comp) m = !m;
        }
        T out = (T)0; bool op = false;
        if (m) {
            if (a.accum_op >= 0) {
                if (wp && tp) { out = op_apply<T>(a.accum_op, a.wval[i], a.tval[i]); op = true; }
                else if (wp) { out = a.wval[i]; op = true; }
                else if (tp) { out = a.tval[i]; op = true; }
            } else if (tp) { out = a.tval[i]; op = true; }
        } else if (!a.replace && wp) { out = a.wval[i]; op = true; }
        if (op) a.oval[i] = out;
        if (a.opres) a.opres[i] = op;
    }
}
template <typename T> static void launch_finalize_typed(const VecFinalizeArgs &g) {
    VecFinalizeTyped<T> a{};
    a.n = g.n; a.wval = (const T *)g.wval; a.wpres = g.wpres; a.w_exists = g.w_exists; a.tval = (const T *)g.tval; a.tpres = g.tpres;
    a.mval = g.mval; a.mpres = g.mpres; a.mtc = g.mtc; a.has_mask = g.has_mask; a.mask_comp = g.mask_comp; a.mask_struct = g.mask_struct;
    a.replace = g.replace; a.accum_op = g.accum_op; a.oval = (T *)g.oval; a.opres = g.opres;
    vec_finalize_typed_kernel<T><<<vgrid(g.n), 256, 0, G.stream>>>(a); GB_LAUNCHED();
}
static bool finalize_typed(const VecFinalizeArgs &g) {
    // one type throughout, whole-vector write, per-position T, accumulator (if any) of that type with a same-type result
    if (g.wtc != g.ttc || g.t_scalar || g.region) return false;
    if (g.accum_op >= 0 && (g.accum_tc != g.wtc || g.accum_ztc != g.wtc || g.accum_op >= OP_EQ)) return false;
    switch (g.wtc) {
        case TC_BOOL: launch_finalize_typed<bool>(g); return true;
        case TC_INT8: launch_finalize_typed<int8_t>(g); return true;
        case TC_INT16: launch_finalize_typed<int16_t>(g); return true;
        case TC_INT32: launch_finalize_typed<int32_t>(g); return true;
        case TC_INT64: launch_finalize_typed<int64_t>(g); return true;
        case TC_UINT8: launch_finalize_typed<uint8_t>(g); return true;
        case TC_UINT16: launch_finalize_typed<uint16_t>(g); return true;
        case TC_UINT32: launch_finalize_typed<uint32_t>(g); return true;
        case TC_UINT64: launch_finalize_typed<uint64_t>(g); return true;
        case TC_FP32: launch_finalize_typed<float>(g); return true;
        case TC_FP64: launch_finalize_typed<double>(g); return true;
        default: return false;
    }
}

GrB_Info vector_write(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const DescFlags &f,
                      const void *tval, const uint8_t *tpres, int ttc, bool t_scalar, const uint8_t *region,
                      DevBuf<void> &&own_val, DevBuf<uint8_t> &&own_pres) {
    std::string *err = &w->err;
    const int64_t n = (int64_t)w->n;
    const int wtc = w->type->code;
    if (!mask && f.mask_comp) {
        // w<!NULL>: the complement of "no mask" lets nothing through -- w keeps its entries, or loses all of
        // them under GrB_REPLACE (GraphBLAS C API 1.3 section 4.3; SuiteSparse's quick-mask exit)
        own_val.reset(); own_pres.reset();
        if (f.replace) {
            vector_invalidate_device(w);
            w->hi.clear(); w->hx.clear(); w->pi.clear(); w->px.clear(); w->host_valid = true;
        }
        return GrB_SUCCESS;
    }
    const bool need_final = mask != nullptr || accum != nullptr || region != nullptr || t_scalar || !own_val;
    if (!need_final) {      // w takes T's buffers
        if (wtc != ttc) {
            DevBuf<void> cv;
            GB_TRY(dev_cast_values(cv, wtc, tval, ttc, n, err));
            own_val = std::move(cv);
        }
        vector_adopt_device(w, own_val.release(), own_pres.release());
        CU_TRY(cudaGetLastError(), err);
        return GrB_SUCCESS;
    }
    const bool w_empty = w->host_valid && w->hi.empty() && w->pi.empty();   // nothing to merge with
    if (!w_empty) GB_TRY(vector_ensure_device(w));
    if (mask) GB_TRY(vector_ensure_device(mask));
    VecFinalizeArgs fa{};
    fa.n = n; fa.wval = w->dval; fa.wpres = w->dpres; fa.wtc = wtc; fa.w_exists = w_empty ? 0 : 1;
    fa.tval = tval; fa.tpres = tpres; fa.ttc = ttc; fa.t_scalar = t_scalar ? 1 : 0;
    if (mask) { fa.mval = mask->dval; fa.mpres = mask->dpres; fa.mtc = mask->type->code; fa.has_mask = 1; }
    fa.mask_comp = f.mask_comp; fa.mask_struct = f.mask_struct; fa.replace = f.replace;
    fa.accum_op = accum ? accum->opcode : -1;
    fa.accum_tc = accum ? accum->xtype->code : 0; fa.accum_ztc = accum ? accum->ztype->code : 0;
    fa.region = region;
    DevBuf<void> oval; DevBuf<uint8_t> opres;
    GB_TRY(oval.alloc((size_t)n * tc_size(wtc) + 16, err));
    fa.oval = oval;
    // a full w stays full under an accumulator (and a mask that does not replace), and a full T over the whole
    // vector without a mask gives a full result: no presence bytes, and the next mxv sees a dense operand
    // (SSSP: v = min(v, A' min.+ v))
    const bool w_full = !w_empty && w->dpres == nullptr;
    const bool out_full = (w_full && !(mask && f.replace) && (accum != nullptr || (region != nullptr && tpres == nullptr))) ||
                          (tpres == nullptr && !mask && !region);
    if (!out_full) { GB_TRY(opres.alloc((size_t)n, err)); fa.opres = opres; }
    if (!finalize_typed(fa)) { vec_finalize_kernel<<<vgrid(n), 256, 0, G.stream>>>(fa); GB_LAUNCHED(); }
    own_val.reset(); own_pres.reset();
    vector_adopt_device(w, oval.release(), opres.release());
    CU_TRY(cudaGetLastError(), err);
    return GrB_SUCCESS;
}

// ------------------------------------------------------------------ T = u (op) v,  T = f(u),  T = op(x, u), T = op(u, y)
enum { EW_ADD = 0, EW_MULT = 1, EW_UNARY = 2, EW_BIND1 = 3, EW_BIND2 = 4 };
struct EwiseArgs {
    int64_t n; int mode; int op; int xtc, ztc;       // op's operand type (x and y share it for builtins) and result type
    const void *uval; const uint8_t *upres; int utc;
    const void *vval; const uint8_t *vpres; int vtc;
    Sc scalar;                                        // bound operand, already of type xtc
    void *tval; uint8_t *tpres;
};
__global__ void vec_ewise_kernel(const EwiseArgs a) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * blockDim.x) {
        const bool up = a.upres ? a.upres[i] != 0 : true;
        Sc z; z.u = 0; bool tp = false;
        if (a.mode == EW_ADD || a.mode == EW_MULT) {
            const bool vp = a.vpres ? a.vpres[i] != 0 : true;
            if (up && vp) {
                z = sc_binop(a.op, a.xtc, sc_cast(sc_load(a.utc, a.uval, i), a.utc, a.xtc), sc_cast(sc_load(a.vtc, a.vval, i), a.vtc, a.xtc));
                tp = true;
            } else if (a.mode == EW_ADD && up) { z = sc_cast(sc_load(a.utc, a.uval, i), a.utc, a.ztc); tp = true; }
            else if (a.mode == EW_ADD && vp) { z = sc_cast(sc_load(a.vtc, a.vval, i), a.vtc, a.ztc); tp = true; }
        } else if (up) {
            const Sc x = sc_cast(sc_load(a.utc, a.uval, i), a.utc, a.xtc);
            z = a.mode == EW_UNARY ? sc_unop(a.op, a.xtc, x) : (a.mode == EW_BIND1 ? sc_binop(a.op, a.xtc, a.scalar, x) : sc_binop(a.op, a.xtc, x, a.scalar));
            tp = true;
        }
        if (tp) sc_store(a.ztc, a.tval, i, z);
        if (a.tpres) a.tpres[i] = tp;
    }
}

#define GB_VEC_OK(v, fn) do { if (!(v)) return gb_fail(GrB_NULL_POINTER, nullptr, "%s: NULL vector", fn); \
    if (!gb_valid_vector(v)) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "%s: invalid vector handle", fn); } while (0)
#define GB_NEED_DEVICE(w, fn) do { if (!G.have_device) return gb_fail(GrB_PANIC, &(w)->err, "%s: no CUDA device: libb200grb computes only on the GPU (no CPU fallback)", fn); } while (0)

static GrB_Info binop_ok(const GrB_BinaryOp op, const GrB_BinaryOp accum, const char *fn) {
    if (!op) return gb_fail(GrB_NULL_POINTER, nullptr, "%s: NULL operator", fn);
    if (op->magic != GB_MAGIC || (accum && accum->magic != GB_MAGIC)) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "%s: invalid operator", fn);
    if (op->opcode == OP_USER || (accum && accum->opcode == OP_USER))
        return gb_fail(GrB_INVALID_VALUE, nullptr, "%s: user-defined operators are host function pointers and cannot run on the GPU", fn);
    return GrB_SUCCESS;
}

static GrB_Info vec_ewise(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_BinaryOp op, const GrB_Vector u,
                          const GrB_Vector v, const GrB_Descriptor desc, int mode, const char *fn) {
    GB_VEC_OK(w, fn); GB_VEC_OK(u, fn); GB_VEC_OK(v, fn);
    if (mask) GB_VEC_OK(mask, fn);
    GB_TRY(binop_ok(op, accum, fn));
    if (u->n != v->n || w->n != u->n || (mask && mask->n != w->n)) return gb_fail(GrB_DIMENSION_MISMATCH, &w->err, "%s: dimensions do not match", fn);
    GB_NEED_DEVICE(w, fn);
    GB_TRY(vector_ensure_device(u)); GB_TRY(vector_ensure_device(v));
    const int64_t n = (int64_t)w->n;
    EwiseArgs a{};
    a.n = n; a.mode = mode; a.op = op->opcode; a.xtc = op->xtype->code; a.ztc = op->ztype->code;
    a.uval = u->dval; a.upres = u->dpres; a.utc = u->type->code; a.vval = v->dval; a.vpres = v->dpres; a.vtc = v->type->code;
    DevBuf<void> tval; DevBuf<uint8_t> tpres;
    GB_TRY(tval.alloc((size_t)n * tc_size(a.ztc) + 16, &w->err));
    const bool t_full = mode == EW_ADD ? (!u->dpres || !v->dpres) : (!u->dpres && !v->dpres);
    if (!t_full) GB_TRY(tpres.alloc((size_t)n, &w->err));
    a.tval = tval; a.tpres = tpres;
    vec_ewise_kernel<<<vgrid(n), 256, 0, G.stream>>>(a); GB_LAUNCHED();
    return vector_write(w, mask, accum, desc_flags(desc), a.tval, a.tpres, a.ztc, false, nullptr, std::move(tval), std::move(tpres));
}
extern "C" GrB_Info GrB_Vector_eWiseAdd_BinaryOp(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_BinaryOp op,
                                                  const GrB_Vector u, const GrB_Vector v, const GrB_Descriptor desc) {
    GB_LOCK; GB_CHECK_INIT; return vec_ewise(w, mask, accum, op, u, v, desc, EW_ADD, "GrB_Vector_eWiseAdd_BinaryOp");
}
extern "C" GrB_Info GrB_Vector_eWiseAdd_Monoid(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_Monoid op,
                                                const GrB_Vector u, const GrB_Vector v, const GrB_Descriptor desc) {
    GB_LOCK; GB_CHECK_INIT;
    if (!op) return gb_fail(GrB_NULL_POINTER, nullptr, "GrB_Vector_eWiseAdd_Monoid: NULL monoid");
    return vec_ewise(w, mask, accum, op->op, u, v, desc, EW_ADD, "GrB_Vector_eWiseAdd_Monoid");
}
extern "C" GrB_Info GrB_Vector_eWiseAdd_Semiring(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_Semiring op,
                                                  const GrB_Vector u, const GrB_Vector v, const GrB_Descriptor desc) {
    GB_LOCK; GB_CHECK_INIT;
    if (!op) return gb_fail(GrB_NULL_POINTER, nullptr, "GrB_Vector_eWiseAdd_Semiring: NULL semiring");
    return vec_ewise(w, mask, accum, op->add->op, u, v, desc, EW_ADD, "GrB_Vector_eWiseAdd_Semiring");
}
extern "C" GrB_Info GrB_Vector_eWiseMult_BinaryOp(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_BinaryOp op,
                                                   const GrB_Vector u, const GrB_Vector v, const GrB_Descriptor desc) {
    GB_LOCK; GB_CHECK_INIT;
    return vec_ewise(w, mask, accum, op, u, v, desc, EW_MULT, "GrB_Vector_eWiseMult_BinaryOp");
}
extern "C" GrB_Info GrB_Vector_eWiseMult_Monoid(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_Monoid op,
                                                 const GrB_Vector u, const GrB_Vector v, const GrB_Descriptor desc) {
    GB_LOCK; GB_CHECK_INIT;
    if (!op) return gb_fail(GrB_NULL_POINTER, nullptr, "GrB_Vector_eWiseMult_Monoid: NULL monoid");
    return vec_ewise(w, mask, accum, op->op, u, v, desc, EW_MULT, "GrB_Vector_eWiseMult_Monoid");
}
extern "C" GrB_Info GrB_Vector_eWiseMult_Semiring(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_Semiring op,
                                                   const GrB_Vector u, const GrB_Vector v, const GrB_Descriptor desc) {
    GB_LOCK; GB_CHECK_INIT;
    if (!op) return gb_fail(GrB_NULL_POINTER, nullptr, "GrB_Vector_eWiseMult_Semiring: NULL semiring");
    return vec_ewise(w, mask, accum, op->mul, u, v, desc, EW_MULT, "GrB_Vector_eWiseMult_Semiring");
}

// ------------------------------------------------------------------ apply
static GrB_Info vec_apply(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, int mode, int opcode, int xtc, int ztc, Sc scalar,
                          const GrB_Vector u, const GrB_Descriptor desc, const char *fn) {
    GB_VEC_OK(w, fn); GB_VEC_OK(u, fn);
    if (mask) GB_VEC_OK(mask, fn);
    if (accum && accum->opcode == OP_USER) return gb_fail(GrB_INVALID_VALUE, nullptr, "%s: user-defined accumulators cannot run on the GPU", fn);
    if (w->n != u->n || (mask && mask->n != w->n)) return gb_fail(GrB_DIMENSION_MISMATCH, &w->err, "%s: dimensions do not match", fn);
    GB_NEED_DEVICE(w, fn);
    GB_TRY(vector_ensure_device(u));
    const int64_t n = (int64_t)w->n;
    EwiseArgs a{};
    a.n = n; a.mode = mode; a.op = opcode; a.xtc = xtc; a.ztc = ztc; a.scalar = scalar;
    a.uval = u->dval; a.upres = u->dpres; a.utc = u->type->code;
    DevBuf<void> tval; DevBuf<uint8_t> tpres;
    GB_TRY(tval.alloc((size_t)n * tc_size(ztc) + 16, &w->err));
    if (u->dpres) GB_TRY(tpres.alloc((size_t)n, &w->err));
    a.tval = tval; a.tpres = tpres;
    vec_ewise_kernel<<<vgrid(n), 256, 0, G.stream>>>(a); GB_LAUNCHED();
    return vector_write(w, mask, accum, desc_flags(desc), a.tval, a.tpres, ztc, false, nullptr, std::move(tval), std::move(tpres));
}
extern "C" GrB_Info GrB_Vector_apply(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_UnaryOp op, const GrB_Vector u, const GrB_Descriptor desc) {
    GB_LOCK; GB_CHECK_INIT;
    if (!op) return gb_fail(GrB_NULL_POINTER, nullptr, "GrB_Vector_apply: NULL operator");
    if (op->magic != GB_MAGIC) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "GrB_Vector_apply: invalid operator");
    Sc none; none.u = 0;
    return vec_apply(w, mask, accum, EW_UNARY, op->opcode, op->xtype->code, op->ztype->code, none, u, desc, "GrB_Vector_apply");
}
static GrB_Info vec_bind(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_BinaryOp op, int first, const void *x, int xtc_in,
                         const GrB_Vector u, const GrB_Descriptor desc, const char *fn) {
    GB_TRY(binop_ok(op, accum, fn));
    const int xtc = op->xtype->code;
    // xtc_in >= 0: x points at a C value of that type; < 0: at a carrier (GxB_Scalar) of type -1 - xtc_in
    const Sc s = xtc_in >= 0 ? sc_cast(sc_load(xtc_in, x, 0), xtc_in, xtc) : sc_cast(*(const Sc *)x, -1 - xtc_in, xtc);
    return vec_apply(w, mask, accum, first ? EW_BIND1 : EW_BIND2, op->opcode, xtc, op->ztype->code, s, u, desc, fn);
}
#define GB_VEC_TYPED(TN, CT, TC) \
    extern "C" GrB_Info GrB_Vector_apply_BinaryOp1st_##TN(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_BinaryOp op, CT x, const GrB_Vector u, const GrB_Descriptor desc) { \
        GB_LOCK; GB_CHECK_INIT; return vec_bind(w, mask, accum, op, 1, &x, TC, u, desc, "GrB_Vector_apply_BinaryOp1st_" #TN); } \
    extern "C" GrB_Info GrB_Vector_apply_BinaryOp2nd_##TN(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_BinaryOp op, const GrB_Vector u, CT y, const GrB_Descriptor desc) { \
        GB_LOCK; GB_CHECK_INIT; return vec_bind(w, mask, accum, op, 0, &y, TC, u, desc, "GrB_Vector_apply_BinaryOp2nd_" #TN); } \
    extern "C" GrB_Info GrB_Vector_assign_##TN(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, CT x, const GrB_Index *I, GrB_Index ni, const GrB_Descriptor desc) { \
        GB_LOCK; GB_CHECK_INIT; return vec_assign_scalar(w, mask, accum, &x, TC, I, ni, desc, "GrB_Vector_assign_" #TN); } \
    extern "C" GrB_Info GrB_Vector_reduce_##TN(CT *c, const GrB_BinaryOp accum, const GrB_Monoid m, const GrB_Vector u, const GrB_Descriptor d) { \
        (void)d; GB_LOCK; GB_CHECK_INIT; return vec_reduce(c, TC, accum, m, u, "GrB_Vector_reduce_" #TN); }

// ------------------------------------------------------------------ index lists (GrB_ALL, explicit, GxB_RANGE / STRIDE / BACKWARDS)
extern "C" const GrB_Index *GrB_ALL;
// Expands (I, ni) over a dimension of `dim` positions.  all = true: every position in order (no list needed).
GrB_Info index_list(const GrB_Index *I, GrB_Index ni, uint64_t dim, bool *all, std::vector<uint64_t> &out, std::string *err, const char *fn) {
    *all = false; out.clear();
    if (!I) return gb_fail(GrB_NULL_POINTER, err, "%s: NULL index list", fn);
    if (I == GrB_ALL) { *all = true; return GrB_SUCCESS; }
    if (ni == GxB_RANGE || ni == GxB_STRIDE || ni == GxB_BACKWARDS) {
        const int64_t lo = (int64_t)I[0], hi = (int64_t)I[1];
        const int64_t inc = ni == GxB_RANGE ? 1 : (ni == GxB_STRIDE ? (int64_t)I[2] : -(int64_t)I[2]);
        if (inc == 0) return GrB_SUCCESS;
        if (inc > 0) for (int64_t k = lo; k <= hi; k += inc) out.push_back((uint64_t)k);
        else for (int64_t k = lo; k >= hi; k += inc) out.push_back((uint64_t)k);
    } else out.assign(I, I + ni);
    for (uint64_t k : out) if (k >= dim) return gb_fail(GrB_INDEX_OUT_OF_BOUNDS, err, "%s: index %llu out of bounds (dimension %llu)", fn, (unsigned long long)k, (unsigned long long)dim);
    if (out.size() == dim) { bool iota = true; for (uint64_t k = 0; k < dim && iota; ++k) iota = out[k] == k; if (iota) { *all = true; out.clear(); } }
    return GrB_SUCCESS;
}
static GrB_Info upload_indices(const std::vector<uint64_t> &idx, DevBuf<uint64_t> &d, std::string *err) {
    GB_TRY(d.alloc(idx.size(), err));
    CU_TRY(cudaMemcpyAsync(d, idx.data(), idx.size() * sizeof(uint64_t), cudaMemcpyHostToDevice, G.stream), err);
    CU_TRY(cudaStreamSynchronize(G.stream), err);          // idx is a caller-owned temporary
    return GrB_SUCCESS;
}
__global__ void region_mark_kernel(const uint64_t *idx, int64_t k, uint8_t *region) {
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < k; q += (int64_t)gridDim.x * blockDim.x) region[idx[q]] = 1;
}
// T(idx[q]) = u(q): the scatter of GrB_assign; later duplicates win is not defined by the spec (we take any)
__global__ void vec_scatter_u_kernel(const uint64_t *idx, int64_t k, const void *uval, const uint8_t *upres, int tc, void *tval, uint8_t *tpres, uint8_t *region) {
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < k; q += (int64_t)gridDim.x * blockDim.x) {
        const uint64_t i = idx[q];
        const bool up = upres ? upres[q] != 0 : true;
        if (up) sc_store(tc, tval, i, sc_load(tc, uval, q));
        tpres[i] = up; region[i] = 1;
    }
}
// T(q) = u(idx[q]): GrB_extract
__global__ void vec_gather_u_kernel(const uint64_t *idx, int64_t k, const void *uval, const uint8_t *upres, int tc, void *tval, uint8_t *tpres) {
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < k; q += (int64_t)gridDim.x * blockDim.x) {
        const uint64_t i = idx[q];
        const bool up = upres ? upres[i] != 0 : true;
        if (up) sc_store(tc, tval, q, sc_load(tc, uval, i));
        tpres[q] = up;
    }
}

static GrB_Info vec_assign_scalar(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const void *x, int xtc, const GrB_Index *I, GrB_Index ni,
                                  const GrB_Descriptor desc, const char *fn) {
    GB_VEC_OK(w, fn);
    if (mask) GB_VEC_OK(mask, fn);
    if (accum && accum->opcode == OP_USER) return gb_fail(GrB_INVALID_VALUE, nullptr, "%s: user-defined accumulators cannot run on the GPU", fn);
    if (mask && mask->n != w->n) return gb_fail(GrB_DIMENSION_MISMATCH, &w->err, "%s: mask dimension does not match", fn);
    bool all; std::vector<uint64_t> idx;
    GB_TRY(index_list(I, ni, w->n, &all, idx, &w->err, fn));
    GB_NEED_DEVICE(w, fn);
    // T: one value (of w's type) standing for every position of the region
    const int wtc = w->type->code;
    DevBuf<void> tval;
    GB_TRY(tval.alloc(16, &w->err));
    uint64_t word[2] = {0, 0};
    sc_store(wtc, word, 0, sc_cast(sc_load(xtc, x, 0), xtc, wtc));
    CU_TRY(cudaMemcpyAsync(tval, word, 8, cudaMemcpyHostToDevice, G.stream), &w->err);
    CU_TRY(cudaStreamSynchronize(G.stream), &w->err);
    DevBuf<uint8_t> region;
    if (!all) {
        GB_TRY(region.alloc((size_t)w->n, &w->err));
        CU_TRY(cudaMemsetAsync(region, 0, (size_t)w->n, G.stream), &w->err);
        if (!idx.empty()) {
            DevBuf<uint64_t> didx;
            GB_TRY(upload_indices(idx, didx, &w->err));
            region_mark_kernel<<<vgrid((int64_t)idx.size()), 256, 0, G.stream>>>(didx, (int64_t)idx.size(), region); GB_LAUNCHED();
        }
    }
    return vector_write(w, mask, accum, desc_flags(desc), tval, nullptr, wtc, true, region, std::move(tval));
}

extern "C" GrB_Info GrB_Vector_assign(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_Vector u, const GrB_Index *I, GrB_Index ni,
                                      const GrB_Descriptor desc) {
    GB_LOCK; GB_CHECK_INIT;
    const char *fn = "GrB_Vector_assign";
    GB_VEC_OK(w, fn); GB_VEC_OK(u, fn);
    if (mask) GB_VEC_OK(mask, fn);
    if (accum && accum->opcode == OP_USER) return gb_fail(GrB_INVALID_VALUE, nullptr, "%s: user-defined accumulators cannot run on the GPU", fn);
    if (mask && mask->n != w->n) return gb_fail(GrB_DIMENSION_MISMATCH, &w->err, "%s: mask dimension does not match", fn);
    bool all; std::vector<uint64_t> idx;
    GB_TRY(index_list(I, ni, w->n, &all, idx, &w->err, fn));
    if ((all ? w->n : (uint64_t)idx.size()) != u->n) return gb_fail(GrB_DIMENSION_MISMATCH, &w->err, "%s: u has %llu positions, the index list %llu", fn,
                                                                     (unsigned long long)u->n, (unsigned long long)(all ? w->n : idx.size()));
    GB_NEED_DEVICE(w, fn);
    GB_TRY(vector_ensure_device(u));
    const int utc = u->type->code;
    if (all) {
        if (w == u && !mask && !accum) return GrB_SUCCESS;
        return vector_write(w, mask, accum, desc_flags(desc), u->dval, u->dpres, utc, false, nullptr);
    }
    DevBuf<void> tval; DevBuf<uint8_t> tpres, region;
    const size_t n = (size_t)w->n;
    GB_TRY(tval.alloc(n * tc_size(utc) + 16, &w->err));
    GB_TRY(tpres.alloc(n, &w->err));
    GB_TRY(region.alloc(n, &w->err));
    CU_TRY(cudaMemsetAsync(tpres, 0, n, G.stream), &w->err);
    CU_TRY(cudaMemsetAsync(region, 0, n, G.stream), &w->err);
    if (!idx.empty()) {
        DevBuf<uint64_t> didx;
        GB_TRY(upload_indices(idx, didx, &w->err));
        vec_scatter_u_kernel<<<vgrid((int64_t)idx.size()), 256, 0, G.stream>>>(didx, (int64_t)idx.size(), u->dval, u->dpres, utc, tval, tpres, region); GB_LAUNCHED();
    }
    return vector_write(w, mask, accum, desc_flags(desc), tval, tpres, utc, false, region, std::move(tval), std::move(tpres));
}

extern "C" GrB_Info GrB_Vector_extract(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_Vector u, const GrB_Index *I, GrB_Index ni,
                                       const GrB_Descriptor desc) {
    GB_LOCK; GB_CHECK_INIT;
    const char *fn = "GrB_Vector_extract";
    GB_VEC_OK(w, fn); GB_VEC_OK(u, fn);
    if (mask) GB_VEC_OK(mask, fn);
    if (accum && accum->opcode == OP_USER) return gb_fail(GrB_INVALID_VALUE, nullptr, "%s: user-defined accumulators cannot run on the GPU", fn);
    if (mask && mask->n != w->n) return gb_fail(GrB_DIMENSION_MISMATCH, &w->err, "%s: mask dimension does not match", fn);
    if (I && I != GrB_ALL && ni == GxB_RANGE && I[0] <= I[1] && I[1] < u->n && I[1] - I[0] + 1 == w->n && w != u && G.have_device) {
        // a contiguous range (the slice v[a:b] of reference: pygraphblas/base.py:216-252): two device copies, no index list
        GB_TRY(vector_ensure_device(u));
        const size_t n = (size_t)w->n, sz = (size_t)tc_size(u->type->code);
        DevBuf<void> tval; DevBuf<uint8_t> tpres;
        GB_TRY(tval.alloc(n * sz + 16, &w->err));
        CU_TRY(cudaMemcpyAsync(tval, (const uint8_t *)u->dval + (size_t)I[0] * sz, n * sz, cudaMemcpyDeviceToDevice, G.stream), &w->err);
        if (u->dpres) {
            GB_TRY(tpres.alloc(n, &w->err));
            CU_TRY(cudaMemcpyAsync(tpres, u->dpres + I[0], n, cudaMemcpyDeviceToDevice, G.stream), &w->err);
        }
        return vector_write(w, mask, accum, desc_flags(desc), tval, tpres, u->type->code, false, nullptr, std::move(tval), std::move(tpres));
    }
    bool all; std::vector<uint64_t> idx;
    GB_TRY(index_list(I, ni, u->n, &all, idx, &w->err, fn));
    if ((all ? u->n : (uint64_t)idx.size()) != w->n) return gb_fail(GrB_DIMENSION_MISMATCH, &w->err, "%s: w has %llu positions, the index list %llu", fn,
                                                                     (unsigned long long)w->n, (unsigned long long)(all ? u->n : idx.size()));
    GB_NEED_DEVICE(w, fn);
    GB_TRY(vector_ensure_device(u));
    const int utc = u->type->code;
    if (all) {
        if (w == u && !mask && !accum) return GrB_SUCCESS;
        return vector_write(w, mask, accum, desc_flags(desc), u->dval, u->dpres, utc, false, nullptr);
    }
    DevBuf<void> tval; DevBuf<uint8_t> tpres;
    const size_t n = (size_t)w->n;
    GB_TRY(tval.alloc(n * tc_size(utc) + 16, &w->err));
    GB_TRY(tpres.alloc(n, &w->err));
    if (!idx.empty()) {
        DevBuf<uint64_t> didx;
        GB_TRY(upload_indices(idx, didx, &w->err));
        vec_gather_u_kernel<<<vgrid((int64_t)idx.size()), 256, 0, G.stream>>>(didx, (int64_t)idx.size(), u->dval, u->dpres, utc, tval, tpres); GB_LAUNCHED();
    }
    return vector_write(w, mask, accum, desc_flags(desc), tval, tpres, utc, false, nullptr, std::move(tval), std::move(tpres));
}

// ------------------------------------------------------------------ reduce to a scalar
// Two-level fold on the carrier: threads -> warp (shuffles) -> CTA (shared) -> per-CTA partials -> one last CTA.
struct ReduceArgs { int64_t n; const void *val; const uint8_t *pres; int vtc; int op; int mtc; Sc *part; uint8_t *part_has; int stage2; };
__device__ __forceinline__ void red_join(int op, int mtc, Sc &a, int &ah, Sc b, int bh) {
    if (bh) { a = ah ? sc_binop(op, mtc, a, b) : b; ah = 1; }
}
__global__ void __launch_bounds__(256) vec_reduce_kernel(const ReduceArgs a) {
    __shared__ unsigned long long s_v[8]; __shared__ int s_h[8];
    Sc acc; acc.u = 0; int has = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * blockDim.x) {
        if (a.stage2) red_join(a.op, a.mtc, acc, has, a.part[i], a.part_has[i]);
        else if (!a.pres || a.pres[i]) red_join(a.op, a.mtc, acc, has, sc_cast(sc_load(a.vtc, a.val, i), a.vtc, a.mtc), 1);
    }
    for (int o = 16; o > 0; o >>= 1) {
        Sc y; y.u = __shfl_xor_sync(0xffffffffu, (unsigned long long)acc.u, o);
        const int yh = __shfl_xor_sync(0xffffffffu, has, o);
        red_join(a.op, a.mtc, acc, has, y, yh);
    }
    if ((threadIdx.x & 31) == 0) { s_v[threadIdx.x >> 5] = acc.u; s_h[threadIdx.x >> 5] = has; }
    __syncthreads();
    if (threadIdx.x == 0) {
        Sc r; r.u = 0; int rh = 0;
        for (int q = 0; q < 8; ++q) { Sc y; y.u = s_v[q]; red_join(a.op, a.mtc, r, rh, y, s_h[q]); }
        Sc *out = a.stage2 ? a.part + a.n : a.part;              // stage 2 writes its single result after the partials
        uint8_t *oh = a.stage2 ? a.part_has + a.n : a.part_has;
        out[a.stage2 ? 0 : blockIdx.x] = r; oh[a.stage2 ? 0 : blockIdx.x] = (uint8_t)rh;
    }
}
GrB_Info dev_reduce_values(const void *val, const uint8_t *pres, int vtc, int64_t n, int op, int mtc, Sc *out, bool *has, std::string *err) {
    out->u = 0; *has = false;
    if (n <= 0) return GrB_SUCCESS;
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n, 256 * 8), (int64_t)G.num_sms * 8));
    ReduceArgs a{};
    a.n = n; a.val = val; a.pres = pres; a.vtc = vtc; a.op = op; a.mtc = mtc;
    DevBuf<Sc> part; DevBuf<uint8_t> part_has;
    GB_TRY(part.alloc((size_t)grid + 1, err));
    GB_TRY(part_has.alloc((size_t)grid + 1, err));
    a.part = part; a.part_has = part_has;
    vec_reduce_kernel<<<grid, 256, 0, G.stream>>>(a); GB_LAUNCHED();
    ReduceArgs b = a; b.n = grid; b.stage2 = 1;
    vec_reduce_kernel<<<1, 256, 0, G.stream>>>(b); GB_LAUNCHED();
    uint8_t rh = 0;
    CU_TRY(cudaMemcpyAsync(out, a.part + grid, sizeof(Sc), cudaMemcpyDeviceToHost, G.stream), err);
    CU_TRY(cudaMemcpyAsync(&rh, a.part_has + grid, 1, cudaMemcpyDeviceToHost, G.stream), err);
    CU_TRY(cudaStreamSynchronize(G.stream), err);
    *has = rh != 0;
    return GrB_SUCCESS;
}
static GrB_Info vec_reduce(void *c, int ctc, const GrB_BinaryOp accum, const GrB_Monoid monoid, const GrB_Vector u, const char *fn) {
    if (!G.have_device) return gb_fail(GrB_PANIC, nullptr, "%s: no CUDA device: libb200grb computes only on the GPU (no CPU fallback)", fn);
    if (!c || !monoid) return gb_fail(GrB_NULL_POINTER, nullptr, "%s: NULL argument", fn);
    GB_VEC_OK(u, fn);
    if (monoid->magic != GB_MAGIC) return gb_fail(GrB_UNINITIALIZED_OBJECT, nullptr, "%s: invalid monoid", fn);
    const GrB_BinaryOp op = monoid->op;
    if (op->opcode == OP_USER || (accum && accum->opcode == OP_USER)) return gb_fail(GrB_INVALID_VALUE, nullptr, "%s: user-defined operators cannot run on the GPU", fn);
    GB_TRY(vector_ensure_device(u));
    const int mtc = op->ztype->code;
    Sc r; bool rh = false;
    GB_TRY(dev_reduce_values(u->dval, u->dpres, u->type->code, (int64_t)u->n, op->opcode, mtc, &r, &rh, &u->err));
    const Sc acc = rh ? r : sc_monoid_identity(op->opcode, mtc);
    Sc out = sc_cast(acc, mtc, ctc);
    if (accum) {
        const int atc = accum->xtype->code;
        const Sc old = sc_cast(sc_load(ctc, c, 0), ctc, atc);
        out = sc_cast(sc_binop(accum->opcode, atc, old, sc_cast(acc, mtc, atc)), accum->ztype->code, ctc);
    }
    sc_store(ctc, c, 0, out);
    return GrB_SUCCESS;
}

GB_VEC_TYPED(BOOL, bool, TC_BOOL) GB_VEC_TYPED(INT8, int8_t, TC_INT8) GB_VEC_TYPED(INT16, int16_t, TC_INT16) GB_VEC_TYPED(INT32, int32_t, TC_INT32)
GB_VEC_TYPED(INT64, int64_t, TC_INT64) GB_VEC_TYPED(UINT8, uint8_t, TC_UINT8) GB_VEC_TYPED(UINT16, uint16_t, TC_UINT16)
GB_VEC_TYPED(UINT32, uint32_t, TC_UINT32) GB_VEC_TYPED(UINT64, uint64_t, TC_UINT64) GB_VEC_TYPED(FP32, float, TC_FP32) GB_VEC_TYPED(FP64, double, TC_FP64)

// GxB_Scalar forms used by Vector.apply_first / apply_second (vector.py:1131-1178)
extern "C" GrB_Info GxB_Vector_apply_BinaryOp1st(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_BinaryOp op, const GxB_Scalar x,
                                                  const GrB_Vector u, const GrB_Descriptor desc) {
    GB_LOCK; GB_CHECK_INIT;
    if (!x || x->magic != GB_MAGIC || !x->has) return gb_fail(GrB_INVALID_VALUE, nullptr, "GxB_Vector_apply_BinaryOp1st: empty or invalid scalar");
    return vec_bind(w, mask, accum, op, 1, &x->v, -1 - x->type->code, u, desc, "GxB_Vector_apply_BinaryOp1st");
}
extern "C" GrB_Info GxB_Vector_apply_BinaryOp2nd(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_BinaryOp op, const GrB_Vector u,
                                                  const GxB_Scalar y, const GrB_Descriptor desc) {
    GB_LOCK; GB_CHECK_INIT;
    if (!y || y->magic != GB_MAGIC || !y->has) return gb_fail(GrB_INVALID_VALUE, nullptr, "GxB_Vector_apply_BinaryOp2nd: empty or invalid scalar");
    return vec_bind(w, mask, accum, op, 0, &y->v, -1 - y->type->code, u, desc, "GxB_Vector_apply_BinaryOp2nd");
}
